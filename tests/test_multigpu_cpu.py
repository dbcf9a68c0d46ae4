"""N>1 host logic on CPU: the strip-sharding driver (gfxexp_b200/multigpu.py) run with world_size 2 over gloo,
with the CPU oracle as the compute backend, must composite exactly the single-process frame (SURVEY.md §8e)."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, FRAMES = 96, 64, 3


class OracleBackend:
    """Same interface as multigpu.GpuBackend, on top of tests/oracle_lib (zero-copy numpy views)."""

    def __init__(self, oframe):
        from tests import oracle_lib as O
        self.O = O
        self.oframe = oframe
        self._views = {}

    def light_dist(self, frame_index):
        pass  # static scene: the oracle builds its distributions at scene creation

    def gbuffer(self, params):
        self.oframe.gbuffer(params, 2)

    def restir(self, params, pass_id):
        self.oframe.restir(params, pass_id, 2)

    def tensor(self, buffer_id, index=0):
        key = (buffer_id, index)
        if key not in self._views:
            nbytes = C.c_size_t()
            ptr = self.O.lib().orc_buffer_ptr(self.oframe.h, buffer_id, index, C.byref(nbytes))
            raw = (C.c_float * (nbytes.value // 4)).from_address(ptr)
            self._views[key] = torch.from_numpy(np.frombuffer(raw, dtype=np.float32))
        return self._views[key]

    def new_tensor(self, numel):
        return torch.empty(numel, dtype=torch.float32)


def _worker(rank, world, port, result_path, H=H, boundaries=None):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gfxexp_b200 import abi, multigpu, scenes
    from tests import oracle_lib as O
    scene = scenes.tiny_city_scene()
    oscene = O.OracleScene(scene)
    oframe = O.OracleFrame(oscene, W, H)
    p = abi.default_frame_params(scene, W, H)
    driver = multigpu.StripDriver(OracleBackend(oframe), p, W, H, rank, world, halo=24, boundaries=boundaries)
    outs = []
    for f in range(FRAMES):
        driver.render_frame(f, num_spatial_passes=2)
        outs.append(driver.composited.clone().numpy())
    if rank == 0:
        np.save(result_path, np.stack(outs))
    dist.barrier()
    dist.destroy_process_group()


def _moving_camera(scene, frame):
    from gfxexp_b200 import abi
    cam = abi.make_camera(scene, W, H)
    cam.position[1] += 0.12 * frame   # vertical motion: reprojected pixels cross the strip seams
    cam.position[0] += 0.05 * frame
    return cam


def _worker_moving(rank, world, port, result_path):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gfxexp_b200 import abi, multigpu, scenes
    from tests import oracle_lib as O
    scene = scenes.tiny_city_scene()
    oframe = O.OracleFrame(O.OracleScene(scene), W, H)
    p = abi.default_frame_params(scene, W, H)
    driver = multigpu.StripDriver(OracleBackend(oframe), p, W, H, rank, world, halo=24, max_motion_rows=24)
    outs = []
    for f in range(FRAMES):
        p.prevCamera = _moving_camera(scene, max(f - 1, 0))
        p.camera = _moving_camera(scene, f)
        driver.render_frame(f, num_spatial_passes=1)
        outs.append(driver.composited.clone().numpy())
    if rank == 0:
        np.save(result_path, np.stack(outs))
    dist.barrier()
    dist.destroy_process_group()


def test_strips_equal_single_process_with_a_moving_camera(tmp_path, oracle):
    """temporal reuse follows the motion vectors across the strip seams: with the motion inside the halo the sharded frames
    still equal the single-process frames bit for bit"""
    from gfxexp_b200 import abi, engine, scenes
    result = str(tmp_path / "moving.npy")
    mp.spawn(_worker_moving, args=(2, _free_port(), result), nprocs=2, join=True)
    got = np.load(result)
    scene = scenes.tiny_city_scene()
    oframe = oracle.OracleFrame(oracle.OracleScene(scene), W, H)
    p = abi.default_frame_params(scene, W, H)
    for f in range(FRAMES):
        p.prevCamera = _moving_camera(scene, max(f - 1, 0))
        p.camera = _moving_camera(scene, f)
        for kind, pass_id in engine.restir_frame_passes(p, f, 1):
            oframe.gbuffer(p) if kind == "gbuffer" else oframe.restir(p, pass_id)
        want = oframe.buffer(abi.BUF_BEAUTY_ACCUM).reshape(-1)
        assert np.array_equal(got[f].view(np.uint32), want.view(np.uint32)), f"frame {f}: sharded frame differs"


def test_strip_driver_refuses_what_the_halo_cannot_cover():
    from gfxexp_b200 import abi, multigpu, scenes
    scene = scenes.tiny_city_scene()

    class Dummy:
        def new_tensor(self, n):
            return torch.empty(n)
    p = abi.default_frame_params(scene, 64, 64)
    p.spatialNeighborRadius = 30.0
    with pytest.raises(ValueError):     # radius 30 > halo 24
        multigpu.StripDriver(Dummy(), p, 64, 64, 0, 2)
    p.spatialNeighborRadius = 20.0
    with pytest.raises(ValueError):     # motion beyond the halo
        multigpu.StripDriver(Dummy(), p, 64, 64, 0, 2, max_motion_rows=30)
    d = multigpu.StripDriver(Dummy(), p, 64, 64, 0, 2)
    p.enableTemporalReuse = 1
    cam = abi.make_camera(scene, 64, 64)
    cam.position[0] += 1.0
    p.prevCamera = abi.make_camera(scene, 64, 64)
    p.camera = cam
    with pytest.raises(ValueError):     # a moving camera without a stated motion bound
        d.render_frame(1)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# 4 ranks: the two middle ranks exchange seams on both sides; boundaries: cost-balanced strips of unequal height (all-gather-v)
@pytest.mark.parametrize("world,H,boundaries", [(2, 64, None), (4, 128, None), (2, 64, [0, 40, 64]), (3, 128, [0, 56, 88, 128])])
def test_strips_equal_single_process(tmp_path, oracle, world, H, boundaries):
    from gfxexp_b200 import abi, engine, scenes
    result = str(tmp_path / "composited.npy")
    mp.spawn(_worker, args=(world, _free_port(), result, H, boundaries), nprocs=world, join=True)
    got = np.load(result)

    scene = scenes.tiny_city_scene()
    oscene = oracle.OracleScene(scene)
    oframe = oracle.OracleFrame(oscene, W, H)
    p = abi.default_frame_params(scene, W, H)
    for f in range(FRAMES):
        for kind, pass_id in engine.restir_frame_passes(p, f, 2):
            if kind == "gbuffer":
                oframe.gbuffer(p)
            else:
                oframe.restir(p, pass_id)
        want = oframe.buffer(abi.BUF_BEAUTY_ACCUM).reshape(-1)
        assert np.array_equal(got[f].view(np.uint32), want.view(np.uint32)), f"frame {f}: sharded frame differs"


def test_balanced_boundaries():
    from gfxexp_b200 import multigpu
    cost = np.r_[np.full(300, 0.15), np.full(780, 1.0)]           # a sky above the geometry
    b = multigpu.balanced_boundaries(cost, 8, 24)
    assert b[0] == 0 and b[-1] == 1080 and all(v % 8 == 0 for v in b) and all(b[i + 1] - b[i] >= 24 for i in range(8))
    per = [cost[b[i]:b[i + 1]].sum() for i in range(8)]
    assert max(per) / (sum(per) / 8) < 1.05, per                  # within 5 % of equal work ...
    equal = [cost[i * 135:(i + 1) * 135].sum() for i in range(8)]
    assert max(equal) / (sum(equal) / 8) > 1.25                   # ... where equal heights are 25 % off
    assert multigpu.balanced_boundaries(np.ones(192), 2, 24) == [0, 96, 192]
    assert multigpu.balanced_boundaries(np.r_[np.zeros(150), np.ones(42)], 4, 24) == [0, 120, 144, 168, 192]  # the halo floor
    with pytest.raises(ValueError):
        multigpu.balanced_boundaries(np.ones(64), 4, 24)


def test_strip_partition_rejects_ragged_heights():
    from gfxexp_b200 import abi, multigpu, scenes
    scene = scenes.tiny_city_scene()
    p = abi.default_frame_params(scene, 64, 50)

    class Dummy:
        def new_tensor(self, n):
            return torch.empty(n)
    with pytest.raises(ValueError):
        multigpu.StripDriver(Dummy(), p, 64, 50, 0, 4)
    p = abi.default_frame_params(scene, 64, 64)
    with pytest.raises(ValueError):     # 16 rows per rank < 24 halo rows: a seam would have to cross two ranks
        multigpu.StripDriver(Dummy(), p, 64, 64, 0, 4)


# ---- the NRC frame sharded by strips (the oracle's restatement of gfx_nrc_shard), world_size 2 over gloo ---------------------
NRC_W, NRC_H, NRC_FRAMES = 64, 48, 3


def _nrc_frame(O, oframe, onet, p, frame, rows=None, seed_tile=None):
    """one NRC frame on the oracle (network included), on `rows` = (y0, y1) or the whole frame; the perFrameRng() draws are a
    function of the frame index.  Frame 0 starts a new sequence, or continues one whose last frame had `seed_tile`."""
    from gfxexp_b200 import abi
    from tests import nrc_records
    rng = np.random.default_rng(500 + frame)
    offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
    w, n = oframe.W, oframe.W * oframe.H
    p.frameIndex, p.bufferIndex, p.numAccumFrames = frame, frame % 2, frame
    p.tileOriginY, p.tileRows = 0, 0
    oframe.gbuffer(p)
    if rows is not None:
        p.tileOriginY, p.tileRows = rows[0], rows[1] - rows[0]
    seeded = frame == 0 and seed_tile is not None
    if seeded:
        st = oframe.linear_buffer(abi.BUF_NRC_STATE, copy=False)
        st[:] = nrc_records.seeded_state(st, p.bufferIndex, seed_tile)
    oframe.nrc_preprocess(p, offsets[0], offsets[1], frame == 0 and not seeded)
    oframe.pathtrace(p, abi.PT_NRC)
    q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
    ti = oframe.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    suffix = oframe.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL)[:, 0]
    lo, hi = (rows[0] * w, rows[1] * w) if rows is not None else (0, n)
    pix = lo + np.flatnonzero((ti[lo:hi, 3] & 1).astype(bool))
    sfx = n + np.flatnonzero(((suffix >> 23) & 1).astype(bool))
    idx = np.concatenate([pix, sfx])
    pred = oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)
    if len(idx):
        pred[idx] = onet.infer(q[idx])
    oframe.nrc_accumulate(p)
    oframe.nrc_propagate(p)
    oframe.nrc_shuffle(p)
    tq, tt = oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 1), oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 1)
    for step in range(4):
        sl = slice(step * 16384, (step + 1) * 16384)
        onet.train(tq[sl], tt[sl])
    p.tileOriginY, p.tileRows = 0, 0


def _nrc_setup(scene_name="tiny_city_scene", w=NRC_W, h=NRC_H):
    from gfxexp_b200 import abi, engine, scenes
    from tests import oracle_lib as O
    scene = getattr(scenes, scene_name)()
    oframe = O.OracleFrame(O.OracleScene(scene), w, h)
    onet = O.OracleNrc(2, 1e-2)
    onet.set_params(engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 4
    p.radianceScale = 2.0
    return O, oframe, onet, p


def _worker_nrc(rank, world, port, result_path, scene_name, w, h, frames, seed_tile):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gfxexp_b200 import abi
    O, oframe, onet, p = _nrc_setup(scene_name, w, h)
    oframe.nrc_shard(rank, world)
    rows = (rank * h // world, (rank + 1) * h // world)
    out = {}
    for f in range(frames):
        _nrc_frame(O, oframe, onet, p, f, rows, seed_tile)
        out[f"beauty{f}"] = oframe.buffer(abi.BUF_BEAUTY_ACCUM)[rows[0]:rows[1]].copy()
        out[f"state{f}"] = oframe.linear_buffer(abi.BUF_NRC_STATE)[:8, 0].copy()
        out[f"records{f}"] = oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0).copy()
        out[f"targets{f}"] = oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0).copy()
    out["weights"] = onet.get_master()
    np.savez(result_path + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()


def _nrc_strips_equal_single_process(tmp_path, scene_name, w, h, frames, seed_tile=None):
    """runs the frames sharded over two ranks and unsharded, asserts they agree and returns the unsharded state words"""
    from gfxexp_b200 import abi
    result = str(tmp_path / "nrc")
    mp.spawn(_worker_nrc, args=(2, _free_port(), result, scene_name, w, h, frames, seed_tile), nprocs=2, join=True)
    O, oframe, onet, p = _nrc_setup(scene_name, w, h)
    got = [np.load(result + f".{r}.npz") for r in range(2)]
    states = []
    for f in range(frames):
        _nrc_frame(O, oframe, onet, p, f, seed_tile=seed_tile)
        st = oframe.linear_buffer(abi.BUF_NRC_STATE)[:8, 0]
        states.append(st)
        ntrain = min(int(st[f % 2]), abi.NRC_TRAIN_BUFFER_SIZE)
        assert ntrain > 30, "vacuous: no training vertices"
        beauty = oframe.buffer(abi.BUF_BEAUTY_ACCUM)
        for r in range(2):
            rows = slice(r * h // 2, (r + 1) * h // 2)
            assert np.array_equal(got[r][f"beauty{f}"].view(np.uint32), beauty[rows].view(np.uint32)), f"frame {f} rank {r}: image"
            assert np.array_equal(got[r][f"state{f}"], st), f"frame {f} rank {r}: counters / tile sizes"
            assert np.array_equal(got[r][f"records{f}"][:ntrain].view(np.uint32),
                                  oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain].view(np.uint32)), f"frame {f} rank {r}: records"
            assert np.array_equal(got[r][f"targets{f}"][:ntrain].view(np.uint32),
                                  oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain].view(np.uint32)), f"frame {f} rank {r}: targets"
    want = onet.get_master()
    for r in range(2):
        assert np.array_equal(got[r]["weights"].view(np.uint32), want.view(np.uint32)), f"rank {r}: trained weights"
    return states


def test_nrc_strips_equal_single_process(tmp_path):
    """the numbering of the training vertices over the ranks (one count per rank and commit round exchanged), the merge of the
    records and the replicated training reproduce the unsharded frame bit for bit: images, counters and tile sizes, all
    records, the trained weights of both ranks"""
    _nrc_strips_equal_single_process(tmp_path, "tiny_city_scene", NRC_W, NRC_H, NRC_FRAMES)


def test_nrc_strips_equal_single_process_past_the_buffer(tmp_path):
    """the same with small_city_scene at 1920x1080 and 4x4 tiles: the ranks number their vertices past the 131 072 records, each drops its own and
    ends those suffixes with a query, and the next frame's controller acts on the count past the buffer"""
    from gfxexp_b200 import abi
    states = _nrc_strips_equal_single_process(tmp_path, "small_city_scene", 1920, 1080, 2, seed_tile=4)
    assert states[0][0] > abi.NRC_TRAIN_BUFFER_SIZE and tuple(states[0][2:4]) == (4, 4), states[0]
    assert tuple(states[1][4:6]) == (7, 7), states[1]
