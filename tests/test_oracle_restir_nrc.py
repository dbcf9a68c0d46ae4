"""ReSTIR DI + NRC as one estimator (GFX_PT_NRC_INDIRECT and the additive gfx_nrc_accumulate) on the CPU oracle
(tests/oracle_restir_nrc.py):

  the indirect-only path tracer follows GFX_PT_NRC's paths and writes its training data bit for bit - records, state block,
  inference queries, terminal infos, RNG, shuffled records - so the cache learns what it learns in the old frame
  it traces one shadow ray fewer per non-training primary hit that drew a light sample, and no other ray fewer
  on a plane under a uniform environment every bounce ray escapes and its environment term belongs to ReSTIR DI: the combined
  frame's beauty is the DI-only beauty, bit for bit
  with fixed network weights it estimates what GFX_PT_NRC estimates (Student-t bars over repeats, with negative controls)
  with the indirect switch off the restatement is the bump oracle's GFX_PT_NRC, bit for bit
  sharded over two ranks (gloo) it equals the unsharded frame"""
import os
import sys

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_lib
from tests import oracle_restir_nrc as RN
from tests.test_gpu_furnace import _furnace_scene

W, H = 96, 64


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype.itemsize == 4 else a


def _same(a, b, tag):
    ga, gb = _bits(a), _bits(b)
    if not np.array_equal(ga, gb):
        bad = np.argwhere(ga != gb)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first {bad[:4].tolist()}")


SCENES = {"city": scenes.small_city_scene, "city_env": scenes.small_city_scene_env, "city_bumped": scenes.small_city_scene_bumped}
_scene_cache = {}


def _oscene(name):
    if name not in _scene_cache:
        scene = SCENES[name]()
        _scene_cache[name] = (scene, RN.OracleScene(scene))
    return _scene_cache[name]


def _params(scene, max_path_length, bump):
    p = abi.default_frame_params(scene, W, H)
    p.maxPathLength = max_path_length
    p.enableBumpMapping = 1 if bump else 0
    p.radianceScale = 2.0
    return p


def _training_data(of, p):
    """everything the frame hands to the cache's training and to the inference, in bits"""
    n = W * H
    ti = of.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    q = of.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
    suffix = of.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL)
    has_query = (ti[:, 3] & 1).astype(bool)
    suffix_query = ((suffix[:, 0] >> 23) & 1).astype(bool)
    ntrain = min(int(of.linear_buffer(abi.BUF_NRC_STATE)[p.bufferIndex, 0]), abi.NRC_TRAIN_BUFFER_SIZE)
    return {
        "state": of.linear_buffer(abi.BUF_NRC_STATE),
        "rng": of.buffer(abi.BUF_RNG),
        "terminal info": ti,
        "pixel queries": q[:n][has_query],
        "suffix terminals": suffix,
        "suffix queries": q[n:n + len(suffix)][suffix_query],
        "train queries": of.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain],
        "train targets": of.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain],
        "vertex infos": of.linear_buffer(abi.BUF_NRC_TRAIN_VERTEX_INFO)[:ntrain],
    }


@pytest.mark.parametrize("scene_name,bump", [("city", False), ("city_env", False), ("city_bumped", True), ("city_bumped", False)])
@pytest.mark.parametrize("max_path_length", [2, 5, 0])
def test_same_paths_and_training_data(scene_name, bump, max_path_length):
    scene, oscene = _oscene(scene_name)
    p = _params(scene, max_path_length, bump)
    frames = {v: RN.OracleFrame(oscene, W, H) for v in (abi.PT_NRC, abi.PT_NRC_INDIRECT)}
    rng = np.random.default_rng(5)
    for f in range(2):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, f
        offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
        rays, data = {}, {}
        for v, of in frames.items():
            of.gbuffer(p)
            of.nrc_preprocess(p, offsets[0], offsets[1], f == 0)
            rays[v] = of.pathtrace(p, v)
            data[v] = _training_data(of, p)
        for k in data[abi.PT_NRC]:
            _same(data[abi.PT_NRC_INDIRECT][k], data[abi.PT_NRC][k], f"frame {f} {k}")
        # the rays: GFX_PT_NRC traces no ray the indirect variant skips, the indirect variant skips one shadow ray per
        # non-training primary hit that drew a light sample
        assert frames[abi.PT_NRC].skipped_shadow_rays == 0
        skipped = frames[abi.PT_NRC_INDIRECT].skipped_shadow_rays
        assert skipped > W * H // 4
        assert rays[abi.PT_NRC_INDIRECT] == rays[abi.PT_NRC] - skipped
        for v, of in frames.items():
            of.nrc_propagate(p)
            of.nrc_shuffle(p)
        for buf in (abi.BUF_NRC_TRAIN_QUERY, abi.BUF_NRC_TRAIN_TARGET):
            _same(frames[abi.PT_NRC_INDIRECT].linear_buffer(buf, 1), frames[abi.PT_NRC].linear_buffer(buf, 1), f"frame {f} shuffled {buf}")
        _same(frames[abi.PT_NRC_INDIRECT].linear_buffer(abi.BUF_NRC_STATE), frames[abi.PT_NRC].linear_buffer(abi.BUF_NRC_STATE),
              f"frame {f} state after the shuffle")
    # the rendering radiance differs: the indirect variant leaves out the primary vertex's direct light
    c1 = frames[abi.PT_NRC].linear_buffer(abi.BUF_NRC_FRAME_CONTRIBUTION)
    c5 = frames[abi.PT_NRC_INDIRECT].linear_buffer(abi.BUF_NRC_FRAME_CONTRIBUTION)
    assert np.isfinite(c5).all() and c5.sum() < c1[np.isfinite(c1).all(axis=1)].sum()


def test_one_training_step_sees_the_same_records():
    """the network after one training step on each variant's shuffled records: the same master weights"""
    scene, oscene = _oscene("city")
    p = _params(scene, 5, False)
    nets = {}
    for v in (abi.PT_NRC, abi.PT_NRC_INDIRECT):
        of = RN.OracleFrame(oscene, W, H)
        of.gbuffer(p)
        of.nrc_preprocess(p, 123, 456, True)
        of.pathtrace(p, v)
        of.nrc_propagate(p)
        of.nrc_shuffle(p)
        net = oracle_lib.OracleNrc(2, 1e-2)
        params = engine.random_nrc_params(net.num_params, net.num_matrix_weights, grid_amplitude=0.1)
        net.set_params(params)
        batch = abi.NRC_TRAIN_BUFFER_SIZE // 8   # one of the four training steps' quarters of the 65536 shuffled records
        net.train(of.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 1)[:batch], of.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 1)[:batch])
        nets[v] = net.get_master()
    _same(nets[abi.PT_NRC_INDIRECT], nets[abi.PT_NRC], "master weights")


@pytest.mark.parametrize("unbiased", [False, True])
def test_furnace_combined_frame_is_the_di_frame(unbiased):
    """a plane under a uniform environment: the bounce rays all escape, their environment term is ReSTIR DI's, so the
    indirect-only radiance is 0 and the combined beauty is the DI beauty, bit for bit"""
    scene = _furnace_scene((scenes.BSDF_LAMBERT, 0.8, 0.8, 0.8), -28.0)
    oscene = RN.OracleScene(scene)
    p = abi.default_frame_params(scene, W, H)
    p.enableEnvLight, p.envLightPowerCoeff, p.maxPathLength = 1, 1.5, 5
    di, combined = RN.OracleFrame(oscene, W, H), RN.OracleFrame(oscene, W, H)
    for f in range(3):
        p.numAccumFrames = f
        for of in (di, combined):
            for kind, pid in engine.restir_frame_passes(p, f, 1, True, unbiased):
                if kind == "gbuffer":
                    of.gbuffer(p)
                else:
                    of.restir(p, pid)
        combined.nrc_preprocess(p, 7 * f, 11 * f, f == 0)
        combined.pathtrace(p, abi.PT_NRC_INDIRECT)
        assert not combined.linear_buffer(abi.BUF_NRC_FRAME_CONTRIBUTION).any()
        assert not (combined.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)[:, 3] & 1).any()
        combined.nrc_accumulate(p)
        _same(combined.buffer(abi.BUF_BEAUTY_ACCUM), di.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} beauty")
        di.buffer(abi.BUF_RNG, copy=False)[:] = combined.buffer(abi.BUF_RNG)  # the NRC paths drew from the pixels' RNGs
    assert di.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3].mean() > 0.1


def test_pt_nrc_is_the_bump_oracles_restatement():
    """the indirect switch sits in a copy of the bump oracle's NRC path tracer: with it off, the copy must stay that path
    tracer, bit for bit (every buffer the frame writes, with and without bump mapping)"""
    scene, oscene = _oscene("city_bumped")
    for bump in (False, True):
        p = _params(scene, 5, bump)
        a, b = RN.OracleFrame(oscene, W, H), RN.OracleFrame(oscene, W, H)
        for f in range(2):
            p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, f
            for of in (a, b):
                of.gbuffer(p)
                of.nrc_preprocess(p, 17 + f, 29 * f, f == 0)
            rays_a = a.pathtrace(p, abi.PT_NRC)
            rays_b = b.bump_pathtrace_nrc(p)
            assert rays_a == rays_b
            for buf in (abi.BUF_NRC_FRAME_CONTRIBUTION, abi.BUF_NRC_TERMINAL_INFO, abi.BUF_NRC_INFERENCE_QUERY,
                        abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL, abi.BUF_NRC_TRAIN_VERTEX_INFO, abi.BUF_NRC_STATE):
                _same(a.linear_buffer(buf), b.linear_buffer(buf), f"bump {bump} frame {f} buffer {buf}")
            for buf in (abi.BUF_NRC_TRAIN_QUERY, abi.BUF_NRC_TRAIN_TARGET):
                _same(a.linear_buffer(buf, 0), b.linear_buffer(buf, 0), f"bump {bump} frame {f} buffer {buf}")
            _same(a.buffer(abi.BUF_RNG), b.buffer(abi.BUF_RNG), f"bump {bump} frame {f} rng")


# ---- unbiasedness: the combined frame estimates what GFX_PT_NRC estimates ---------------------------------------------------
UW, UH, REPEATS = 96, 64, 16
FALSE_ALARM = 1e-4   # two-sided, per class and colour channel


def _one_bounce_scene(env: bool):
    """a floor, a red wall behind it and a 3 x 3 emitter 1.6 above the floor facing down: the floor and the wall see the emitter
    directly and each other's light after one bounce, and BSDF samples from both hit the emitter (the implicit terms of path
    length 2 that the combined frame leaves to ReSTIR DI)"""
    mats = np.zeros(3, dtype=scenes.MATERIAL_DTYPE)
    mats["bsdfType"] = scenes.BSDF_LAMBERT
    mats[0]["p0"] = (0.85, 0.85, 0.85)
    mats[1]["p0"] = (0.9, 0.35, 0.2)
    mats[2]["emittance"] = (6.0, 6.0, 5.0)
    mats[2]["hasEmittance"] = 1
    floor = scenes.make_plane(1, 8.0, 0)
    wall = scenes.make_plane(1, 8.0, 1)
    light = scenes.make_quad_light(3.0, 2)
    instances = [scenes.make_instance([0]), scenes.make_instance([1], translate=(0.0, 4.0, -3.0), pitch_deg=90.0),
                 scenes.make_instance([2], translate=(0.5, 1.6, -1.0))]
    eye, target = np.array([0.0, 2.2, 4.5]), np.array([0.0, 0.6, -2.0])
    scene = scenes.Scene([floor, wall, light], mats, instances, eye.astype(np.float32), scenes.look_at_orientation(eye, target),
                         np.radians(60.0), "one_bounce")
    if env:
        sky = np.ones((16, 32, 4), dtype=np.float32)
        sky[..., :3] = (0.2, 0.25, 0.35)
        scene.env_map = sky
    return scene


def _infer(of, net):
    """the fixed cache's predictions of this frame's pixel queries"""
    n = of.W * of.H
    ti = of.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    idx = np.flatnonzero((ti[:n, 3] & 1).astype(bool))
    if len(idx):
        q = of.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
        of.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[idx] = net.infer(q[idx])


def _estimates(oscene, net, scene, seed):
    """one repeat from fresh RNG states: the images of the combined frame, of GFX_PT_NRC, of ReSTIR DI alone and of the old
    mixture (frame 1 of the old frame), and the pixel classes (G-buffer instance slot; -1 for a miss)"""
    p = abi.default_frame_params(scene, UW, UH)
    p.maxPathLength = 5
    p.radianceScale = 2.0
    offsets = [[int(v) for v in np.random.default_rng(seed + f).integers(0, 2 ** 32, 2)] for f in range(2)]

    def restir(of, f):
        p.numAccumFrames = f
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, True):
            of.gbuffer(p) if kind == "gbuffer" else of.restir(p, pid)

    def nrc(of, f, variant):
        of.nrc_preprocess(p, offsets[f][0], offsets[f][1], f == 0)
        of.pathtrace(p, variant)
        _infer(of, net)
        of.nrc_accumulate(p)

    out = {}
    of = RN.OracleFrame(oscene, UW, UH, seed=seed)
    restir(of, 0)
    out["D"] = of.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3]
    nrc(of, 0, abi.PT_NRC_INDIRECT)
    out["combined"] = of.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3]
    cls = of.buffer(abi.BUF_GBUFFER0, 0)[..., 0].astype(np.int64)
    cls[cls == 0xFFFFFFFF] = -1
    of = RN.OracleFrame(oscene, UW, UH, seed=seed + 1)
    p.frameIndex, p.bufferIndex, p.numAccumFrames = 0, 0, 0
    of.gbuffer(p)
    nrc(of, 0, abi.PT_NRC)
    out["N"] = of.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3]
    of = RN.OracleFrame(oscene, UW, UH, seed=seed + 2)
    for f in range(2):
        restir(of, f)
        nrc(of, f, abi.PT_NRC)
    out["old mixture"] = of.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3]
    return out, cls


def _welch(a, b):
    """|mean a - mean b| in standard errors per class and channel ([R, classes, 3] each), and the Student-t bound"""
    from scipy import stats
    r = a.shape[0]
    se = np.sqrt(a.var(0, ddof=1) / r + b.var(0, ddof=1) / r)
    return np.abs(a.mean(0) - b.mean(0)) / np.maximum(se, 1e-12), stats.t.ppf(1 - FALSE_ALARM / 2, 2 * r - 2)


@pytest.mark.parametrize("env", [False, True])
def test_combined_frame_is_unbiased(env):
    """With fixed network weights and unbiased ReSTIR DI, the combined frame D + I and GFX_PT_NRC's frame N estimate the same
    pixel values: per class of pixels (floor, wall, emitter), their frame means over 16 repeats with fresh RNG states agree within
    Student-t bars.  Negative controls fail the same bound: N + D counts the direct light twice, and the old frame's image after
    two frames, (1 - w)^2 N_0 + w (1 - w) D_1 + w N_1, weighs the indirect light by 3/4."""
    scene = _one_bounce_scene(env)
    oscene = RN.OracleScene(scene)
    net = oracle_lib.OracleNrc(2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, net.num_matrix_weights, seed=3, grid_amplitude=0.1))
    means = {k: [] for k in ("combined", "N", "N + D", "old mixture")}
    for r in range(REPEATS):
        est, cls = _estimates(oscene, net, scene, 9000 + 10 * r)
        est["N + D"] = est["N"] + est["D"]
        classes = [c for c in range(len(scene.instances)) if (cls == c).sum() >= 20]
        for k in means:
            means[k].append([est[k][cls == c].mean(0) for c in classes])
    means = {k: np.array(v, dtype=np.float64) for k, v in means.items()}
    assert len(classes) >= 2
    z, bound = _welch(means["combined"], means["N"])
    assert (z < bound).all(), f"combined against GFX_PT_NRC: {z} standard errors, bound {bound:.2f}; means " \
                              f"{means['combined'].mean(0)} against {means['N'].mean(0)}"
    for control in ("N + D", "old mixture"):
        z, bound = _welch(means[control], means["N"])
        assert (z > bound).any(), f"the negative control {control} passes: {z} standard errors, bound {bound:.2f}"


# ---- the combined frame sharded by strips (the oracle's restatement of gfx_nrc_shard), world_size 2 over gloo ---------------
SW, SH, SFRAMES = 64, 48, 3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _strip_setup():
    scene = scenes.tiny_city_scene()
    of = RN.OracleFrame(RN.OracleScene(scene), SW, SH)
    net = oracle_lib.OracleNrc(2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, net.num_matrix_weights, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, SW, SH)
    p.maxPathLength = 4
    p.radianceScale = 2.0
    return of, net, p


def _strip_frame(of, net, p, f, rows=None):
    """one combined frame: the ReSTIR DI passes on the whole frame (every rank computes the same), then GFX_PT_NRC_INDIRECT, the
    inference of this rank's rows and the additive accumulation on `rows` = (y0, y1), propagation, shuffle and 4 training
    steps"""
    rng = np.random.default_rng(700 + f)
    offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
    p.tileOriginY, p.tileRows = 0, 0
    p.numAccumFrames = f
    for kind, pid in engine.restir_frame_passes(p, f, 1, True, False):
        of.gbuffer(p, 2) if kind == "gbuffer" else of.restir(p, pid, 2)
    if rows is not None:
        p.tileOriginY, p.tileRows = rows[0], rows[1] - rows[0]
    of.nrc_preprocess(p, offsets[0], offsets[1], f == 0)
    of.pathtrace(p, abi.PT_NRC_INDIRECT, 2)
    n = SW * SH
    q = of.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
    ti = of.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    suffix = of.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL)[:, 0]
    lo, hi = (rows[0] * SW, rows[1] * SW) if rows is not None else (0, n)
    idx = np.concatenate([lo + np.flatnonzero((ti[lo:hi, 3] & 1).astype(bool)), n + np.flatnonzero(((suffix >> 23) & 1).astype(bool))])
    if len(idx):
        of.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[idx] = net.infer(q[idx])
    of.nrc_accumulate(p)
    of.nrc_propagate(p)
    of.nrc_shuffle(p)
    tq, tt = of.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 1), of.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 1)
    for step in range(4):
        net.train(tq[step * 16384:(step + 1) * 16384], tt[step * 16384:(step + 1) * 16384])
    p.tileOriginY, p.tileRows = 0, 0


def _strip_worker(rank, world, port, result_path):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    of, net, p = _strip_setup()
    of.nrc_shard(rank, world)
    rows = (rank * SH // world, (rank + 1) * SH // world)
    out = {}
    for f in range(SFRAMES):
        _strip_frame(of, net, p, f, rows)
        # the next frame's ReSTIR DI passes run on the whole frame: every rank takes the other strips' RNG states, which only
        # their own path tracer advanced
        import torch
        rng_state = of.buffer(abi.BUF_RNG, copy=False)
        mine = torch.from_numpy(rng_state[rows[0]:rows[1]].view(np.int64).copy())
        strips = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(strips, mine)
        for r in range(world):
            rng_state[r * SH // world:(r + 1) * SH // world] = strips[r].numpy().view(np.uint64)
        out[f"beauty{f}"] = of.buffer(abi.BUF_BEAUTY_ACCUM)[rows[0]:rows[1]].copy()
        out[f"state{f}"] = of.linear_buffer(abi.BUF_NRC_STATE)[:8, 0].copy()
        out[f"targets{f}"] = of.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0).copy()
    out["weights"] = net.get_master()
    np.savez(result_path + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()


def test_combined_strips_equal_single_process(tmp_path):
    """GFX_PT_NRC_INDIRECT under gfx_nrc_shard: two ranks over gloo, each tracing and accumulating its strip, reproduce the
    unsharded combined frame bit for bit - images, counters and tile sizes, propagated records, trained weights"""
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    result = str(tmp_path / "combined")
    mp.spawn(_strip_worker, args=(2, port, result), nprocs=2, join=True)
    got = [np.load(result + f".{r}.npz") for r in range(2)]
    of, net, p = _strip_setup()
    for f in range(SFRAMES):
        _strip_frame(of, net, p, f)
        st = of.linear_buffer(abi.BUF_NRC_STATE)[:8, 0]
        ntrain = min(int(st[f % 2]), abi.NRC_TRAIN_BUFFER_SIZE)
        assert ntrain > 30, "vacuous: no training vertices"
        beauty = of.buffer(abi.BUF_BEAUTY_ACCUM)
        for r in range(2):
            rows = slice(r * SH // 2, (r + 1) * SH // 2)
            _same(got[r][f"beauty{f}"], beauty[rows], f"frame {f} rank {r}: image")
            _same(got[r][f"state{f}"], st, f"frame {f} rank {r}: counters / tile sizes")
            _same(got[r][f"targets{f}"][:ntrain], of.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], f"frame {f} rank {r}: targets")
    for r in range(2):
        _same(got[r]["weights"], net.get_master(), f"rank {r}: trained weights")
