"""ReSTIR DI + NRC as one estimator on the GPU (GFX_PT_NRC_INDIRECT, the additive gfx_nrc_accumulate, StripDriver(combined=True),
gfx_headless restir_nrc):

  the combined frame is bit-exact to the CPU oracle (tests/oracle_restir_nrc.py): image, path-tracer outputs, training records
  before and after the propagation, shuffled records, state block
  its training data and the weights trained on them are those of the old frame (combined=False), at 1920x1080 too
  strips without gfx_nrc_shard are refused as for GFX_PT_NRC
  gfx_stats_read's ray count drops by exactly the shadow rays of the non-training primary hits that the oracle counts
  StripDriver(combined=True) is the frame of the context-level launches, on 1 GPU and (skipped otherwise) on 2
  the C++ host's restir_nrc renderer equals the Python host"""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, multigpu, scenes
from tests import oracle_restir_nrc as RN
from tests import test_gpu_nrc_frame as NRC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")
W, H = 160, 96
HASH, TRI = abi.NRC_POSITION_ENCODING_HASH_GRID, abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE


def _same(got, want, tag):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    g = g.view(np.uint32) if g.dtype.itemsize == 4 else g
    w = w.view(np.uint32) if w.dtype.itemsize == 4 else w
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first {bad[:4].tolist()}")


def _state(words):
    """the state block without the target averages, which the shuffle sums with float atomics in no fixed order (they only
    feed a display), and without the last word, the strip launch size, which the oracle does not keep"""
    w = np.array(words[:abi.NRC_STATE_NUM_INFERENCE_QUERIES + 1])
    w[abi.NRC_STATE_TARGET_AVG:abi.NRC_STATE_TARGET_AVG + 6] = 0
    return w


def _offsets(f):
    rng = np.random.default_rng(2000 + f)
    return [int(rng.integers(0, 2 ** 32)) for _ in range(2)]


def _net(ctx, encoding):
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2, position_encoding=encoding)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, grid_amplitude=0.1, seed=31))
    return net


def _setup(ctx, scene, w, h, bump):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 5
    p.radianceScale = 2.0
    p.enableBumpMapping = 1 if bump else 0
    return p


def _context_frame(ctx, net, p, f, unbiased, variant, train=True):
    """one ReSTIR DI + NRC frame through the context's launches (the single-GPU frame of StripDriver.render_restir_nrc_frame)"""
    ctx.build_light_distributions(f % 2)
    for kind, pid in engine.restir_frame_passes(p, f, 1, True, unbiased):
        ctx.gbuffer(p) if kind == "gbuffer" else ctx.restir(p, pid)
    off = _offsets(f)
    ctx.nrc_preprocess(p, off[0], off[1], f == 0)
    ctx.pathtrace(p, variant)
    ctx.nrc_frame_infer(net)
    ctx.nrc_accumulate(p)
    if train:
        ctx.nrc_propagate(p)
        ctx.nrc_shuffle(p)
        ctx.nrc_frame_train(net)


SCENES = {"city": scenes.small_city_scene, "city_env": scenes.small_city_scene_env, "city_bumped": scenes.small_city_scene_bumped}


@pytest.mark.parametrize("scene_name,bump,unbiased,encoding", [
    ("city", False, False, HASH), ("city", False, True, TRI), ("city_env", False, True, HASH), ("city_env", False, False, TRI),
    ("city_bumped", True, False, HASH), ("city_bumped", True, True, HASH)])
def test_combined_frames_bit_exact_to_oracle(gfx_ctx, scene_name, bump, unbiased, encoding):
    scene = SCENES[scene_name]()
    p = _setup(gfx_ctx, scene, W, H, bump)
    oframe = RN.OracleFrame(RN.OracleScene(scene), W, H)
    net = _net(gfx_ctx, encoding)
    for f in range(4):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, unbiased):
            if kind == "gbuffer":
                gfx_ctx.gbuffer(p)
                oframe.gbuffer(p)
            else:
                gfx_ctx.restir(p, pid)
                oframe.restir(p, pid)
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} ReSTIR DI beauty")
        off = _offsets(f)
        gfx_ctx.nrc_preprocess(p, off[0], off[1], f == 0)
        oframe.nrc_preprocess(p, off[0], off[1], f == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC_INDIRECT)
        oframe.pathtrace(p, abi.PT_NRC_INDIRECT)
        ntrain, _, _ = NRC._compare_pathtrace(gfx_ctx, oframe, p, f"frame {f}")
        _same(_state(gfx_ctx.download_linear(abi.BUF_NRC_STATE)), _state(oframe.linear_buffer(abi.BUF_NRC_STATE)), f"frame {f} state")
        gfx_ctx.nrc_frame_infer(net)
        oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:] = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        gfx_ctx.nrc_accumulate(p)
        oframe.nrc_accumulate(p)
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} combined beauty")
        gfx_ctx.nrc_propagate(p)
        oframe.nrc_propagate(p)
        _same(gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain],
              f"frame {f} propagated targets")
        gfx_ctx.nrc_shuffle(p)
        oframe.nrc_shuffle(p)
        for buf in (abi.BUF_NRC_TRAIN_QUERY, abi.BUF_NRC_TRAIN_TARGET):
            _same(gfx_ctx.download_linear(buf, 1), oframe.linear_buffer(buf, 1), f"frame {f} shuffled {buf}")
        gfx_ctx.nrc_frame_train(net)
    beauty = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3]
    assert np.isfinite(beauty).all() and beauty.mean() > 1e-3
    net.close()


def _frames(ctx, scene, w, h, variant, frames, unbiased=False, encoding=HASH):
    """the images, the training data of the last frame and the trained master weights of `frames` context-level frames"""
    p = _setup(ctx, scene, w, h, False)
    net = _net(ctx, encoding)
    images = []
    for f in range(frames):
        p.numAccumFrames = f
        _context_frame(ctx, net, p, f, unbiased, variant, train=False)
        ntrain = min(int(ctx.download_linear(abi.BUF_NRC_STATE)[p.bufferIndex, 0]), abi.NRC_TRAIN_BUFFER_SIZE)
        data = {"state": _state(ctx.download_linear(abi.BUF_NRC_STATE)), "rng": ctx.download(abi.BUF_RNG),
                "terminal info": ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO),
                "suffix terminals": ctx.download_linear(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL),
                "vertex infos": ctx.download_linear(abi.BUF_NRC_TRAIN_VERTEX_INFO)[:ntrain],
                "train queries": ctx.download_linear(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain],
                "train targets": ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain]}
        ctx.nrc_propagate(p)
        ctx.nrc_shuffle(p)
        ctx.nrc_frame_train(net)
        images.append(ctx.download(abi.BUF_BEAUTY_ACCUM))
    weights = net.read(abi.NRC_READ_MASTER)
    net.close()
    return images, data, weights


@pytest.mark.parametrize("w,h", [(W, H), (1920, 1080)])
def test_same_training_data_and_weights_as_the_old_frame(gfx_ctx, w, h):
    scene = scenes.small_city_scene()
    frames = 4 if w == W else 2
    old_images, old, old_weights = _frames(gfx_ctx, scene, w, h, abi.PT_NRC, frames)
    new_images, new, new_weights = _frames(gfx_ctx, scene, w, h, abi.PT_NRC_INDIRECT, frames)
    for k in old:
        _same(new[k], old[k], f"{w}x{h} {k}")
    _same(new_weights, old_weights, f"{w}x{h} trained master weights")
    assert not np.array_equal(new_images[-1].view(np.uint32), old_images[-1].view(np.uint32))


def test_strips_without_shard_are_refused(gfx_ctx):
    scene = scenes.small_city_scene()
    p = _setup(gfx_ctx, scene, W, H, False)
    gfx_ctx.build_light_distributions(0)
    gfx_ctx.gbuffer(p)
    gfx_ctx.nrc_preprocess(p, 1, 2, True)
    p.tileOriginY, p.tileRows = 0, H // 2
    for variant, name in ((abi.PT_NRC, "GFX_PT_NRC)"), (abi.PT_NRC_INDIRECT, "GFX_PT_NRC_INDIRECT)")):
        with pytest.raises(Exception) as e:
            gfx_ctx.pathtrace(p, variant)
        assert name in str(e.value) and "strips need gfx_nrc_shard" in str(e.value), str(e.value)


def test_strip_driver_combined_is_the_context_frame(gfx_ctx):
    scene = scenes.small_city_scene()
    want, _, want_weights = _frames(gfx_ctx, scene, W, H, abi.PT_NRC_INDIRECT, 3)
    p = _setup(gfx_ctx, scene, W, H, False)
    net = _net(gfx_ctx, HASH)
    driver = multigpu.StripDriver(gfx_ctx, p, W, H, 0, 1)
    driver.enable_nrc(net, overlap_training=False)
    for f in range(3):
        p.numAccumFrames = f
        driver.render_restir_nrc_frame(f, _offsets(f), combined=True)
        gfx_ctx.synchronize()
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), want[f], f"frame {f} StripDriver(combined=True) beauty")
    _same(net.read(abi.NRC_READ_MASTER), want_weights, "trained master weights")
    net.close()


W2, H2, FRAMES2 = 320, 192, 3


def _worker(rank, world, port, result_path):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    scene = scenes.small_city_scene()
    ctx = engine.Context(rank)
    p = _setup(ctx, scene, W2, H2, False)
    net = _net(ctx, HASH)
    driver = multigpu.StripDriver(ctx, p, W2, H2, rank, world)
    driver.enable_nrc(net)
    outs = []
    for f in range(FRAMES2):
        p.numAccumFrames = f
        driver.render_restir_nrc_frame(f, _offsets(f), combined=True)
        torch.cuda.synchronize()
        outs.append(driver.composited.cpu().numpy().copy())
    driver.wait_training()
    np.save(result_path + f".weights.{rank}.npy", net.read(abi.NRC_READ_MASTER))
    if rank == 0:
        np.save(result_path + ".frames.npy", np.stack(outs))
    dist.barrier()
    net.close()
    driver.comm.close()
    dist.destroy_process_group()
    ctx.close()


def test_combined_strips_on_two_gpus_equal_one(tmp_path, gfx_ctx):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    result = str(tmp_path / "restir_nrc")
    mp.spawn(_worker, args=(2, port, result), nprocs=2, join=True)
    got = np.load(result + ".frames.npy")
    want, _, want_weights = _frames(gfx_ctx, scenes.small_city_scene(), W2, H2, abi.PT_NRC_INDIRECT, FRAMES2)
    for f in range(FRAMES2):
        _same(got[f].reshape(-1), want[f].reshape(-1), f"frame {f}: 2-GPU combined frame")
    for rank in range(2):
        _same(np.load(result + f".weights.{rank}.npy"), want_weights, f"rank {rank} weights")


@pytest.mark.parametrize("renderer", ["restir_nrc", "restir_nrc_unbiased"])
def test_cpp_host_matches_python_host(gfx_ctx, tmp_path, renderer):
    w, h, frames = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path, out_path, params_path = (str(tmp_path / n) for n in ("scene.bin", "out.raw", "nrc.f16"))
    scenes.save_scene_bin(scene, scene_path, w, h)
    probe = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    params = engine.random_nrc_params(probe.num_params, 64 * 64 * 2 + 16 * 64, grid_amplitude=0.1)
    probe.close()
    params.tofile(params_path)
    res = subprocess.run([HOST, scene_path, renderer, str(w), str(h), str(frames), out_path, params_path],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    assert json.loads(res.stdout.strip().splitlines()[-1])["renderer"] == renderer
    got = np.fromfile(out_path, dtype=np.float32).reshape(h, w, 4)

    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    p = abi.default_frame_params(scene, w, h)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    net.set_params(params)
    rs = np.random.RandomState(72139121)  # std::mt19937 perFrameRng(72139121)
    for f in range(frames):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, renderer.endswith("unbiased")):
            gfx_ctx.gbuffer(p) if kind == "gbuffer" else gfx_ctx.restir(p, pid)
        off = [int(v) for v in rs.randint(0, 2 ** 32, size=2, dtype=np.uint64)]
        gfx_ctx.nrc_preprocess(p, off[0], off[1], f == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC_INDIRECT)
        gfx_ctx.nrc_frame_infer(net)
        gfx_ctx.nrc_accumulate(p)
        gfx_ctx.nrc_propagate(p)
        gfx_ctx.nrc_shuffle(p)
        gfx_ctx.nrc_frame_train(net)
    want = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)
    net.close()
    _same(got, want, f"{renderer}: C++ host image")
    assert np.isfinite(got).all() and got[..., :3].mean() > 1e-4


@pytest.mark.parametrize("scene_name,bump", [("city", False), ("city_env", False), ("city_bumped", True)])
def test_rays_counter_drops_by_the_skipped_shadow_rays(gfx_ctx, scene_name, bump):
    """the work the variant saves: from the same state, gfx_stats_read's ray count of GFX_PT_NRC_INDIRECT is GFX_PT_NRC's less
    one shadow ray per non-training primary hit whose light sample contributes (the oracle counts those pixels)"""
    scene = SCENES[scene_name]()
    rays = {}
    for variant in (abi.PT_NRC, abi.PT_NRC_INDIRECT):
        p = _setup(gfx_ctx, scene, W, H, bump)
        gfx_ctx.build_light_distributions(0)
        gfx_ctx.gbuffer(p)
        gfx_ctx.nrc_preprocess(p, 1234, 5678, True)
        gfx_ctx.synchronize()
        gfx_ctx.read_stats(reset=True)
        gfx_ctx.pathtrace(p, variant)
        gfx_ctx.synchronize()
        rays[variant] = gfx_ctx.read_stats(reset=True)[0]
    oframe = RN.OracleFrame(RN.OracleScene(scene), W, H)
    oframe.gbuffer(p)
    oframe.nrc_preprocess(p, 1234, 5678, True)
    oframe.pathtrace(p, abi.PT_NRC_INDIRECT)
    skipped = oframe.skipped_contributing_shadow_rays
    assert skipped > W * H // 8
    assert rays[abi.PT_NRC] - rays[abi.PT_NRC_INDIRECT] == skipped, (rays, skipped)
