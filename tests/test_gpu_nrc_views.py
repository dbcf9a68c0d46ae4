"""GPU parity of the NRC cache's "Directly Visualized Prediction" display (GFX_PT_NRC_VISUALIZE_PREDICTION, the reference's
visualizePrediction ray-gen + the W*H inference of neural_radiance_caching_main.cpp:2371-2387): the queries and terminal
infos equal the oracle's bit for bit, the inference covers exactly pad128(W*H) rows, running the display between frames
changes nothing an NRC sequence computes, the rejections, and the C++ host's `-view prediction` image."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, imageio, scenes
from tests import oracle_views as V

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")
SENTINEL = np.uint32(0x7FC0DEAD)  # a NaN no kernel produces


def _same(got, want, tag):
    g, w = np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32)
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first {bad[:4].tolist()}")


def _setup(ctx, scene, w, h, encoding=abi.NRC_POSITION_ENCODING_HASH_GRID):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2, position_encoding=encoding)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, seed=23, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, w, h)
    p.radianceScale = 2.0
    return net, p


def _offsets(f):
    rng = np.random.default_rng(500 + f)
    return [int(rng.integers(0, 2 ** 32)) for _ in range(2)]


def _sentinel_queries(ctx):
    q = ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)
    q.view(np.uint32)[:] = SENTINEL
    ctx.upload(abi.BUF_NRC_INFERENCE_QUERY, 0, q)


@pytest.mark.parametrize("w,h", [(192, 108), (1920, 1080)])
@pytest.mark.parametrize("scene_name", ["small_interior_scene", "small_city_scene_textured", "small_city_scene_env"])
def test_visualize_pass_matches_oracle(gfx_ctx, scene_name, w, h):
    scene = getattr(scenes, scene_name)()
    net, p = _setup(gfx_ctx, scene, w, h)
    oframe = V.ViewsFrame(scene, w, h)
    n = w * h
    misses = 0
    for f in range(2):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.nrc_frame(net, p, f, _offsets(f), train=True)   # a full NRC frame first
        _sentinel_queries(gfx_ctx)
        gfx_ctx.pathtrace(p, abi.PT_NRC_VISUALIZE_PREDICTION)
        oframe.gbuffer(p)
        oframe.nrc_visualize_prediction(p)
        ti_g = gfx_ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO)
        _same(ti_g, oframe.linear_buffer(abi.BUF_NRC_TERMINAL_INFO), f"frame {f} terminal info")
        hit = (ti_g[:, 3] & 1).astype(bool)
        assert np.array_equal(hit, gfx_ctx.download(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0].reshape(-1) != 0xFFFFFFFF)
        q_g = gfx_ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)
        _same(q_g[:n][hit], oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)[:n][hit], f"frame {f} queries of the hits")
        assert (q_g[:n][~hit].view(np.uint32) == SENTINEL).all(), "a miss row was written"
        assert (q_g[n:].view(np.uint32) == SENTINEL).all(), "a row past the pixels was written"
        st = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
        assert st[abi.NRC_STATE_NUM_INFERENCE_QUERIES] == (n + 127) // 128 * 128
        misses += int((~hit).sum())
    if scene_name == "small_city_scene_env":
        assert misses > 0
    net.close()


@pytest.mark.parametrize("encoding", [abi.NRC_POSITION_ENCODING_HASH_GRID, abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE])
@pytest.mark.parametrize("w,h", [(192, 108), (1920, 1080)])
def test_frame_infer_after_visualize_pass(gfx_ctx, encoding, w, h):
    """gfx_nrc_frame_infer after the pass predicts exactly pad128(W*H) rows, bit-identical to gfx_nrc_infer on them"""
    import torch
    net, p = _setup(gfx_ctx, scenes.small_city_scene_env(), w, h, encoding)
    gfx_ctx.build_light_distributions(0)
    gfx_ctx.nrc_frame(net, p, 0, _offsets(0), train=True)
    gfx_ctx.pathtrace(p, abi.PT_NRC_VISUALIZE_PREDICTION)
    capacity, count = abi.nrc_query_capacity(w, h), (w * h + 127) // 128 * 128
    sentinel = np.full((capacity, 3), SENTINEL, dtype=np.uint32).view(np.float32)
    gfx_ctx.upload(abi.BUF_NRC_INFERRED_RADIANCE, 0, sentinel)
    gfx_ctx.nrc_frame_infer(net)
    got = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
    _same(got[count:], sentinel[count:], "rows past pad128(W*H)")
    queries = torch.from_numpy(gfx_ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)[:count]).cuda()
    direct = torch.empty((count, 3), device="cuda")
    net.infer(queries, direct, count)
    torch.cuda.synchronize()
    _same(got[:count], direct.cpu().numpy(), "frame inference vs gfx_nrc_infer")
    net.close()


def test_visualization_leaves_the_sequence_unchanged(gfx_ctx):
    """four NRC frames with pass + inference + present after each give the bits of the same four frames without them"""
    scene = scenes.small_city_scene()
    w, h = 160, 96

    def run(with_views):
        net, p = _setup(gfx_ctx, scene, w, h)
        for f in range(4):
            p.numAccumFrames = f
            gfx_ctx.build_light_distributions(f % 2)
            gfx_ctx.nrc_frame(net, p, f, _offsets(f), train=True)
            if with_views:
                gfx_ctx.present(mode=abi.PRESENT_NRC_PATH_LENGTH, flags=abi.PRESENT_NRC_TRAINING_PATHS, frame_params=p)
                gfx_ctx.nrc_visualize_prediction(net, p)
                gfx_ctx.present(mode=abi.PRESENT_NRC_PREDICTION, frame_params=p)
        gfx_ctx.synchronize()
        out = {"beauty": gfx_ctx.download(abi.BUF_BEAUTY_ACCUM),
               "state": gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:8],
               "weights": net.read(abi.NRC_READ_MASTER)}
        for i in range(2):
            out[f"train query {i}"] = gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_QUERY, i)
            out[f"train target {i}"] = gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, i)
        out["vertex info"] = gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_VERTEX_INFO)
        net.close()
        return out

    plain, viewed = run(False), run(True)
    for k in plain:
        _same(viewed[k], plain[k], k)


def test_rejections(gfx_ctx):
    scene = scenes.tiny_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(64, 32)
    p = abi.default_frame_params(scene, 64, 32)
    gfx_ctx.gbuffer(p)
    lib, h = gfx_ctx.lib, gfx_ctx.h
    # no NRC buffers yet
    assert lib.gfx_pathtrace_launch(h, None, C.byref(p), abi.PT_NRC_VISUALIZE_PREDICTION) == -4
    for mode, flags in [(abi.PRESENT_NRC_PREDICTION, 0), (abi.PRESENT_NRC_PATH_LENGTH, 0), (abi.PRESENT_COLOR, abi.PRESENT_NRC_TRAINING_PATHS)]:
        pp = abi.GfxPresentParams(abi.BUF_BEAUTY_ACCUM, 0, mode, flags, 1.0, 1.0, C.pointer(p), 0.1, 0.5)
        assert lib.gfx_present_launch(h, None, C.byref(pp)) == -4, (mode, flags)
    # a new mode or flag without the frame parameters
    for mode, flags in [(abi.PRESENT_FLOW, 0), (abi.PRESENT_COLOR, abi.PRESENT_REGIR_CELLS), (abi.PRESENT_NRC_PREDICTION, 0),
                        (abi.PRESENT_NORMAL, abi.PRESENT_NRC_TRAINING_PATHS)]:
        pp = abi.GfxPresentParams(abi.BUF_BEAUTY_ACCUM, 0, mode, flags, 1.0, 1.0, None, 0.1, 0.5)
        assert lib.gfx_present_launch(h, None, C.byref(pp)) == -1, (mode, flags)
    pp = abi.GfxPresentParams(abi.BUF_BEAUTY_ACCUM, 0, 5, 0, 1.0, 1.0, C.pointer(p), 0.1, 0.5)
    assert lib.gfx_present_launch(h, None, C.byref(pp)) == -1
    # a sharded context: the handle is only stored by gfx_nrc_shard, and the pass refuses before any collective
    comm = C.c_uint64(0)
    assert lib.gfx_nrc_shard(h, C.addressof(comm), 0, 2) == 0
    assert lib.gfx_pathtrace_launch(h, None, C.byref(p), abi.PT_NRC_VISUALIZE_PREDICTION) == -6
    assert lib.gfx_nrc_shard(h, None, 0, 1) == 0
    assert lib.gfx_pathtrace_launch(h, None, C.byref(p), abi.PT_NRC_VISUALIZE_PREDICTION) == 0
    gfx_ctx.synchronize()


def test_cpp_host_prediction_view_matches_python_host(gfx_ctx, tmp_path):
    W, H, FRAMES = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path, png_path, params_path = (str(tmp_path / n) for n in ("scene.bin", "view.png", "nrc.f16"))
    scenes.save_scene_bin(scene, scene_path, W, H)
    params = engine.random_nrc_params(64 * 64 * 2 + 16 * 64 + 991232, 64 * 64 * 2 + 16 * 64, seed=41, grid_amplitude=0.1)
    params.tofile(params_path)
    res = subprocess.run([HOST, scene_path, "nrc", str(W), str(H), str(FRAMES), png_path, params_path, "-view", "prediction"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    got = imageio.read_png(png_path)

    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    net.set_params(params)
    rs = np.random.RandomState(72139121)  # std::mt19937 perFrameRng(72139121)
    for f in range(FRAMES):
        p.numAccumFrames = f
        p.resetFlowBuffer = 1 if f == 0 else 0
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.nrc_frame(net, p, f, [int(v) for v in rs.randint(0, 2 ** 32, size=2, dtype=np.uint64)], train=True)
    gfx_ctx.nrc_visualize_prediction(net, p)
    want = gfx_ctx.present(mode=abi.PRESENT_NRC_PREDICTION, frame_params=p)
    net.close()
    assert np.array_equal(got, want), "C++ host view differs from the Python host view"
    assert (want & 0xFFFFFF).any()
    # the views that do not apply to a renderer are refused
    res = subprocess.run([HOST, scene_path, "pathtrace", str(W), str(H), "1", png_path, "-view", "prediction"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 2 and "-view prediction" in res.stderr
