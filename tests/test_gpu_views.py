"""GPU parity of the debug views of gfx_present_launch (NRC prediction, rendering path length, motion vectors, training-path
tint, ReGIR cells): every mode and flag gives the RGBA8 image of the oracle's present fed the same device buffers, with and
without FLIP_Y; the existing COLOR / NORMAL modes are unaffected by the new fields."""
import ctypes as C

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_views as V

pytestmark = pytest.mark.gpu
TM = abi.PRESENT_TONE_MAP | abi.PRESENT_SRGB_GAMMA


def _inputs(ctx, p):
    b = p.bufferIndex
    return dict(terminal_info=ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO),
                inferred_radiance=ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE),
                inference_query=ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY),
                gbuffer1=ctx.download(abi.BUF_GBUFFER1, b), gbuffer2=ctx.download(abi.BUF_GBUFFER2, b).view(np.float32),
                rgba=ctx.download(abi.BUF_BEAUTY_ACCUM))


def _check(ctx, oracle, p, cases, tag):
    ins = _inputs(ctx, p)
    for mode, flags, brightness, alpha in cases:
        for flip in (0, abi.PRESENT_FLIP_Y):
            got = ctx.present(abi.BUF_BEAUTY_ACCUM, 0, mode, flags | flip, brightness, alpha, frame_params=p,
                              motion_vector_scale=0.1, motion_vector_offset=0.5)
            want = V.present_views(p, mode, flags | flip, brightness_scale=brightness, alpha_override=alpha,
                                        motion_vector_scale=0.1, motion_vector_offset=0.5, **ins)
            bad = np.argwhere(got != want)
            assert len(bad) == 0, f"{tag}: mode {mode} flags {flags | flip}: {len(bad)} pixels differ, first {bad[:3].tolist()}"
            assert (got != 0).any()


@pytest.mark.parametrize("w,h", [(1920, 1080), (100, 37)])
def test_views_bit_exact(gfx_ctx, oracle, w, h):
    scene = scenes.small_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, seed=5, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, w, h)
    p.radianceScale = 2.0
    p.regirGridDim[:] = [0, 0, 0]
    for f in range(2):
        p.numAccumFrames = f
        p.resetFlowBuffer = 1 if f == 0 else 0
        if f == 1:  # a moving camera
            p.prevCamera = p.camera
            cam = abi.GfxCamera.from_buffer_copy(p.camera)
            cam.position[0] += 0.4
            cam.position[2] -= 0.3
            p.camera = cam
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.nrc_frame(net, p, f, [0x2545F491 + f, 0x9E3779B9 * (f + 1) & 0xFFFFFFFF], train=True)
    gfx_ctx.synchronize()
    assert (gfx_ctx.download(abi.BUF_GBUFFER1, p.bufferIndex) != 0).any()
    after_frame = [(abi.PRESENT_NRC_PATH_LENGTH, 0, 1.0, 1.0), (abi.PRESENT_NRC_PATH_LENGTH, TM | abi.PRESENT_NRC_TRAINING_PATHS, 1.0, -1.0),
                   (abi.PRESENT_FLOW, 0, 1.0, 1.0), (abi.PRESENT_FLOW, TM, 2.0, 0.5),
                   (abi.PRESENT_COLOR, TM | abi.PRESENT_NRC_TRAINING_PATHS, 2.0, 1.0),
                   (abi.PRESENT_COLOR, TM | abi.PRESENT_REGIR_CELLS, 2.0, 1.0),
                   (abi.PRESENT_COLOR, abi.PRESENT_REGIR_CELLS | abi.PRESENT_NRC_TRAINING_PATHS, 1.0, -1.0),
                   (abi.PRESENT_NRC_PREDICTION, TM, 4.0, 1.0)]
    _check(gfx_ctx, oracle, p, after_frame, "after an NRC frame")
    p.regirGridDim[:] = [7, 3, 5]
    _check(gfx_ctx, oracle, p, [(abi.PRESENT_COLOR, TM | abi.PRESENT_REGIR_CELLS, 2.0, 1.0)], "7x3x5 cells")
    gfx_ctx.nrc_visualize_prediction(net, p)
    gfx_ctx.synchronize()
    _check(gfx_ctx, oracle, p, [(abi.PRESENT_NRC_PREDICTION, TM, 4.0, 1.0), (abi.PRESENT_NRC_PREDICTION, 0, 1.0, -1.0),
                                (abi.PRESENT_NRC_PREDICTION, TM | abi.PRESENT_NRC_TRAINING_PATHS, 1.0, 1.0),
                                (abi.PRESENT_NRC_PATH_LENGTH, 0, 1.0, 1.0)], "after the visualisation pass")
    net.close()


def test_existing_modes_ignore_the_new_fields(gfx_ctx, oracle):
    """COLOR / NORMAL without the new flags give the oracle's plain present whatever the trailing fields hold"""
    scene = scenes.tiny_city_scene()
    w, h = 100, 37
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    p = abi.default_frame_params(scene, w, h)
    gfx_ctx.build_light_distributions(0)
    gfx_ctx.gbuffer(p)
    gfx_ctx.pathtrace(p, abi.PT_BASELINE)
    beauty, normal = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), gfx_ctx.download(abi.BUF_NORMAL_ACCUM)
    for src, mode in [(abi.BUF_BEAUTY_ACCUM, abi.PRESENT_COLOR), (abi.BUF_NORMAL_ACCUM, abi.PRESENT_NORMAL)]:
        want = oracle.present(beauty if mode == abi.PRESENT_COLOR else normal, mode, TM | abi.PRESENT_FLIP_Y, 2.0, 1.0)
        for frame in (None, p):
            got = gfx_ctx.present(src, 0, mode, TM | abi.PRESENT_FLIP_Y, 2.0, 1.0, frame_params=frame,
                                  motion_vector_scale=float("nan"), motion_vector_offset=7.0)
            assert np.array_equal(got, want)
    assert C.sizeof(abi.GfxPresentParams) == 40
