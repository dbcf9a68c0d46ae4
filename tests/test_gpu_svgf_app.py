"""GPU parity: the SVGF app's own frame (svgf/svgf_main.cpp:1980-2172) - its path tracer GFX_PT_SVGF with specular
mollification, temporal accumulation, the filter or the feedbackNoisyLighting pass, background and TAA - against the CPU
oracle (oracle/svgf_app.cpp), bit for bit after every frame: RNG, beauty, albedo and every SVGF plane."""
import json
import os
import subprocess

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_svgf_app as OA

pytestmark = pytest.mark.gpu

SVGF_BUFFERS = [(abi.BUF_SVGF_LIGHTING_VARIANCE, 2), (abi.BUF_SVGF_MOMENTS, 2), (abi.BUF_SVGF_PREV_LIGHTING, 1),
                (abi.BUF_SVGF_ALBEDO, 1), (abi.BUF_SVGF_DEPTH, 2), (abi.BUF_SVGF_FINAL, 2)]
FRAME_BUFFERS = [abi.BUF_RNG, abi.BUF_BEAUTY_ACCUM, abi.BUF_ALBEDO_ACCUM]


def _same(got, want):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


def _run(gfx_ctx, scene, w, h, frames, pan=0.0, env_rotation=0.0, max_path_length=5, **kw):
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OA.Frame(scene, w, h)
    sv = OA.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightRotation = env_rotation
    p.maxPathLength = max_path_length
    for frame in range(frames):
        cam = abi.make_camera(scene, w, h)
        cam.position[0] += pan * frame
        p.prevCamera = p.camera if frame > 0 else cam
        p.camera = cam
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, **kw):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
            if kind == "gbuffer":
                fr.gbuffer(p)
            elif kind == "pathtrace":
                fr.pathtrace(p, pass_id)
            elif kind == "svgf":
                sv.run(p, pass_id, stage)
        gfx_ctx.synchronize()
        for buf in FRAME_BUFFERS:
            got, want = gfx_ctx.download(buf), fr.buffer(buf)
            assert _same(got, want), f"frame {frame}: buffer {buf} differs at {np.count_nonzero(got != want)} elements"
        for buf, count in SVGF_BUFFERS:
            for idx in range(count):
                got, want = gfx_ctx.download(buf, idx), sv.buffer(buf, idx)
                assert _same(got, want), \
                    f"frame {frame}: SVGF buffer {buf}[{idx}] differs at {np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))} elements"
    final = gfx_ctx.download(abi.BUF_SVGF_FINAL, (frames - 1) % 2)
    assert np.isfinite(final).all()
    return p, final


CASES = {
    "city_static": (scenes.small_city_scene, 192, 108, 4, 0.0, {}),
    "city_pan": (scenes.tiny_city_scene, 160, 90, 3, 0.06, {}),
    "interior_pbr": (scenes.small_interior_scene, 160, 90, 3, 0.0, {}),
    "city_textured": (scenes.small_city_scene_textured, 160, 90, 3, 0.04, {}),
    "length2": (scenes.tiny_city_scene, 160, 90, 3, 0.0, {"max_path_length": 2}),
    "length8": (scenes.tiny_city_scene, 160, 90, 3, 0.0, {"max_path_length": 8}),
    "no_mollification": (scenes.small_city_scene, 160, 90, 3, 0.0, {"mollify": False}),
    "svgf_off_temporal_on": (scenes.tiny_city_scene, 160, 90, 4, 0.04, {"enable_svgf": False}),
    "svgf_off_temporal_off": (scenes.tiny_city_scene, 160, 90, 3, 0.0, {"enable_svgf": False, "temporal_accumulation": False}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_svgf_app_frame_bit_exact(gfx_ctx, case):
    make, w, h, frames, pan, kw = CASES[case]
    _run(gfx_ctx, make(), w, h, frames, pan, **kw)


def test_svgf_app_with_environment_light(gfx_ctx):
    """NEE and the miss program sample the environment; sky pixels get their colour from fillBackground only"""
    scene = scenes.small_city_scene_env()
    _, final = _run(gfx_ctx, scene, 160, 90, 3, 0.04, env_rotation=0.7)
    gb0 = gfx_ctx.download(abi.BUF_GBUFFER0, 0)
    sky = gb0[..., 0] == 0xFFFFFFFF
    assert sky.sum() > 100 and final[sky][:, :3].mean() > 0.05
    assert np.all(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[sky][:, :3] == 0)
    assert np.all(gfx_ctx.download(abi.BUF_ALBEDO_ACCUM)[sky] == 0)


def test_svgf_app_strip_equals_full_frame(gfx_ctx):
    scene = scenes.small_city_scene()
    w, h = 160, 90
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.build_light_distributions(0)
    p = abi.default_frame_params(scene, w, h)
    p.svgfFlags |= abi.SVGF_MOLLIFY_SPECULAR
    out = []
    for y0, rows in ((0, 0), (37, 29)):
        gfx_ctx.create_frame(w, h)  # the same RNG seed for both runs
        p.tileOriginY, p.tileRows = 0, 0
        gfx_ctx.gbuffer(p)
        p.tileOriginY, p.tileRows = y0, rows
        gfx_ctx.pathtrace(p, abi.PT_SVGF)
        gfx_ctx.synchronize()
        out.append([gfx_ctx.download(b) for b in FRAME_BUFFERS])
    for full, strip in zip(*out):
        assert _same(full[37:66], strip[37:66])


def test_svgf_app_denoises(gfx_ctx):
    """on a static camera the filtered image is closer to the mean of 96 frames of the variant's own raw beauty than the
    1-spp input is"""
    scene = scenes.small_city_scene()
    w, h = 192, 108
    p, final = _run(gfx_ctx, scene, w, h, 4)
    noisy = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3].copy()
    acc = np.zeros_like(noisy, dtype=np.float64)
    for k in range(96):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, 4 + k):
            if kind in ("light_dist", "gbuffer", "pathtrace"):
                engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
        acc += gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3]
    converged = (acc / 96).astype(np.float32)

    def mse(img):
        return float(np.mean((np.clip(img[..., :3], 0, 4) - np.clip(converged, 0, 4)) ** 2))
    assert mse(final) < 0.5 * mse(noisy), (mse(final), mse(noisy))


def test_svgf_app_1080p_strip_against_oracle(gfx_ctx):
    """1920x1080: frames 0 and 1 of GFX_PT_SVGF on a 48-row strip of the oracle equal the GPU's rows"""
    scene = scenes.small_city_scene()
    w, h, y0, rows = 1920, 1080, 516, 48
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OA.Frame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    for frame in range(2):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame):
            if kind in ("light_dist", "gbuffer", "pathtrace"):
                engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
        gfx_ctx.synchronize()
        p.tileOriginY, p.tileRows = y0, rows
        fr.gbuffer(p)
        fr.pathtrace(p, abi.PT_SVGF)
        p.tileOriginY, p.tileRows = 0, 0
        for buf in FRAME_BUFFERS:
            got, want = gfx_ctx.download(buf)[y0:y0 + rows], fr.buffer(buf)[y0:y0 + rows]
            assert _same(got, want), f"frame {frame}: buffer {buf} differs"


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")


@pytest.mark.parametrize("out_kind", ["raw", "png"])
def test_cpp_host_svgf_matches_python_host(gfx_ctx, tmp_path, out_kind):
    W, H, FRAMES = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path = str(tmp_path / "scene.bin")
    scenes.save_scene_bin(scene, scene_path, W, H)
    out_path = str(tmp_path / f"out.{out_kind}")
    res = subprocess.run([HOST, scene_path, "svgf", str(W), str(H), str(FRAMES), out_path], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stderr
    info = json.loads(res.stdout.strip().splitlines()[-1])
    assert info["renderer"] == "svgf" and info["kernel_launches"] > 0
    # the Python host: the same loop on the scene file's defaults
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    for f in range(FRAMES):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, f):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
    gfx_ctx.synchronize()
    index = (FRAMES - 1) % 2
    want = gfx_ctx.download(abi.BUF_SVGF_FINAL, index)
    if out_kind == "raw":
        got = np.fromfile(out_path, dtype=np.float32).reshape(H, W, 4)
        assert _same(got, want), "svgf: C++ host image differs from the Python host image"
        assert np.isfinite(got).all() and got[..., :3].mean() > 1e-4
    else:
        from gfxexp_b200 import imageio
        assert np.array_equal(imageio.read_png(out_path), gfx_ctx.present(abi.BUF_SVGF_FINAL, index, frame_params=p))
