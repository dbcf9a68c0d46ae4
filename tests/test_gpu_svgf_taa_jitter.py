"""GPU parity of the SVGF app's frame with its TAA sub-pixel jitter (GFX_SVGF_SUBPIXEL_JITTER, svgf_main.cpp:1410-1424,
2005-2008) against the CPU oracle (oracle/svgf_taa_jitter.cpp), bit for bit after every frame: RNG, beauty, albedo, the four G-buffer planes and every
SVGF plane.  Runs of 20 frames or more wrap the offset index at taaHistoryLength 16; one run uses length 4."""
import json
import os
import subprocess

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_svgf_taa_jitter as OJ

pytestmark = pytest.mark.gpu

SVGF_BUFFERS = [(abi.BUF_SVGF_LIGHTING_VARIANCE, 2), (abi.BUF_SVGF_MOMENTS, 2), (abi.BUF_SVGF_PREV_LIGHTING, 1),
                (abi.BUF_SVGF_ALBEDO, 1), (abi.BUF_SVGF_DEPTH, 2), (abi.BUF_SVGF_FINAL, 2)]
FRAME_BUFFERS = [abi.BUF_RNG, abi.BUF_BEAUTY_ACCUM, abi.BUF_ALBEDO_ACCUM]
GBUFFERS = [abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3]


def _same(got, want):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


def _run(gfx_ctx, scene, w, h, frames, pan=0.0, env_rotation=0.0, taa_history_length=16, **kw):
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OJ.Frame(scene, w, h)
    sv = OJ.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightRotation = env_rotation
    p.taaHistoryLength = taa_history_length
    for frame in range(frames):
        cam = abi.make_camera(scene, w, h)
        cam.position[0] += pan * frame
        p.prevCamera = p.camera if frame > 0 else cam
        p.camera = cam
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, taa_jitter=True, **kw):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
            if kind == "gbuffer":
                fr.gbuffer(p)
            elif kind == "pathtrace":
                fr.pathtrace(p, pass_id)
            elif kind == "svgf":
                sv.run(p, pass_id, stage)
        gfx_ctx.synchronize()
        for buf in GBUFFERS:
            got, want = gfx_ctx.download(buf, p.bufferIndex), fr.buffer(buf, p.bufferIndex)
            assert _same(got, want), f"frame {frame}: G-buffer {buf} differs at {np.count_nonzero(got != want)} elements"
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
    "city_static": (scenes.small_city_scene, 128, 72, 20, 0.0, {}),
    "city_pan": (scenes.tiny_city_scene, 128, 72, 20, 0.04, {}),
    "city_env_pan": (scenes.small_city_scene_env, 128, 72, 20, 0.04, {"env_rotation": 0.7}),
    "city_textured": (scenes.small_city_scene_textured, 128, 72, 20, 0.04, {}),
    "svgf_off_temporal_on": (scenes.tiny_city_scene, 128, 72, 20, 0.04, {"enable_svgf": False}),
    "taa_length_4": (scenes.tiny_city_scene, 128, 72, 9, 0.04, {"taa_history_length": 4}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_svgf_taa_jitter_frame_bit_exact(gfx_ctx, case):
    make, w, h, frames, pan, kw = CASES[case]
    _run(gfx_ctx, make(), w, h, frames, pan, **kw)


def test_svgf_taa_jitter_strip_equals_full_frame(gfx_ctx):
    """the jitter draws no random numbers: a strip's G-buffer and path tracer rows equal the full frame's"""
    scene = scenes.small_city_scene()
    w, h = 160, 90
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.build_light_distributions(0)
    p = abi.default_frame_params(scene, w, h)
    p.frameIndex = 5
    p.svgfFlags |= abi.SVGF_MOLLIFY_SPECULAR | abi.SVGF_SUBPIXEL_JITTER
    out = []
    for y0, rows in ((0, 0), (37, 29)):
        gfx_ctx.create_frame(w, h)  # the same RNG seed for both runs
        p.tileOriginY, p.tileRows = y0, rows
        gfx_ctx.gbuffer(p)
        gfx_ctx.pathtrace(p, abi.PT_SVGF)
        gfx_ctx.synchronize()
        out.append([gfx_ctx.download(b, 0) for b in GBUFFERS] + [gfx_ctx.download(b) for b in FRAME_BUFFERS])
    for full, strip in zip(*out):
        assert _same(full[37:66], strip[37:66])


def test_svgf_taa_jitter_1080p_strip_against_oracle(gfx_ctx):
    """1920x1080: frames 0 to 2 (offsets (0, 0), (1/2, 1/3), (1/4, 2/3)) on a 48-row strip of the oracle equal the GPU's rows"""
    scene = scenes.small_city_scene()
    w, h, y0, rows = 1920, 1080, 516, 48
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OJ.Frame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    for frame in range(3):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, taa_jitter=True):
            if kind in ("light_dist", "gbuffer", "pathtrace"):
                engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
        gfx_ctx.synchronize()
        p.tileOriginY, p.tileRows = y0, rows
        fr.gbuffer(p)
        fr.pathtrace(p, abi.PT_SVGF)
        p.tileOriginY, p.tileRows = 0, 0
        for buf in GBUFFERS:
            got, want = gfx_ctx.download(buf, p.bufferIndex)[y0:y0 + rows], fr.buffer(buf, p.bufferIndex)[y0:y0 + rows]
            assert _same(got, want), f"frame {frame}: G-buffer {buf} differs"
        for buf in FRAME_BUFFERS:
            got, want = gfx_ctx.download(buf)[y0:y0 + rows], fr.buffer(buf)[y0:y0 + rows]
            assert _same(got, want), f"frame {frame}: buffer {buf} differs"


def test_svgf_taa_jitter_with_enable_jittering_is_refused(gfx_ctx):
    scene = scenes.tiny_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(64, 40)
    p = abi.default_frame_params(scene, 64, 40)
    p.svgfFlags |= abi.SVGF_SUBPIXEL_JITTER
    p.enableJittering = 1
    with pytest.raises(engine.GfxError, match="status -1: .*enableJittering"):
        gfx_ctx.gbuffer(p)
    with pytest.raises(engine.GfxError, match="status -1: .*enableJittering"):
        gfx_ctx.svgf(p, abi.SVGF_FILL_BACKGROUND, 5)
    p.enableJittering = 0
    gfx_ctx.gbuffer(p)
    gfx_ctx.svgf(p, abi.SVGF_FILL_BACKGROUND, 5)
    gfx_ctx.synchronize()


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")


def test_cpp_host_svgf_taa_jitter_matches_python_host(gfx_ctx, tmp_path):
    W, H, FRAMES = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path = str(tmp_path / "scene.bin")
    scenes.save_scene_bin(scene, scene_path, W, H)
    out_path = str(tmp_path / "out.raw")
    res = subprocess.run([HOST, scene_path, "svgf", str(W), str(H), str(FRAMES), out_path, "-taa-jitter"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    info = json.loads(res.stdout.strip().splitlines()[-1])
    assert info["renderer"] == "svgf"
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    for f in range(FRAMES):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, f, taa_jitter=True):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
    gfx_ctx.synchronize()
    want = gfx_ctx.download(abi.BUF_SVGF_FINAL, (FRAMES - 1) % 2)
    got = np.fromfile(out_path, dtype=np.float32).reshape(H, W, 4)
    assert _same(got, want), "svgf -taa-jitter: C++ host image differs from the Python host image"
    # and the jitter changed the image
    gfx_ctx.create_frame(W, H)
    for f in range(FRAMES):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, f):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
    gfx_ctx.synchronize()
    assert not _same(gfx_ctx.download(abi.BUF_SVGF_FINAL, (FRAMES - 1) % 2), want)
