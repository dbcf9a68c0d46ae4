"""GPU parity of the SVGF app's debug views (gfx_svgf_debug_visualize, debugVisualize of svgf/gpu_kernels/visualize.cu) against
the CPU oracle (oracle/svgf_views.cpp), bit for bit: all seven views after every frame of SVGF-app runs, each at the point of the
frame where the app launches it (svgf_main.cpp:2138-2145, 2175-2185), together with RNG, beauty, albedo and every SVGF plane.
Also: the views leave the frame untouched, strips, 1080p, the present, the C++ host and the refusals."""
import json
import os
import subprocess

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_lib as O
from tests import oracle_svgf_views as OV

pytestmark = pytest.mark.gpu

SVGF_BUFFERS = [(abi.BUF_SVGF_LIGHTING_VARIANCE, 2), (abi.BUF_SVGF_MOMENTS, 2), (abi.BUF_SVGF_PREV_LIGHTING, 1),
                (abi.BUF_SVGF_ALBEDO, 1), (abi.BUF_SVGF_DEPTH, 2), (abi.BUF_SVGF_FINAL, 2)]
FRAME_BUFFERS = [abi.BUF_RNG, abi.BUF_BEAUTY_ACCUM, abi.BUF_ALBEDO_ACCUM]
EARLY_VIEWS = (abi.SVGF_VIEW_NOISY_BEAUTY, abi.SVGF_VIEW_VARIANCE)
LATE_VIEWS = (abi.SVGF_VIEW_FILTERED_VARIANCE, abi.SVGF_VIEW_ALBEDO, abi.SVGF_VIEW_NORMAL, abi.SVGF_VIEW_MOTION_VECTOR,
              abi.SVGF_VIEW_SAMPLE_COUNT)
STAGES = 5  # the app's numFilteringStages, which it passes to every view launch, SVGF on or off (svgf_main.cpp:2127, 2184)


def _same(got, want):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


def _compare_view(gfx_ctx, sv, p, view, stages, frame):
    gfx_ctx.svgf_debug_visualize(p, view, num_filtering_stages=stages)
    sv.debug_visualize(p, view, 0.5, 0.1, stages)
    gfx_ctx.synchronize()
    got, want = gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE), sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)
    assert _same(got, want), \
        f"frame {frame}: view {view} differs at {np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))} elements"
    return got


def _run(gfx_ctx, scene, w, h, frames, pan=0.0, env_rotation=0.0, modulate=False, svgf_off_from=None, **kw):
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OV.Frame(scene, w, h)
    sv = OV.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightRotation = env_rotation
    if modulate:
        p.svgfFlags |= abi.SVGF_MODULATE_ALBEDO
    launched = set()
    views = {}
    for frame in range(frames):
        cam = abi.make_camera(scene, w, h)
        cam.position[0] += pan * frame
        p.prevCamera = p.camera if frame > 0 else cam
        p.camera = cam
        if svgf_off_from is not None:
            kw["enable_svgf"] = frame < svgf_off_from
        before = gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE) if frame > 0 else None
        early = False
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, view=abi.SVGF_VIEW_NOISY_BEAUTY, **kw):
            if kind == "svgf_view":  # the app's first launch point: Noisy Beauty, then Variance
                assert stage == STAGES
                early = True
                for view in EARLY_VIEWS:
                    views[view] = _compare_view(gfx_ctx, sv, p, view, stage, frame)
                    launched.add(view)
                continue
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
            if kind == "gbuffer":
                fr.gbuffer(p)
            elif kind == "pathtrace":
                fr.pathtrace(p, pass_id)
            elif kind == "svgf":
                sv.run(p, pass_id, stage)
        if before is not None and not early:
            # SVGF off: the app never launches Noisy Beauty or Variance, and the buffer keeps what it held on both sides
            gfx_ctx.synchronize()
            assert _same(gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE), before)
            assert _same(sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE), before)
        gfx_ctx.synchronize()
        for buf in FRAME_BUFFERS:
            got, want = gfx_ctx.download(buf), fr.buffer(buf)
            assert _same(got, want), f"frame {frame}: buffer {buf} differs"
        for buf, count in SVGF_BUFFERS:
            for idx in range(count):
                got, want = gfx_ctx.download(buf, idx), sv.buffer(buf, idx)
                assert _same(got, want), f"frame {frame}: SVGF buffer {buf}[{idx}] differs"
        for view in LATE_VIEWS:  # the app's second launch point, after albedo modulation + TAA
            views[view] = _compare_view(gfx_ctx, sv, p, view, STAGES, frame)
            launched.add(view)
    return p, sv, views, launched


CASES = {
    "city_static": (scenes.small_city_scene, 192, 108, 4, 0.0, {}),
    "city_pan": (scenes.tiny_city_scene, 160, 90, 3, 0.06, {}),
    "city_textured": (scenes.small_city_scene_textured, 160, 90, 3, 0.04, {}),
    "city_env_pan": (scenes.small_city_scene_env, 160, 90, 3, 0.04, {"env_rotation": 0.7}),
    "taa_jitter": (scenes.tiny_city_scene, 128, 72, 5, 0.04, {"taa_jitter": True}),
    "modulate_albedo": (scenes.small_city_scene, 160, 90, 3, 0.04, {"modulate": True}),
    "svgf_off_temporal_on": (scenes.tiny_city_scene, 160, 90, 4, 0.04, {"enable_svgf": False}),
    "svgf_switched_off": (scenes.tiny_city_scene, 160, 90, 4, 0.04, {"svgf_off_from": 2}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_svgf_views_bit_exact(gfx_ctx, case):
    make, w, h, frames, pan, kw = CASES[case]
    _, _, views, launched = _run(gfx_ctx, make(), w, h, frames, pan, **kw)
    assert launched == (set(LATE_VIEWS) if kw.get("enable_svgf") is False else set(EARLY_VIEWS) | set(LATE_VIEWS))
    for view, img in views.items():
        assert np.all(img[..., 3] == 1)
    if case == "svgf_switched_off":
        # SVGF off in the last frames: Filtered Variance shows lighting plane 1 as the last filtered frame left it
        frozen = gfx_ctx.download(abi.BUF_SVGF_LIGHTING_VARIANCE, 1)[..., 3]
        assert np.count_nonzero(frozen) > 100
        assert _same(views[abi.SVGF_VIEW_FILTERED_VARIANCE][..., 0], np.sqrt(frozen))
    if case == "city_env_pan":
        # the sky's motion vectors come from fillBackground's prevScreenPos, which reprojects directions only: the camera
        # translates, so the sky stays near the neutral 0.5 while the geometry moves
        gb0 = gfx_ctx.download(abi.BUF_GBUFFER0, (frames - 1) % 2)
        sky = (gb0[..., 0] == 0xFFFFFFFF)
        assert sky.sum() > 100
        assert np.all(views[abi.SVGF_VIEW_NORMAL][sky][:, :3] == 0.5)
        assert np.all(views[abi.SVGF_VIEW_ALBEDO][sky][:, :3] == 1)
        motion = views[abi.SVGF_VIEW_MOTION_VECTOR][..., :2]
        assert np.abs(motion[sky] - 0.5).max() < 1e-3 and np.abs(motion[~sky] - 0.5).max() > 0.01


def test_svgf_views_present_equals_oracle(gfx_ctx):
    """gfx_present_launch(COLOR) of the debug buffer with the app's display flags equals the oracle's present of its buffer"""
    scene = scenes.small_city_scene_env()
    w, h = 160, 90
    p, sv, _, _ = _run(gfx_ctx, scene, w, h, 2, 0.04, env_rotation=0.7)
    for view in EARLY_VIEWS + LATE_VIEWS:
        # both planes at the end of the frame: the early views too are defined there
        gfx_ctx.svgf_debug_visualize(p, view)
        sv.debug_visualize(p, view)
        flags = engine.svgf_view_present_flags(view)
        got = gfx_ctx.present(abi.BUF_SVGF_DEBUG_VISUALIZE, 0, flags=flags, frame_params=p)
        want = O.present(sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE), abi.PRESENT_COLOR, flags)
        assert np.array_equal(got, want), f"view {view}: present differs at {np.count_nonzero(got != want)} pixels"


def test_svgf_views_leave_the_frame_untouched(gfx_ctx):
    """a sequence with a view after every frame leaves RNG, beauty, albedo and every SVGF plane as the same sequence without"""
    scene = scenes.tiny_city_scene()
    w, h, frames = 128, 72, 4
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    out = []
    for with_views in (False, True):
        gfx_ctx.create_frame(w, h)
        p = abi.default_frame_params(scene, w, h)
        for frame in range(frames):
            cam = abi.make_camera(scene, w, h)
            cam.position[0] += 0.04 * frame
            p.prevCamera = p.camera if frame > 0 else cam
            p.camera = cam
            view = frame % 7 if with_views else None
            for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, view=view):
                engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
            if with_views:
                for v in range(7):
                    gfx_ctx.svgf_debug_visualize(p, v)
        gfx_ctx.synchronize()
        out.append([gfx_ctx.download(b) for b in FRAME_BUFFERS] +
                   [gfx_ctx.download(b, i) for b, n in SVGF_BUFFERS for i in range(n)])
    for a, b in zip(*out):
        assert _same(a, b)


def test_svgf_views_strip_writes_its_rows(gfx_ctx):
    scene = scenes.small_city_scene()
    w, h, y0, rows = 160, 90, 37, 29
    p, _, _, _ = _run(gfx_ctx, scene, w, h, 2, 0.04)
    sentinel = np.full((h, w, 4), -7.0, dtype=np.float32)
    for view in range(7):
        p.tileOriginY, p.tileRows = 0, 0
        gfx_ctx.svgf_debug_visualize(p, view)
        gfx_ctx.synchronize()
        full = gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE)
        gfx_ctx.upload(abi.BUF_SVGF_DEBUG_VISUALIZE, 0, sentinel)
        p.tileOriginY, p.tileRows = y0, rows
        gfx_ctx.svgf_debug_visualize(p, view)
        gfx_ctx.synchronize()
        strip = gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE)
        assert _same(strip[y0:y0 + rows], full[y0:y0 + rows]), f"view {view}"
        assert np.all(strip[:y0] == -7) and np.all(strip[y0 + rows:] == -7), f"view {view}"
    p.tileOriginY, p.tileRows = 0, 0


def test_svgf_views_1080p_strip_against_oracle(gfx_ctx):
    """1920x1080, frames 0 and 1: every view of the GPU's planes on a 48-row strip equals the oracle's view of those planes, with
    the normal and prevScreenPos from the oracle's own G-buffer of the strip"""
    scene = scenes.small_city_scene()
    w, h, y0, rows = 1920, 1080, 516, 48
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    fr = OV.Frame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    for frame in range(2):
        cam = abi.make_camera(scene, w, h)
        cam.position[0] += 0.04 * frame
        p.prevCamera = p.camera if frame > 0 else cam
        p.camera = cam
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame):
            engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
        gfx_ctx.synchronize()
        p.tileOriginY, p.tileRows = y0, rows
        fr.gbuffer(p)
        fr.pathtrace(p, abi.PT_SVGF)
        normal, psp = fr.view_inputs(p)
        p.tileOriginY, p.tileRows = 0, 0
        for buf in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER3):
            assert _same(gfx_ctx.download(buf, p.bufferIndex)[y0:y0 + rows], fr.buffer(buf, p.bufferIndex)[y0:y0 + rows])
        for buf in FRAME_BUFFERS:  # the path tracer's output on the strip, which the temporal pass turns into the planes
            assert _same(gfx_ctx.download(buf)[y0:y0 + rows], fr.buffer(buf)[y0:y0 + rows]), f"frame {frame}: buffer {buf}"
        planes = (gfx_ctx.download(abi.BUF_SVGF_LIGHTING_VARIANCE, 0), gfx_ctx.download(abi.BUF_SVGF_LIGHTING_VARIANCE, 1),
                  gfx_ctx.download(abi.BUF_SVGF_ALBEDO), normal, psp, gfx_ctx.download(abi.BUF_SVGF_MOMENTS, p.bufferIndex))
        for view in range(7):
            gfx_ctx.svgf_debug_visualize(p, view)
            gfx_ctx.synchronize()
            got = gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE)[y0:y0 + rows]
            want = OV.view_planes(*planes, view, bool(p.svgfFlags & abi.SVGF_MODULATE_ALBEDO), rows=(y0, y0 + rows))
            assert _same(got, want[y0:y0 + rows]), f"frame {frame}: view {view} differs"


def test_svgf_views_errors(gfx_ctx):
    fresh = engine.Context(0)
    try:
        p = abi.default_frame_params(scenes.tiny_city_scene(), 32, 16)
        with pytest.raises(engine.GfxError, match="status -4"):
            fresh.svgf_debug_visualize(p, abi.SVGF_VIEW_ALBEDO)
    finally:
        fresh.close()
    scene = scenes.tiny_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(32, 16)
    p = abi.default_frame_params(scene, 32, 16)
    with pytest.raises(engine.GfxError, match="status -1"):  # not allocated before the first view
        gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE)
    for view in (7, -1):
        with pytest.raises(engine.GfxError, match="status -1"):
            gfx_ctx.svgf_debug_visualize(p, view)
    gfx_ctx.svgf_debug_visualize(p, abi.SVGF_VIEW_ALBEDO)
    gfx_ctx.synchronize()
    assert gfx_ctx.download(abi.BUF_SVGF_DEBUG_VISUALIZE).shape == (16, 32, 4)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")
HOST_VIEWS = {"noisy": abi.SVGF_VIEW_NOISY_BEAUTY, "variance": abi.SVGF_VIEW_VARIANCE,
              "filtered-variance": abi.SVGF_VIEW_FILTERED_VARIANCE, "albedo": abi.SVGF_VIEW_ALBEDO,
              "normal": abi.SVGF_VIEW_NORMAL, "motion": abi.SVGF_VIEW_MOTION_VECTOR, "samples": abi.SVGF_VIEW_SAMPLE_COUNT}


def test_cpp_host_svgf_views_match_python_host(gfx_ctx, tmp_path):
    from gfxexp_b200 import imageio
    W, H, FRAMES = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path = str(tmp_path / "scene.bin")
    scenes.save_scene_bin(scene, scene_path, W, H)
    for name, view in HOST_VIEWS.items():
        out_path = str(tmp_path / f"{name}.png")
        res = subprocess.run([HOST, scene_path, "svgf", str(W), str(H), str(FRAMES), out_path, "-view", name],
                             capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stderr
        assert json.loads(res.stdout.strip().splitlines()[-1])["renderer"] == "svgf"
        gfx_ctx.upload_scene(scene)
        gfx_ctx.build_bvh()
        gfx_ctx.create_frame(W, H)
        p = abi.default_frame_params(scene, W, H)
        for f in range(FRAMES):
            for kind, pass_id, stage in engine.svgf_app_frame_passes(p, f, view=view):
                engine.run_svgf_app_pass(gfx_ctx, p, kind, pass_id, stage)
        gfx_ctx.synchronize()
        want = gfx_ctx.present(abi.BUF_SVGF_DEBUG_VISUALIZE, 0, flags=engine.svgf_view_present_flags(view), frame_params=p)
        assert np.array_equal(imageio.read_png(out_path), want), f"-view {name}: C++ host image differs from the Python host's"
    # the new names belong to the svgf renderer
    for renderer in ("pathtrace", "restir"):
        res = subprocess.run([HOST, scene_path, renderer, str(W), str(H), "1", str(tmp_path / "x.png"), "-view", "albedo"],
                             capture_output=True, text=True, timeout=300)
        assert res.returncode == 2 and "svgf" in res.stderr
