"""CPU checks of the oracle's TAA sub-pixel jitter (GFX_SVGF_SUBPIXEL_JITTER, svgf_main.cpp:1410-1424, 2005-2008): the
offset table against a numpy restatement of the app's float loop, the sample position (x + ox, y + 1 - oy) against a
rectangle with known edges, motion vectors measured from the sample, the anti-aliasing it buys, and no effect without TAA."""
import numpy as np

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_svgf_taa_jitter as OJ
from tests import svgf_jitter_scenes as JS

MISS = 0xFFFFFFFF


def _halton_f32(base, idx):
    """computeHaltonSequence (svgf_main.cpp:1410-1421), every step rounded to float32"""
    rec = np.float32(1.0) / np.float32(base)
    ret, scale = np.float32(0.0), np.float32(1.0)
    while idx:
        scale = np.float32(scale * rec)
        ret = np.float32(ret + np.float32(np.float32(idx % base) * scale))
        idx //= base
    return ret


def _run(scene, w, h, frames, taa_jitter, svgf=True, on_frame=None, flags_off=0, **kw):
    fr = OJ.Frame(scene, w, h)
    sv = OJ.Svgf(fr) if svgf else None
    p = abi.default_frame_params(scene, w, h)
    p.svgfFlags &= ~flags_off
    for f in range(frames):
        for kind, pid, stage in engine.svgf_app_frame_passes(p, f, taa_jitter=taa_jitter, **kw):
            if kind == "gbuffer":
                fr.gbuffer(p)
            elif kind == "pathtrace":
                fr.pathtrace(p, pid)
            elif kind == "svgf" and sv is not None:
                sv.run(p, pid, stage)
        if on_frame is not None:
            on_frame(f, p, fr, sv)
    return p, fr, sv


def test_offsets_equal_the_apps_table():
    for i in range(256):
        want = (_halton_f32(2, i), _halton_f32(3, i))
        got = OJ.subpixel_offset(i)
        assert np.float32(got[0]).view(np.uint32) == want[0].view(np.uint32), (i, got, want)
        assert np.float32(got[1]).view(np.uint32) == want[1].view(np.uint32), (i, got, want)
    assert OJ.subpixel_offset(0) == (0.0, 0.0)
    assert OJ.subpixel_offset(1) == (np.float32(0.5), np.float32(1) / np.float32(3))
    assert OJ.subpixel_offset(2) == (np.float32(0.25), np.float32(2) * (np.float32(1) / np.float32(3)))


def test_sample_position_convention():
    """hit or miss in the rectangle's edge columns and rows follows the sample position (x + ox, y + 1 - oy), with
    (ox, oy) = subPixelOffsets[frameIndex % 16]; 16 frames visit every offset of the cycle"""
    scene = JS.rect_scene()
    rows = np.arange(int(JS.TOP) + 1, int(JS.BOTTOM))     # rows fully inside vertically
    cols = np.arange(int(JS.LEFT) + 1, int(JS.RIGHT))
    seen = set()

    def check(f, p, fr, sv):
        ox, oy = OJ.subpixel_offset(f % 16)
        hit = fr.buffer(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] != MISS
        xl, xr, yt, yb = int(JS.LEFT), int(JS.RIGHT), int(JS.TOP), int(JS.BOTTOM)
        assert np.all(hit[rows, xl] == (xl + ox >= JS.LEFT)), (f, ox)
        assert np.all(hit[rows, xr] == (xr + ox < JS.RIGHT)), (f, ox)
        assert np.all(hit[yt, cols] == (yt + 1 - oy >= JS.TOP)), (f, oy)
        assert np.all(hit[yb, cols] == (yb + 1 - oy < JS.BOTTOM)), (f, oy)
        assert np.all(hit[rows[0]:rows[-1] + 1, cols[0]:cols[-1] + 1])
        seen.add((bool(hit[rows[0], xl]), bool(hit[yt, cols[0]])))
    _run(scene, JS.W, JS.H, 16, True, svgf=False, on_frame=check)
    assert len(seen) == 4, "the 16 offsets must put both edges' samples on both sides"


def test_static_camera_motion_vectors_vanish():
    """with a static camera the motion vector of every hit is 0 to within 1e-3 px: the current raster position is the
    sample's, not the pixel centre's (which would leave (0.5 - ox, oy - 0.5), e.g. (0.25, 0.17) px at frame 2)"""
    scene = scenes.tiny_city_scene()
    w, h = 64, 40
    moved = []

    def check(f, p, fr, sv):
        gb0 = fr.buffer(abi.BUF_GBUFFER0, p.bufferIndex)
        mv = fr.buffer(abi.BUF_GBUFFER1, p.bufferIndex)
        hit = gb0[..., 0] != MISS
        assert hit.sum() > 500
        assert np.abs(mv[hit]).max() <= 1e-3, (f, float(np.abs(mv[hit]).max()))
        moved.append(fr.buffer(abi.BUF_GBUFFER2, p.bufferIndex)[..., :3].copy())
    _run(scene, w, h, 4, True, svgf=False, on_frame=check)
    assert not np.array_equal(moved[1], moved[2]), "the jitter must move the primary hits"


def _final(taa_jitter, frames=64):
    scene = JS.rect_scene()
    p, fr, sv = _run(scene, JS.W, JS.H, frames, taa_jitter)
    return sv.buffer(abi.BUF_SVGF_FINAL, p.bufferIndex)[..., :3].astype(np.float64)


def test_jitter_anti_aliases_edges():
    """An emitting rectangle against the empty background (0.001), static camera, TAA on, 64 frames.  Over the 56 pixels the
    rectangle's edges cross, the mean absolute error of GFX_BUF_SVGF_FINAL against coverage x radiance + (1 - coverage) x
    background is 1.037 without the jitter and 0.165 with it (radiance 10 / pi = 3.18); the test asks for at most half.
    Pixels the rectangle covers fully or not at all keep their value in both runs: the TAA's bilinear history fetch lands a
    few 1e-6 from the pixel centre, which is all an edge pixel next door can leak into them."""
    cov = JS.coverage()[..., None]
    radiance = np.float32(JS.EMITTANCE) / np.float32(np.pi)
    want = cov * radiance + (1 - cov) * 0.001
    plain, jittered = _final(False), _final(True)
    edge = (cov[..., 0] > 0) & (cov[..., 0] < 1)
    inner, outer = cov[..., 0] == 1, cov[..., 0] == 0
    assert edge.sum() == 56 and inner.sum() > 100 and outer.sum() > 100
    err_plain = float(np.abs(plain - want)[edge].mean())
    err_jittered = float(np.abs(jittered - want)[edge].mean())
    assert err_jittered <= 0.5 * err_plain, (err_plain, err_jittered)
    for img in (plain, jittered):
        assert np.allclose(img[outer], 0.001, rtol=0, atol=1e-5)
        assert np.allclose(img[inner], radiance, rtol=1e-4, atol=0)


def test_no_effect_without_taa():
    """the flag applies only with GFX_SVGF_ENABLE_TEMPORAL_AA: without it every buffer is the same bits as without the flag"""
    scene = scenes.small_city_scene_env()
    w, h = 64, 40
    runs = []
    for jitter in (False, True):
        p, fr, sv = _run(scene, w, h, 3, jitter, flags_off=abi.SVGF_ENABLE_TAA)
        bufs = [fr.buffer(b, i) for b in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3)
                for i in (0, 1)]
        bufs += [fr.buffer(b) for b in (abi.BUF_RNG, abi.BUF_BEAUTY_ACCUM, abi.BUF_ALBEDO_ACCUM)]
        bufs += [sv.buffer(b, i) for b, n in ((abi.BUF_SVGF_LIGHTING_VARIANCE, 2), (abi.BUF_SVGF_MOMENTS, 2),
                                              (abi.BUF_SVGF_PREV_LIGHTING, 1), (abi.BUF_SVGF_ALBEDO, 1),
                                              (abi.BUF_SVGF_DEPTH, 2), (abi.BUF_SVGF_FINAL, 2)) for i in range(n)]
        runs.append(bufs)
    for a, b in zip(*runs):
        assert np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
