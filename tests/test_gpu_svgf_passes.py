"""The device's SVGF passes one at a time on seeded synthetic frames (tests/svgf_scenes.py): bit for bit against the oracle at
small and odd sizes and on the threshold set, within the float64 restatement's per-pixel bars (tests/svgf_ref.py) at 1920x1080 and
on row windows of 3840x2160, strip launches of fewer than 8 rows equal to the full frame, and the two filters refused, with no
kernel launched, on frames one pixel wide or high."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import svgf_ref, svgf_scenes as S

pytestmark = pytest.mark.gpu

TA, FB, TAA, MOD = (abi.SVGF_ENABLE_TEMPORAL_ACCUMULATION, abi.SVGF_FEEDBACK_1ST, abi.SVGF_ENABLE_TAA,
                    abi.SVGF_MODULATE_ALBEDO)
FULL = TA | FB | TAA | MOD
CONFIGS = [(FULL, 16, 5), (FULL & ~FB, 4, 4), (TA | MOD, 1, 3), (TAA, 16, 5), (0, 4, 3)]


@pytest.fixture(scope="module")
def oscene(oracle):
    from gfxexp_b200 import scenes
    return oracle.OracleScene(scenes.tiny_city_scene(), build_bvh=False)


def _planes(side):
    return [side.get(b, i).view(np.uint32) for b, n in S.ALL_PLANES for i in range(n)]


@pytest.mark.parametrize("thresholds", [False, True], ids=["general", "thresholds"])
@pytest.mark.parametrize("size", [(2, 2), (3, 5), (7, 3), (5, 17), (33, 9), (97, 61)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_passes_bit_exact_with_oracle(gfx_ctx, oracle, oscene, size, thresholds):
    W, H = size
    for k, (flags, hist, stages) in enumerate(CONFIGS):
        dev, orc = S.DeviceSide(gfx_ctx, W, H), S.OracleSide(oracle, oscene, W, H)
        sc = S.SyntheticScene(W, H, 7, thresholds)

        def on_pass(p, pass_id, stage):
            assert dev.run(p, pass_id, stage) == 0 and orc.run(p, pass_id, stage) == 0
            gfx_ctx.synchronize()
            for (buf, idx), got, want in zip([(b, i) for b, n in S.ALL_PLANES for i in range(n)], _planes(dev), _planes(orc)):
                assert np.array_equal(got, want), f"{W}x{H} flags {flags} frame {p.frameIndex} pass {pass_id}.{stage}: " \
                    f"buffer {buf}[{idx}] differs at {np.count_nonzero(got != want)} elements"

        S.run_frames([dev, orc], sc, 4, flags, hist, stages, on_pass, first_frame=k % 2)


def _against_restatement(gfx_ctx, W, H, frames, windows, halo, stages=5):
    """the device against the restatement on row windows (lo, hi): each restated on rows lo - halo .. hi + halo - 1"""
    dev = S.DeviceSide(gfx_ctx, W, H)
    sc = S.SyntheticScene(W, H, 11)
    refs = []
    for lo, hi in windows:
        y0 = max(0, lo - halo)
        refs.append((svgf_ref.SvgfRef(W, H, y0, min(H, hi + halo) - y0), (lo, hi)))

    def on_pass(p, pass_id, stage):
        planes = {(b, i): dev.get(b, i) for b, n in S.ALL_PLANES for i in range(n)}
        assert dev.run(p, pass_id, stage) == 0
        gfx_ctx.synchronize()
        for ref, rows in refs:
            for (b, i), a in planes.items():
                ref.load(b, i, a)
            outs = S.ref_pass(ref, p, pass_id, stage)
            S.compare_outputs(dev, ref, outs, p.bufferIndex, f"{W}x{H} rows {rows} frame {p.frameIndex} pass {pass_id}.{stage}",
                              rows)

    S.run_frames([dev], sc, frames, FULL, 16, stages, on_pass, first_frame=1)
    # with SVGF off the app copies lighting plane 0 to the previous lighting (feedbackNoisyLighting)
    p = S.frame_params(W, H, frames + 1, FULL)
    for ref, rows in refs:
        ref.load(abi.BUF_SVGF_LIGHTING_VARIANCE, 0, dev.get(abi.BUF_SVGF_LIGHTING_VARIANCE, 0))
    assert dev.run(p, abi.SVGF_FEEDBACK_NOISY_LIGHTING, 0) == 0
    for ref, rows in refs:
        S.compare_outputs(dev, ref, ref.feedback_noisy_lighting(), p.bufferIndex, "feedback", rows)


# Per-pass isolation needs one pass's footprint of halo around a window: the reprojection's motion (zoom 0.03 x H / 2 rows + 3)
# and the last a-trous stage's 16 + 1 rows.  The windows take the top and bottom edges and the middle, where x < W/2 and
# y < H/2 switch sides.
def test_passes_within_restatement_bars_1080p(gfx_ctx):
    H = 1080
    _against_restatement(gfx_ctx, 1920, H, 2, [(0, 64), (H // 2 - 32, H // 2 + 32), (H - 64, H)], 24)


def test_passes_within_restatement_bars_4k_windows(gfx_ctx):
    H = 2160
    _against_restatement(gfx_ctx, 3840, H, 2, [(0, 32), (H // 2 - 16, H // 2 + 16), (H - 32, H)], 40)


def test_strips_equal_full_frame(gfx_ctx):
    """launches on strips of 3 and 5 rows (fewer than a block's 8) of a frame 45 pixels wide (not a multiple of 32) write what
    the full-frame launches write"""
    W, H = 45, 23
    strips = []
    y = 0
    while y < H:
        n = 3 if len(strips) % 2 == 0 else 5
        strips.append((y, min(n, H - y)))
        y += n
    results = []
    for strip in (False, True):
        dev = S.DeviceSide(gfx_ctx, W, H)
        sc = S.SyntheticScene(W, H, 13, thresholds=True)
        after = []

        def on_pass(p, pass_id, stage):
            for y0, rows in (strips if strip else [(0, 0)]):
                p.tileOriginY, p.tileRows = y0, rows
                assert dev.run(p, pass_id, stage) == 0
            p.tileOriginY, p.tileRows = 0, 0
            gfx_ctx.synchronize()
            after.append(_planes(dev))

        S.run_frames([dev], sc, 3, FULL, 16, 5, on_pass)
        results.append(after)
    for k, (full, tiled) in enumerate(zip(*results)):
        for a, b in zip(full, tiled):
            assert np.array_equal(a, b), f"pass {k}: the strips differ from the full frame"


@pytest.mark.parametrize("size", [(1, 1), (1, 6), (6, 1)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_filters_refuse_frames_under_2x2(gfx_ctx, size):
    """W == 1 or H == 1: the depth gradient's neighbour would be pixel -1 or row -1; both filters return
    GFX_ERR_INVALID_ARGUMENT with an error string, launch nothing and leave every plane as it was"""
    W, H = size
    dev = S.DeviceSide(gfx_ctx, W, H)
    sc = S.SyntheticScene(W, H, 2)
    for buf, idx, arr in sc.history():
        dev.put(buf, idx, arr)
    p = S.frame_params(W, H, 0, FULL)
    for buf, arr in {**sc.gbuffers(0), **sc.shading(0)}.items():
        dev.put(buf, 0, arr)
    assert dev.run(p, abi.SVGF_TEMPORAL_ACCUMULATE, 0) == 0
    gfx_ctx.synchronize()
    before = _planes(dev)
    launches = gfx_ctx.kernel_launches
    for pass_id, stage in [(abi.SVGF_ESTIMATE_VARIANCE, 0)] + [(abi.SVGF_ATROUS, s) for s in range(5)]:
        assert dev.run(p, pass_id, stage) == -1
        assert b"2x2" in gfx_ctx.lib.gfx_last_error_string(gfx_ctx.h)
    gfx_ctx.synchronize()
    assert gfx_ctx.kernel_launches == launches
    assert all(np.array_equal(a, b) for a, b in zip(before, _planes(dev)))
    assert dev.run(p, abi.SVGF_FILL_BACKGROUND, 5) == 0 and dev.run(p, abi.SVGF_MODULATE_TAA, 5) == 0
    gfx_ctx.synchronize()
    assert gfx_ctx.kernel_launches == launches + 2
