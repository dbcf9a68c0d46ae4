"""The oracle's SVGF passes (oracle/denoise.cpp) against the float64 restatement of the reference (tests/svgf_ref.py), one pass
at a time on seeded synthetic frames (tests/svgf_scenes.py): each pass reads the oracle's float32 planes, and its outputs must lie
within the restatement's per-pixel bars; sample counts, accept flags and every plane a pass leaves alone (sky pixels) exactly.
No GPU."""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import svgf_ref, svgf_scenes as S

SIZES = [(2, 2), (3, 5), (7, 3), (5, 17), (31, 7), (33, 9), (97, 61)]
TA, FB, TAA, MOD = (abi.SVGF_ENABLE_TEMPORAL_ACCUMULATION, abi.SVGF_FEEDBACK_1ST, abi.SVGF_ENABLE_TAA,
                    abi.SVGF_MODULATE_ALBEDO)
# every combination of the four switches; the TAA history length and the number of filter stages (the plane parity of the
# background and TAA passes) take every value across them
CONFIGS = [((TA if k & 1 else 0) | (FB if k & 2 else 0) | (TAA if k & 4 else 0) | (MOD if k & 8 else 0),
            (16, 4, 1)[k % 3], (5, 4, 3)[(k // 3) % 3]) for k in range(16)]
FULL = TA | FB | TAA | MOD
GFX_ERR_INVALID_ARGUMENT = -1


@pytest.fixture(scope="module")
def oscene(oracle):
    return oracle.OracleScene(scenes.tiny_city_scene(), build_bvh=False)


def _run(oracle, oscene, W, H, frames, flags, hist, stages, seed=1, thresholds=False, first_frame=1):
    side = S.OracleSide(oracle, oscene, W, H)
    sc = S.SyntheticScene(W, H, seed, thresholds)
    ref = svgf_ref.SvgfRef(W, H)

    def on_pass(p, pass_id, stage):
        S.load_all(ref, side)
        assert side.run(p, pass_id, stage) == 0
        outs = S.ref_pass(ref, p, pass_id, stage)
        S.compare_outputs(side, ref, outs, p.bufferIndex, f"{W}x{H} frame {p.frameIndex} pass {pass_id}.{stage}")

    S.run_frames([side], sc, frames, flags, hist, stages, on_pass, first_frame)
    return ref


@pytest.mark.parametrize("config", range(len(CONFIGS)))
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_passes_equal_restatement(oracle, oscene, size, config):
    flags, hist, stages = CONFIGS[config]
    ref = _run(oracle, oscene, *size, 3, flags, hist, stages, first_frame=(config // 2) % 2)
    assert ref.margins["normal"] >= 8.5e-4    # the generator keeps the normal test 1e-3 (relative) from 0.85


@pytest.mark.parametrize("size", [(3, 5), (33, 9), (97, 61)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_passes_on_thresholds(oracle, oscene, size):
    """the threshold set: the distance test at exactly 0.1f, normals either side of 0.85 by 2e-6, prevScreenPos 0, 1.0 and
    just under, exact pixel centres (fDelta 0, zero-weight neighbours still accepted), counts of exactly 4, depth 1.0"""
    for flags, hist, stages in ((FULL, 16, 5), (FULL & ~FB, 4, 4), (TA | MOD, 1, 3)):
        ref = _run(oracle, oscene, *size, 4, flags, hist, stages, seed=3, thresholds=True)
        assert ref.margins["normal"] >= 2e-6
        if size[0] * size[1] > 100:
            assert ref.margins["normal"] < 1e-4   # the near-0.85 normals met their previous neighbours


def test_threshold_set_sits_on_the_thresholds():
    sq = S.DIST_EXACT * S.DIST_EXACT
    assert sq == np.float32(0.1) and not sq > np.float32(0.1)
    above = np.nextafter(S.DIST_EXACT, np.float32(1))
    assert above * above > np.float32(0.1)
    for W in (32, 33, 97, 1920, 3840):   # prevScreenPos just under 1.0: the float under it where the division can land there
        m = S.SyntheticScene._under_one(W)
        r = (np.float32(W - 1) + np.float32(0.5) - m) / np.float32(W)
        assert r < 1 and r >= 1 - 2 ** -22 and (W != 32 or r == np.nextafter(np.float32(1), np.float32(0)))
    W = 33
    sc = S.SyntheticScene(W, 9, 3, True)
    n0 = S.shading_ref.decode_vector(sc.codes[:1])[0]
    dots = [float(S.shading_ref.decode_vector(np.array([q]))[0] @ n0) for q in sc.code_near]
    assert dots[0] > 0.85 > dots[1] and max(abs(d - 0.85) for d in dots) < 1e-4


def test_stale_variance_reaches_neighbours(oracle, oscene):
    """a reference quirk, kept: a pixel that turns from geometry into sky keeps its last filtered lighting in plane 1 (a-trous
    stages skip sky pixels, and the temporal pass only clears plane 0), and the next frame's stage 1 reads that stale variance
    in its neighbours' 3x3 localMeanStdDev, which has no depth test"""
    W, H = 9, 7
    side = S.OracleSide(oracle, oscene, W, H)
    sc = S.SyntheticScene(W, H, 5)
    ref = svgf_ref.SvgfRef(W, H)
    seen = {}

    def on_pass(p, pass_id, stage):
        S.load_all(ref, side)
        if p.frameIndex == 1 and pass_id == abi.SVGF_ATROUS and stage == 1:
            stale = ref.lighting[1][3, 4, 3]
            seen["stale"] = stale
            assert stale > 0 and stale == seen["frame0"]
            without = svgf_ref.SvgfRef(W, H)
            S.load_all(without, side)
            without.lighting[1][3, 4, 3] = 0.0
            seen["without"] = without.atrous(p, 1)["lighting0"][0][3, 3]
        assert side.run(p, pass_id, stage) == 0
        outs = S.ref_pass(ref, p, pass_id, stage)
        S.compare_outputs(side, ref, outs, p.bufferIndex, f"frame {p.frameIndex} pass {pass_id}.{stage}")
        if p.frameIndex == 0 and pass_id == abi.SVGF_ATROUS and stage == 4:
            seen["frame0"] = side.get(abi.BUF_SVGF_LIGHTING_VARIANCE, 1).view(np.float32)[3, 4, 3]
        if p.frameIndex == 1 and pass_id == abi.SVGF_ATROUS and stage == 1:
            seen["with"] = side.get(abi.BUF_SVGF_LIGHTING_VARIANCE, 0).view(np.float32)[3, 3]

    # pixel (4, 3) is geometry on frame 0 and sky on frame 1; its neighbour (3, 3) is geometry on both
    labels = sc.labels

    def pinned_labels(frame):
        lab, sky = labels(frame)
        sky[2:5, 2:7] = False
        sky[3, 4] = frame == 1
        return lab, sky
    sc.labels = pinned_labels
    S.run_frames([side], sc, 2, FULL, 16, 5, on_pass)
    assert not np.allclose(seen["with"][:3], seen["without"][:3], rtol=1e-6, atol=0), \
        "the stale variance must change the neighbour's filtered lighting"


@pytest.mark.parametrize("size", [(1, 1), (1, 6), (6, 1)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_refuses_filters_on_frames_under_2x2(oracle, oscene, size):
    """the depth gradient's neighbour x + (x < W/2 ? 1 : -1) is pixel -1 at W = 1 (row -1 at H = 1): both filters refuse the
    frame and leave every plane as it was; the other passes run"""
    W, H = size
    side = S.OracleSide(oracle, oscene, W, H)
    sc = S.SyntheticScene(W, H, 2)
    for buf, idx, arr in sc.history():
        side.put(buf, idx, arr)
    p = S.frame_params(W, H, 0, FULL)
    for buf, arr in {**sc.gbuffers(0), **sc.shading(0)}.items():
        side.put(buf, 0, arr)
    assert side.run(p, abi.SVGF_TEMPORAL_ACCUMULATE, 0) == 0
    before = [side.get(b, i).copy() for b, n in S.SVGF_PLANES for i in range(n)]
    assert side.run(p, abi.SVGF_ESTIMATE_VARIANCE, 0) == GFX_ERR_INVALID_ARGUMENT
    for stage in range(5):
        assert side.run(p, abi.SVGF_ATROUS, stage) == GFX_ERR_INVALID_ARGUMENT
    after = [side.get(b, i) for b, n in S.SVGF_PLANES for i in range(n)]
    assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, after))
    assert side.run(p, abi.SVGF_FILL_BACKGROUND, 5) == 0
    assert side.run(p, abi.SVGF_MODULATE_TAA, 5) == 0
