"""The oracle's ReSTIR DI passes against the float64 restatement of the reference (tests/restir_ref.py), pass by pass on
seeded synthetic frames (tests/restir_scenes.py), and its estimators against the direct-lighting integral.

Pass by pass: every pass of a frame's launch list runs on the oracle's own float32 inputs; the RNG state, M, atInfinity and
the held light sample must equal the restatement's, sumWeights, recPDFEstimate, targetDensity and beauty must lie within the
restatement's bars.  Pixels with a decision inside its float32 bar are steered and left out; fewer than 1 % of the pixels
compared in a test may be steered."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import restir_ref, restir_scenes as S

STEER_LIMIT = 0.01


@pytest.fixture(scope="module")
def scene_pair(oracle):
    sc = S.scene()
    return sc, oracle.OracleScene(sc), restir_ref.Scene64(sc)


def _run(oracle, scene_pair, W, H, frame, configure, spatial_passes, temporal, unbiased, seed=1):
    sc, oscene, s64 = scene_pair
    orc = S.OracleSide(oracle, oscene, W, H)
    frames = S.SyntheticFrames(W, H, seed)
    S.setup_frame([orc], frames, s64, frame)
    p = S.frame_params(sc, W, H, frame, cam_step=(0.05, 0.0, 0.02))   # a moving camera: prevCamera != camera
    configure(p)
    ref = restir_ref.RestirRef(s64, W, H)
    for pass_id in S.frame_launches(p, frame, spatial_passes, temporal, unbiased):
        ref.load(orc)
        out = S.ref_pass(ref, p, pass_id)
        orc.run(p, pass_id)
        restir_ref.compare(orc, ref, out, f"{W}x{H} frame {frame} pass {pass_id}")
    assert ref.steered_pixels <= STEER_LIMIT * ref.compared_pixels + 1, \
        f"{ref.steered_pixels} of {ref.compared_pixels} pixels steered"
    return ref


def _cfg(log2=5, neighbors=4, ld=1, reuse_vis=1):
    def f(p):
        p.log2NumCandidateSamples = log2
        p.numSpatialNeighbors = neighbors
        p.useLowDiscrepancyNeighbors = ld
        p.reuseVisibility = reuse_vis
        p.spatialNeighborRadius = 3.0
    return f


@pytest.mark.parametrize("size", S.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("unbiased", [False, True], ids=["biased", "unbiased"])
def test_passes_equal_restatement(oracle, scene_pair, size, unbiased):
    W, H = size
    _run(oracle, scene_pair, W, H, 1, _cfg(), 1, True, unbiased)


@pytest.mark.parametrize("log2", [0, 1, 5, 6, 8])
@pytest.mark.parametrize("reuse_vis", [0, 1])
def test_candidate_counts(oracle, scene_pair, log2, reuse_vis):
    _run(oracle, scene_pair, 9, 9, 1, _cfg(log2=log2, reuse_vis=reuse_vis), 1, True, log2 % 2 == 1)


@pytest.mark.parametrize("log2", [0, 1, 5])
def test_initial_ris_only(oracle, scene_pair, log2):
    """at 1 and 2 candidates many pixels have no live candidate: recPDFEstimate = 0 / 0 must become 0"""
    _run(oracle, scene_pair, 33, 17, 0, _cfg(log2=log2), 0, False, False)


def _lcg_back(state: int, steps: int) -> int:
    """the PCG32 state `steps` draws before `state`"""
    inv = pow(int(restir_ref.PCG_MUL), -1, 1 << 64)
    for _ in range(steps):
        state = ((state - 1) * inv) % (1 << 64)
    return state


def test_dead_temporal_candidate_drawing_zero(oracle, scene_pair):
    """Reservoir::update(sample, 0, u) with u = 0 exactly and sumW > 0 must not accept (u < 0 / sumW is false).  Every state
    below 2^36 draws 0 (rot = 0 and bits 36..58 of the xorshift are zero), so the RNG is wound back from such a state by the
    initial pass's 4 N draws; the temporal neighbour is the pixel itself in an identical previous G-buffer with
    recPDFEstimate = 0, a weight of exactly 0."""
    sc, oscene, s64 = scene_pair
    W, H = 9, 9
    orc = S.OracleSide(oracle, oscene, W, H)
    frames = S.SyntheticFrames(W, H, 9)
    S.setup_frame([orc], frames, s64, 1)
    g = frames.gbuffers(1)
    g[abi.BUF_GBUFFER1] = np.zeros((H, W, 2), np.float32)
    for buf, arr in g.items():
        orc.put(buf, 0, arr)
        orc.put(buf, 1, arr)
    raw, info = frames.reservoirs(s64, 0)
    info[..., 0] = 0.0
    orc.put(abi.BUF_RESERVOIR_INFO, 0, info)
    orc.put(abi.BUF_RESERVOIR, 0, raw)
    rng = np.random.default_rng(4)
    states = np.array([_lcg_back(int(v), 4 * 32) for v in rng.integers(0, 1 << 36, W * H)], np.uint64).reshape(H, W)
    orc.put(abi.BUF_RNG, 0, states)
    p = S.frame_params(sc, W, H, 1)
    _cfg()(p)
    p.currentReservoirIndex = 1
    ref = restir_ref.RestirRef(s64, W, H)
    ref.load(orc)
    out = ref.initial_and_temporal(p, True, False)
    orc.run(p, abi.RESTIR_INITIAL_AND_TEMPORAL_BIASED)
    assert (out["rec"] > 0).sum() > W * H // 4, "too few pixels with a live reservoir to reach the case"
    restir_ref.compare(orc, ref, out, "zero draw on a dead temporal candidate")


@pytest.mark.parametrize("neighbors", [1, 4, 10])
@pytest.mark.parametrize("ld", [0, 1], ids=["random", "low_discrepancy"])
@pytest.mark.parametrize("passes", [1, 2, 5])
@pytest.mark.parametrize("unbiased", [False, True], ids=["biased", "unbiased"])
def test_spatial_settings(oracle, scene_pair, neighbors, ld, passes, unbiased):
    _run(oracle, scene_pair, 17, 11, 1, _cfg(log2=3, neighbors=neighbors, ld=ld), passes, True, unbiased)


def test_row_strips(oracle, scene_pair):
    """launches on strips of 3 rows: each strip's pixels equal the restatement's"""
    sc, oscene, s64 = scene_pair
    W, H = 13, 11
    orc = S.OracleSide(oracle, oscene, W, H)
    frames = S.SyntheticFrames(W, H, 5)
    S.setup_frame([orc], frames, s64, 1)
    p = S.frame_params(sc, W, H, 1)
    _cfg()(p)
    ref = restir_ref.RestirRef(s64, W, H)
    for pass_id in S.frame_launches(p, 1, 1, True, False):
        for y0 in range(0, H, 3):
            p.tileOriginY, p.tileRows = y0, 3
            ref.load(orc)
            out = S.ref_pass(ref, p, pass_id)
            orc.run(p, pass_id)
            restir_ref.compare(orc, ref, out, f"strip {y0} pass {pass_id}")
        p.tileOriginY, p.tileRows = 0, 0


def test_stream_length_saturates(oracle, scene_pair):
    """M near 2^31 into biased spatial passes of 15 neighbours: the combined M saturates at 2^31 - 1 and an area-light sample
    stays an area-light sample (a 31-bit M field wrapped into the atInfinity bit before)"""
    sc, oscene, s64 = scene_pair
    W, H = 9, 9
    orc = S.OracleSide(oracle, oscene, W, H)
    frames = S.SyntheticFrames(W, H, 3)
    S.setup_frame([orc], frames, s64, 1)
    p = S.frame_params(sc, W, H, 1)
    _cfg(neighbors=15)(p)
    p.spatialNeighborRadius = 2.0
    raw, info = frames.reservoirs(s64, 0)
    raw[1, ..., 3] = np.uint32((1 << 31) - 5)                      # every area sample, M = 2^31 - 5
    info[..., 0] = 1.0
    orc.put(abi.BUF_RESERVOIR, 0, raw)
    orc.put(abi.BUF_RESERVOIR_INFO, 0, info)
    ref = restir_ref.RestirRef(s64, W, H)
    p.currentReservoirIndex = 0
    ref.load(orc)
    out = ref.spatial(p, False)
    orc.run(p, abi.RESTIR_SPATIAL_BIASED)
    assert (out["m_raw"] > restir_ref.M31).any()
    got = orc.get(abi.BUF_RESERVOIR, 1)[1, ..., 3].reshape(-1)[out["idx"]]
    assert not (got >> 31).any(), "an area-light sample came back flagged atInfinity"
    assert ((got & restir_ref.M31) == np.minimum(out["m_raw"], restir_ref.M31)).all()
    restir_ref.compare(orc, ref, out, "saturation")
