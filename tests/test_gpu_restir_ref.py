"""The device's original ReSTIR DI passes on seeded synthetic frames (tests/restir_scenes.py): bit for bit against the oracle
on every launch form - the PHASE 0 megakernel (reuseVisibility = 0), the two-phase candidate loop (<= 32 candidates), the
lock-step loop (> 32 candidates, or an environment light) and strip launches - the saturated stream length, a 1920x1080
frame within the float64 restatement's bars (tests/restir_ref.py) on row windows, and the device's estimators at 512x512
against the direct-lighting integral (tests/restir_unbiased.py)."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import restir_ref, restir_scenes as S

pytestmark = pytest.mark.gpu

PLANES = [(abi.BUF_RNG, 0), (abi.BUF_RESERVOIR, 0), (abi.BUF_RESERVOIR, 1), (abi.BUF_RESERVOIR_INFO, 0),
          (abi.BUF_RESERVOIR_INFO, 1), (abi.BUF_BEAUTY_ACCUM, 0)]
# (log2 candidates, reuseVisibility, environment): two-phase, PHASE 0, lock-step by count, lock-step by the environment,
# a single candidate
FORMS = {"two_phase": (5, 1, False), "phase0": (5, 0, False), "lock_step": (6, 1, False), "env": (3, 1, True),
         "one_candidate": (0, 1, False)}


@pytest.fixture(scope="module")
def scenes_(oracle):
    out = {}
    for env in (False, True):
        sc = S.scene(env)
        out[env] = (sc, oracle.OracleScene(sc), restir_ref.Scene64(sc))
    return out


def _upload_scene(ctx, sc):
    ctx.upload_scene(sc)
    ctx.build_bvh()
    ctx.build_light_distributions()


def _cfg(p, log2, reuse_vis, neighbors=4, ld=1):
    p.log2NumCandidateSamples = log2
    p.reuseVisibility = reuse_vis
    p.numSpatialNeighbors = neighbors
    p.useLowDiscrepancyNeighbors = ld
    p.spatialNeighborRadius = 3.0


def _same(dev, orc, what):
    for buf, idx in PLANES:
        got, want = dev.get(buf, idx).view(np.uint32), orc.get(buf, idx).view(np.uint32)
        assert np.array_equal(got, want), f"{what}: buffer {buf}[{idx}] differs at {np.count_nonzero(got != want)} words"


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("size", S.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_passes_bit_exact_with_oracle(gfx_ctx, oracle, scenes_, form, size):
    log2, reuse_vis, env = FORMS[form]
    sc, oscene, s64 = scenes_[env]
    _upload_scene(gfx_ctx, sc)
    W, H = size
    for unbiased, passes, ld in ((False, 1, 1), (True, 2, 0)):
        dev, orc = S.DeviceSide(gfx_ctx, W, H), S.OracleSide(oracle, oscene, W, H)
        S.setup_frame([dev, orc], S.SyntheticFrames(W, H, 2), s64, 1)
        p = S.frame_params(sc, W, H, 1, cam_step=(0.05, 0.0, 0.02))
        _cfg(p, log2, reuse_vis, 10 if unbiased else 4, ld)
        for pass_id in S.frame_launches(p, 1, passes, True, unbiased):
            dev.run(p, pass_id)
            orc.run(p, pass_id)
            _same(dev, orc, f"{form} {W}x{H} unbiased={unbiased} pass {pass_id}")


def test_strips_bit_exact_with_oracle(gfx_ctx, oracle, scenes_):
    """launches on strips of 3 and 5 rows (fewer than a block's 8) equal the oracle's full-frame passes"""
    sc, oscene, s64 = scenes_[False]
    _upload_scene(gfx_ctx, sc)
    W, H = 45, 23
    dev, orc = S.DeviceSide(gfx_ctx, W, H), S.OracleSide(oracle, oscene, W, H)
    S.setup_frame([dev, orc], S.SyntheticFrames(W, H, 4), s64, 1)
    p = S.frame_params(sc, W, H, 1)
    _cfg(p, 5, 1)
    for pass_id in S.frame_launches(p, 1, 1, True, False):
        y, k = 0, 0
        while y < H:
            p.tileOriginY, p.tileRows = y, min(3 if k % 2 == 0 else 5, H - y)
            dev.run(p, pass_id)
            y, k = y + p.tileRows, k + 1
        p.tileOriginY, p.tileRows = 0, 0
        orc.run(p, pass_id)
        _same(dev, orc, f"strips pass {pass_id}")


def test_stream_length_saturates_bit_exact(gfx_ctx, oracle, scenes_):
    sc, oscene, s64 = scenes_[False]
    _upload_scene(gfx_ctx, sc)
    W, H = 9, 9
    dev, orc = S.DeviceSide(gfx_ctx, W, H), S.OracleSide(oracle, oscene, W, H)
    frames = S.SyntheticFrames(W, H, 3)
    S.setup_frame([dev, orc], frames, s64, 1)
    raw, info = frames.reservoirs(s64, 0)
    raw[1, ..., 3] = np.uint32((1 << 31) - 5)
    info[..., 0] = 1.0
    for s in (dev, orc):
        s.put(abi.BUF_RESERVOIR, 0, raw)
        s.put(abi.BUF_RESERVOIR_INFO, 0, info)
    p = S.frame_params(sc, W, H, 1)
    _cfg(p, 5, 1, 15)
    p.currentReservoirIndex = 0
    dev.run(p, abi.RESTIR_SPATIAL_BIASED)
    orc.run(p, abi.RESTIR_SPATIAL_BIASED)
    _same(dev, orc, "saturation")
    m = dev.get(abi.BUF_RESERVOIR, 1)[1, ..., 3]
    hit = dev.get(abi.BUF_GBUFFER0, 1)[..., 0] != S.SKY
    assert not (m[hit] >> 31).any() and (m[hit] == restir_ref.M31).any()


def test_1080p_within_restatement_bars(gfx_ctx, scenes_):
    """a 1920x1080 synthetic frame on the device, each pass against the restatement on three row windows"""
    sc, _, s64 = scenes_[False]
    _upload_scene(gfx_ctx, sc)
    W, H = 1920, 1080
    dev = S.DeviceSide(gfx_ctx, W, H)
    S.setup_frame([dev], S.SyntheticFrames(W, H, 8), s64, 1)
    p = S.frame_params(sc, W, H, 1)
    _cfg(p, 5, 1)
    ref = restir_ref.RestirRef(s64, W, H)
    for pass_id in S.frame_launches(p, 1, 1, True, True):
        ref.load(dev)
        outs = []
        for y0 in (0, H // 2 - 4, H - 8):
            p.tileOriginY, p.tileRows = y0, 8
            outs.append(S.ref_pass(ref, p, pass_id))
        p.tileOriginY, p.tileRows = 0, 0
        dev.run(p, pass_id)
        for out in outs:
            restir_ref.compare(dev, ref, out, f"1080p pass {pass_id}")
    assert ref.steered_pixels <= 0.01 * ref.compared_pixels + 1


# ---- the device's estimators against the direct-lighting integral at 512x512 (tests/restir_unbiased.py) ----------------------
def _initial(log2):
    def cfg(p):
        p.log2NumCandidateSamples = log2
        p.enableTemporalReuse = 0
        p.enableSpatialReuse = 0
        p.numSpatialNeighbors = 0
    return cfg


def _reuse(neighbors, unbiased=True, passes=1):
    def cfg(p):
        p.log2NumCandidateSamples = 3
        p.enableTemporalReuse = 1
        p.enableSpatialReuse = 1 if passes else 0
        p.numSpatialNeighbors = neighbors if passes else 0
        p.useUnbiasedEstimator = 1 if unbiased else 0
        p.useLowDiscrepancyNeighbors = 1
        p.spatialNeighborRadius = 5.0
    return cfg


UNBIASED_CASES = {
    "initial_1": (False, _initial(0), 1, 0, {}), "initial_32": (False, _initial(5), 1, 0, {}),
    "initial_256": (False, _initial(8), 1, 0, {}), "initial_env_4": (True, _initial(2), 1, 0, {}),
    "temporal": (False, _reuse(4, passes=0), 3, 0, {}), "spatial_1x4": (False, _reuse(4), 3, 1, {}),
    "spatial_3x10": (False, _reuse(10, passes=3), 3, 3, {}), "env_spatial_1x4": (True, _reuse(4), 3, 1, {}),
    "rearch": (False, _initial(5), 3, 0, {"rearch": True}),
    "checker_biased": (False, _reuse(4, False), 3, 1, {"checker": True}),
    "checker_unbiased": (False, _reuse(4), 3, 1, {"checker": True}),
}


@pytest.mark.parametrize("case", list(UNBIASED_CASES))
def test_unbiased_at_512(gfx_ctx, scenes_, case):
    from tests import restir_unbiased as RU
    env, cfg, frames, passes, kw = UNBIASED_CASES[case]
    sc, _, s64 = scenes_[env]
    _upload_scene(gfx_ctx, sc)
    means = RU.frame_means(lambda w, h: S.DeviceSide(gfx_ctx, w, h), sc, 512, 512, cfg, frames, passes, 16, **kw)
    integrals = np.array([RU.integral(s64, S.CAM, cls=c) for c in range(means.shape[1])])
    RU.check(means, integrals, f"{case} at 512x512")
