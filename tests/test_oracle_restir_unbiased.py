"""The oracle's ReSTIR DI estimators against the direct-lighting integral (tests/restir_unbiased.py), a check that depends on no
reading of the reference's kernels: initial RIS, unbiased temporal and spatial reuse and the rearchitected renderer's
unbiased configuration on one shading point, with and without the environment; biased and unbiased reuse on a checkerboard of
two shading points that testNeighbor keeps apart; and the measured effect of two reference quirks of the unbiased spatial pass.
"""
import numpy as np
import pytest

from tests import restir_ref, restir_scenes as S, restir_unbiased as RU

W = H = 32
REPEATS = 16


@pytest.fixture(scope="module")
def scenes_(oracle):
    out = {}
    for env in (False, True):
        sc = S.scene(env)
        s64 = restir_ref.Scene64(sc)
        out[env] = (sc, oracle.OracleScene(sc), s64, np.array([RU.integral(s64, S.CAM, cls=c) for c in (0, 1)]))
    return out


def _means(oracle, scenes_, env, configure, frames=1, passes=0, **kw):
    sc, oscene, _, integrals = scenes_[env]
    means = RU.frame_means(lambda w, h: S.OracleSide(oracle, oscene, w, h), sc, W, H, configure, frames, passes, REPEATS, **kw)
    return means, integrals[:means.shape[1]]


def _initial(log2):
    def cfg(p):
        p.log2NumCandidateSamples = log2
        p.enableTemporalReuse = 0
        p.enableSpatialReuse = 0
        p.numSpatialNeighbors = 0
    return cfg


def _reuse(neighbors, unbiased=True, ld=1, passes=1):
    def cfg(p):
        p.log2NumCandidateSamples = 3
        p.enableTemporalReuse = 1
        p.enableSpatialReuse = 1 if passes else 0
        p.numSpatialNeighbors = neighbors if passes else 0
        p.useUnbiasedEstimator = 1 if unbiased else 0
        p.useLowDiscrepancyNeighbors = ld
        p.spatialNeighborRadius = 5.0
    return cfg


@pytest.mark.parametrize("log2", [0, 1, 5, 6, 8])
def test_initial_ris_is_unbiased(oracle, scenes_, log2):
    RU.check(*_means(oracle, scenes_, False, _initial(log2)), f"initial RIS, 2^{log2} candidates")


@pytest.mark.parametrize("log2", [0, 1, 2, 5])
def test_initial_ris_with_environment_is_unbiased(oracle, scenes_, log2):
    """the first 0.25 N candidates sample the environment (for N < 4 with probability 0.25 N)"""
    RU.check(*_means(oracle, scenes_, True, _initial(log2)), f"initial RIS with the environment, 2^{log2} candidates")


@pytest.mark.parametrize("passes,neighbors", [(0, 4), (1, 4), (1, 10), (2, 4), (3, 4)])
def test_unbiased_reuse_is_unbiased(oracle, scenes_, passes, neighbors):
    """temporal reuse, then `passes` spatial passes of low-discrepancy neighbours, unbiased estimator"""
    RU.check(*_means(oracle, scenes_, False, _reuse(neighbors, passes=passes), 3, passes),
             f"unbiased reuse, {passes} spatial passes x {neighbors}")


def test_unbiased_reuse_with_environment_is_unbiased(oracle, scenes_):
    RU.check(*_means(oracle, scenes_, True, _reuse(4), 3, 1), "unbiased reuse with the environment")


def test_rearchitected_unbiased_is_unbiased(oracle, scenes_):
    """restir_rearch_frame_passes with the unbiased estimator: presampled lights, per-pixel RIS, pairwise MIS"""
    means, integrals = _means(oracle, scenes_, False, _initial(5), 3, rearch=True)
    RU.check(means, integrals, "rearchitected unbiased")


@pytest.mark.parametrize("unbiased", [False, True], ids=["biased", "unbiased"])
def test_checkerboard_matches_each_class(oracle, scenes_, unbiased):
    """two shading points 50 degrees apart: unbiased reuse by its MIS weights, biased reuse because testNeighbor's normal test
    rejects every neighbour of the other class"""
    means, integrals = _means(oracle, scenes_, False, _reuse(4, unbiased), 3, 1, checker=True)
    assert abs(integrals[0] - integrals[1]).max() > 0.2 * integrals[0].max()
    RU.check(means, integrals, f"checkerboard, {'unbiased' if unbiased else 'biased'}")


# ---- two reference quirks of the unbiased spatial pass, measured -------------------------------------------------------------
def test_random_neighbours_redrawn_for_mis_bias_the_checkerboard(oracle, scenes_):
    """With random neighbours the MIS loop draws its offsets again from an RNG that has moved on
    (optix_restir_di_kernels.cu:461-471 against :366-376), so it weighs other pixels than the ones the sample came from.  On the
    checkerboard, where those pixels often are of the other class, the estimate is biased; low-discrepancy neighbours (same
    offsets twice) are not."""
    means, integrals = _means(oracle, scenes_, False, _reuse(4, ld=0), 3, 1, checker=True)
    z, bound = RU.t_scores(means, integrals)
    assert (z > bound).any(), f"the quirk no longer shows: {z} standard errors"
    rel = np.abs(means.mean(0) - integrals) / integrals
    assert rel.max() > 0.01


def test_prev_camera_in_spatial_mis(oracle, scenes_):
    """The spatial MIS loop takes current-frame neighbours' view direction from prevCamera (optix_restir_di_kernels.cu:487).
    The numerator and denominator of the MIS weight use the same target function, so the weights still sum to one wherever a
    neighbour's target is positive; with a camera moving 0.2 m per frame over a glossy point the mean stays on the integral."""
    means, integrals = _means(oracle, scenes_, False, _reuse(4), 3, 1, cam_step=(0.2, 0.0, 0.1))
    integrals = np.array([RU.integral(scenes_[False][2], S.CAM + 2 * np.array([0.2, 0.0, 0.1]))])
    RU.check(means, integrals, "moving camera")
