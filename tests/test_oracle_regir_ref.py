"""The oracle's ReGIR against the float64 restatement of the reference (tests/regir_ref.py) and against the direct-lighting
integral (tests/restir_unbiased.py).

Pass by pass, on the oracle's own float32 state: the build of a new grid from the slot seeds, a temporal build over the
previous frame's slots, a temporal build over crafted previous slots (M on both sides of the 20x cap, M = 0, recPDFEstimate =
0, samples at infinity) and access histories at the edge of the idle-cell rule, and the access update.  Slot RNG states, M
and atInfinity must equal the restatement's, the other slot fields lie within its bars; at most 1 % of the slots compared
may be steered.

Then: a grid re-created mid-run (a frame resize, a new grid) keeps every slot finite and the cells the camera sees live, the
lpCos quirk of the cell target, and the frame mean at maxPathLength 2 against the integral, including the cell-centre bias
of small cells."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import regir_ref, regir_scenes as RS, restir_ref, restir_scenes as S, restir_unbiased as RU

STEER_LIMIT = 0.01
W, H = 16, 8


@pytest.fixture(scope="module")
def scenes_(oracle):
    out = {}
    for name, sc in (("plain", RS.scene()), ("flat", RS.flat_scene())):
        out[name] = (sc, oracle.OracleScene(sc), restir_ref.Scene64(sc))
    return out


def _cells(grid, seed, n=24):
    """the first 8 cells (the first 4096 slots), the last one and n seeded others"""
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(min(8, grid.num_cells)), [grid.num_cells - 1],
                                     rng.integers(0, grid.num_cells, n)]))


def _run_builds(oracle, scenes_, scene, grid, log2_slot, crafted=True):
    sc, oscene, s64 = scenes_[scene]
    side = RS.OracleSide(oracle, oscene, W, H)
    p = RS.params(sc, W, H, grid, log2_slot=log2_slot)
    if scene == "plain":
        RS.pad_box(p)
    g = regir_ref.Grid(p)
    cells = _cells(g, log2_slot)
    ref = regir_ref.RegirRef(s64)
    # frame 0: the grid is created by this build, from the slot seeds, with every cell live
    ref.grid = g
    ref.slots = [np.zeros((g.num_cells * regir_ref.SLOTS, 16), np.uint32) for _ in (0, 1)]
    n = g.num_cells * regir_ref.SLOTS
    ref.rng = np.zeros(n, np.uint64)
    first = regir_ref.mt19937_64(regir_ref.SEED, min(n, 8 * regir_ref.SLOTS) if n > 1 << 17 else n)
    ref.rng[:len(first)] = first
    ref.last = np.full(g.num_cells, 0xFFFFFFFF, np.uint32)
    cells0 = cells[cells < len(first) // regir_ref.SLOTS]
    RS.set_frame(p, 0)
    RS.check_build(side, ref, p, 0, False, cells0, "frame 0")
    # frame 1: temporal reuse over frame 0's slots
    RS.set_frame(p, 1)
    ref.load(side, p)
    RS.check_build(side, ref, p, 1, True, cells, "frame 1")
    if crafted:
        # frame 2: crafted previous slots and access histories around the idle rule
        RS.set_frame(p, 2)
        n_cand = 1 << log2_slot
        side.put_linear(abi.BUF_REGIR_SLOTS, 1, RS.crafted_slots(g, n_cand, log2_slot + 7), p)
        # frame - lastAccess in uint32: 0, 1, 3 (lastAccess = -1), 8 (live), 9 and 2^32 - 3 (idle)
        last = np.array([2, 1, 0xFFFFFFFF, 0xFFFFFFFA, 0xFFFFFFF9, 5], np.uint32)
        side.put_linear(abi.BUF_REGIR_LAST_ACCESS, 0, last[np.arange(g.num_cells) % 6], p)
        ref.load(side, p)
        out = RS.check_build(side, ref, p, 2, True, cells, "frame 2, crafted slots")
        assert g.num_cells == 1 or 0 < len(out["live_cells"]) < len(cells), "both live and idle cells"
        # a frame index near 2^32: frame - lastAccess = 2^32 - 1 (lastAccess = -1), 8, 9 and 2^32 - 7
        f = (1 << 32) - 2
        RS.set_frame(p, f)
        last = np.array([0xFFFFFFFF, f - 8, f - 9, 5], np.uint32)
        side.put_linear(abi.BUF_REGIR_LAST_ACCESS, 0, last[np.arange(g.num_cells) % 4], p)
        ref.load(side, p)
        out = RS.check_build(side, ref, p, f, True, cells, "frame 2^32 - 2")
        assert g.num_cells == 1 or 0 < len(out["live_cells"]) < len(cells), "both live and idle cells"
    assert ref.steered <= STEER_LIMIT * ref.compared + 1, f"{ref.steered} of {ref.compared} slots steered"
    return side, ref, p


@pytest.mark.parametrize("grid", list(RS.GRIDS), ids=list(RS.GRIDS))
def test_build_equals_restatement(oracle, scenes_, grid):
    _run_builds(oracle, scenes_, "plain", RS.GRIDS[grid], 3)


@pytest.mark.parametrize("log2_slot", [0, 1, 2, 5, 8])
def test_candidate_counts(oracle, scenes_, log2_slot):
    _run_builds(oracle, scenes_, "plain", RS.GRIDS["5x3x6" if log2_slot % 2 else "8x4x8"], log2_slot)


def test_flat_grid(oracle, scenes_):
    """a scene of height 0: every cell has height 0, and samples lie on the cells' lower and upper faces at once"""
    _run_builds(oracle, scenes_, "flat", (4, 2, 4), 3)


def test_slot_seeds(oracle, scenes_):
    """the slot RNGs of a new grid are std::mt19937_64(591842031321323413)'s outputs in slot order: after the first build
    (4 N draws per slot) the first 4096 and the last 64 states equal the seeds advanced by 4 N PCG32 steps"""
    sc, oscene, _ = scenes_["plain"]
    side = RS.OracleSide(oracle, oscene, W, H)
    p = RS.params(sc, W, H, (5, 3, 6))
    RS.set_frame(p, 0)
    side.build(p, 0, False)
    n = 90 * regir_ref.SLOTS
    want = regir_ref.mt19937_64(regir_ref.SEED, n)
    st = want.copy()
    for _ in range(4 * 8):
        st, _u = restir_ref.pcg_draw(st)
    got = side.get_linear(abi.BUF_REGIR_SLOT_RNG, 0, p).reshape(-1)
    sel = np.r_[0:4096, n - 64:n]
    restir_ref._exact(got[sel], st[sel], "slot RNG after the first build", sel)


def test_update_access(oracle, scenes_):
    """lastAccessFrameIndices takes the frame index where a cell was accessed, numActiveCells counts those cells; 90 cells
    leave the tail of the last 32-cell group empty"""
    sc, oscene, s64 = scenes_["plain"]
    side = RS.OracleSide(oracle, oscene, W, H)
    p = RS.params(sc, W, H, (5, 3, 6))
    RS.set_frame(p, 3)
    side.build(p, 3, False)
    acc = np.random.default_rng(2).choice(np.array([0, 0, 1, 7, 1 << 20], np.uint32), 90)
    side.put_linear(abi.BUF_REGIR_CELL_ACCESSES, 0, acc, p)
    side.put_linear(abi.BUF_REGIR_NUM_ACTIVE_CELLS, 0, np.array([5, 11], np.uint32), p)
    ref = regir_ref.RegirRef(s64)
    ref.load(side, p)
    out = ref.update_access(p, 3)
    side.update(p, 3)
    regir_ref.compare_update(side, out, p, "update access")
    assert out["active"][1] == 11 + (acc > 0).sum()


# ---- a grid re-created mid-run ---------------------------------------------------------------------------------------------------
def test_recreated_by_resize(oracle, scenes_):
    """the frame re-created at 80 x 36 on frame 10 (a new sequence): its new grid starts with lastAccessFrameIndices = 9 and
    builds every cell from that frame on"""
    sc, oscene, _ = scenes_["plain"]
    RS.check_recreation(lambda w, h: RS.OracleSide(oracle, oscene, w, h), sc, {10: "resize"})


def test_recreated_by_new_grid(oracle, scenes_):
    """a new regirGridDim on frame 12, temporal reuse on: the new grid's never-built previous slots (M = 0) weigh nothing"""
    sc, oscene, _ = scenes_["plain"]
    RS.check_recreation(lambda w, h: RS.OracleSide(oracle, oscene, w, h), sc, {12: (5, 3, 6)})


def test_environment_pole_keeps_slots_finite(oracle):
    """An environment candidate drawn at v = 0 exactly (uPos1 = 0, one draw in 2^23) is the pole, which the sampler gives
    areaPDensity 0 and no emittance: the reference's weight 0 / 0 made the slot's sumWeights NaN, and temporal reuse carried it
    on.  Slot 23978 of the sky scene draws it among its first 64 candidates of frame 0 at 2^8 candidates."""
    sc = RS.scene(True)
    side = RS.OracleSide(oracle, oracle.OracleScene(sc), W, H)
    p = RS.params(sc, W, H, RS.GRIDS["5x3x6"], log2_slot=8)
    for f in range(3):
        RS.set_frame(p, f)
        side.build(p, f, f > 0)
        s = regir_ref.Slots(side.get_linear(abi.BUF_REGIR_SLOTS, p.bufferIndex, p))
        assert np.isfinite(s.sumw).all(), f"frame {f}: {np.flatnonzero(~np.isfinite(s.sumw))} hold a non-finite sumWeights"
        assert s.rec[23978] > 0


# ---- the frame at maxPathLength 2, per pixel ------------------------------------------------------------------------------------
NW, NH = 48, 32


def _nee_case(oracle, scenes_, grid, log2_cell, randomize, seed):
    sc, oscene, s64 = scenes_["plain"]
    side = RS.OracleSide(oracle, oscene, NW, NH)
    p = RS.params(sc, NW, NH, RS.GRIDS[grid], log2_slot=2, log2_cell=log2_cell, randomize=randomize)
    g = regir_ref.Grid(p)
    gb0 = RS.gbuffer(sc, NW, NH, seed).reshape(-1, 4)
    gb0[: NW * NH // 4] = RS.face_points(g, NW * NH // 4, seed)   # 1 / 64 of the pixels on a face
    RS.put_gbuffer([side], gb0.reshape(NH, NW, 4))
    side.put(abi.BUF_RNG, 0, np.random.default_rng(seed).integers(0, 1 << 62, (NH, NW), dtype=np.int64).astype(np.uint64))
    ref = regir_ref.NeeRef(s64)
    for f in range(2):
        RS.set_frame(p, f)
        side.build(p, f, f > 0)
        before = side.get_linear(abi.BUF_REGIR_CELL_ACCESSES, 0, p).reshape(-1).astype(np.int64)
        out = ref.frame(side, p)
        side.pathtrace(p)
        regir_ref.compare_frame(side, ref, out, p, before, f"{grid} frame {f}")
        side.update(p, f)
    assert ref.steered <= STEER_LIMIT * ref.compared + 1, f"{ref.steered} of {ref.compared} pixels steered"


@pytest.mark.parametrize("grid", list(RS.GRIDS), ids=list(RS.GRIDS))
@pytest.mark.parametrize("randomize", [True, False], ids=["jitter", "no_jitter"])
def test_nee_equals_restatement(oracle, scenes_, grid, randomize):
    _nee_case(oracle, scenes_, grid, 2, randomize, 11)


@pytest.mark.parametrize("log2_cell", [0, 1, 3, 5])
def test_nee_cell_candidates(oracle, scenes_, log2_cell):
    _nee_case(oracle, scenes_, "8x4x8", log2_cell, True, 20 + log2_cell)


def test_pathtrace_needs_a_build(oracle, scenes_):
    sc, oscene, _ = scenes_["plain"]
    side = RS.OracleSide(oracle, oscene, W, H)
    with pytest.raises(RuntimeError, match="regir_build_cells first"):
        side.pathtrace(RS.params(sc, W, H, (5, 3, 6)))


# ---- the lpCos quirk --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", ["8x4x8", "5x3x6"])
def test_cell_target_cosine(oracle, scenes_, grid):
    """below a squared half diagonal of 1 (8 x 4 x 8: 0.64) the held targets carry the cell-centre cosine; above it
    (5 x 3 x 6: 1.33) none do, so samples behind the cell centre keep a target"""
    sc, oscene, s64 = scenes_["plain"]
    side = RS.OracleSide(oracle, oscene, W, H)
    p = RS.params(sc, W, H, RS.GRIDS[grid])
    RS.set_frame(p, 0)
    side.build(p, 0, False)
    g = regir_ref.Grid(p)
    s = regir_ref.Slots(side.get_linear(abi.BUF_REGIR_SLOTS, 0, p))
    live = np.flatnonzero(s.rec > 0)
    c = g.centres(live // regir_ref.SLOTS)
    d = s.pos[live] - c
    dist2 = (d * d).sum(-1)
    cos = (-d * s.nrm[live]).sum(-1) / np.sqrt(dist2)
    outside = ((np.abs(d) > g.half + 1e-5)).any(-1)
    with_cos = (s.le[live] / np.pi * (cos / dist2)[:, None]).mean(-1)
    without = (s.le[live] / np.pi / dist2[:, None]).mean(-1)
    sel = outside & (np.abs(cos) < 0.9)
    assert sel.sum() > 1000
    t = s.target[live][sel]
    if g.uses_cosine:
        np.testing.assert_allclose(t, with_cos[sel], rtol=1e-4)
        assert (cos[sel] > 0).all(), "a live slot holds a sample behind its cell centre"
    else:
        np.testing.assert_allclose(t, without[sel], rtol=1e-4)
        assert (cos[sel] < 0).any(), "no live slot holds a sample behind its cell centre"


# ---- the frame mean at maxPathLength 2 against the integral ------------------------------------------------------------------------
UW = UH = 32
REPEATS = 16
POINT = (0.3, 0.2)


def _means(oracle, sc, oscene, p, point, frames):
    return RS.frame_means(lambda w, h: RS.OracleSide(oracle, oscene, w, h), sc, UW, UH, p, point, frames, REPEATS)


@pytest.fixture(scope="module")
def unbiased_scenes(oracle):
    out = {}
    for env in (False, True):
        sc = RS.scene(env)
        s64 = restir_ref.Scene64(sc)
        x = RS.decoded_floor_point(*POINT)
        out[env] = (sc, oracle.OracleScene(sc), s64, x, RU.integral(s64, S.CAM, point=x))
    return out


@pytest.mark.parametrize("grid,log2_slot,log2_cell,randomize,frames", [
    ("1x1x1", 0, 0, True, 1), ("1x1x1", 3, 2, True, 1), ("1x1x1", 8, 5, False, 1), ("5x3x6", 3, 2, True, 1),
    ("5x3x6", 1, 3, False, 1), ("5x3x6", 3, 2, True, 8), ("1x1x1", 2, 1, True, 8)])
def test_large_cells_are_unbiased(oracle, unbiased_scenes, grid, log2_slot, log2_cell, randomize, frames):
    """cells whose squared half diagonal exceeds 1 ignore the cosine, so every emitter is in the target's support"""
    sc, oscene, _, x, integral = unbiased_scenes[False]
    p = RS.params(sc, UW, UH, RS.GRIDS[grid], log2_slot=log2_slot, log2_cell=log2_cell, randomize=randomize)
    RU.check(_means(oracle, sc, oscene, p, x, frames), integral[None], f"{grid}, 2^{log2_slot} x 2^{log2_cell}")


@pytest.mark.parametrize("frames", [1, 8])
def test_large_cells_with_sky_are_unbiased(oracle, unbiased_scenes, frames):
    sc, oscene, _, x, integral = unbiased_scenes[True]
    p = RS.params(sc, UW, UH, RS.GRIDS["5x3x6"], log2_slot=3, log2_cell=2)
    RU.check(_means(oracle, sc, oscene, p, x, frames), integral[None], "with the sky")


def test_cell_centre_bias(oracle, unbiased_scenes):
    """Small cells take the cosine at the cell centre.  Over 10 x 4 x 8 the cells of column 9 have centres at x = 3.6, behind
    the vertical emitter's plane x = 3.5 (it faces -x); a floor point at x = 3.2 in front of it jitters into column 9 half of
    the time, and there that emitter has a target only where it lies inside the cell itself.  The mean is the integral over
    that support (regir_ref.expected_nee), not the full integral.  (Over 8 x 4 x 8 a centre lies on the plane itself, so the
    sign of the cosine would be left to float32 rounding.)"""
    sc, oscene, s64, _, _ = unbiased_scenes[False]
    x = RS.decoded_floor_point(3.2, 0.0)
    p = RS.params(sc, UW, UH, RS.GRIDS["10x4x8"], log2_slot=0, log2_cell=2)
    g = regir_ref.Grid(p)
    assert np.isclose(g.centres([9])[0][0], 3.6) and g.uses_cosine
    means = _means(oracle, sc, oscene, p, x, 1)
    expected = regir_ref.expected_nee(s64, g, x, S.CAM, True)
    full = RU.integral(s64, S.CAM, point=x)
    RU.check(means, expected[None], "the cell-centre bias")
    z, bound = RU.t_scores(means, full[None])
    assert (z > bound).all() and (full - expected).min() > 0.05 * full.min(), \
        f"the full integral {full} is not told apart from the biased one {expected}"
