"""The device's ReGIR against the oracle bit for bit on synthetic inputs, against the float64 restatement of the reference
(tests/regir_ref.py) at 1080p on the default grid, and against the direct-lighting integral at 512 x 512.

Bit for bit: builds over every grid of tests/regir_scenes.py (crafted previous slots, access histories around the idle rule
and near 2^32), path-traced frames on G-buffers of every triangle and the sky, access updates, with and without the sky, with
cell randomization on and off, and the re-creation sequences of tests/test_oracle_regir_ref.py."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import regir_ref, regir_scenes as RS, restir_ref, restir_scenes as S, restir_unbiased as RU

pytestmark = pytest.mark.gpu
W, H = 64, 36
STEER_LIMIT = 0.01
POINT = (0.3, 0.2)


def _same(got, want, tag):
    g = np.ascontiguousarray(got).view(np.uint32 if np.asarray(got).dtype.itemsize == 4 else np.uint64)
    w = np.ascontiguousarray(want).view(g.dtype)
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first at {bad[0].tolist()}")


@pytest.fixture(scope="module", params=[False, True], ids=["plain", "sky"])
def pair(request, gfx_ctx, oracle):
    sc = RS.scene(request.param)
    gfx_ctx.upload_scene(sc)
    gfx_ctx.build_bvh()
    gfx_ctx.build_light_distributions(0)
    return sc, oracle.OracleScene(sc), restir_ref.Scene64(sc)


def _sides(gfx_ctx, oracle, oscene, w, h):
    return RS.DeviceSide(gfx_ctx, w, h), RS.OracleSide(oracle, oscene, w, h)


def _compare_all(dev, orc, p, tag):
    for buf in (abi.BUF_REGIR_SLOTS,):
        for i in (0, 1):
            _same(dev.get_linear(buf, i, p), orc.get_linear(buf, i, p), f"{tag}: slots {i}")
    for buf, name in ((abi.BUF_REGIR_SLOT_RNG, "slot RNG"), (abi.BUF_REGIR_CELL_ACCESSES, "accesses"),
                      (abi.BUF_REGIR_LAST_ACCESS, "last access")):
        _same(dev.get_linear(buf, 0, p), orc.get_linear(buf, 0, p), f"{tag}: {name}")
    _same(dev.get_linear(abi.BUF_REGIR_NUM_ACTIVE_CELLS, 0, p), orc.get_linear(abi.BUF_REGIR_NUM_ACTIVE_CELLS, 0, p),
          f"{tag}: numActiveCells")
    _same(dev.get(abi.BUF_RNG), orc.get(abi.BUF_RNG), f"{tag}: pixel RNG")
    _same(dev.get(abi.BUF_BEAUTY_ACCUM), orc.get(abi.BUF_BEAUTY_ACCUM), f"{tag}: beauty")


@pytest.mark.parametrize("grid", list(RS.GRIDS), ids=list(RS.GRIDS))
@pytest.mark.parametrize("log2_slot,log2_cell,randomize", [(3, 2, True), (0, 0, False), (8, 5, True), (5, 3, False)])
def test_frames_equal_oracle(gfx_ctx, oracle, pair, grid, log2_slot, log2_cell, randomize):
    """with the sky and 2^8 candidates, slot 23978 draws the environment's pole on frame 0 (areaPDensity 0)"""
    sc, oscene, _ = pair
    if grid == "default" and log2_slot != 3:
        pytest.skip("the oracle's builds of 4 M slots run once, at 2^3 candidates")
    sides = _sides(gfx_ctx, oracle, oscene, W, H)
    p = RS.params(sc, W, H, RS.GRIDS[grid], log2_slot=log2_slot, log2_cell=log2_cell, randomize=randomize, max_path_length=3)
    RS.put_gbuffer(sides, RS.gbuffer(sc, W, H, log2_slot))
    rng = np.random.default_rng(log2_cell).integers(0, 1 << 62, (H, W), dtype=np.int64).astype(np.uint64)
    g = regir_ref.Grid(p)
    frames = [0, 1, 2, "crafted", 3, (1 << 32) - 2, (1 << 32) - 1]
    for f in frames:
        if f == "crafted":
            slots = RS.crafted_slots(g, 1 << log2_slot, log2_slot)
            last = np.array([2, 1, 0xFFFFFFFF, 0xFFFFFFFA, 0xFFFFFFF9, 5], np.uint32)[np.arange(g.num_cells) % 6]
            for s in sides:
                s.put_linear(abi.BUF_REGIR_SLOTS, 0, slots, p)
                s.put_linear(abi.BUF_REGIR_LAST_ACCESS, 0, last, p)
            continue
        RS.set_frame(p, f)
        for s in sides:
            if f == 0:
                s.put(abi.BUF_RNG, 0, rng)
            s.build(p, f, f != 0)
            s.pathtrace(p)
        _compare_all(*sides, p, f"{grid} frame {f}")
        for s in sides:
            s.update(p, f)
        _compare_all(*sides, p, f"{grid} frame {f} after the access update")


@pytest.mark.parametrize("events", [{10: "resize"}, {12: (5, 3, 6)}], ids=["resize", "new_grid"])
def test_recreation_on_device(gfx_ctx, oracle, pair, events):
    """the re-creation sequences on the device: lastAccessFrameIndices = F - 1, every slot finite, every seen cell live, and
    the oracle's bits on every frame"""
    sc, oscene, _ = pair
    RS.check_recreation(lambda w, h: RS.DeviceSide(gfx_ctx, w, h), sc, events)
    frames = {}
    for which, side_for in (("device", lambda w, h: RS.DeviceSide(gfx_ctx, w, h)),
                            ("oracle", lambda w, h: RS.OracleSide(oracle, oscene, w, h))):
        for f, side, p, _ in RS.protocol(side_for, sc, events):
            side.pathtrace(p)
            frames[which, f] = (side.get_linear(abi.BUF_REGIR_SLOTS, p.bufferIndex, p), side.get(abi.BUF_BEAUTY_ACCUM),
                                side.get_linear(abi.BUF_REGIR_LAST_ACCESS, 0, p))
    for f in range(18):
        for k, name in enumerate(("slots", "beauty", "last access")):
            _same(frames["device", f][k], frames["oracle", f][k], f"frame {f} {name}")


def test_fullsize_build_within_restatement(gfx_ctx, oracle, pair):
    """a 1920 x 1080 frame on the default grid: the device's build of frames 0 to 2 against the restatement on a seeded
    1/16 of the cells (and the first 8, whose seeds are restated too), and every pixel of its path-traced frames"""
    sc, _, s64 = pair
    if getattr(sc, "env_map", None) is not None:
        pytest.skip("environment candidates are held to the oracle bit for bit, not restated")
    w, h = 1920, 1080
    dev = RS.DeviceSide(gfx_ctx, w, h)
    p = RS.pad_box(RS.params(sc, w, h, (0, 0, 0)))
    g = regir_ref.Grid(p)
    ref = regir_ref.RegirRef(s64)
    ref.grid = g
    n = g.num_cells * regir_ref.SLOTS
    ref.slots = [np.zeros((n, 16), np.uint32) for _ in (0, 1)]
    ref.rng = np.zeros(n, np.uint64)
    ref.rng[:4096] = regir_ref.mt19937_64(regir_ref.SEED, 4096)
    ref.last = np.full(g.num_cells, 0xFFFFFFFF, np.uint32)
    RS.set_frame(p, 0)
    RS.check_build(dev, ref, p, 0, False, np.arange(8), "1080p frame 0")
    cells = np.unique(np.concatenate([np.arange(8), np.random.default_rng(5).choice(g.num_cells, g.num_cells // 16, replace=False)]))
    gb0 = RS.gbuffer(sc, w, h, 3).reshape(-1, 4)
    gb0[: w * h // 16] = RS.face_points(g, w * h // 16, 3)
    RS.put_gbuffer([dev], gb0.reshape(h, w, 4))
    dev.put(abi.BUF_RNG, 0, np.random.default_rng(3).integers(0, 1 << 62, (h, w), dtype=np.int64).astype(np.uint64))
    nee = regir_ref.NeeRef(s64)
    for f in (0, 1, 2):
        RS.set_frame(p, f)
        if f:
            ref.load(dev, p)
            RS.check_build(dev, ref, p, f, True, cells, f"1080p frame {f}")
        before = dev.get_linear(abi.BUF_REGIR_CELL_ACCESSES, 0, p).reshape(-1).astype(np.int64)
        out = nee.frame(dev, p)
        dev.pathtrace(p)
        regir_ref.compare_frame(dev, nee, out, p, before, f"1080p frame {f}")
        dev.update(p, f)
    assert ref.steered <= STEER_LIMIT * ref.compared + 1, f"{ref.steered} of {ref.compared} slots steered"
    assert nee.steered <= STEER_LIMIT * nee.compared + 1, f"{nee.steered} of {nee.compared} pixels steered"


UW = UH = 512
REPEATS = 8


@pytest.mark.parametrize("grid,log2_slot,log2_cell,randomize,frames", [
    ("1x1x1", 3, 2, True, 1), ("5x3x6", 0, 5, False, 1), ("5x3x6", 3, 2, True, 8)])
def test_large_cells_are_unbiased(gfx_ctx, pair, grid, log2_slot, log2_cell, randomize, frames):
    sc, _, s64 = pair
    x = RS.decoded_floor_point(*POINT)
    integral = RU.integral(s64, S.CAM, point=x)
    p = RS.params(sc, UW, UH, RS.GRIDS[grid], log2_slot=log2_slot, log2_cell=log2_cell, randomize=randomize)
    means = RS.frame_means(lambda w, h: RS.DeviceSide(gfx_ctx, w, h), sc, UW, UH, p, x, frames, REPEATS)
    RU.check(means, integral[None], f"{grid}, 2^{log2_slot} x 2^{log2_cell}")


def test_cell_centre_bias(gfx_ctx, pair):
    sc, _, s64 = pair
    if getattr(sc, "env_map", None) is not None:
        pytest.skip("pinned without the sky")
    x = RS.decoded_floor_point(3.2, 0.0)
    p = RS.params(sc, UW, UH, RS.GRIDS["10x4x8"], log2_slot=0, log2_cell=2)
    means = RS.frame_means(lambda w, h: RS.DeviceSide(gfx_ctx, w, h), sc, UW, UH, p, x, 1, REPEATS)
    expected = regir_ref.expected_nee(s64, regir_ref.Grid(p), x, S.CAM, True)
    RU.check(means, expected[None], "the cell-centre bias")
