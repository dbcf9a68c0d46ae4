"""Seeded ReGIR inputs over tests/restir_scenes.py's 36-triangle scene, and the two systems under test - TEST INFRASTRUCTURE
for tests/test_oracle_regir_ref.py and tests/test_gpu_regir_ref.py.

The ReGIR path tracer reads only G-buffer 0, (instance, geometry instance, primitive, quantised barycentrics), and recomputes
the surface point from the triangle.  gbuffer() writes it directly: points on every triangle of the scene (the floor, which is
the scene box's lower face, the emitters, and the box's faces, many of them seen from behind), and sky pixels.
point_gbuffer() puts every pixel on one floor point, so a frame's mean estimates that point's direct lighting.

Grids: 1 x 1 x 1, 5 x 3 x 6 (90 cells, not a multiple of 32), 8 x 4 x 8, 10 x 4 x 8, the default (dimensions 0 -> 32 x 8 x 32)
and, on the flat scene (floor only, a box of height 0), 4 x 2 x 4 with a cell height of 0.  Over the scene's box
[-4, 4] x [0, 3] x [-4, 4] the squared half diagonal of a cell is 34.25, 1.33 and 9.3 (flat) for the large grids and 0.64,
0.55 and 0.066 for the small ones, so both branches of sampleIntensity's `lpCos > minSquaredDistance` run.
"""
from __future__ import annotations

import numpy as np

from gfxexp_b200 import abi, scenes
from tests import light_scenes, regir_ref, restir_scenes as S

F32 = np.float32
SKY = 0xFFFFFFFF
GRIDS = {"1x1x1": (1, 1, 1), "5x3x6": (5, 3, 6), "8x4x8": (8, 4, 8), "10x4x8": (10, 4, 8), "default": (0, 0, 0)}
LARGE_CELLS = ("1x1x1", "5x3x6")
SMALL_CELLS = ("8x4x8", "10x4x8", "default")
# the floor quad of restir_scenes.scene() is geometry 0: triangle 1 is p0 + b (p2 - p0) + c (p3 - p0) over
# p0 = (-4, 0, -4), p2 = (4, 0, 4), p3 = (4, 0, -4)
FLOOR_GEOM, FLOOR_TRI1 = 0, 1


def scene(with_env: bool = False) -> scenes.Scene:
    return S.scene(with_env)


def flat_scene() -> scenes.Scene:
    """the floor and an emitter quad in its plane: the scene's box, and so every cell, has height 0 (as in a furnace plane)"""
    tm = light_scenes.tri_mesh
    meshes = [tm(S._quad((0, 0, 0), (0, 0, 4), (4, 0, 0)), S.DS3), tm(S._quad((0.5, 0.0, -0.5), (0.6, 0, 0), (0, 0, 0.6)), S.EMIT_A)]
    return scenes.Scene(meshes, S._materials(), [scenes.make_instance([0, 1])], S.CAM.astype(F32),
                        scenes.look_at_orientation(tuple(S.CAM), (0.0, 0.0, 0.0)).astype(F32), 0.8, name="regir_flat")


def params(sc, W, H, grid, frame=0, log2_slot=3, log2_cell=2, randomize=True, max_path_length=2):
    p = S.frame_params(sc, W, H, frame)
    p.regirGridDim = (abi.c_u32 * 3)(*grid)
    p.regirLog2NumCandidatesPerLightSlot = log2_slot
    p.regirLog2NumCandidatesPerCell = log2_cell
    p.regirEnableCellRandomization = 1 if randomize else 0
    p.maxPathLength = max_path_length
    p.numAccumFrames = 0
    return p


def pad_box(p):
    """the grid over [-4.1, 4.1] x [0, 3.3] x [-4.1, 4.1] instead of the scene's box: the ceiling emitter lies on the box's
    upper face and the vertical emitter on faces of the default grid, where float32 rounding alone decides isOutsideCell"""
    p.sceneAabbMin = (abi.c_f * 3)(-4.1, 0.0, -4.1)
    p.sceneAabbMax = (abi.c_f * 3)(4.1, 3.3, 4.1)
    return p


def set_frame(p, frame):
    p.frameIndex, p.bufferIndex = frame, frame % 2


def floor_bc(x, z):
    """(b, c) on the floor's triangle 1 of the point (x, 0, z), x >= z"""
    b = (z + 4) / 8
    return b, (x + 4) / 8 - b


def quantise(v):
    return np.round(np.asarray(v, np.float64) * 65535).astype(np.uint32)


def decoded_floor_point(x, z):
    """the float64 position of the floor point (x, 0, z) after the G-buffer's 16-bit barycentrics"""
    b, c = floor_bc(x, z)
    qb, qc = quantise(b), quantise(c)
    b, c = float(F32(qb / F32(65535))), float(F32(qc / F32(65535)))
    p0, p2, p3 = np.array([-4.0, 0, -4]), np.array([4.0, 0, 4]), np.array([4.0, 0, -4])
    return (1 - b - c) * p0 + b * p2 + c * p3


def point_gbuffer(W, H, x, z) -> np.ndarray:
    b, c = floor_bc(x, z)
    gb0 = np.zeros((H, W, 4), np.uint32)
    gb0[..., 1] = FLOOR_GEOM
    gb0[..., 2] = FLOOR_TRI1
    gb0[..., 3] = quantise(b) | (quantise(c) << 16)
    return gb0


def gbuffer(sc, W, H, seed) -> np.ndarray:
    """points on every triangle, 10 % sky, a third of them on the floor (the box's lower face)"""
    rng = np.random.default_rng(seed)
    n = W * H
    tris = [(g, t) for g, mesh in enumerate(sc.meshes) for t in range(len(mesh.triangles))]
    pick = rng.integers(0, len(tris), n)
    floor = rng.random(n) < 0.33
    geom = np.where(floor, FLOOR_GEOM, [tris[k][0] for k in pick])
    prim = np.where(floor, rng.integers(0, 2, n), [tris[k][1] for k in pick])
    b = rng.random(n)
    c = rng.random(n) * (1 - b)
    gb0 = np.zeros((n, 4), np.uint32)
    gb0[:, 1], gb0[:, 2] = geom, prim
    gb0[:, 3] = quantise(b) | (quantise(c) << 16)
    gb0[rng.random(n) < 0.1, 0] = SKY
    return gb0.reshape(H, W, 4)


def face_points(grid: regir_ref.Grid, n: int, seed: int) -> np.ndarray:
    """G-buffer-0 rows [n, 4] of floor points 1e-3 of a cell to either side of the grid's x and z cell faces, and one in 16 on
    the face itself (as near as 16-bit barycentrics get; those within their bar are steered)"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4), np.uint32)
    for j in range(n):
        axis = 0 if j % 2 == 0 else 2
        k = rng.integers(1, max(int(grid.dim[axis]), 2))
        off = 0.0 if j // 2 % 16 == 0 else (1e-3 if j // 2 % 2 else -1e-3)   # one in 16 on the face
        face = grid.origin[axis] + k * grid.size[axis] + off * grid.size[axis]
        other = rng.uniform(-3.9, 3.9)
        x, z = (face, other) if axis == 0 else (other, face)
        if x < z:                                      # the floor's triangle 1 holds x >= z; mirror into it
            x, z = z, x
        b, c = floor_bc(np.clip(x, -3.99, 3.99), np.clip(z, -3.99, 3.99))
        out[j, 1], out[j, 2], out[j, 3] = FLOOR_GEOM, FLOOR_TRI1, quantise(b) | (quantise(c) << 16)
    return out


def crafted_slots(grid: regir_ref.Grid, n_cand: int, seed: int) -> np.ndarray:
    """a previous slot plane [S, 16]: live slots with M on both sides of the 20x cap (20 N - 1, 20 N, 20 N + 1) and far
    above it, M = 0 (a slot never built), recPDFEstimate = 0, and samples at infinity"""
    rng = np.random.default_rng(seed)
    s = grid.num_cells * regir_ref.SLOTS
    cap = 20 * n_cand
    m = rng.choice(np.array([1, n_cand, cap - 1, cap, cap + 1, 50 * cap, 0], np.uint32), s)
    inf = rng.random(s) < 0.15
    d = rng.normal(size=(s, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    pos = np.where(inf[:, None], d, rng.uniform(-3, 3, (s, 3)))
    raw = np.zeros((s, 16), np.uint32)
    raw[:, 0:3] = rng.uniform(1, 10, (s, 3)).astype(F32).view(np.uint32)
    raw[:, 3] = np.where(m > 0, rng.uniform(0.01, 5, s), 0.0).astype(F32).view(np.uint32)
    raw[:, 4:7] = pos.astype(F32).view(np.uint32)
    raw[:, 7] = m | (inf.astype(np.uint32) << 31)
    raw[:, 8:11] = (-d).astype(F32).view(np.uint32)
    raw[:, 11] = np.where((m > 0) & (rng.random(s) > 0.1), rng.uniform(0.01, 3, s), 0.0).astype(F32).view(np.uint32)
    raw[:, 12] = rng.uniform(0.01, 1, s).astype(F32).view(np.uint32)
    return raw


# ---- the systems under test ------------------------------------------------------------------------------------------------
class OracleSide:
    def __init__(self, oracle, oscene, W, H):
        self.frame = oracle.OracleFrame(oscene, W, H)

    def put(self, buf, idx, arr):
        v = self.frame.buffer(buf, idx, copy=False)
        v[...] = np.ascontiguousarray(arr).view(v.dtype).reshape(v.shape)

    def get(self, buf, idx=0):
        return self.frame.buffer(buf, idx)

    def put_linear(self, buf, idx, arr, p):
        v = self.frame.linear_buffer(buf, idx, copy=False, params=p)
        v[...] = np.ascontiguousarray(arr).view(v.dtype).reshape(v.shape)

    def get_linear(self, buf, idx, p):
        return self.frame.linear_buffer(buf, idx, params=p)

    def build(self, p, frame, temporal):
        self.frame.regir_build_cells(p, frame, temporal)

    def update(self, p, frame):
        self.frame.regir_update_access(p, frame)

    def pathtrace(self, p):
        self.frame.pathtrace(p, abi.PT_REGIR)

    def gbuffer(self, p):
        self.frame.gbuffer(p)


class DeviceSide:
    def __init__(self, ctx, W, H):
        self.ctx = ctx
        ctx.create_frame(W, H)

    def put(self, buf, idx, arr):
        self.ctx.upload(buf, idx, np.ascontiguousarray(arr))

    def get(self, buf, idx=0):
        self.ctx.synchronize()
        return self.ctx.download(buf, idx)

    def put_linear(self, buf, idx, arr, p):
        self.ctx.upload(buf, idx, np.ascontiguousarray(arr))

    def get_linear(self, buf, idx, p):
        self.ctx.synchronize()
        return self.ctx.download_linear(buf, idx, params=p)

    def build(self, p, frame, temporal):
        self.ctx.regir_build_cells(p, frame, temporal)

    def update(self, p, frame):
        self.ctx.regir_update_access(p, frame)

    def pathtrace(self, p):
        self.ctx.pathtrace(p, abi.PT_REGIR)

    def gbuffer(self, p):
        self.ctx.gbuffer(p)


def put_gbuffer(sides, gb0):
    for s in sides:
        for i in (0, 1):
            s.put(abi.BUF_GBUFFER0, i, gb0)


def frame_means(make_side, sc, W, H, p, point, frames, repeats):
    """[repeats, 1, 3]: the mean beauty of the last of `frames` ReGIR frames with every pixel at the floor point `point`; each
    repeat reseeds the pixel RNGs and the slot RNGs (pixels share slots, so they are correlated within a repeat)"""
    out = []
    for r in range(repeats):
        side = make_side(W, H)
        put_gbuffer([side], point_gbuffer(W, H, point[0], point[2]))
        set_frame(p, 0)
        side.build(p, 0, False)                 # creates the grid; the slot RNGs are reseeded below
        grid = regir_ref.Grid(p)
        seeds = np.random.default_rng(1000 + r)
        side.put_linear(abi.BUF_REGIR_SLOT_RNG, 0,
                        seeds.integers(0, 1 << 62, grid.num_cells * regir_ref.SLOTS, dtype=np.int64).astype(np.uint64), p)
        side.put(abi.BUF_RNG, 0, seeds.integers(0, 1 << 62, (H, W), dtype=np.int64).astype(np.uint64))
        for f in range(frames):
            set_frame(p, f)
            side.build(p, f, f > 0)
            side.pathtrace(p)
            side.update(p, f)
        out.append([side.get(abi.BUF_BEAUTY_ACCUM, 0)[..., :3].reshape(-1, 3).mean(0)])
    return np.array(out)


# ---- shared test steps -----------------------------------------------------------------------------------------------------------
def check_build(side, ref: "regir_ref.RegirRef", p, frame, temporal, cells, what):
    """one build on `side` against the restatement of the same build on the side's state before it"""
    out = ref.build(p, frame, temporal, cells)
    side.build(p, frame, temporal)
    regir_ref.compare_build(side, ref, out, p, what)
    return out


def protocol(side_for, sc, events, frames=18, grid=(8, 4, 8)):
    """frames 0 .. frames - 1 of regir_main.cpp's loop on a camera's G-buffer: build (temporal unless a new sequence), path trace,
    access update.  `events[f]` is "resize" (a new 80 x 36 frame, a new sequence) or a new grid; yields (frame, side, p,
    created) after the build, created when that build made a new grid; the caller path-traces"""
    side = side_for(64, 36)
    p = params(sc, 64, 36, grid, max_path_length=2)
    for f in range(frames):
        new_sequence = f == 0
        ev = events.get(f)
        if ev == "resize":
            side = side_for(80, 36)
            p = params(sc, 80, 36, tuple(p.regirGridDim), max_path_length=2)
            new_sequence = True
        elif ev is not None:
            p.regirGridDim = (abi.c_u32 * 3)(*ev)
        set_frame(p, f)
        side.gbuffer(p)
        side.build(p, f, not new_sequence)
        yield f, side, p, f == 0 or ev is not None
        side.update(p, f)


def check_recreation(side_for, sc, events):
    """every slot finite on every frame; a grid created by the build of frame F starts with lastAccessFrameIndices = F - 1,
    and from F on every cell the camera sees has a live slot"""
    created_at = None
    for f, side, p, created in protocol(side_for, sc, events):
        if created:
            created_at = f
            last = side.get_linear(abi.BUF_REGIR_LAST_ACCESS, 0, p).reshape(-1)
            assert (last == np.uint32((f - 1) & 0xFFFFFFFF)).all(), f"frame {f}: a new grid's lastAccessFrameIndices {np.unique(last)}"
        side.pathtrace(p)
        slots = regir_ref.Slots(np.concatenate([side.get_linear(abi.BUF_REGIR_SLOTS, i, p) for i in (0, 1)]))
        assert np.isfinite(slots.sumw).all(), f"frame {f}: {int((~np.isfinite(slots.sumw)).sum())} slots hold a non-finite sumWeights"
        cur = regir_ref.Slots(side.get_linear(abi.BUF_REGIR_SLOTS, p.bufferIndex, p))
        seen = np.flatnonzero(side.get_linear(abi.BUF_REGIR_CELL_ACCESSES, 0, p).reshape(-1) > 0)
        live = (cur.rec.reshape(-1, regir_ref.SLOTS) > 0).any(1)
        assert len(seen) and live[seen].all(), f"frame {f}: {int((~live[seen]).sum())} of {len(seen)} seen cells have no live slot"
        assert np.isfinite(side.get(abi.BUF_BEAUTY_ACCUM)[..., :3]).all()
    assert created_at is not None
