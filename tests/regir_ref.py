"""ReGIR's cell reservoirs restated in float64 - TEST INFRASTRUCTURE for tests/test_oracle_regir_ref.py and
tests/test_gpu_regir_ref.py.

Written from the reference, not from oracle/regir.inl or gfxexp_b200/csrc/regir.cu:
  build_cell_reservoirs.cu:6-69      sampleIntensity, with its `lpCos > minSquaredDistance` as written: lpCos is still 1
                                     there, so the cell-centre cosine is taken when the squared half diagonal of a cell is
                                     below 1 and assumed to be 1 otherwise
  build_cell_reservoirs.cu:71-225    buildCellReservoirsAndTemporalReuse: the idle-cell rule in uint32 arithmetic, streaming
                                     RIS over 2^k candidates, the finite check, the temporal merge with its 20x cap and length
                                     correction
  build_cell_reservoirs.cu:235-248   updateLastAccessFrameIndices and numActiveCells
  optix_pathtracing_kernels.cu:18-82 sampleFromCell's cell lookup (calcCellLinearIndex, regir_shared.h:731-742) as a
                                     probability over the jitter, for the expected value of a frame (expected_nee)
  regir_shared.h:7, 95-132           512 slots per cell; Reservoir
  regir_main.cpp:1073-1112           the grid over the scene's box (32 x 8 x 32 when a dimension is 0) and the slot seeds of
                                     std::mt19937_64(591842031321323413)
Two departures of this project are restated as the project defines them (DESIGN.md): a grid created by the build of frame F
starts with lastAccessFrameIndices = F - 1 (the reference's startup fill -1 is the case F = 0), and a previous slot with M = 0
contributes weight 0 to the temporal merge instead of 0 / 0.

Area-light candidates come from tests/restir_ref.Scene64 (the flat CDF pick and squareToTriangle); PCG32 is replayed in
integers in the oracle's draw order (uLight, uPos0, uPos1, then the update's u).  Environment candidates are not restated
pass by pass: frames with a sky are held to the oracle bit for bit (tests/test_gpu_regir_ref.py) and the estimator with it to
the direct-lighting integral (tests/restir_unbiased.py).

Margins and bars follow tests/restir_ref.py (U = 2^-24).  Decisions, each steered when inside its bar:
  * light pick: (16 + n) U against the float64 CDF boundaries;
  * isOutsideCell, per face: the float32 cell centre and half size carry a few U of |origin| + |centre| + |half|, the
    sample position a few U of |position|; bar 16 U (|origin| + |centre| + |half| + |position|), only when that face decides;
  * the sign of the cell-centre cosine (small cells only): 16 U;
  * Reservoir::update's u < w / sumW: (2 K + i + 2) U + 2 cond, relative to the ratio.
Continuous outputs (sumWeights, recPDFEstimate, targetDensity) carry (3 K + n + 8) U plus 3 cond, where cond is the
float32 conditioning of the cell target: 8 U / |cos| for the cosine and 16 U |centre| / dist for the cancellation of
position - centre.
"""
from __future__ import annotations

import numpy as np

from tests import restir_ref
from tests.restir_ref import K_CHAIN, M31, U, pcg_draw

SLOTS = 512                            # kNumLightSlotsPerCell (regir_shared.h:7)
SEED = 591842031321323413              # regir_main.cpp:1105
IDLE_AFTER = 8                         # frameIndex - lastAccessFrameIndex > 8 (build_cell_reservoirs.cu:80)
U32 = 0xFFFFFFFF


# ---- std::mt19937_64 -----------------------------------------------------------------------------------------------------------
def mt19937_64(seed: int, n: int) -> np.ndarray:
    """the first n outputs of std::mt19937_64(seed), from the generator's definition (C++ [rand.eng.mers])"""
    mask = (1 << 64) - 1
    mt = [seed & mask]
    for i in range(1, 312):
        mt.append((6364136223846793005 * (mt[-1] ^ (mt[-1] >> 62)) + i) & mask)
    out = np.empty(n, np.uint64)
    k = 312
    for j in range(n):
        if k == 312:
            for i in range(312):
                x = (mt[i] & 0xFFFFFFFF80000000) | (mt[(i + 1) % 312] & 0x7FFFFFFF)
                mt[i] = mt[(i + 156) % 312] ^ (x >> 1) ^ (0xB5026F5AA96619E9 if x & 1 else 0)
            k = 0
        y = mt[k]
        k += 1
        y ^= (y >> 29) & 0x5555555555555555
        y ^= (y << 17) & 0x71D67FFFEDA60000
        y ^= (y << 37) & 0xFFF7EEE000000000
        y ^= y >> 43
        out[j] = y
    return out


# ---- the grid ------------------------------------------------------------------------------------------------------------------
class Grid:
    """regir_main.cpp:1109-1112 over the frame's scene box, in float64 from the float32 parameters"""

    def __init__(self, p):
        dim = [int(v) for v in p.regirGridDim]
        if 0 in dim:
            dim = [32, 8, 32]
        self.dim = np.array(dim, np.int64)
        self.num_cells = int(np.prod(self.dim))
        lo = np.asarray(p.sceneAabbMin[:], np.float32).astype(np.float64)
        hi = np.asarray(p.sceneAabbMax[:], np.float32).astype(np.float64)
        self.origin = lo
        self.size = (hi - lo) / self.dim
        self.half = 0.5 * self.size
        self.min_sq = float(np.sum(self.half ** 2))
        self.uses_cosine = 1.0 > self.min_sq          # `lpCos > minSquaredDistance` with lpCos = 1

    def cell_coords(self, cells):
        cells = np.asarray(cells, np.int64)
        dx, dy = self.dim[0], self.dim[1]
        return np.stack([cells % dx, (cells % (dx * dy)) // dx, cells // (dx * dy)], -1)

    def centres(self, cells):
        return self.origin + (self.cell_coords(cells) + 0.5) * self.size

    def index_probabilities(self, point, randomize: bool):
        """{cell: probability} of calcCellLinearIndex(point + jitter) over the uniform jitter of sampleFromCell: per axis
        t = (x - origin) / size + o, o uniform in [-0.5, 0.5); C's float -> uint32 saturates below 0, then the clamp to dim - 1"""
        per_axis = []
        for a in range(3):
            t = (point[a] - self.origin[a]) / self.size[a] if self.size[a] > 0 else (np.inf if point[a] > self.origin[a] else 0.0)
            probs = {}
            if not randomize or not np.isfinite(t):
                probs[int(np.clip(np.floor(t) if np.isfinite(t) else (self.dim[a] - 1 if t > 0 else 0), 0, self.dim[a] - 1))] = 1.0
            else:
                for i in range(int(np.floor(t - 0.5)), int(np.floor(t + 0.5)) + 1):
                    w = max(0.0, min(i + 1.0, t + 0.5) - max(float(i), t - 0.5))
                    if w > 0:
                        c = int(np.clip(i, 0, self.dim[a] - 1))
                        probs[c] = probs.get(c, 0.0) + w
            per_axis.append(probs)
        out = {}
        for ix, px in per_axis[0].items():
            for iy, py in per_axis[1].items():
                for iz, pz in per_axis[2].items():
                    out[int(iz * self.dim[0] * self.dim[1] + iy * self.dim[0] + ix)] = px * py * pz
        return out


# ---- sampleIntensity (build_cell_reservoirs.cu:6-69), area samples ------------------------------------------------------------
def sample_intensity(grid: Grid, centre, pos, nrm, le):
    """-> (contribution [n, 3], steered, conditioning, cosine taken); centre [n, 3] or [3]"""
    centre = np.broadcast_to(centre, pos.shape)
    lo, hi = centre - grid.half, centre + grid.half
    below, above = pos - lo, hi - pos                     # both >= 0 on an axis where the sample is inside
    face = np.minimum(np.abs(below), np.abs(above))
    bar = 16 * U * (np.abs(grid.origin) + np.abs(centre) + grid.half + np.abs(pos))
    out_axis = (below < 0) | (above < 0)
    outside = out_axis.any(-1)
    clearly_out = (out_axis & (face >= bar)).any(-1)
    steer = ~clearly_out & (face < bar).any(-1)         # a flat grid's exact zeros decide exactly
    d = pos - centre
    dist2 = np.sum(d * d, -1)
    dist = np.sqrt(dist2)
    perp = np.sum(-d * nrm, -1)
    with np.errstate(divide="ignore", invalid="ignore"):
        cos = perp / dist
    use_cos = outside & grid.uses_cosine
    lpcos = np.where(use_cos, cos, 1.0)
    d2 = np.where(outside, dist2, grid.min_sq)
    with np.errstate(divide="ignore", invalid="ignore"):
        cont = np.where((lpcos > 0)[:, None], le / np.pi * (lpcos / d2)[:, None], 0.0)
        cond = np.where(use_cos, 8 * U / np.abs(cos), 0.0) + np.where(outside, 16 * U * np.abs(centre).max(-1) / dist, 0.0)
    steer |= use_cos & (np.abs(cos) < 16 * U)
    return cont, steer, np.where(lpcos > 0, cond, 0.0), use_cos


# ---- slots ---------------------------------------------------------------------------------------------------------------------
class Slots:
    """one slot plane [S, 16] uint32 (Reservoir<LightSample> + ReservoirInfo, one 64-byte record) in float64"""

    def __init__(self, raw: np.ndarray):
        raw = raw.reshape(-1, 16)
        f = raw.view(np.float32).astype(np.float64)
        self.le, self.sumw = f[:, 0:3], f[:, 3]
        self.pos = f[:, 4:7]
        self.m = (raw[:, 7] & M31).astype(np.int64)
        self.inf = (raw[:, 7] >> 31).astype(bool)
        self.nrm, self.rec, self.target = f[:, 8:11], f[:, 11], f[:, 12]


def idle(frame: int, last) -> np.ndarray:
    """the idle-cell rule in uint32: frameIndex - lastAccessFrameIndex > 8"""
    return ((np.uint64(frame) - np.asarray(last, np.uint64)) & np.uint64(U32)) > IDLE_AFTER


def _rel_bar(n):
    return (3 * K_CHAIN + n + 8) * U


class RegirRef:
    """the build and the access update on a system's float32 state (load()); each returns the expected outputs"""

    def __init__(self, s64: restir_ref.Scene64):
        self.s64 = s64
        self.steered = 0
        self.compared = 0

    def load(self, side, p):
        self.grid = Grid(p)
        self.slots = [side.get_linear(abi_buf("SLOTS"), i, p).copy() for i in (0, 1)]
        self.rng = side.get_linear(abi_buf("SLOT_RNG"), 0, p).reshape(-1).copy()
        self.last = side.get_linear(abi_buf("LAST_ACCESS"), 0, p).reshape(-1).copy()
        self.accesses = side.get_linear(abi_buf("CELL_ACCESSES"), 0, p).reshape(-1).copy()
        self.active = side.get_linear(abi_buf("NUM_ACTIVE_CELLS"), 0, p).reshape(-1).copy()

    # ---- buildCellReservoirsAndTemporalReuse ------------------------------------------------------------------------------
    def build(self, p, frame: int, temporal: bool, cells=None) -> dict:
        """the slots of `cells` (default all) after the build of `frame`"""
        g, s64 = self.grid, self.s64
        cells = np.arange(g.num_cells) if cells is None else np.asarray(cells, np.int64)
        live_cells = cells[~idle(frame, self.last[cells])]
        idx = (live_cells[:, None] * SLOTS + np.arange(SLOTS)[None]).reshape(-1)
        P = len(idx)
        centre = np.repeat(g.centres(live_cells), SLOTS, 0)
        rng = self.rng[idx].astype(np.uint64)
        n_cand = 1 << p.regirLog2NumCandidatesPerLightSlot
        sumw = np.zeros(P)
        sel = dict(pos=np.zeros((P, 3)), nrm=np.zeros((P, 3)), le=np.zeros((P, 3)))
        inf = np.zeros(P, bool)
        sel_target = np.zeros(P)
        steer = np.zeros(P, bool)
        cond = np.zeros(P)
        for i in range(n_cand):
            rng, ul = pcg_draw(rng)
            rng, u0 = pcg_draw(rng)
            rng, u1 = pcg_draw(rng)
            rng, u = pcg_draw(rng)
            k, lpos, lnrm, le, dens, pick_margin = s64.sample(ul, u0, u1)
            steer |= pick_margin < (16 + s64.n_lights) * U
            cont, st, cd, _ = sample_intensity(g, centre, lpos, lnrm, le)
            steer |= st
            cond = np.maximum(cond, cd)
            td = cont.mean(-1)
            w = td / dens
            sumw = sumw + w
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = w / sumw
            acc = u < ratio
            steer |= (w > 0) & (np.abs(u - ratio) < ((2 * K_CHAIN + i + 2) * U + 2 * cond) * ratio)
            for key, val in (("pos", lpos), ("nrm", lnrm), ("le", le)):
                sel[key] = np.where(acc[:, None], val, sel[key])
            sel_target = np.where(acc, td, sel_target)
        m = np.full(P, n_cand, np.int64)
        with np.errstate(divide="ignore", invalid="ignore"):
            rec = sumw / (sel_target * m)
        bad = ~np.isfinite(rec)
        rec[bad] = 0.0
        sel_target[bad] = 0.0
        n_terms = n_cand
        if temporal:
            prev = Slots(self.slots[(p.bufferIndex + 1) % 2])
            empty = rec == 0.0
            sumw[empty] = 0.0
            for key in sel:
                sel[key][empty] = 0.0
            pm = np.minimum(prev.m[idx], 20 * n_cand)
            with np.errstate(divide="ignore", invalid="ignore"):
                w = np.where(prev.m[idx] > 0, pm / prev.m[idx] * prev.sumw[idx], 0.0)
            rng, u = pcg_draw(rng)
            sumw = sumw + w
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = w / sumw
            acc = u < ratio
            steer |= (w > 0) & (np.abs(u - ratio) < ((2 * K_CHAIN + n_cand + 2) * U + 2 * cond) * ratio)
            for key, src in (("pos", prev.pos), ("nrm", prev.nrm), ("le", prev.le)):
                sel[key] = np.where(acc[:, None], src[idx], sel[key])
            inf = acc & prev.inf[idx]
            sel_target = np.where(acc, prev.target[idx], sel_target)
            m = n_cand + pm
            with np.errstate(divide="ignore", invalid="ignore"):
                rec = (1.0 / m) * sumw / sel_target
            bad = ~np.isfinite(rec)
            rec[bad] = 0.0
            sel_target[bad] = 0.0
            n_terms += 2
        return dict(idx=idx, cells=cells, live_cells=live_cells, rng=rng, m=m, inf=inf, pos=sel["pos"], le=sel["le"],
                    sumw=sumw, rec=rec, target=sel_target, steer=steer, cond=cond, n_terms=n_terms, buf=p.bufferIndex & 1)

    # ---- updateLastAccessFrameIndices --------------------------------------------------------------------------------------
    def update_access(self, p, frame: int) -> dict:
        touched = self.accesses > 0
        last = np.where(touched, np.uint32(frame & U32), self.last).astype(np.uint32)
        active = self.active.copy()
        active[p.bufferIndex & 1] += np.uint32(touched.sum())
        return dict(last=last, active=active)


def abi_buf(name: str) -> int:
    from gfxexp_b200 import abi
    return getattr(abi, "BUF_REGIR_" + name)


# ---- comparison ------------------------------------------------------------------------------------------------------------
def compare_build(side, ref: RegirRef, out: dict, p, what: str) -> int:
    """a system's slots, slot RNGs and access counts after a build against the restated ones; returns the steered count"""
    idx, steer = out["idx"], out["steer"]
    keep = ~steer
    ref.steered += int(steer.sum())
    ref.compared += len(idx)
    raw = side.get_linear(abi_buf("SLOTS"), out["buf"], p).reshape(-1, 16)
    rng = side.get_linear(abi_buf("SLOT_RNG"), 0, p).reshape(-1)
    # idle cells keep their slots and RNG states bit for bit, and every cell's access count is reset
    idle_cells = np.setdiff1d(out["cells"], out["live_cells"])
    if len(idle_cells):
        islots = (idle_cells[:, None] * SLOTS + np.arange(SLOTS)[None]).reshape(-1)
        restir_ref._exact(raw[islots], ref.slots[out["buf"]].reshape(-1, 16)[islots], f"{what}: an idle cell's slots", islots)
        restir_ref._exact(rng[islots], ref.rng[islots], f"{what}: an idle cell's slot RNG", islots)
    acc = side.get_linear(abi_buf("CELL_ACCESSES"), 0, p).reshape(-1)[out["cells"]]
    restir_ref._exact(acc, np.zeros_like(acc), f"{what}: perCellNumAccesses after the build", out["cells"])
    got = Slots(raw[idx])
    k = idx[keep]
    restir_ref._exact(rng[idx][keep], out["rng"][keep], f"{what}: slot RNG state", k)
    restir_ref._exact(got.m[keep], out["m"][keep], f"{what}: M", k)
    restir_ref._exact(got.inf[keep], out["inf"][keep], f"{what}: atInfinity", k)
    restir_ref._close(got.pos[keep], out["pos"][keep], 1e-4, f"{what}: the held light sample", k, absolute=True)
    restir_ref._close(got.le[keep], out["le"][keep], 1e-6, f"{what}: the held emittance", k)
    bar = _rel_bar(out["n_terms"]) + 3 * out["cond"][keep]
    restir_ref._close(got.sumw[keep], out["sumw"][keep], bar, f"{what}: sumWeights", k)
    restir_ref._close(got.rec[keep], out["rec"][keep], bar, f"{what}: recPDFEstimate", k)
    restir_ref._close(got.target[keep], out["target"][keep], bar, f"{what}: targetDensity", k)
    return int(steer.sum())


def compare_update(side, out: dict, p, what: str):
    last = side.get_linear(abi_buf("LAST_ACCESS"), 0, p).reshape(-1)
    restir_ref._exact(last, out["last"], f"{what}: lastAccessFrameIndices", np.arange(len(last)))
    active = side.get_linear(abi_buf("NUM_ACTIVE_CELLS"), 0, p).reshape(-1)
    restir_ref._exact(active, out["active"], f"{what}: numActiveCells", np.arange(2))


# ---- the expected value of a frame at maxPathLength 2 ----------------------------------------------------------------------
def cell_target_mask(grid: Grid, cell: int):
    """the support of cell `cell`'s target as a mask over area-light points (pos, nrm) -> bool"""
    centre = grid.centres([cell])[0]

    def mask(pos, nrm):
        cont, _, _, _ = sample_intensity(grid, centre, pos, nrm, np.ones_like(pos))
        return cont[:, 0] > 0
    return mask


def expected_nee(s64, grid: Grid, point, cam, randomize: bool, **integral_kw) -> np.ndarray:
    """sum over the cells the jitter reaches of P(cell) x the direct lighting of the point over that cell's target support:
    two-stage RIS with a target that is zero on part of the emitters estimates the integral over the rest"""
    from tests import restir_unbiased
    total = np.zeros(3)
    for cell, prob in grid.index_probabilities(point, randomize).items():
        total += prob * restir_unbiased.integral(s64, cam, point=point, mask=cell_target_mask(grid, cell), **integral_kw)
    return total


# ---- sampleFromCell / performNextEventEstimation<true> and the frame at maxPathLength 2 (optix_pathtracing_kernels.cu) -----
def surface_points(scene, gb0):
    """computeSurfacePoint from G-buffer 0 (instance, geometry, primitive, 16-bit barycentrics) in float64: position, geometric
    normal, shading normal and material of each pixel; the scene's instances have identity transforms"""
    inst = scene.instances[0]
    assert np.allclose(np.asarray(inst.transform, np.float64)[:, :3], np.eye(3)) and not np.asarray(inst.transform)[:, 3].any()
    geom, prim = gb0[:, 1].astype(np.int64), gb0[:, 2].astype(np.int64)
    b = (gb0[:, 3] & 0xFFFF).astype(np.float32) / np.float32(65535)
    c = (gb0[:, 3] >> 16).astype(np.float32) / np.float32(65535)
    b, c = b.astype(np.float64), c.astype(np.float64)
    a = 1 - (b + c)
    pos, ng, ns, mat = (np.zeros((len(gb0), 3)), np.zeros((len(gb0), 3)), np.zeros((len(gb0), 3)), np.zeros(len(gb0), np.int64))
    for g in np.unique(geom):
        mesh = scene.meshes[inst.mesh_slots[g]]
        sel = geom == g
        tri = mesh.triangles.astype(np.int64)[prim[sel]]
        v = mesh.positions.astype(np.float64)[tri]
        n = mesh.normals.astype(np.float64)[tri]
        w = np.stack([a[sel], b[sel], c[sel]], -1)[..., None]
        pos[sel] = (w * v).sum(1)
        e = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
        ng[sel] = e / np.linalg.norm(e, axis=-1, keepdims=True)
        sn = (w * n).sum(1)
        ns[sel] = sn / np.linalg.norm(sn, axis=-1, keepdims=True)
        mat[sel] = mesh.material
    return pos, ng, ns, mat


def _cell_axis(t, dim, bar):
    """calcCellLinearIndex on one axis: C's float -> uint32 saturates (negative and NaN -> 0, +inf -> max), then the clamp to
    dim - 1; the index changes at the integers 1 .. dim - 1, steered within `bar` of one"""
    with np.errstate(invalid="ignore"):
        i = np.where(np.isnan(t) | (t < 0), 0.0, np.where(np.isinf(t), float(dim - 1), np.floor(np.minimum(t, 2.0 ** 33))))
    i = np.minimum(i, dim - 1).astype(np.int64)
    near = np.clip(np.round(t), 1, max(dim - 1, 1))
    steer = np.isfinite(t) & (dim > 1) & (np.abs(t - near) < bar)
    return i, steer


class NeeRef:
    """the ReGIR frame at maxPathLength 2 (first-hit emission + one ReGIR next-event estimation) per pixel, on a system's
    float32 G-buffer 0, pixel RNGs and slots; sky pixels show the 0.001 background (scenes without a sky)"""

    def __init__(self, s64: restir_ref.Scene64):
        self.s64 = s64
        self.steered = 0
        self.compared = 0

    def frame(self, side, p) -> dict:
        from gfxexp_b200 import abi
        s64, g = self.s64, Grid(p)
        assert getattr(s64.scene, "env_map", None) is None and p.maxPathLength == 2
        buf = p.bufferIndex & 1
        gb0 = side.get(abi.BUF_GBUFFER0, buf).reshape(-1, 4)
        rng_all = side.get(abi.BUF_RNG, 0).reshape(-1).astype(np.uint64)
        slots = Slots(side.get_linear(abi_buf("SLOTS"), buf, p))
        idx = np.flatnonzero(gb0[:, 0] != U32)
        P = len(idx)
        cam = np.asarray(p.camera.position[:], np.float32).astype(np.float64)
        pos, ng, ns, mat = surface_points(s64.scene, gb0[idx])
        v = cam - pos
        dist = np.linalg.norm(v, axis=-1)
        fh = np.sum(v * ng, -1)
        steer = np.abs(fh) < 16 * U * dist
        front = np.where(fh >= 0, 1.0, -1.0)
        sp = restir_ref.ShadingPoints.__new__(restir_ref.ShadingPoints)
        t, _ = restir_ref.shading_ref.make_coordinate_system(ns)
        sp.pos = restir_ref.offset_ray_origin(pos.astype(np.float32), front[:, None] * ng)
        sp.n, sp.t = ns, t
        sp.b = np.cross(ns, t)
        sp.vout_local = sp.to_local(v / dist[:, None])
        sp.mat, sp.s64, sp.dist = mat, s64, dist
        # emission, decided by vOutLocal.z > 0 (bar 16 U)
        le = s64.emittance[mat]
        contrib = np.where((sp.vout_local[:, 2] > 0)[:, None], le / np.pi, 0.0)
        steer |= (np.abs(sp.vout_local[:, 2]) < 16 * U) & le.any(-1)
        rng = rng_all[idx].copy()
        # the cell: three jitter draws, then calcCellLinearIndex
        q = sp.pos.copy()
        if p.regirEnableCellRandomization:
            for a in range(3):
                rng, u = pcg_draw(rng)
                q[:, a] = q[:, a] + g.size[a] * (u - 0.5)
        cell = np.zeros(P, np.int64)
        stride = 1
        for a in range(3):
            with np.errstate(divide="ignore", invalid="ignore"):
                ta = (q[:, a] - g.origin[a]) / g.size[a]
            bar = 64 * U * (np.abs(q[:, a]) + np.abs(g.origin[a]) + g.size[a]) / max(g.size[a], 1e-30)
            ia, st = _cell_axis(ta, int(g.dim[a]), bar)
            steer |= st
            cell += ia * stride
            stride *= int(g.dim[a])
        accesses = np.bincount(cell[~steer], minlength=g.num_cells)
        # resampling of 2^k slots of the cell
        n_res = 1 << p.regirLog2NumCandidatesPerCell
        sumw = np.zeros(P)
        m_total = np.zeros(P, np.int64)
        sel = dict(pos=np.zeros((P, 3)), nrm=np.zeros((P, 3)), le=np.zeros((P, 3)))
        inf = np.zeros(P, bool)
        sel_td = np.zeros(P)
        lobe = sp.lobe_bar()
        for i in range(n_res):
            rng, u = pcg_draw(rng)
            slot = cell * SLOTS + np.minimum(np.floor(u * SLOTS), SLOTS - 1).astype(np.int64)
            m = slots.m[slot]
            m_total += m                                   # dead slots still count their M
            live = slots.rec[slot] != 0.0
            cont, _ = sp.direct(slots.pos[slot], slots.nrm[slot], slots.le[slot], slots.inf[slot], False)
            lobe = np.maximum(lobe, np.where(live, sp.lobe_bar() + sp.cond, 0.0))
            td = cont.mean(-1)
            w = td * slots.rec[slot] * m
            uu = np.zeros(P)
            if live.any():
                rng_l, u_l = pcg_draw(rng[live])
                rng[live] = rng_l
                uu[live] = u_l
            sumw = np.where(live, sumw + w, sumw)
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = w / sumw
            acc = live & (uu < ratio)
            steer |= live & (w > 0) & (np.abs(uu - ratio) < ((2 * K_CHAIN + i + 2) * U + 2 * lobe) * ratio)
            for key, src in (("pos", slots.pos), ("nrm", slots.nrm), ("le", slots.le)):
                sel[key] = np.where(acc[:, None], src[slot], sel[key])
            inf = np.where(acc, slots.inf[slot], inf)
            sel_td = np.where(acc, td, sel_td)
        with np.errstate(divide="ignore", invalid="ignore"):
            est = (1.0 / m_total) * sumw / sel_td
        est = np.where(np.isfinite(est), est, 0.0)
        go = est > 0
        if go.any():
            sub = restir_ref.ShadingPoints.__new__(restir_ref.ShadingPoints)
            sub.__dict__.update({k: (val[go] if isinstance(val, np.ndarray) else val) for k, val in sp.__dict__.items()})
            cont, amb = sub.direct(sel["pos"][go], sel["nrm"][go], sel["le"][go], inf[go], True)   # tmax 0.9999 dist / 1e10
            contrib[go] += cont * est[go][:, None]
            steer[go] |= amb
        rng, _ = pcg_draw(rng)                               # sampleThroughput's two draws; then the path ends at length 2
        rng, _ = pcg_draw(rng)
        return dict(idx=idx, rng=rng, beauty=contrib, steer=steer, lobe=lobe, n_terms=n_res + 4, accesses=accesses,
                    n_steered_accesses=int(steer.sum()), sky=np.flatnonzero(gb0[:, 0] == U32))


def compare_frame(side, ref: NeeRef, out: dict, p, accesses_before, what: str) -> int:
    """a system's beauty, pixel RNGs and per-cell access counts after a ReGIR path-tracing launch against the restated ones"""
    from gfxexp_b200 import abi
    idx, steer = out["idx"], out["steer"]
    keep = ~steer
    ref.steered += int(steer.sum())
    ref.compared += len(idx)
    beauty = side.get(abi.BUF_BEAUTY_ACCUM, 0).reshape(-1, 4).astype(np.float64)
    restir_ref._exact(beauty[out["sky"], :3], np.full((len(out["sky"]), 3), np.float32(0.001)).astype(np.float64),
                      f"{what}: sky background", out["sky"])
    rng = side.get(abi.BUF_RNG, 0).reshape(-1)[idx]
    restir_ref._exact(rng[keep], out["rng"][keep], f"{what}: pixel RNG", idx[keep])
    bar = _rel_bar(out["n_terms"]) + 3 * out["lobe"][keep]
    restir_ref._close(beauty[idx[keep], :3], out["beauty"][keep], bar[:, None], f"{what}: beauty", idx[keep])
    got = side.get_linear(abi_buf("CELL_ACCESSES"), 0, p).reshape(-1).astype(np.int64) - accesses_before
    want = out["accesses"]
    bad = (got < want) | (got > want + out["n_steered_accesses"])
    assert not bad.any() and got.sum() == len(idx), \
        f"{what}: perCellNumAccesses off at {int(bad.sum())} cells, {int(got.sum())} accesses for {len(idx)} pixels"
    return int(steer.sum())
