"""The original ReSTIR DI passes restated in float64 - TEST INFRASTRUCTURE for tests/test_oracle_restir_ref.py and
tests/test_gpu_restir_ref.py.

Written from restir_di/gpu_kernels/optix_restir_di_kernels.cu and restir_di_shared.h, not from oracle/render.cpp or
gfxexp_b200/csrc/restir.cu:
  optix_restir_di_kernels.cu:14-287   performInitialRIS / performInitialAndTemporalRIS{Biased,Unbiased}
  optix_restir_di_kernels.cu:303-547  performSpatialRIS{Biased,Unbiased}
  optix_restir_di_kernels.cu:559-637  shading
  restir_di_shared.h:106-139          Reservoir (a full uint32_t stream length)
  restir_di_shared.h:320-516          sampleLight<false> for area lights (the pick is the flat CDF of tests/light_ref.py)
  restir_di_shared.h:518-582          performDirectLighting, evaluateVisibility (tmax = 0.9999 dist, 1e10 at infinity)
  restir_di_shared.h:747-771          testNeighbor
  common_shared.h:116-138             PCG32RNG, replayed exactly in integers with the reference's draw order
The BSDFs and decoders are tests/shading_ref.py's.  Visibility is a brute-force float64 ray / triangle test over every
triangle of the scene.  The environment light is not restated pass by pass: frames with one are held to the oracle bit for bit
(tests/test_gpu_restir_ref.py), and the oracle's and the device's estimators with it to the direct-lighting integral
(tests/restir_unbiased.py).

Each pass runs on the float32 inputs of a system under test (load()), so a pass is compared in isolation.  Every discrete
decision gets a margin and a first-order float32 bar; a pixel with any decision inside its bar is *steered*: it is left out
of the comparison and counted, and the tests bound how many there are.  U = 2^-24 is float32's unit roundoff.
  * light pick: |ul - C_k| against the float64 CDF boundaries C_k.  The float32 pick rescales ul by three float32
    integrals and subtracts float32 CDFs built by sequential sums; each step moves ul by a few U at most, and the scan of
    n weights by n U.  Bar: (16 + n) U.
  * Reservoir::update's u < w / sumW: the float32 weight is a chain of K <= 64 roundings (the BRDF's powers and square
    roots, G, the densities), sumW adds one U per term, so the ratio carries (2 K + n + 1) U, n the number of updates.
  * testNeighbor: |d' - d| / d against 0.1 with d, d' float32 lengths (4 U each, amplified by d / |d' - d| ~ 10), the dot
    product of two decoded normals against 0.9 (polar decoding: 8 U per component).  Bars 64 U and 32 U.
  * frontHit: dot(vOut, n_g) = 0, bar 16 U |vOut|; shading's emission test vOutLocal.z > 0, bar 16 U.
  * neighbour coordinates: the truncation of x + 0.5 + delta at the nonzero integers ((-1, 1) truncates to 0); bar
    16 U (|x| + 1 + |delta|) plus, for random neighbours, 16 U radius for sqrt and the float32 sin / cos.
  * visibility: a triangle decides the ray when its barycentrics and its distance (against 0 and 0.9999 dist) clear
    1e-5: float32 vertices and origins of magnitude <= 20 over edges >= 0.1 give barycentric errors of 20 / 0.1 x 8 U.
Continuous outputs are compared with a relative bar of (3 K + n + 8) U, n the number of terms in the longest sum, plus
three times the GGX lobe term (16 U / alpha, see Scene64) of the materials a pass evaluates; the acceptance ratio's bar
takes twice that term as well.
"""
from __future__ import annotations

import numpy as np

from gfxexp_b200 import abi
from tests import light_ref, shading_ref

U = 2.0 ** -24
K_CHAIN = 64
PCG_MUL = np.uint64(6364136223846793005)
M31 = (1 << 31) - 1
SKY = 0xFFFFFFFF
VIS_BAR = 1e-5


# ---- PCG32 (common_shared.h:116-138) ---------------------------------------------------------------------------------------
def pcg_draw(state: np.ndarray):
    """(next state, getFloat0cTo1o) for every state of the array"""
    with np.errstate(over="ignore"):
        new = state * PCG_MUL + np.uint64(1)
    xs = (((state >> np.uint64(18)) ^ state) >> np.uint64(27)) & np.uint64(0xFFFFFFFF)
    rot = state >> np.uint64(59)
    out = ((xs >> rot) | (xs << ((np.uint64(32) - rot) & np.uint64(31)))) & np.uint64(0xFFFFFFFF)
    return new, (out >> np.uint64(9)).astype(np.float64) * 2.0 ** -23


def halton(base: int, i: int) -> float:
    """the radical inverse of i in base, in float64"""
    r, s = 0.0, 1.0
    while i:
        s /= base
        r += (i % base) * s
        i //= base
    return r


def neighbor_deltas() -> np.ndarray:
    """restir_di_main.cpp:1534-1540: concentricSampleDisk(Halton2(i), Halton3(i)), i < 1024"""
    u0 = np.array([halton(2, i) for i in range(1024)])
    u1 = np.array([halton(3, i) for i in range(1024)])
    return np.stack(shading_ref.concentric_sample_disk(u0, u1), -1)


def offset_ray_origin(p32: np.ndarray, n: np.ndarray) -> np.ndarray:
    """common_device.cuh:112-140 on float32 positions: integer steps of the float bits, a float offset near the origin"""
    p32 = np.asarray(p32, np.float32)
    off = np.trunc(256.0 * n).astype(np.int64)
    bits = p32.view(np.int32).astype(np.int64) + np.where(p32 < 0, -1, 1) * off
    p1 = bits.astype(np.int32).view(np.float32).astype(np.float64)
    p2 = p32.astype(np.float64) + n / 65536.0
    return np.where(np.abs(p32) < 1.0 / 32.0, p2, p1)


def _dot(a, b):
    return np.sum(a * b, -1)


def _int_margin(v, keep_zero=True):
    """distance of v to the nearest integer at which C's (int) truncation changes (every nonzero integer)"""
    r = np.round(v)
    r = np.where(r == 0, np.where(v >= 0, 1.0, -1.0), r) if keep_zero else r
    return np.abs(v - r)


class Scene64:
    """the emitters, triangles and materials of a scenes.Scene in float64"""

    def __init__(self, scene):
        self.scene = scene
        self.em = light_ref.emitters(scene)
        self.cdf = np.concatenate([[0.0], np.cumsum(self.em.prob)])
        self.n_lights = len(self.em.prob)
        tris = []
        for inst in scene.instances:
            xf = np.asarray(inst.transform, np.float64)
            for slot in inst.mesh_slots:
                mesh = scene.meshes[slot]
                p = mesh.positions.astype(np.float64)[mesh.triangles.astype(np.int64)]
                tris.append(p @ xf[:, :3].T + xf[:, 3])
        self.tris = np.concatenate(tris)
        self.e1 = self.tris[:, 1] - self.tris[:, 0]
        self.e2 = self.tris[:, 2] - self.tris[:, 0]
        m = scene.materials
        self.bsdfs = [shading_ref.setup(int(m["bsdfType"][k]), m["p0"][k], m["p1"][k], m["p2"][k]) for k in range(len(m))]
        self.emittance = np.where(m["hasEmittance"][:, None] != 0, m["emittance"].astype(np.float64), 0.0)
        # GGX's D = alpha^2 / (pi (m_x^2 + m_y^2 + alpha^2 m_z^2)^2) turns an absolute error of ~4 U in the half vector into a
        # relative one of ~16 U / alpha near its peak
        self.lobe_bar = np.array([0.0 if b.type == 0 else 16 * U / b.roughness ** 2 for b in self.bsdfs])

    # -- sampleLight<false> for area lights -------------------------------------------------------------------------------
    def sample(self, ul, u0, u1):
        """-> (light index, position, normal, emittance, area density, pick margin)"""
        k = np.clip(np.searchsorted(self.cdf, ul, side="right") - 1, 0, self.n_lights - 1)
        inner = self.cdf[1:-1]
        margin = np.min(np.abs(ul[:, None] - inner[None, :]), axis=1) if inner.size else np.full(ul.shape, np.inf)
        a, b, c = light_ref.square_to_triangle(u0, u1)
        w = self.em.world[k]
        pos = a[:, None] * w[:, 0] + b[:, None] * w[:, 1] + c[:, None] * w[:, 2]
        nrm = self.em.normals[k]
        n = a[:, None] * nrm[:, 0] + b[:, None] * nrm[:, 1] + c[:, None] * nrm[:, 2]
        n = np.einsum("pij,pj->pi", self.em.normal_matrix[k], n)
        n /= np.linalg.norm(n, axis=-1, keepdims=True)
        return k, pos, n, self.em.emittance[k], self.em.density[k], margin

    # -- brute-force visibility -------------------------------------------------------------------------------------------
    def visible(self, org, d, tmax):
        """(visible, ambiguous) of rays org + t d, 0 < t < tmax, |d| = 1, against every triangle (Moller-Trumbore in float64)"""
        vis = np.ones(org.shape[0], bool)
        amb = np.zeros(org.shape[0], bool)
        for s in range(0, org.shape[0], 2048):
            o, dd, tm = org[s:s + 2048, None], d[s:s + 2048, None], tmax[s:s + 2048, None]
            pv = np.cross(dd, self.e2[None])
            det = _dot(self.e1[None], pv)
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                tv = o - self.tris[None, :, 0]
                uu = _dot(tv, pv) * inv
                qv = np.cross(tv, self.e1[None])
                vv = _dot(dd, qv) * inv
                t = _dot(self.e2[None], qv) * inv
                # margins in units of their bars: barycentrics, t > 0 (the float32 plane distance of an origin carries
                # ~8 U |org|, far below offsetRayOrigin's step) and t < 0.9999 tmax
                m = np.minimum(np.minimum(uu, vv), 1 - uu - vv) / VIS_BAR
                m = np.minimum(m, t / (8 * U * (np.abs(o).max(-1) + 1)))
                m = np.minimum(m, (tm * 0.9999 - t) / (VIS_BAR * tm))
            m = np.where(np.isfinite(m), m, -np.inf)
            vis[s:s + 2048] = ~(m > 1).any(1)
            amb[s:s + 2048] = (np.abs(m) <= 1).any(1) & vis[s:s + 2048]
        return vis, amb


class ShadingPoints:
    """the common prologue of the passes for pixels idx of one G-buffer (optix_restir_di_kernels.cu:21-56)"""

    def __init__(self, s64: Scene64, gb: dict, idx, cam_pos):
        gb2, gb3 = gb[2].reshape(-1, 4)[idx], gb[3].reshape(-1, 4)[idx]
        p32 = gb2[:, :3].view(np.float32)
        p = p32.astype(np.float64)
        ng = shading_ref.decode_vector(gb2[:, 3])
        v = cam_pos[None] - p
        fh = _dot(v, ng)
        self.front_margin = np.abs(fh) / (16 * U * np.linalg.norm(v, axis=-1))
        front = np.where(fh >= 0, 1.0, -1.0)
        self.pos = offset_ray_origin(p32, front[:, None] * ng)
        self.dist = np.linalg.norm(v, axis=-1)
        vout = v / self.dist[:, None]
        self.n = shading_ref.decode_vector(gb3[:, 0])
        self.t = shading_ref.decode_vector(gb3[:, 1])
        self.b = np.cross(self.n, self.t)
        self.vout_local = self.to_local(vout)
        self.mat = np.where(gb3[:, 3] == SKY, 0, gb3[:, 3]).astype(np.int64)   # sky rows are gathered, then masked out
        self.s64 = s64

    def to_local(self, v):
        return np.stack([_dot(self.t, v), _dot(self.b, v), _dot(self.n, v)], -1)

    def lobe_bar(self):
        return self.s64.lobe_bar[self.mat]

    def steered(self):
        return self.front_margin < 1

    def direct(self, pos_l, nrm_l, le, at_inf, with_vis: bool):
        """performDirectLighting<_, with_vis>: (contribution [P, 3], ambiguous visibility).  self.cond is the contribution's
        relative float32 conditioning: a cosine computed with an absolute error of ~8 U carries 8 U / cos"""
        d = np.where(at_inf[:, None], pos_l, pos_l - self.pos)
        dist2 = _dot(d, d)
        dist = np.sqrt(dist2)
        with np.errstate(divide="ignore", invalid="ignore"):
            d = d / dist[:, None]
        dl = self.to_local(d)
        lp_cos = _dot(-d, nrm_l)
        sp_cos = dl[:, 2]
        amb = np.zeros(len(dist), bool)
        vis = np.ones(len(dist), bool)
        live = lp_cos > 0
        if with_vis and live.any():
            tmax = np.where(at_inf, 1e10, dist)
            v, a = self.s64.visible(self.pos[live], d[live], tmax[live])
            vis[live], amb[live] = v, a
        out = np.zeros((len(dist), 3))
        for m in np.unique(self.mat[live & vis]):
            sel = live & vis & (self.mat == m)
            fs = shading_ref.evaluate(self.s64.bsdfs[m], self.vout_local[sel], dl[sel])
            with np.errstate(divide="ignore", invalid="ignore"):
                g = lp_cos[sel] * np.abs(sp_cos[sel]) / dist2[sel]
            out[sel] = fs * (le[sel] / np.pi) * g[:, None]
        with np.errstate(divide="ignore"):
            cond = 8 * U * (1 / np.abs(lp_cos) + 1 / np.abs(sp_cos) + 1 / np.abs(self.vout_local[:, 2]))
        self.cond = np.where(out.any(-1), cond, 0.0)
        return out, amb


def weight(c):
    return c.mean(-1)


class Reservoirs:
    """one reservoir plane set in float64: the sample (position, normal, emittance, atInfinity), sumW, M, and the info"""

    def __init__(self, raw: np.ndarray, info: np.ndarray):
        a, b, c = (raw[k].reshape(-1, 4) for k in range(3))
        self.le = a[:, :3].view(np.float32).astype(np.float64)
        self.sumw = a[:, 3].view(np.float32).astype(np.float64)
        self.pos = b[:, :3].view(np.float32).astype(np.float64)
        self.m = (b[:, 3] & M31).astype(np.int64)
        self.inf = (b[:, 3] >> 31).astype(bool)
        self.nrm = c[:, :3].view(np.float32).astype(np.float64)
        info = info.reshape(-1, 2).astype(np.float64)
        self.rec, self.target = info[:, 0], info[:, 1]


def _rel_bar(n):
    return (3 * K_CHAIN + n + 8) * U


def _select(cond, a, b):
    return np.where(cond[:, None] if a.ndim == 2 else cond, a, b)


class RestirRef:
    """the passes on a W x H frame; load() takes a system's float32 planes, each pass returns the expected outputs"""

    def __init__(self, s64: Scene64, W: int, H: int):
        self.s64, self.W, self.H = s64, W, H
        self.deltas = neighbor_deltas()
        self.steered_pixels = 0
        self.compared_pixels = 0

    def load(self, side):
        self.gb = {i: {k: side.get(b, i) for k, b in enumerate((abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2,
                                                                 abi.BUF_GBUFFER3))} for i in (0, 1)}
        self.rng = side.get(abi.BUF_RNG, 0).reshape(-1).astype(np.uint64)
        self.res = [Reservoirs(side.get(abi.BUF_RESERVOIR, i), side.get(abi.BUF_RESERVOIR_INFO, i)) for i in (0, 1)]
        self.beauty = side.get(abi.BUF_BEAUTY_ACCUM, 0).reshape(-1, 4).astype(np.float64)

    def _pixels(self, p, buf):
        y0 = p.tileOriginY
        y1 = min(self.H, y0 + p.tileRows) if p.tileRows else self.H
        idx = np.arange(y0 * self.W, y1 * self.W)
        return idx[self.gb[buf][0].reshape(-1, 4)[idx, 0] != SKY]

    @staticmethod
    def _cam(c):
        return np.asarray(c.position[:], np.float32).astype(np.float64)

    # ---- testNeighbor -------------------------------------------------------------------------------------------------------
    def _test_neighbor(self, buf, nbx, nby, dist, normal, cam_pos, geometry):
        inb = (nbx >= 0) & (nbx < self.W) & (nby >= 0) & (nby < self.H)
        nb = np.where(inb, nby * self.W + nbx, 0)
        ok = inb & (self.gb[buf][0].reshape(-1, 4)[nb, 0] != SKY)
        steer = np.zeros(len(nb), bool)
        if geometry:
            npos = self.gb[buf][2].reshape(-1, 4)[nb, :3].view(np.float32).astype(np.float64)
            nn = shading_ref.decode_vector(self.gb[buf][3].reshape(-1, 4)[nb, 0])
            nd = np.linalg.norm(cam_pos[None] - npos, axis=-1)
            rel = np.abs(nd - dist) / dist
            dp = _dot(normal, nn)
            ok &= ~(rel > 0.1) & ~(dp < 0.9)
            steer = inb & ((np.abs(rel - 0.1) < 64 * U) | (np.abs(dp - 0.9) < 32 * U))
        return ok, nb, steer

    def _neighbor_coord(self, p, x, y, n_idx, rng, live):
        radius = float(np.float32(p.spatialNeighborRadius))
        if p.useLowDiscrepancyNeighbors:
            d = self.deltas[(p.spatialNeighborBaseIndex + n_idx) % 1024]
            dx = np.full(len(x), radius * d[0])
            dy = np.full(len(x), radius * d[1])
            bar_extra = 0.0
        else:
            rng[live], u0 = pcg_draw(rng[live])
            rng[live], u1 = pcg_draw(rng[live])
            r = np.zeros(len(x))
            a = np.zeros(len(x))
            r[live] = radius * np.sqrt(u0)
            a[live] = 2 * np.pi * u1
            dx, dy = r * np.cos(a), r * np.sin(a)
            bar_extra = 16 * U * radius
        vx, vy = x + 0.5 + dx, y + 0.5 + dy
        steer = ((_int_margin(vx) < 16 * U * (np.abs(x) + 1 + np.abs(dx)) + bar_extra)
                 | (_int_margin(vy) < 16 * U * (np.abs(y) + 1 + np.abs(dy)) + bar_extra))
        return np.trunc(vx).astype(np.int64), np.trunc(vy).astype(np.int64), steer

    # ---- performInitialAndTemporalRIS ---------------------------------------------------------------------------------------
    def initial_and_temporal(self, p, temporal: bool, unbiased: bool) -> dict:
        s64 = self.s64
        buf, cur = p.bufferIndex & 1, p.currentReservoirIndex & 1
        idx = self._pixels(p, buf)
        P = len(idx)
        cam = self._cam(p.camera)
        sp = ShadingPoints(s64, self.gb[buf], idx, cam)
        steer = sp.steered()
        lobe = sp.lobe_bar()
        rng = self.rng[idx].copy()
        n_cand = 1 << p.log2NumCandidateSamples
        sumw = np.zeros(P)
        sel_k = np.full(P, -1)
        sel = dict(pos=np.zeros((P, 3)), nrm=np.zeros((P, 3)), le=np.zeros((P, 3)))
        sel_target = np.zeros(P)
        no_inf = np.zeros(P, bool)
        for i in range(n_cand):
            rng, ul = pcg_draw(rng)
            rng, u0 = pcg_draw(rng)
            rng, u1 = pcg_draw(rng)
            rng, u = pcg_draw(rng)
            k, lpos, lnrm, le, dens, pick_margin = s64.sample(ul, u0, u1)
            steer |= pick_margin < (16 + s64.n_lights) * U
            cont, _ = sp.direct(lpos, lnrm, le, no_inf, False)
            lobe = np.maximum(lobe, sp.lobe_bar() + sp.cond)
            td = weight(cont)
            with np.errstate(divide="ignore", invalid="ignore"):
                w = td / dens
            sumw = sumw + w
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = w / sumw
            acc = u < ratio
            steer |= (w > 0) & (np.abs(u - ratio) < ((2 * K_CHAIN + i + 2) * U + 2 * lobe) * ratio)
            sel_k = np.where(acc, k, sel_k)
            for key, val in (("pos", lpos), ("nrm", lnrm), ("le", le)):
                sel[key] = _select(acc, val, sel[key])
            sel_target = np.where(acc, td, sel_target)
        m = np.full(P, n_cand, np.int64)
        with np.errstate(divide="ignore", invalid="ignore"):
            rec = sumw / (sel_target * m)
        bad = ~np.isfinite(rec)
        rec[bad] = 0.0
        sel_target[bad] = 0.0
        if p.reuseVisibility:
            live = sel_target > 0
            d = sel["pos"] - sp.pos
            dist = np.linalg.norm(d, axis=-1)
            with np.errstate(divide="ignore", invalid="ignore"):
                vis, amb = s64.visible(sp.pos[live], (d / dist[:, None])[live], dist[live])
            steer[live] |= amb
            occl = np.zeros(P, bool)
            occl[live] = ~vis
            rec[occl] = 0.0
            sel_target[occl] = 0.0
        inf = np.zeros(P, bool)
        n_terms = n_cand
        if temporal:
            prev_buf, prev_res = (buf + 1) % 2, (cur + 1) % 2
            self_m = m.copy()
            empty = rec == 0.0
            sumw[empty] = 0.0
            for key in sel:
                sel[key][empty] = 0.0
            sel_k[empty] = -1
            m_cap = 20 * self_m
            x, y = idx % self.W, idx // self.W
            mv = self.gb[buf][1].reshape(-1, 2)[idx].astype(np.float64)
            vx, vy = x + 0.5 - mv[:, 0], y + 0.5 - mv[:, 1]
            steer |= (_int_margin(vx) < 4 * U * (x + 1 + np.abs(mv[:, 0]))) | (_int_margin(vy) < 4 * U * (y + 1 + np.abs(mv[:, 1])))
            nbx, nby = np.trunc(vx).astype(np.int64), np.trunc(vy).astype(np.int64)
            ok, nb, st = self._test_neighbor(prev_buf, nbx, nby, sp.dist, sp.n, cam, not unbiased)
            steer |= st
            prev = self.res[prev_res]
            nb_sel = np.zeros(P, bool)
            nb_m = np.minimum(prev.m[nb], m_cap)
            if ok.any():
                cont, _ = sp.direct(prev.pos[nb], prev.nrm[nb], prev.le[nb], prev.inf[nb], False)
                lobe = np.maximum(lobe, np.where(ok, sp.lobe_bar() + sp.cond, 0.0))
                td = weight(cont)
                w = td * prev.rec[nb] * nb_m
                rng_ok, u = pcg_draw(rng[ok])
                rng[ok] = rng_ok
                uu = np.zeros(P)
                uu[ok] = u
                sumw = np.where(ok, sumw + w, sumw)
                with np.errstate(divide="ignore", invalid="ignore"):
                    ratio = w / sumw
                acc = ok & (uu < ratio)
                steer |= ok & (w > 0) & (np.abs(uu - ratio) < ((2 * K_CHAIN + 4) * U + 2 * lobe) * ratio)
                nb_sel = acc
                for key, src in (("pos", prev.pos), ("nrm", prev.nrm), ("le", prev.le)):
                    sel[key] = _select(acc, src[nb], sel[key])
                inf = np.where(acc, prev.inf[nb], inf)
                sel_target = np.where(acc, td, sel_target)
                sel_k = np.where(acc, -2, sel_k)
            m = np.where(ok, self_m + nb_m, self_m)
            n_terms += 1
            if unbiased:
                cont, _ = sp.direct(sel["pos"], sel["nrm"], sel["le"], inf, False)
                lobe = np.maximum(lobe, sp.lobe_bar() + sp.cond)
                td_self = weight(cont)
                num = td_self
                den = td_self * self_m
                if ok.any():
                    nsp = ShadingPoints(s64, self.gb[prev_buf], nb, self._cam(p.prevCamera))
                    cont, _ = nsp.direct(sel["pos"], sel["nrm"], sel["le"], inf, False)
                    lobe = np.maximum(lobe, np.where(ok, nsp.lobe_bar() + nsp.cond, 0.0))
                    td_nb = weight(cont)
                    steer |= ok & nsp.steered()
                    den = np.where(ok, den + td_nb * nb_m, den)
                    num = np.where(ok & nb_sel, td_nb, num)
                with np.errstate(divide="ignore", invalid="ignore"):
                    wfe = num / den
            else:
                wfe = 1.0 / m
            with np.errstate(divide="ignore", invalid="ignore"):
                rec = wfe * sumw / sel_target
            bad = ~np.isfinite(rec)
            rec[bad] = 0.0
            sel_target[bad] = 0.0
        out = dict(idx=idx, res=cur, rng=rng, m=np.minimum(m, M31), inf=inf, pos=sel["pos"], sumw=sumw, rec=rec,
                   target=sel_target, steer=steer, n_terms=n_terms, m_raw=m, lobe=lobe)
        return out

    # ---- performSpatialRIS --------------------------------------------------------------------------------------------------
    def spatial(self, p, unbiased: bool) -> dict:
        s64 = self.s64
        buf, src = p.bufferIndex & 1, p.currentReservoirIndex & 1
        dst = (src + 1) % 2
        idx = self._pixels(p, buf)
        P = len(idx)
        cam = self._cam(p.camera)
        sp = ShadingPoints(s64, self.gb[buf], idx, cam)
        steer = sp.steered()
        lobe = sp.lobe_bar()
        rng = self.rng[idx].copy()
        x, y = idx % self.W, idx // self.W
        R = self.res[src]
        take = R.rec[idx] > 0
        sel = dict(pos=np.where(take[:, None], R.pos[idx], 0.0), nrm=np.where(take[:, None], R.nrm[idx], 0.0),
                   le=np.where(take[:, None], R.le[idx], 0.0))
        inf = take & R.inf[idx]
        sumw = np.where(take, R.sumw[idx], 0.0)
        sel_target = np.where(take, R.target[idx], 0.0)
        self_m = R.m[idx]
        m = self_m.copy()
        sel_n = np.full(P, -1)
        all_live = np.ones(P, bool)
        n_nb = p.numSpatialNeighbors
        for n_idx in range(n_nb):
            nbx, nby, st = self._neighbor_coord(p, x, y, n_idx, rng, all_live)
            ok, nb, st2 = self._test_neighbor(buf, nbx, nby, sp.dist, sp.n, cam, not unbiased)
            ok &= (nbx != x) | (nby != y)
            steer |= st | (st2 & ((nbx != x) | (nby != y)))
            cont, _ = sp.direct(R.pos[nb], R.nrm[nb], R.le[nb], R.inf[nb], False)
            lobe = np.maximum(lobe, np.where(ok, sp.lobe_bar() + sp.cond, 0.0))
            td = weight(cont)
            w = td * R.rec[nb] * R.m[nb]
            u = np.zeros(P)
            if ok.any():
                rng_ok, u_ok = pcg_draw(rng[ok])
                rng[ok] = rng_ok
                u[ok] = u_ok
            sumw = np.where(ok, sumw + w, sumw)
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = w / sumw
            acc = ok & (u < ratio)
            steer |= ok & (w > 0) & (np.abs(u - ratio) < ((2 * K_CHAIN + n_idx + 3) * U + 2 * lobe) * ratio)
            for key, srcv in (("pos", R.pos), ("nrm", R.nrm), ("le", R.le)):
                sel[key] = _select(acc, srcv[nb], sel[key])
            inf = np.where(acc, R.inf[nb], inf)
            sel_target = np.where(acc, td, sel_target)
            sel_n = np.where(acc, n_idx, sel_n)
            m = np.where(ok, m + R.m[nb], m)
        m_raw = m
        m = np.minimum(m, M31)   # the combined stream length saturates at 2^31 - 1 (DESIGN.md); the reference's uint32_t wraps at 2^32
        if unbiased:
            wfe = np.zeros(P)
            live = sel_target > 0
            cont, amb = sp.direct(sel["pos"], sel["nrm"], sel["le"], inf, bool(p.reuseVisibility))
            lobe = np.maximum(lobe, sp.lobe_bar() + sp.cond)
            steer |= live & amb
            td_self = weight(cont)
            visibility = np.ones(P, bool)
            if p.reuseVisibility:
                visibility = td_self > 0
            num = td_self
            den = td_self * self_m
            for n_idx in range(n_nb):
                nbx, nby, st = self._neighbor_coord(p, x, y, n_idx, rng, live)
                ok = live & (nbx >= 0) & (nbx < self.W) & (nby >= 0) & (nby < self.H) & ((nbx != x) | (nby != y))
                steer |= live & st
                nb = np.where(ok, nby * self.W + nbx, 0)
                ok &= self.gb[buf][0].reshape(-1, 4)[nb, 0] != SKY
                if not ok.any():
                    continue
                nsp = ShadingPoints(s64, self.gb[buf], nb, self._cam(p.prevCamera))
                cont, amb = nsp.direct(sel["pos"], sel["nrm"], sel["le"], inf, bool(p.reuseVisibility))
                lobe = np.maximum(lobe, np.where(ok, nsp.lobe_bar() + nsp.cond, 0.0))
                steer |= ok & (amb | nsp.steered())
                td_nb = weight(cont)
                den = np.where(ok, den + td_nb * R.m[nb], den)
                num = np.where(ok & (sel_n == n_idx), td_nb, num)
            with np.errstate(divide="ignore", invalid="ignore"):
                wfe = np.where(live, num / den, 0.0)
            if p.reuseVisibility:
                wfe = np.where(visibility, wfe, 0.0)
        else:
            with np.errstate(divide="ignore"):
                wfe = 1.0 / m
        with np.errstate(divide="ignore", invalid="ignore"):
            rec = wfe * sumw / sel_target
        bad = ~np.isfinite(rec)
        rec[bad] = 0.0
        target = np.where(bad, 0.0, sel_target)
        return dict(idx=idx, res=dst, rng=rng, m=np.minimum(m, M31), inf=inf, pos=sel["pos"], sumw=sumw, rec=rec,
                    target=target, steer=steer, n_terms=n_nb + 1 + int(unbiased) * (n_nb + 1), m_raw=m_raw, lobe=lobe)

    # ---- shading ------------------------------------------------------------------------------------------------------------
    def shading(self, p) -> dict:
        s64 = self.s64
        buf, cur = p.bufferIndex & 1, p.currentReservoirIndex & 1
        idx = self._pixels(p, buf)
        cam = self._cam(p.camera)
        sp = ShadingPoints(s64, self.gb[buf], idx, cam)
        steer = sp.steered()
        R = self.res[cur]
        contrib = np.where((sp.vout_local[:, 2] > 0)[:, None], s64.emittance[sp.mat] / np.pi, 0.0)
        # the emission test vOutLocal.z > 0: a dot product of unit vectors, bar 16 U
        steer |= (np.abs(sp.vout_local[:, 2]) < 16 * U) & s64.emittance[sp.mat].any(-1)
        rec = R.rec[idx]
        live = (rec > 0) & np.isfinite(rec)
        vis_done = bool(p.reuseVisibility) and (not p.enableTemporalReuse or (p.enableSpatialReuse and p.useUnbiasedEstimator))
        cont, amb = sp.direct(R.pos[idx], R.nrm[idx], R.le[idx], R.inf[idx], not vis_done)
        steer |= live & amb
        lobe = sp.lobe_bar() + sp.cond
        contrib = contrib + np.where(live[:, None], rec[:, None] * cont, 0.0)
        cw = 1.0 / (1 + p.numAccumFrames)
        prev = self.beauty[idx, :3] if p.numAccumFrames > 0 else 0.0
        beauty = (1 - cw) * prev + cw * contrib
        return dict(idx=idx, beauty=beauty, steer=steer, n_terms=4, lobe=lobe)


# ---- comparison ------------------------------------------------------------------------------------------------------------
def compare(side, ref: RestirRef, out: dict, what: str):
    """a system's outputs of one pass against the restated ones on the unsteered pixels; returns the steered count"""
    idx, steer = out["idx"], out["steer"]
    keep = ~steer
    ref.steered_pixels += int(steer.sum())
    ref.compared_pixels += len(idx)
    bar = _rel_bar(out["n_terms"]) + 3 * out["lobe"][keep]
    if "beauty" in out:
        got = side.get(abi.BUF_BEAUTY_ACCUM, 0).reshape(-1, 4)[idx, :3].astype(np.float64)
        _close(got[keep], out["beauty"][keep], bar[:, None], f"{what}: beauty", idx[keep])
        return int(steer.sum())
    raw = side.get(abi.BUF_RESERVOIR, out["res"])
    b = raw[1].reshape(-1, 4)[idx]
    a = raw[0].reshape(-1, 4)[idx]
    info = side.get(abi.BUF_RESERVOIR_INFO, out["res"]).reshape(-1, 2)[idx].astype(np.float64)
    rng = side.get(abi.BUF_RNG, 0).reshape(-1)[idx]
    k = idx[keep]
    _exact(rng[keep], out["rng"][keep], f"{what}: RNG state", k)
    _exact((b[:, 3] & M31)[keep].astype(np.int64), out["m"][keep], f"{what}: M", k)
    _exact((b[:, 3] >> 31)[keep].astype(bool), out["inf"][keep], f"{what}: atInfinity", k)
    pos = b[:, :3].view(np.float32).astype(np.float64)
    _close(pos[keep], out["pos"][keep], 1e-4, f"{what}: the held light sample", k, absolute=True)
    _close(a[:, 3].view(np.float32).astype(np.float64)[keep], out["sumw"][keep], bar, f"{what}: sumWeights", k)
    _close(info[keep, 0], out["rec"][keep], bar, f"{what}: recPDFEstimate", k)
    _close(info[keep, 1], out["target"][keep], bar, f"{what}: targetDensity", k)
    return int(steer.sum())


def _exact(got, want, what, pix):
    bad = got != want
    if bad.any():
        j = int(np.argmax(bad))
        raise AssertionError(f"{what} differs at {int(bad.sum())} pixels; first at pixel {int(pix[j])}: "
                             f"got {got[j]!r}, restated {want[j]!r}")


def _close(got, want, bar, what, pix, absolute=False):
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    tol = bar if absolute else bar * np.abs(want) + 1e-30
    bad = ~(np.abs(got - want) <= tol)
    if bad.ndim > 1:
        bad = bad.any(-1)
    if bad.any():
        j = int(np.argmax(bad))
        raise AssertionError(f"{what} off its bar at {int(bad.sum())} pixels; first at pixel {int(pix[j])}: "
                             f"got {got[j]!r}, restated {want[j]!r}")
