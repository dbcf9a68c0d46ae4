"""The G-buffer pass restated in float64 - TEST INFRASTRUCTURE for tests/test_oracle_gbuffer_ref.py and
tests/test_gpu_gbuffer_ref.py.

Written from restir_di/gpu_kernels/optix_gbuffer_kernels.cu and restir_di_shared.h, not from oracle/render.cpp or
gfxexp_b200/csrc/gbuffer.cu:
  optix_gbuffer_kernels.cu:5-110     setupGBuffers RG: the ray through (x + jx, y + jy) with vh = 2 tan(fovY / 2) per pixel, the
                                     enableJittering sample (two PCG32 draws, the state written back), the motion vector from
                                     the pixel centre, resetFlowBuffer and the NaN position, the running means of albedo / normal
  optix_gbuffer_kernels.cu:112-199   setupGBuffers CH: barycentric attributes, object -> world, the normal through the inverse
                                     transpose of the instance's transform (OptiX's transformNormalFromObjectToWorldSpace; the
                                     scene's Instance.normal_matrix is not read), the tangent's Gram-Schmidt step, the
                                     non-finite-normal fallback, the bump frame, the DH-reflectance albedo
  optix_gbuffer_kernels.cu:201-243   setupGBuffers MS: position = direction, envLightRotation, u wrapped to [0, 1)
  restir_di_shared.h:51-59           calcScreenPosition, with its invert(orientation)
  svgf_main.cpp:1410-1424, 2005-2008 the SVGF app's TAA sample (halton(2, i), 1 - halton(3, i)), i = frameIndex % history; the
                                     motion vector is then taken from the sample (oracle/svgf_taa_jitter.cpp derives this)
The decoders and the BSDFs' DH-reflectance estimate are tests/shading_ref.py's, the texture filter and the bump frame
tests/texture_ref.py's, PCG32 and the radical inverse tests/restir_ref.py's.  The closest hit is brute force over every
world-space triangle (Moller-Trumbore in float64).  The previous position is computed twice: as curToPrevTransform . P, and as
the previous frame's transform . P_obj (which checks scenes.move_instance); both must give the motion vector.

A system under test runs the pass in float32.  Every discrete decision gets a margin and a first-order float32 bar, and a pixel
with a decision inside its bar is *steered*: left out of the comparison and counted.  U = 2^-24.
  * closest hit: a triangle decides a ray when its smallest barycentric clears bc_bar = 64 U (|O| + |P|) / h, h the
    triangle's smallest altitude (float32 vertices, origin and direction move the barycentrics by that much); a pixel is
    steered when a triangle inside that bar lies in front of the nearest hit, or when the two nearest hits are within
    1e-5 of each other in relative distance;
  * the miss program's u = phi / 2 pi wrapped: steered within 64 U of an integer;
  * the height map's gather footprint: steered within the texture-coordinate bar of its 255.5 / 256 step.
Continuous outputs get first-order bars: the position 64 U (|P| + |O| + t / max(|cos|, 0.01)) plus the transform's
magnitude, the barycentrics (position bar) / h, attributes that much times their spread over the triangle, directions that
plus 64 U times the normal matrix's condition number, divided by the length of the projected tangent for the tangent, and
the motion vector the position and 32 U |P| terms through the projection's Jacobian.  The encoded planes add their
quantisation: a truncated 16-bit polar pair decodes within 1.1e-4 of its vector, a UNORM16 within 1 / 65535 below its value.
The 8-bit weights of the bilinear filter may flip within the texture-coordinate bar: such a pixel's texture value gets an
allowance of one weight step (2 / 256 of its texel spread) instead of being steered.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from gfxexp_b200 import abi
from tests import restir_ref, shading_ref, texture_ref

U = 2.0 ** -24
SKY = 0xFFFFFFFF
Q_VEC = 1.1e-4          # sqrt(5) pi / 65535: a truncated (phi, theta) pair
Q_16 = 1.0 / 65535
T_BAR = 1e-5
NAN_TANGENT = 0xFFFF0000  # encodeVector of a NaN vector: theta = acos(clamp(NaN)) = acos(-1) = pi, phi = NaN -> 0


def _dot(a, b):
    return np.sum(a * b, -1)


def _normalize(v):
    with np.errstate(divide="ignore", invalid="ignore"):
        return v / np.linalg.norm(v, axis=-1, keepdims=True)


# ---- camera (restir_di_shared.h:44-59) ---------------------------------------------------------------------------------
@dataclass
class Camera64:
    position: np.ndarray
    orientation: np.ndarray
    aspect: float
    fov_y: float

    @staticmethod
    def of(cam: abi.GfxCamera) -> "Camera64":
        return Camera64(np.array(cam.position[:], np.float64), np.array(cam.orientation[:], np.float64).reshape(3, 3),
                        float(cam.aspect), float(cam.fovY))

    @property
    def vh(self):
        return 2 * np.tan(self.fov_y / 2)

    def direction(self, fx, fy):
        v = np.stack([self.aspect * self.vh * (0.5 - fx), self.vh * (0.5 - fy), np.ones_like(fx)], -1)
        return _normalize(v @ self.orientation.T)

    def view(self, p):
        return (p - self.position) @ np.linalg.inv(self.orientation).T

    def screen_position(self, p):
        """calcScreenPosition: (sx, sy) in [0, 1]^2 for a point in front of the camera"""
        v = self.view(p)
        with np.errstate(divide="ignore", invalid="ignore"):
            zx, zy = v[..., 0] / v[..., 2], v[..., 1] / v[..., 2]
        h = self.vh
        w = self.aspect * h
        return np.stack([1 - (zx + 0.5 * w) / w, 1 - (zy + 0.5 * h) / h], -1)

    def screen_jacobian_bar(self, p, W, H, dp):
        """first-order bound of W, H * screen_position(p) under a perturbation |dp| of p, plus the rounding of the projection"""
        v = self.view(p)
        z = np.abs(v[..., 2])
        with np.errstate(divide="ignore", invalid="ignore"):
            k = (1 + np.abs(v[..., 0] / v[..., 2]) + np.abs(v[..., 1] / v[..., 2])) / z
            e = dp + 32 * U * (np.linalg.norm(p, axis=-1) + np.linalg.norm(self.position))
            return (W / (self.aspect * self.vh) + H / self.vh) * k * e + 16 * U * (W + H)


# ---- the sample of a pixel ---------------------------------------------------------------------------------------------
def taa_sample(p):
    """(jx, jy) of GFX_SVGF_SUBPIXEL_JITTER with GFX_SVGF_ENABLE_TEMPORAL_AA, or None"""
    if not (p.svgfFlags & abi.SVGF_SUBPIXEL_JITTER) or not (p.svgfFlags & abi.SVGF_ENABLE_TAA):
        return None
    i = p.frameIndex % (p.taaHistoryLength or 16)
    return restir_ref.halton(2, i), 1 - restir_ref.halton(3, i)


# ---- the scene in float64 ----------------------------------------------------------------------------------------------
class Scene64:
    """every world-space triangle of a scenes.Scene with its (instance, mesh, primitive), the meshes' vertex attributes, and
    each instance's transform, inverse-transpose normal matrix and curToPrev in float64"""

    def __init__(self, scene, prev_instances=None):
        self.scene = scene
        tris, ids = [], []
        self.xf, self.nm, self.c2p, self.prev_xf = [], [], [], []
        for k, inst in enumerate(scene.instances):
            xf = np.asarray(inst.transform, np.float64)
            self.xf.append(xf)
            self.nm.append(np.linalg.inv(xf[:, :3]).T)
            self.c2p.append(np.asarray(inst.cur_to_prev, np.float64))
            prev = (prev_instances or scene.instances)[k]
            self.prev_xf.append(np.asarray(prev.transform, np.float64))
            for slot in inst.mesh_slots:
                mesh = scene.meshes[slot]
                p = mesh.positions.astype(np.float64)[mesh.triangles.astype(np.int64)]
                tris.append(p @ xf[:, :3].T + xf[:, 3])
                n = len(mesh.triangles)
                ids.append(np.stack([np.full(n, k), np.full(n, slot), np.arange(n)], 1))
        self.tris = np.concatenate(tris)
        self.ids = np.concatenate(ids)
        self.e1 = self.tris[:, 1] - self.tris[:, 0]
        self.e2 = self.tris[:, 2] - self.tris[:, 0]
        cr = np.linalg.norm(np.cross(self.e1, self.e2), axis=-1)
        longest = np.max(np.linalg.norm(np.stack([self.e1, self.e2, self.e2 - self.e1], 1), axis=-1), 1)
        self.altitude = cr / longest
        self.extent = np.max(np.abs(self.tris), axis=(1, 2))
        m = scene.materials
        self.params = [(int(m["bsdfType"][k]), m["p0"][k], m["p1"][k], m["p2"][k]) for k in range(len(m))]
        self.bsdfs = [shading_ref.setup(*prm) for prm in self.params]

    def closest_hit(self, org, d):
        """-> (triangle index or -1, t, bcB, bcC, steered)"""
        n = len(d)
        idx = np.full(n, -1)
        t_hit = np.full(n, np.inf)
        bb, bc = np.zeros(n), np.zeros(n)
        steer = np.zeros(n, bool)
        step = max(1, 2 ** 20 // len(self.tris))
        for s in range(0, n, step):
            dd = d[s:s + step, None]
            pv = np.cross(dd, self.e2[None])
            det = _dot(self.e1[None], pv)
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                tv = org[None, None] - self.tris[None, :, 0]
                uu = _dot(tv, pv) * inv
                qv = np.cross(tv, self.e1[None])
                vv = _dot(dd, qv) * inv
                t = _dot(self.e2[None], qv) * inv
            bar = 64 * U * (np.linalg.norm(org) + self.extent[None]) / self.altitude[None]
            m = np.minimum(np.minimum(uu, vv), 1 - uu - vv)
            ok = np.isfinite(t) & (t > 0)
            inside = ok & (m > bar)
            amb = ok & (np.abs(m) <= bar)
            tin = np.where(inside, t, np.inf)
            k = np.argmin(tin, 1)
            r = np.arange(len(k))
            t1 = tin[r, k]
            tin[r, k] = np.inf
            t2 = tin.min(1)
            lim = np.where(np.isfinite(t1), t1 * (1 + T_BAR), np.inf)
            st = (np.where(amb, t, np.inf) < lim[:, None]).any(1) | (t2 < t1 * (1 + T_BAR))
            hit = np.isfinite(t1)
            sl = slice(s, s + step)
            idx[sl] = np.where(hit, k, -1)
            t_hit[sl] = t1
            bb[sl], bc[sl] = uu[r, k], vv[r, k]
            steer[sl] = st
        return idx, t_hit, bb, bc, steer


@dataclass
class Reference:
    """the restated pass over the pixels pix (flat indices) of a W x H frame"""
    W: int
    H: int
    pix: np.ndarray
    steered: np.ndarray
    hit: np.ndarray
    ids: np.ndarray                 # [N, 3] instance, mesh, primitive (SKY for a miss)
    mat: np.ndarray
    bc: np.ndarray                  # [N, 2] bcB, bcC (u, v for a miss)
    position: np.ndarray
    prev_position: np.ndarray       # curToPrev . P
    prev_position_obj: np.ndarray   # previous transform . P_obj
    geometric_normal: np.ndarray
    shading_normal: np.ndarray      # the frame's normal (after the bump, not renormalised)
    tangent: np.ndarray
    tex_coord: np.ndarray
    albedo: np.ndarray
    motion: np.ndarray
    motion_obj: np.ndarray
    rng: np.ndarray | None
    bars: dict = field(default_factory=dict)


def gbuffer(s64: Scene64, p, W: int, H: int, rng_in=None, rows=None, bump: bool = False) -> Reference:
    """the pass on rows [y0, y1) (by default the strip p describes); rng_in: the frame's PCG32 states before the pass"""
    if rows is None:
        y0 = p.tileOriginY
        y1 = min(H, p.tileOriginY + p.tileRows) if p.tileRows else H
    else:
        y0, y1 = rows
    ys, xs = np.mgrid[y0:y1, 0:W]
    xs, ys = xs.ravel().astype(np.float64), ys.ravel().astype(np.float64)
    pix = (ys * W + xs).astype(np.int64)
    n = len(pix)
    cam, prev_cam = Camera64.of(p.camera), Camera64.of(p.prevCamera)

    # ray generation (:10-27)
    jx, jy = np.full(n, 0.5), np.full(n, 0.5)
    rng_out = None
    taa = taa_sample(p)
    if taa is not None:
        jx[:], jy[:] = taa
    elif p.enableJittering:
        st = np.asarray(rng_in, np.uint64).reshape(-1)[pix]
        st, jx = restir_ref.pcg_draw(st)
        st, jy = restir_ref.pcg_draw(st)
        rng_out = st
    d = cam.direction((xs + jx) / W, (ys + jy) / H)
    org = cam.position

    tri, t, bcB, bcC, steer = s64.closest_hit(org, d)
    hit = tri >= 0
    ids = np.full((n, 3), SKY, np.int64)
    mat = np.full(n, SKY, np.int64)
    f64 = lambda: np.full((n, 3), np.nan)
    pos, prev_a, prev_b, ng, ns, tan = f64(), f64(), f64(), f64(), f64(), f64()
    tc = np.zeros((n, 2))
    bc = np.zeros((n, 2))
    albedo = np.zeros((n, 3))
    pos_bar = np.full(n, 16 * U)
    dir_bar = np.full(n, 16 * U)
    tan_bar = np.full(n, 16 * U)
    tc_bar = np.full(n, 16 * U)
    alb_bar = np.full(n, 64 * U)

    # closest hit (:112-199)
    h = np.flatnonzero(hit)
    if len(h):
        tr = tri[h]
        inst, slot, prim = s64.ids[tr].T
        ids[h] = s64.ids[tr]
        b, c = bcB[h], bcC[h]
        a = 1 - (b + c)
        bc[h] = np.stack([b, c], 1)
        P_obj = np.zeros((len(h), 3))
        n_obj, t_obj = np.zeros((len(h), 3)), np.zeros((len(h), 3))
        uv, spread_n, spread_t, spread_uv = np.zeros((len(h), 2)), np.zeros(len(h)), np.zeros(len(h)), np.zeros(len(h))
        ng_obj = np.zeros((len(h), 3))
        for ms in np.unique(slot):
            sel = slot == ms
            mesh = s64.scene.meshes[ms]
            vi = mesh.triangles.astype(np.int64)[prim[sel]]
            mat[h[sel]] = mesh.material
            w = np.stack([a[sel], b[sel], c[sel]], 1)[:, :, None]
            pv, nv = mesh.positions.astype(np.float64)[vi], mesh.normals.astype(np.float64)[vi]
            tv, uvv = mesh.tangents.astype(np.float64)[vi], mesh.texcoords.astype(np.float64)[vi]
            P_obj[sel] = np.sum(w * pv, 1)
            n_obj[sel] = np.sum(w * nv, 1)
            t_obj[sel] = np.sum(w * tv, 1)
            uv[sel] = np.sum(w * uvv, 1)
            ng_obj[sel] = np.cross(pv[:, 1] - pv[:, 0], pv[:, 2] - pv[:, 0])
            sp = lambda v: np.max(np.linalg.norm(v - v[:, :1], axis=-1), 1)
            spread_n[sel], spread_t[sel], spread_uv[sel] = sp(nv), sp(tv), sp(uvv)
        xf = np.stack([s64.xf[i] for i in inst])
        nm = np.stack([s64.nm[i] for i in inst])
        c2p = np.stack([s64.c2p[i] for i in inst])
        pxf = np.stack([s64.prev_xf[i] for i in inst])
        mv3 = lambda m, v: np.einsum("kij,kj->ki", m, v)
        P = mv3(xf[:, :, :3], P_obj) + xf[:, :, 3]
        pos[h] = P
        prev_a[h] = mv3(c2p[:, :, :3], P) + c2p[:, :, 3]
        prev_b[h] = mv3(pxf[:, :, :3], P_obj) + pxf[:, :, 3]
        g = _normalize(mv3(nm, ng_obj))
        sn = _normalize(mv3(nm, n_obj))
        tw = mv3(xf[:, :, :3], t_obj)
        tw = _normalize(tw - _dot(sn, tw)[:, None] * sn)
        bad = ~np.isfinite(sn).all(1)
        g[bad], sn[bad], tw[bad] = (0, 0, 1), (0, 0, 1), (1, 0, 0)
        tc[h] = uv

        # bars: the position along the surface, the barycentrics, directions through the normal matrix
        cosv = np.abs(_dot(d[h], g))
        scale = np.abs(xf).max((1, 2))
        pb = 64 * U * (np.linalg.norm(P, axis=-1) + np.linalg.norm(org) + t[h] / np.maximum(cosv, 0.01)
                       + scale * np.linalg.norm(P_obj, axis=-1))
        pos_bar[h] = pb
        bc_err = pb / s64.altitude[tr]
        cond = np.linalg.cond(nm)
        nl = np.linalg.norm(n_obj, axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            db = 64 * U * cond + 2 * bc_err * spread_n / nl
            tperp = np.linalg.norm(mv3(xf[:, :, :3], t_obj) - _dot(sn, mv3(xf[:, :, :3], t_obj))[:, None] * sn, axis=-1)
            tb = (db + 64 * U * cond + 2 * bc_err * spread_t * scale) * np.linalg.norm(mv3(xf[:, :, :3], t_obj), axis=-1) / tperp
        db[bad], tb[bad] = 0.0, 0.0
        # a tangent (nearly) along the normal: exactly there the tangent is NaN on both sides, near it its direction is noise
        near_parallel = np.isfinite(tperp) & (tperp < 1e-3 * np.linalg.norm(mv3(xf[:, :, :3], t_obj), axis=-1)) & ~bad
        steer[h] |= near_parallel & (tperp > 0)
        tb[~np.isfinite(tb)] = 0.0
        dir_bar[h] = db
        tc_bar[h] = bc_err * spread_uv + 16 * U * (1 + np.abs(uv).max(1))

        # BSDF setup, the bump frame, the albedo (:172-184)
        frame_t, frame_n = tw.copy(), sn.copy()
        extra = np.zeros(len(h))
        textures = s64.scene.textures
        mt = s64.scene.material_textures
        bm = s64.scene.bump_maps
        for mm in np.unique(mat[h]):
            sel = np.flatnonzero(mat[h] == mm)
            btype, p0, p1, p2 = s64.params[mm]
            u_, v_ = uv[sel, 0], uv[sel, 1]
            fetched = {}
            if mt is not None:
                for slot_k in range(3):
                    if mt[mm, slot_k] != SKY:
                        tex = textures[int(mt[mm, slot_k])]
                        val, _ = texture_ref.fetch_repeat(tex, u_, v_, np.float64)
                        near = texture_ref.fetch_margin(tex, u_, v_) < tc_bar[h][sel]
                        rng_t = float(np.ptp(tex[..., :3]))
                        extra[sel] += np.where(near, 2 / 256 * rng_t, 0.0) + tc_bar[h][sel] * 2 * max(tex.shape[:2]) * rng_t
                        fetched[slot_k] = val
            if bump:
                kind = abi.BUMP_NORMAL_MAP
                tex = np.array([[[127 / 255, 127 / 255, 1.0, 1.0]]], np.float32)
                if bm is not None and bm[mm, 0] != SKY:
                    tex, kind = textures[int(bm[mm, 0])], int(bm[mm, 1])
                mod = texture_ref.read_modified_normal(tex, kind, u_, v_)
                # the modified normal moves with the texture coordinates (a texel's spread per texel) and by one weight step
                # near the filter's rounding steps; the frame's rotation passes that and the frame's own error on
                spread = 2 * float(np.ptp(tex[..., :3]))
                bump_err = tc_bar[h][sel] * 2 * max(tex.shape[:2]) * spread
                if kind == abi.BUMP_HEIGHT_MAP:
                    steer[h[sel]] |= texture_ref.fetch_margin(tex, u_, v_, gather=True) < tc_bar[h][sel]
                else:
                    bump_err += np.where(texture_ref.fetch_margin(tex, u_, v_) < tc_bar[h][sel], 2 / 256 * spread, 0.0)
                fb = texture_ref.apply_bump_mapping(mod, tw[sel], np.cross(sn[sel], tw[sel]), sn[sel])
                frame_t[sel], frame_n[sel] = fb[:, 0:3], fb[:, 6:9]
                dir_bar[h[sel]] = 4 * (dir_bar[h[sel]] + tb[sel] + bump_err)
            vz = _dot(frame_n[sel], -d[h[sel]])
            if fetched:
                for k_, row in enumerate(sel):
                    q0 = fetched[0][k_, :3] if 0 in fetched else p0
                    q1 = fetched[1][k_, :3] if 1 in fetched else p1
                    q2 = fetched[2][k_, 0] if 2 in fetched else p2
                    albedo[h[row]] = shading_ref.dh_reflectance_estimate(shading_ref.setup(btype, q0, q1, q2),
                                                                         np.array([[0.0, 0.0, vz[k_]]]))[0]
            else:
                albedo[h[sel]] = shading_ref.dh_reflectance_estimate(s64.bsdfs[mm], np.stack([0 * vz, 0 * vz, vz], 1))
        ns[h], tan[h] = frame_n, frame_t
        tan_bar[h] = np.maximum(tb, dir_bar[h])
        ng[h] = g
        alb_bar[h] = 16 * (dir_bar[h] + 8 * U) + 4 * extra + 64 * U

    # miss (:201-243)
    m_ = np.flatnonzero(~hit)
    if len(m_):
        dm = d[m_]
        phi, theta = shading_ref.to_polar_y_up(dm)
        u = (phi + float(np.float32(p.envLightRotation))) / (2 * np.pi)
        steer[m_] |= np.abs(u - np.round(u)) < 64 * U * (1 + np.abs(u))
        u = u - np.floor(u)
        v = theta / np.pi
        pos[m_], prev_a[m_], prev_b[m_] = dm, dm, dm
        ng[m_], ns[m_] = -dm, -dm
        tan[m_] = np.stack([-np.cos(phi), 0 * phi, -np.sin(phi)], 1)
        tc[m_] = np.stack([u, v], 1)
        bc[m_] = np.stack([u, v], 1)
        dir_bar[m_] = tan_bar[m_] = 64 * U
        tc_bar[m_] = 64 * U * (1 + np.abs(u))

    # motion vector (:56-62)
    cur = np.stack([xs + jx, ys + jy], 1) if taa is not None else np.stack([xs + 0.5, ys + 0.5], 1)
    wh = np.array([W, H], np.float64)
    motion = cur - prev_cam.screen_position(prev_a) * wh
    motion_obj = cur - prev_cam.screen_position(prev_b) * wh
    mv_bar = prev_cam.screen_jacobian_bar(prev_a, W, H, pos_bar)
    nanp = np.isnan(prev_a[:, 0])
    zero = nanp | bool(p.resetFlowBuffer)
    motion[zero], motion_obj[zero], mv_bar[zero] = 0.0, 0.0, 0.0

    return Reference(W, H, pix, steer, hit, ids, mat, bc, pos, prev_a, prev_b, ng, ns, tan, tc, albedo, motion, motion_obj,
                     rng_out, dict(position=pos_bar, direction=dir_bar, tangent=tan_bar, tex_coord=tc_bar, albedo=alb_bar,
                                   motion=mv_bar))


# ---- comparison with a system under test's planes ----------------------------------------------------------------------
def _unorm16_ok(q, ref, bar, wrap=False):
    """q = min(trunc(65535 x), 65535) of an x within bar of ref"""
    dec = q / 65535.0
    if wrap:   # texture coordinates: ref is a fraction, compared on the circle
        dd = (ref - dec) % 1.0
        return (dd <= Q_16 + bar) | (dd >= 1 - bar)
    return (dec <= np.minimum(ref, 1.0) + bar) & (dec >= ref - Q_16 - bar)


def _vec_ok(q, ref, bar):
    """encodeVector takes theta = acos(clamp(v.y)) of the vector as it is: a bump frame's normal is not of unit length (the
    texel's length carries over), and near |v.y| = 1 acos amplifies the error of v.y by 1 / sin(theta)"""
    phi, theta = shading_ref.to_polar_y_up(ref)
    s = np.sqrt(np.maximum(0.0, 1 - np.minimum(np.abs(ref[:, 1]), 1.0) ** 2))
    bar = bar + bar / np.maximum(s, np.sqrt(bar))
    return np.linalg.norm(shading_ref.decode_vector(q) - shading_ref.from_polar_y_up(phi, theta), axis=-1) <= Q_VEC + bar


def mismatches(ref: Reference, planes: dict, accum_prev=None, num_accum_frames: int = 0) -> dict:
    """pixels (of the non-steered ones) where each plane leaves its bar.  planes: abi buffer id -> [H, W, ...] array of the
    system under test after the pass; accum_prev: its (albedo, normal) running means before it"""
    keep = ~ref.steered
    pix = ref.pix
    B = ref.bars
    g0 = planes[abi.BUF_GBUFFER0].reshape(-1, 4)[pix].astype(np.int64)
    g1 = planes[abi.BUF_GBUFFER1].reshape(-1, 2)[pix].astype(np.float64)
    g2 = planes[abi.BUF_GBUFFER2].reshape(-1, 4)[pix]
    g3 = planes[abi.BUF_GBUFFER3].reshape(-1, 4)[pix].astype(np.int64)
    out = {}
    out["ids"] = (g0[:, :3] != ref.ids).any(1)
    out["mat"] = g3[:, 3] != ref.mat
    out["bc"] = ~(_unorm16_ok(g0[:, 3] & 0xFFFF, ref.bc[:, 0], B["tex_coord"]) & _unorm16_ok(g0[:, 3] >> 16, ref.bc[:, 1], B["tex_coord"]))
    P = g2[:, :3].view(np.float32).astype(np.float64)
    out["position"] = ~(np.linalg.norm(P - ref.position, axis=-1) <= B["position"])
    out["geometric_normal"] = ~_vec_ok(g2[:, 3], ref.geometric_normal, B["direction"])
    out["shading_normal"] = ~_vec_ok(g3[:, 0], ref.shading_normal, B["direction"])
    nan_t = ~np.isfinite(ref.tangent).all(1)
    with np.errstate(invalid="ignore"):
        t_ok = _vec_ok(g3[:, 1], np.where(nan_t[:, None], 1.0, ref.tangent), B["tangent"])
    out["tangent"] = ~np.where(nan_t, g3[:, 1] == NAN_TANGENT, t_ok)
    frac = ref.tex_coord - np.floor(ref.tex_coord)
    out["tex_coord"] = ~(_unorm16_ok(g3[:, 2] & 0xFFFF, frac[:, 0], B["tex_coord"], True)
                         & _unorm16_ok(g3[:, 2] >> 16, frac[:, 1], B["tex_coord"], True))
    for name, mv in (("motion", ref.motion), ("motion_prev_transform", ref.motion_obj)):
        out[name] = ~(np.abs(g1 - mv).max(1) <= B["motion"])
    a = planes[abi.BUF_ALBEDO_ACCUM].reshape(-1, 4)[pix].astype(np.float64)
    nrm = planes[abi.BUF_NORMAL_ACCUM].reshape(-1, 4)[pix].astype(np.float64)
    w = 1.0 / (1 + num_accum_frames)
    pa = pn = np.zeros((len(pix), 3))
    if num_accum_frames > 0:
        pa = accum_prev[0].reshape(-1, 4)[pix, :3].astype(np.float64)
        pn = accum_prev[1].reshape(-1, 4)[pix, :3].astype(np.float64)
    want_a = (1 - w) * pa + w * ref.albedo
    want_n = (1 - w) * pn + w * ref.shading_normal
    out["albedo"] = ~(np.abs(a[:, :3] - want_a).max(1) <= w * B["albedo"] + 8 * U * (1 + np.abs(pa).max(1)))
    out["normal"] = ~(np.abs(nrm[:, :3] - want_n).max(1) <= w * 2 * B["direction"] + 8 * U * (1 + np.abs(pn).max(1)))
    out["alpha"] = (a[:, 3] != 1) | (nrm[:, 3] != 1)
    if ref.rng is not None:
        out["rng"] = planes[abi.BUF_RNG].reshape(-1)[pix] != ref.rng
    return {k: v & keep for k, v in out.items()}


def report(bad: dict, ref: Reference) -> str:
    lines = [f"{k}: {int(v.sum())} pixels, first {ref.pix[np.flatnonzero(v)[:4]].tolist()}" for k, v in bad.items() if v.any()]
    return "; ".join(lines)
