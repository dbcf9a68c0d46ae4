"""A small emitter scene, seeded synthetic ReSTIR DI frames and the two systems under test - TEST INFRASTRUCTURE for
tests/test_oracle_restir_ref.py and tests/test_gpu_restir_ref.py.

The scene (light_scenes.tri_mesh helpers) is a floor of 8 x 8 m, a down-facing quad emitter 3 m above it, a triangle emitter
facing up (away from the floor), a vertical quad emitter whose lower half a box hides from most of the floor, and the box
itself: 36 triangles.  `with_env` adds a procedural sky.

A frame's G-buffers are written directly (the G-buffer pass is skipped).  They hold:
  * floor points under a camera at (0, 6, 6), positions jittered by up to 1 cm;
  * miss pixels (a disc and 3 % single pixels);
  * points whose geometric normal faces away from the camera (frontHit = -1);
  * shading normals tilted up to 25 degrees from the geometric normal;
  * Lambert and DiffuseAndSpecular materials at smoothness 0, 0.3, 0.6 and 0.95, and an emissive material;
  * patches whose distance to the camera is 0.91 / 0.93 / 1.07 / 1.09 and 0.8 / 1.2 times their neighbours', and whose
    shading normal's dot product with the floor's is 0.88 / 0.92: either side of testNeighbor's 0.1 and 0.9;
  * motion vectors that leave the frame on every side, land in the (-1, 0) band that C's truncation maps to 0, and
    stay >= 0.01 px from the integers at which truncation changes.
Previous-frame reservoirs hold samples of the scene's lights and samples at infinity, recPDFEstimate = 0 on 10 % of them,
and M on both sides of the 20x cap (for 2^5 candidates: 639, 640, 641) and up to 2^31 - 1.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from gfxexp_b200 import abi, scenes
from tests import light_scenes, restir_ref, shading_ref

F32 = np.float32
SKY = 0xFFFFFFFF
EMIT_A, EMIT_B, LAMBERT, DS0, DS3, DS6, DS95, LAMBERT_RED = range(8)
CAM = np.array([0.0, 6.0, 6.0])
M_CHOICES = np.array([1, 5, 31, 32, 33, 639, 640, 641, 5000, 1 << 20, (1 << 31) - 5, (1 << 31) - 1], np.uint32)
SIZES = [(1, 1), (7, 3), (9, 9), (33, 17), (97, 61), (41, 1)]


def _materials() -> np.ndarray:
    m = np.zeros(8, dtype=scenes.MATERIAL_DTYPE)
    m["bsdfType"] = scenes.BSDF_DIFFUSE_AND_SPECULAR
    m["p0"] = (0.6, 0.6, 0.6)
    m["p1"] = (0.04, 0.04, 0.04)
    m["emittance"][EMIT_A] = (12.0, 10.0, 8.0)
    m["emittance"][EMIT_B] = (3.0, 5.0, 9.0)
    m["hasEmittance"][[EMIT_A, EMIT_B]] = 1
    m["bsdfType"][[LAMBERT, LAMBERT_RED]] = scenes.BSDF_LAMBERT
    m["p0"][LAMBERT_RED] = (0.8, 0.2, 0.1)
    for slot, s in ((DS0, 0.0), (DS3, 0.3), (DS6, 0.6), (DS95, 0.95)):
        m["p2"][slot] = s
    return m


def _quad(c, a, b):
    c, a, b = (np.asarray(v, np.float64) for v in (c, a, b))
    p = [c - a - b, c + a - b, c + a + b, c - a + b]
    return [[p[0], p[1], p[2]], [p[0], p[2], p[3]]]


def _box(lo, hi):
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    c, h = (lo + hi) / 2, (hi - lo) / 2
    ex, ey, ez = np.diag(h)
    tris = []
    for n, a, b in ((ex, ey, ez), (ey, ez, ex), (ez, ex, ey)):
        tris += _quad(c + n, a, b) + _quad(c - n, b, a)
    return tris


def scene(with_env: bool = False) -> scenes.Scene:
    tm = light_scenes.tri_mesh
    meshes = [
        tm(_quad((0, 0, 0), (0, 0, 4), (4, 0, 0)), DS3),                        # floor, normal +y
        tm(_quad((0.5, 3.0, -0.5), (0.6, 0, 0), (0, 0, 0.6)), EMIT_A),           # faces down
        tm([[[-2.0, 2.5, 1.0], [-1.0, 2.5, 1.5], [-1.5, 2.5, 0.5]]], EMIT_B),     # faces up, away from the floor
        tm(_quad((3.5, 1.0, 0.0), (0, 0, 0.8), (0, 0.8, 0)), EMIT_A),            # vertical, faces -x
        tm(_box((2.4, 0.0, -0.9), (2.9, 1.0, 0.9)), LAMBERT),                    # hides the lower half of the last one
    ]
    sc = scenes.Scene(meshes, _materials(), [scenes.make_instance([0, 1, 2, 3, 4])], CAM.astype(F32),
                      scenes.look_at_orientation(tuple(CAM), (0.0, 0.0, 0.0)).astype(F32), 0.8, name="restir_synthetic")
    if with_env:
        sc.env_map = scenes.procedural_sky(32, 16, sun_power=20.0, seed=3)
        sc.name += "_env"
    return sc


def encode(v):
    shape = v.shape[:-1]
    v = v.reshape(-1, 3)
    phi, theta = shading_ref.to_polar_y_up(v / np.linalg.norm(v, axis=-1, keepdims=True))
    qp = np.round(phi / (2 * np.pi) * 65535).astype(np.uint32) % 65536
    qt = np.round(theta / np.pi * 65535).astype(np.uint32)
    return (qp | (qt << 16)).reshape(shape)


def _rotate_towards(n, axis, angle):
    """n rotated by `angle` about the unit vector perpendicular to n and axis"""
    k = np.cross(n, axis)
    k /= np.maximum(np.linalg.norm(k, axis=-1, keepdims=True), 1e-12)
    return n * np.cos(angle)[..., None] + np.cross(k, n) * np.sin(angle)[..., None]


def frame_params(sc, W, H, frame, cam_step=(0.0, 0.0, 0.0)):
    p = abi.default_frame_params(sc, W, H)
    p.camera.position = (C.c_float * 3)(*(CAM + frame * np.asarray(cam_step)).astype(F32))
    p.prevCamera.position = (C.c_float * 3)(*(CAM + (frame - 1) * np.asarray(cam_step)).astype(F32))
    p.frameIndex = frame
    p.bufferIndex = frame % 2
    p.resetFlowBuffer = 0
    return p


class SyntheticFrames:
    def __init__(self, W: int, H: int, seed: int = 1):
        self.W, self.H, self.seed = W, H, seed

    def _patch(self, rng, frac):
        W, H = self.W, self.H
        x0, y0 = int(rng.uniform(0, 1 - frac) * W), int(rng.uniform(0, 1 - frac) * H)
        m = np.zeros((H, W), bool)
        m[y0:y0 + max(1, int(round(frac * H))), x0:x0 + max(1, int(round(frac * W)))] = True
        return m

    def gbuffers(self, frame: int, cam=CAM) -> dict:
        W, H = self.W, self.H
        rng = np.random.default_rng(self.seed * 1009 + frame)
        yy, xx = np.mgrid[0:H, 0:W]
        pos = np.stack([-3 + 6 * (xx + 0.5) / W, np.zeros((H, W)), -3 + 6 * (yy + 0.5) / H], -1)
        pos += rng.uniform(-0.01, 0.01, (H, W, 3)) * [1, 0, 1]
        up = np.broadcast_to([0.0, 1.0, 0.0], (H, W, 3)).copy()
        ng = up.copy()
        ng[rng.random((H, W)) < 0.05] = [0.0, -1.0, 0.0]                 # frontHit = -1
        # distance to the camera scaled either side of testNeighbor's 10 %
        scale = np.ones((H, W))
        for f in (0.91, 0.93, 1.07, 1.09, 0.8, 1.2):
            scale[self._patch(rng, 0.15)] = f
        pos = cam + (pos - cam) * scale[..., None]
        # shading normals: tilted up to 25 degrees, patches at dot 0.88 / 0.92 with the floor's
        axis = rng.normal(size=(H, W, 3))
        ns = _rotate_towards(up, axis, np.radians(rng.uniform(0, 25, (H, W))))
        for d in (0.88, 0.92):
            pm = self._patch(rng, 0.2)
            ns[pm] = _rotate_towards(up[pm], axis[pm], np.full(pm.sum(), np.arccos(d)))
        t, _ = shading_ref.make_coordinate_system(ns.reshape(-1, 3))
        mats = rng.choice([LAMBERT, DS0, DS3, DS6, DS95, LAMBERT_RED], (H, W))
        mats[self._patch(rng, 0.1)] = EMIT_A
        sky = rng.random((H, W)) < 0.03
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        sky |= (xx - cx) ** 2 + (yy - cy) ** 2 < (0.1 * max(W, H)) ** 2
        gb0 = np.zeros((H, W, 4), np.uint32)
        gb0[..., 0] = np.where(sky, SKY, 0)
        gb2 = np.zeros((H, W, 4), np.uint32)
        gb2[..., :3] = pos.astype(F32).view(np.uint32)
        gb2[..., 3] = encode(ng)
        gb3 = np.zeros((H, W, 4), np.uint32)
        gb3[..., 0] = encode(ns)
        gb3[..., 1] = encode(t.reshape(H, W, 3))
        gb3[..., 3] = np.where(sky, SKY, mats)
        return {abi.BUF_GBUFFER0: gb0, abi.BUF_GBUFFER1: self.motion(rng), abi.BUF_GBUFFER2: gb2, abi.BUF_GBUFFER3: gb3}

    def motion(self, rng):
        """x + 0.5 - mv: 60 % in frame, the rest off every side or in the (-1, 0) band; fractions in [0.01, 0.99]"""
        W, H = self.W, self.H
        yy, xx = np.mgrid[0:H, 0:W]
        out = np.zeros((H, W, 2), F32)
        for k, (n, c) in enumerate(((W, xx), (H, yy))):
            kind = rng.choice(5, (H, W), p=[0.6, 0.1, 0.1, 0.1, 0.1])
            whole = np.select([kind == 0, kind == 1, kind == 2, kind == 3],
                              [c + rng.integers(-3, 4, (H, W)), rng.integers(-5, -1, (H, W)), n + rng.integers(0, 4, (H, W)),
                               np.zeros((H, W), np.int64)], -1)
            frac = rng.uniform(0.01, 0.99, (H, W))
            v = np.where(whole < 0, whole + 1 - frac, whole + frac)     # kind 4: -1 < v < 0, truncated to column / row 0
            v = np.where(kind == 3, frac, v)
            out[..., k] = (c + 0.5 - v).astype(F32)
        return out

    def rng_states(self) -> np.ndarray:
        return np.random.default_rng(self.seed * 7 + 3).integers(0, 1 << 63, (self.H, self.W), dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)

    def reservoirs(self, s64: "restir_ref.Scene64", which: int) -> tuple:
        """(raw [3, H, W, 4] uint32, info [H, W, 2] float32) of a seeded previous reservoir plane"""
        W, H = self.W, self.H
        n = W * H
        rng = np.random.default_rng(self.seed * 31 + which)
        _, pos, nrm, le, _, _ = s64.sample(rng.random(n), rng.random(n), rng.random(n))
        inf = rng.random(n) < 0.15
        d = rng.normal(size=(n, 3))
        d[:, 1] = np.abs(d[:, 1]) + 0.2
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        pos = np.where(inf[:, None], d, pos)
        nrm = np.where(inf[:, None], -d, nrm)
        le = np.where(inf[:, None], np.pi * np.array([0.5, 0.6, 0.7]), le)
        m = rng.choice(M_CHOICES, n)
        raw = np.zeros((3, n, 4), np.uint32)
        raw[0, :, :3] = le.astype(F32).view(np.uint32)
        raw[0, :, 3] = rng.uniform(0.01, 5, n).astype(F32).view(np.uint32)
        raw[1, :, :3] = pos.astype(F32).view(np.uint32)
        raw[1, :, 3] = m | (inf.astype(np.uint32) << 31)
        raw[2, :, :3] = nrm.astype(F32).view(np.uint32)
        info = np.zeros((n, 2), F32)
        info[:, 0] = np.where(rng.random(n) < 0.1, 0.0, rng.uniform(0.01, 3, n))
        info[:, 1] = rng.uniform(0.01, 1, n)
        return raw.reshape(3, H, W, 4), info.reshape(H, W, 2)


# ---- the systems under test ------------------------------------------------------------------------------------------------
class OracleSide:
    def __init__(self, oracle, oscene, W, H):
        self.frame = oracle.OracleFrame(oscene, W, H)

    def put(self, buf, idx, arr):
        v = self.frame.buffer(buf, idx, copy=False)
        v[...] = np.ascontiguousarray(arr).view(v.dtype).reshape(v.shape)

    def get(self, buf, idx):
        return self.frame.buffer(buf, idx)

    def run(self, p, pass_id):
        self.frame.restir(p, pass_id)

    def run_rearch(self, p, pass_id):
        self.frame.restir_rearch(p, pass_id)


class DeviceSide:
    def __init__(self, ctx, W, H):
        self.ctx = ctx
        ctx.create_frame(W, H)

    def put(self, buf, idx, arr):
        self.ctx.upload(buf, idx, np.ascontiguousarray(arr))

    def get(self, buf, idx):
        self.ctx.synchronize()
        return self.ctx.download(buf, idx)

    def run(self, p, pass_id):
        self.ctx.restir(p, pass_id)

    def run_rearch(self, p, pass_id):
        self.ctx.restir(p, pass_id)


def setup_frame(sides, frames: SyntheticFrames, s64, frame: int, cam=CAM):
    """the G-buffers of `frame` and the frame before, RNG states, both reservoir planes and zero beauty on every side"""
    cur = frame % 2
    planes = [(b, cur, a) for b, a in frames.gbuffers(frame, cam).items()]
    planes += [(b, 1 - cur, a) for b, a in frames.gbuffers(frame - 1, cam).items()]
    planes.append((abi.BUF_RNG, 0, frames.rng_states()))
    for which in (0, 1):
        raw, info = frames.reservoirs(s64, which)
        planes += [(abi.BUF_RESERVOIR, which, raw), (abi.BUF_RESERVOIR_INFO, which, info)]
    planes.append((abi.BUF_BEAUTY_ACCUM, 0, np.zeros((frames.H, frames.W, 4), F32)))
    for buf, idx, arr in planes:
        for s in sides:
            s.put(buf, idx, arr)


def frame_launches(p, frame: int, spatial_passes: int, temporal: bool, unbiased: bool):
    """engine.restir_frame_passes without the G-buffer pass"""
    from gfxexp_b200 import engine
    for kind, pass_id in engine.restir_frame_passes(p, frame, spatial_passes, temporal, unbiased):
        if kind == "restir":
            yield pass_id


def ref_pass(ref: "restir_ref.RestirRef", p, pass_id):
    if pass_id == abi.RESTIR_INITIAL_RIS:
        return ref.initial_and_temporal(p, False, False)
    if pass_id == abi.RESTIR_INITIAL_AND_TEMPORAL_BIASED:
        return ref.initial_and_temporal(p, True, False)
    if pass_id == abi.RESTIR_INITIAL_AND_TEMPORAL_UNBIASED:
        return ref.initial_and_temporal(p, True, True)
    if pass_id == abi.RESTIR_SPATIAL_BIASED:
        return ref.spatial(p, False)
    if pass_id == abi.RESTIR_SPATIAL_UNBIASED:
        return ref.spatial(p, True)
    return ref.shading(p)
