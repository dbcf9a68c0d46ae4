"""Frames of one or two repeated shading points and the direct lighting they integrate - TEST INFRASTRUCTURE for
tests/test_oracle_restir_unbiased.py and tests/test_gpu_restir_ref.py.

Every pixel of the frame holds the same shading point (or, as a checkerboard, one of two points whose shading normals are 50
degrees apart, so testNeighbor's 0.9 normal test keeps them apart), so each pixel estimates that point's direct lighting.
The reference value is a float64 quadrature that reads none of the kernels:
  * area lights: each emitter triangle of tests/restir_scenes.py cut into n^2 sub-triangles, f Le G V at their centroids;
  * the environment: k x k sub-texels per texel of the map, the texture unit's bilinear filter (weights kept to 1/256, clamp
    addressing) at their centres, f L |cos| V times the solid angle 2 pi^2 sin(theta) du dv;
with the brute-force visibility of tests/restir_ref.py.  At n = 96 and k = 16 the quadrature agrees with n = 192 and k = 32 to
2e-6 without and 2.5e-4 with the environment (relative).

sigma comes from R independent repeats of the whole frame with fresh RNG states, because spatial reuse correlates pixels.
The mean of R repeats against the quadrature is a Student-t test with R - 1 degrees of freedom; the bound is its quantile at
1 - 5e-5, a two-sided false-alarm rate of 1e-4 per colour channel and test.
"""
from __future__ import annotations

import numpy as np
from scipy import stats

from gfxexp_b200 import abi, engine
from tests import light_ref, restir_ref, restir_scenes as S

POINT = np.array([0.3, 0.0, 0.2])
UP = np.array([0.0, 1.0, 0.0])
TILTED = np.array([0.0, np.cos(np.radians(50)), np.sin(np.radians(50))])   # dot with UP 0.64 < 0.9
FALSE_ALARM = 1e-4


def _normal(cls):
    return TILTED if cls else UP


def gbuffers(W, H, mat=S.DS3, checker=False, point=POINT) -> dict:
    yy, xx = np.mgrid[0:H, 0:W]
    cls = ((xx + yy) % 2 == 1) if checker else np.zeros((H, W), bool)
    gb0 = np.zeros((H, W, 4), np.uint32)
    gb2 = np.zeros((H, W, 4), np.uint32)
    gb2[..., :3] = np.asarray(point).astype(np.float32).view(np.uint32)
    gb2[..., 3] = S.encode(UP[None])[0]
    gb3 = np.zeros((H, W, 4), np.uint32)
    for c in (0, 1):
        n = _normal(c)
        t = np.cross(n, [0.0, 0.0, 1.0]) if c == 0 else np.array([1.0, 0.0, 0.0])
        gb3[cls == c, 0] = S.encode(n[None])[0]
        gb3[cls == c, 1] = S.encode(t[None] / np.linalg.norm(t))[0]
    gb3[..., 3] = mat
    return {abi.BUF_GBUFFER0: gb0, abi.BUF_GBUFFER1: np.zeros((H, W, 2), np.float32), abi.BUF_GBUFFER2: gb2,
            abi.BUF_GBUFFER3: gb3}, cls


def _repeat(sp, n):
    pts = restir_ref.ShadingPoints.__new__(restir_ref.ShadingPoints)
    pts.__dict__.update({k: np.repeat(v, n, axis=0) if isinstance(v, np.ndarray) else v for k, v in sp.__dict__.items()})
    return pts


def integral(s64, cam, mat=S.DS3, cls=0, n=96, k=16, env_power=1.0, env_rotation=0.0, point=POINT, mask=None):
    """float64 direct lighting of the shading point of class cls seen from cam; mask(position, normal) -> bool, if given,
    keeps only the emitter points it accepts"""
    g, _ = gbuffers(1, 2, mat, True, point)
    gb = {i: v[cls:cls + 1] for i, v in zip(range(4), g.values())}
    sp = restir_ref.ShadingPoints(s64, gb, np.array([0]), cam)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a = np.concatenate([((i + 1 / 3) / n)[(i + j) < n], ((i + 2 / 3) / n)[(i + j) < n - 1]])
    b = np.concatenate([((j + 1 / 3) / n)[(i + j) < n], ((j + 2 / 3) / n)[(i + j) < n - 1]])
    c = 1 - a - b
    em = s64.em
    pts = _repeat(sp, len(a))
    total = np.zeros(3)
    for t in range(len(em.prob)):
        w = em.world[t]
        pos = a[:, None] * w[0] + b[:, None] * w[1] + c[:, None] * w[2]
        nrm = a[:, None] * em.normals[t, 0] + b[:, None] * em.normals[t, 1] + c[:, None] * em.normals[t, 2]
        nrm = nrm @ em.normal_matrix[t].T
        nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
        cont, _ = pts.direct(pos, nrm, np.broadcast_to(em.emittance[t], pos.shape), np.zeros(len(a), bool), True)
        if mask is not None:
            cont = cont * mask(pos, nrm)[:, None]
        total += cont.sum(0) * em.area_world[t] / n ** 2
    env = getattr(s64.scene, "env_map", None)
    if env is not None:
        tex = light_ref.env_texels(env)
        h, w = tex.shape[:2]
        u = (np.arange(w * k) + 0.5) / (w * k)
        v = (np.arange(h * k) + 0.5) / (h * k)
        uu, vv = (x.reshape(-1) for x in np.meshgrid(u, v))
        radiance = env_power * bilinear(tex, uu, vv)
        d = light_ref.env_direction(uu, vv, env_rotation)
        pts = _repeat(sp, len(uu))
        cont, _ = pts.direct(d, -d, np.pi * radiance, np.ones(len(uu), bool), True)
        d_omega = (2 * np.pi / (w * k)) * (np.pi / (h * k)) * np.sin(np.pi * vv)
        total += (cont * d_omega[:, None]).sum(0)
    return total


def bilinear(tex, u, v):
    """tex2DLod with a linear filter and clamp addressing: weights kept to 8 fractional bits"""
    h, w = tex.shape[:2]
    xb, yb = u * w - 0.5, v * h - 0.5
    fx, fy = np.floor(xb), np.floor(yb)
    a = (np.floor((xb - fx) * 256 + 0.5) / 256)[:, None]
    b = (np.floor((yb - fy) * 256 + 0.5) / 256)[:, None]
    x0, x1 = np.clip(fx, 0, w - 1).astype(int), np.clip(fx + 1, 0, w - 1).astype(int)
    y0, y1 = np.clip(fy, 0, h - 1).astype(int), np.clip(fy + 1, 0, h - 1).astype(int)
    return (1 - a) * (1 - b) * tex[y0, x0] + a * (1 - b) * tex[y0, x1] + (1 - a) * b * tex[y1, x0] + a * b * tex[y1, x1]


def frame_means(make_side, sc, W, H, configure, frames, passes, repeats, checker=False, rearch=False, mat=S.DS3,
                cam_step=(0.0, 0.0, 0.0)):
    """[repeats, classes, 3]: the mean beauty of each class after `frames` frames of the launch list"""
    out = []
    for r in range(repeats):
        side = make_side(W, H)
        g, cls = gbuffers(W, H, mat, checker)
        for buf in (0, 1):
            for b, a in g.items():
                side.put(b, buf, a)
        side.put(abi.BUF_RNG, 0, np.random.default_rng(100 + r).integers(0, 1 << 62, (H, W), dtype=np.int64).astype(np.uint64))
        p = S.frame_params(sc, W, H, 0, cam_step)
        configure(p)
        for f in range(frames):
            p.camera.position = S.frame_params(sc, W, H, f, cam_step).camera.position
            p.prevCamera.position = S.frame_params(sc, W, H, f, cam_step).prevCamera.position
            p.numAccumFrames = 0
            if rearch:
                for kind, pass_id in engine.restir_rearch_frame_passes(p, f, True, True, True):
                    if kind == "restir":
                        side.run_rearch(p, pass_id)
            else:
                for kind, pass_id in engine.restir_frame_passes(p, f, passes, bool(p.enableTemporalReuse),
                                                                bool(p.useUnbiasedEstimator)):
                    if kind == "restir":
                        side.run(p, pass_id)
        beauty = side.get(abi.BUF_BEAUTY_ACCUM, 0)[..., :3]
        out.append([beauty[cls == c].mean(0) for c in ((0, 1) if checker else (0,))])
    return np.array(out)


def t_scores(means, integrals):
    """|mean - integral| / (s / sqrt(R)) per class and channel, and the bound of the false-alarm rate"""
    r = means.shape[0]
    sigma = means.std(0, ddof=1) / np.sqrt(r)
    z = np.abs(means.mean(0) - integrals) / np.maximum(sigma, 1e-12)
    return z, stats.t.ppf(1 - FALSE_ALARM / 2, r - 1)


def check(means, integrals, what):
    z, bound = t_scores(means, integrals)
    assert (z < bound).all(), f"{what}: frame means {means.mean(0)} against the integrals {integrals} ({z} standard errors, " \
                              f"bound {bound:.2f})"
