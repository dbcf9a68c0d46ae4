"""Texture filtering and bump mapping restated in numpy from common/common_device.cuh, not from oracle/ or csrc/ - TEST
INFRASTRUCTURE for tests/test_bump_oracle.py (in float32, bit for bit against the oracle) and tests/gbuffer_ref.py (in float64).

  fetch_repeat          tex2DLod with a linear filter and repeat addressing: the fraction kept to 8 bits, four texels blended
  gather_indices        tex2Dgather's footprint: one texel on when the fraction is above 255.5 / 256
  apply_bump_mapping    applyBumpMapping (:176-203): atan of the quotient, the normal not renormalised
  read_modified_normal  readModifiedNormalFromNormalMap (:205-213, y flipped) / readModifiedNormalFromHeightMap (:229-238)
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
HEIGHT_MAP = 1   # GfxBumpMapType: 0 normal map, 1 height map


def fetch_repeat(tex, u, v, dt=F32):
    """-> (blended texels [N, 4], (x0, x1, y0, y1)).  dt = float32 restates the texture unit's arithmetic; dt = float64 takes the
    same 8-bit weights from float64 coordinates"""
    H, W = tex.shape[:2]
    u, v = np.asarray(u, dt), np.asarray(v, dt)
    xB = (u - np.floor(u)) * dt(W) - dt(0.5)
    yB = (v - np.floor(v)) * dt(H) - dt(0.5)
    fx, fy = np.floor(xB), np.floor(yB)
    a = np.floor((xB - fx) * dt(256) + dt(0.5)) * dt(1 / 256)
    b = np.floor((yB - fy) * dt(256) + dt(0.5)) * dt(1 / 256)
    ix, iy = fx.astype(np.int64), fy.astype(np.int64)
    x0, x1, y0, y1 = ix % W, (ix + 1) % W, iy % H, (iy + 1) % H
    w00, w10, w01, w11 = (dt(1) - a) * (dt(1) - b), a * (dt(1) - b), (dt(1) - a) * b, a * b
    out = w00[:, None] * tex[y0, x0] + w10[:, None] * tex[y0, x1] + w01[:, None] * tex[y1, x0] + w11[:, None] * tex[y1, x1]
    return out.astype(dt), (x0, x1, y0, y1)


def fetch_margin(tex, u, v, gather=False):
    """how far (in texture coordinates) u, v lie from the nearest point where the filter's discrete choices change: a step of
    the 8-bit rounding of the fraction (fetch_repeat, every 1 / 256 texel), or the footprint's step at 255.5 / 256
    (gather_indices; the floor's own step is continuous there, the footprint wraps with it)"""
    H, W = tex.shape[:2]
    out = np.full(np.shape(u), np.inf)
    for c, n in ((np.asarray(u, np.float64), W), (np.asarray(v, np.float64), H)):
        xB = (c - np.floor(c)) * n - 0.5
        s = (xB - np.floor(xB)) * 256
        d = np.minimum(np.abs(s - 255.5), s + 0.5) if gather else np.abs(s + 0.5 - np.round(s + 0.5))
        out = np.minimum(out, d / (256 * n))
    return out


def gather_indices(tex, u, v, dt=F32):
    """the footprint of tex2Dgather: floor(xB), one texel on when the fraction is above 255.5 / 256, wrapped"""
    H, W = tex.shape[:2]
    out = []
    for c, n in ((np.asarray(u, dt), W), (np.asarray(v, dt), H)):
        xB = (c - np.floor(c)) * dt(n) - dt(0.5)
        fx = np.floor(xB)
        i = fx.astype(np.int64) + ((xB - fx) * dt(256) > dt(255.5))
        out += [i % n, (i + 1) % n]
    return out[0], out[1], out[2], out[3]


def apply_bump_mapping(n, t, b, nn):
    """applyBumpMapping in float64: the modified normal n in the frame (t, b, nn) -> [N, 9] (tangent, bitangent, normal)"""
    proj = np.hypot(n[:, 0], n[:, 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        tilt = np.arctan(proj / n[:, 2])
        qs, qc = np.sin(tilt / 2), np.cos(tilt / 2)
        qx, qy, qw = -n[:, 1] / proj * qs, n[:, 0] / proj * qs, qc
    mt = np.stack([1 - 2 * qy * qy, 2 * qx * qy, -2 * qy * qw], 1)
    mb = np.stack([2 * qx * qy, 1 - 2 * qx * qx, 2 * qx * qw], 1)
    M = np.stack([t, b, nn], 2)  # columns
    out = np.concatenate([np.einsum("kij,kj->ki", M, mt), np.einsum("kij,kj->ki", M, mb), np.einsum("kij,kj->ki", M, n)], 1)
    return np.where((proj < 1e-3)[:, None], np.concatenate([t, b, nn], 1), out)


def read_modified_normal(tex, kind, u, v):
    """the modified normal in the tangent frame, float64, at float64 texture coordinates -> [N, 3]"""
    if kind == HEIGHT_MAP:
        H, W = tex.shape[:2]
        x0, x1, y0, y1 = gather_indices(tex, u, v, np.float64)
        h = np.stack([tex[y1, x0, 0], tex[y1, x1, 0], tex[y0, x1, 0], tex[y0, x0, 0]], 1).astype(np.float64)
        coeff = 5.0 / 1024
        n = np.stack([-(coeff * W) * (h[:, 1] - h[:, 0]), (coeff * H) * (h[:, 0] - h[:, 3]), np.ones(len(h))], 1)
        return n / np.linalg.norm(n, axis=1, keepdims=True)
    blend, _ = fetch_repeat(tex, u, v, np.float64)
    n = 2 * blend[:, :3] - 1
    n[:, 1] = -n[:, 1]
    return n
