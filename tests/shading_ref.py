"""Float64 numpy restatement of the reference's shading layer, written from common/common_device.cuh (not from
gfxexp_b200/csrc/shading.cuh or oracle/shading.h), and a float64 quadrature of the DiffuseAndSpecular BRDF's directional
albedo.  TEST INFRASTRUCTURE: tests/test_shading_host.py, test_gpu_shading.py and test_gpu_furnace.py hold the float32 code
against it.

  common_device.cuh:14-25    fromPolarYUp / toPolarYUp
  common_device.cuh:27-79    barycentric, vector and texture-coordinate encoders
  common_device.cuh:92-100   makeCoordinateSystem
  common_device.cuh:112-140  offsetRayOrigin (Ray Tracing Gems ch. 6)
  common_device.cuh:285-323  concentricSampleDisk, cosineSampleHemisphere
  common_device.cuh:335-385  LambertBRDF and its setup
  common_device.cuh:443-508  GGXMicrofacetDistribution
  common_device.cuh:532-764  DiffuseAndSpecularBRDF (USE_HEIGHT_CORRELATED_SMITH, no fitted pre-integration)
  common_device.cuh:767-826  SimplePBR_BRDF and the setup of both with BSDFFlags::Regularize

Every function takes float64 arrays of records along axis 0 (directions as (N, 3)) and returns float64.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

PI = np.pi
LUM = np.array([0.2126729, 0.7151522, 0.0721750])  # sRGB_calcLuminance, basic_types.h


# ---- encoders and frames (:14-140) ------------------------------------------------------------------------------------
def from_polar_y_up(phi, theta):  # :14-20
    phi, theta = np.asarray(phi, np.float64), np.asarray(theta, np.float64)
    return np.stack([-np.sin(phi) * np.sin(theta), np.cos(theta), np.cos(phi) * np.sin(theta)], -1)


def to_polar_y_up(v):  # :21-25
    v = np.asarray(v, np.float64)
    theta = np.arccos(np.clip(v[:, 1], -1.0, 1.0))
    phi = np.fmod(np.arctan2(-v[:, 0], v[:, 2]) + 2 * PI, 2 * PI)
    return phi, theta


def decode_vector(q):  # :43-49
    q = np.asarray(q, np.uint32)
    return from_polar_y_up(2 * PI * ((q & 0xFFFF) / 65535.0), PI * ((q >> 16) / 65535.0))


def decode_tex_coords(q):  # :73-79
    q = np.asarray(q, np.uint32)
    return np.stack([(q & 0xFFFF) / 65535.0, (q >> 16) / 65535.0], -1)


def make_coordinate_system(n):  # :92-100
    n = np.asarray(n, np.float64)
    sign = np.where(n[:, 2] >= 0, 1.0, -1.0)
    a = -1 / (sign + n[:, 2])
    b = n[:, 0] * n[:, 1] * a
    t = np.stack([1 + sign * n[:, 0] ** 2 * a, sign * b, -sign * n[:, 0]], -1)
    bt = np.stack([b, sign + n[:, 1] ** 2 * a, -n[:, 1]], -1)
    return t, bt


# ---- warps (:285-323) -------------------------------------------------------------------------------------------------
def concentric_sample_disk(u0, u1):
    sx, sy = 2 * np.asarray(u0, np.float64) - 1, 2 * np.asarray(u1, np.float64) - 1
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(sx >= -sy, np.where(sx > sy, sx, sy), np.where(sx > sy, -sy, -sx))
        th = np.where(sx >= -sy, np.where(sx > sy, sy / sx, 2 - sx / sy), np.where(sx > sy, 6 + sx / sy, 4 + sy / sx))
    th = th * PI / 4
    zero = (sx == 0) & (sy == 0)
    return np.where(zero, 0.0, r * np.cos(th)), np.where(zero, 0.0, r * np.sin(th))


def cosine_sample_hemisphere(u0, u1):
    x, y = concentric_sample_disk(u0, u1)
    return np.stack([x, y, np.sqrt(np.maximum(0.0, 1 - x * x - y * y))], -1)


# ---- BSDFs (:335-826) -------------------------------------------------------------------------------------------------
@dataclass
class Bsdf:
    type: int                # 0 Lambert, 1 DiffuseAndSpecular (SimplePBR after setup)
    diffuse: np.ndarray      # (3,)
    f0: np.ndarray           # (3,)
    roughness: float


def setup(bsdf_type, p0, p1, p2, regularize=False) -> Bsdf:
    """setupBSDFBody (:376-385, :778-826) with 1x1 textures.  The float32 code computes the smoothness in float32; the
    inputs are float32 values, and the clamp 0.999 and the halving are taken at float32 so the roughness matches."""
    f32 = np.float32
    p0, p1 = np.asarray(p0, np.float64), np.asarray(p1, np.float64)
    if bsdf_type == 0:
        return Bsdf(0, p0.copy(), np.zeros(3), 1.0)
    if bsdf_type == 1:
        s = f32(p2) * f32(0.5) if regularize else f32(p2)
        s = min(s, f32(0.999))                              # :795-802: halved before the clamp
        return Bsdf(1, p0.copy(), p1.copy(), 1.0 - float(s))
    s = min(f32(1.0) - f32(p1[1]), f32(0.999))              # :819
    if regularize:
        s = s * f32(0.5)                                    # :821-823: after the clamp
    metallic = float(p1[2])
    base = p0
    return Bsdf(1, base * (1 - metallic), 0.16 * 0.5 ** 2 * (1 - metallic) + base * metallic, 1.0 - float(s))  # :767-776


def _dot(a, b):
    return np.sum(a * b, -1)


def ggx_d(alpha, m):  # :447-452
    temp = m[:, 0] ** 2 + m[:, 1] ** 2 + (m[:, 2] * alpha) ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(m[:, 2] <= 0, 0.0, alpha ** 2 / (PI * temp ** 2))


def ggx_g1(alpha, v, m):  # :453-458
    with np.errstate(divide="ignore", invalid="ignore"):
        temp = alpha ** 2 * (v[:, 0] ** 2 + v[:, 1] ** 2) / v[:, 2] ** 2
        return np.where(_dot(v, m) * v[:, 2] <= 0, 0.0, 2 / (1 + np.sqrt(1 + temp)))


def ggx_g2(alpha, v1, v2, m):  # :459-469
    with np.errstate(divide="ignore", invalid="ignore"):
        l1 = (-1 + np.sqrt(1 + alpha ** 2 * (v1[:, 0] ** 2 + v1[:, 1] ** 2) / v1[:, 2] ** 2)) / 2
        l2 = (-1 + np.sqrt(1 + alpha ** 2 * (v2[:, 0] ** 2 + v2[:, 1] ** 2) / v2[:, 2] ** 2)) / 2
        chi = ((_dot(v1, m) / v1[:, 2]) > 0) & ((_dot(v2, m) / v2[:, 2]) > 0)
        return np.where(chi, 1 / (1 + l1 + l2), 0.0)


def ggx_pdf(alpha, v, m):  # :505-507
    with np.errstate(divide="ignore", invalid="ignore"):
        return ggx_g1(alpha, v, m) * np.abs(_dot(v, m)) * ggx_d(alpha, m) / np.abs(v[:, 2])


def ggx_sample(alpha, v, u0, u1):  # :470-504, visible-normal sampling
    sv = np.stack([alpha * v[:, 0], alpha * v[:, 1], v[:, 2]], -1)
    sv /= np.linalg.norm(sv, axis=-1, keepdims=True)
    d2 = np.sqrt(sv[:, 0] ** 2 + sv[:, 1] ** 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        t1 = np.where((sv[:, 2] < 0.9999)[:, None], np.stack([sv[:, 1] / d2, -sv[:, 0] / d2, 0 * d2], -1), [1.0, 0.0, 0.0])
    t2 = np.stack([t1[:, 1] * sv[:, 2], -t1[:, 0] * sv[:, 2], d2], -1)
    a = 1 / (1 + sv[:, 2])
    r = np.sqrt(u0)
    phi = PI * np.where(u1 < a, u1 / a, 1 + (u1 - a) / (1 - a))
    p1 = r * np.cos(phi)
    p2 = r * np.sin(phi) * np.where(u1 < a, 1.0, sv[:, 2])
    m = p1[:, None] * t1 + p2[:, None] * t2 + np.sqrt(np.maximum(0.0, 1 - p1 ** 2 - p2 ** 2))[:, None] * sv
    m = np.stack([alpha * m[:, 0], alpha * m[:, 1], m[:, 2]], -1)
    m /= np.linalg.norm(m, axis=-1, keepdims=True)
    return m, ggx_d(alpha, m), ggx_pdf(alpha, v, m)


def _lerp(a, b, t):
    return (1 - t) * a + t * b


def _flip(vg, x):
    return np.where((vg[:, 2] >= 0)[:, None], x, -x)


def _weights(b: Bsdf, vg):
    """the one-sample-MIS weights of sampleThroughput / evaluatePDF (:553-564, :711-724)"""
    dv_z = np.abs(vg[:, 2])
    f_d90 = 0.5 * b.roughness + 2 * b.roughness * vg[:, 2] ** 2
    exp_diff_fresnel = _lerp(1.0, f_d90, (1 - dv_z) ** 5)
    wd = float(LUM @ b.diffuse) * exp_diff_fresnel ** 2 * _lerp(1.0, 1 / 1.51, b.roughness)
    ws = _lerp(float(LUM @ b.f0), 1.0, (1 - dv_z) ** 5)
    return wd, ws


def _brdf_value(b: Bsdf, alpha, dl, dv, m, dot_lh, d):
    """the shared tail of sampleThroughput / evaluate (:615-637, :660-687) in the entering frame"""
    g = ggx_g2(alpha, dl, dv, m)
    f = _lerp(b.f0[None, :], 1.0, ((1 - dot_lh) ** 5)[:, None])
    with np.errstate(divide="ignore", invalid="ignore"):
        spec = f * ((d * g) / (4 * dl[:, 2] * dv[:, 2]))[:, None]
    spec = np.where((g == 0)[:, None], 0.0, spec)
    f_d90 = 0.5 * b.roughness + 2 * b.roughness * dot_lh ** 2
    fo = _lerp(1.0, f_d90, (1 - dv[:, 2]) ** 5)
    fi = _lerp(1.0, f_d90, (1 - dl[:, 2]) ** 5)
    diff = b.diffuse[None, :] * (fo * fi * _lerp(1.0, 1 / 1.51, b.roughness) / PI)[:, None]
    return diff + spec


def evaluate(b: Bsdf, vg, vs):  # Lambert :358-363, DiffuseAndSpecular :648-690
    vg, vs = np.asarray(vg, np.float64), np.asarray(vs, np.float64)
    same = vg[:, 2] * vs[:, 2] > 0
    if b.type == 0:
        return np.where(same[:, None], b.diffuse[None, :] / PI, 0.0)
    alpha = b.roughness ** 2
    dv, dl = _flip(vg, vg), _flip(vg, vs)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = (dl + dv) / np.linalg.norm(dl + dv, axis=-1, keepdims=True)
        val = _brdf_value(b, alpha, dl, dv, m, _dot(dl, m), ggx_d(alpha, m))
    return np.where(same[:, None], val, 0.0)


def evaluate_pdf(b: Bsdf, vg, vs):  # Lambert :364-369, DiffuseAndSpecular :691-734
    vg, vs = np.asarray(vg, np.float64), np.asarray(vs, np.float64)
    if b.type == 0:
        return np.where(vg[:, 2] * vs[:, 2] > 0, np.abs(vs[:, 2]) / PI, 0.0)
    alpha = b.roughness ** 2
    dv, dl = _flip(vg, vg), _flip(vg, vs)
    wd, ws = _weights(b, vg)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = (dl + dv) / np.linalg.norm(dl + dv, axis=-1, keepdims=True)
        spec = 1 / (4 * _dot(dl, m)) * ggx_pdf(alpha, dv, m)
        return np.where(wd + ws == 0, 0.0, (dl[:, 2] / PI * wd + spec * ws) / (wd + ws))


def sample_throughput(b: Bsdf, vg, u0, u1):
    """(throughput, vSampled, dirPDensity); Lambert :348-357, DiffuseAndSpecular :532-647"""
    vg = np.asarray(vg, np.float64)
    u0, u1 = np.asarray(u0, np.float64), np.asarray(u1, np.float64)
    n = len(vg)
    if b.type == 0:
        vs = cosine_sample_hemisphere(u0, u1)
        pdf = vs[:, 2] / PI
        vs[:, 2] = np.where(vg[:, 2] <= 0, -vs[:, 2], vs[:, 2])
        return np.broadcast_to(b.diffuse, (n, 3)).copy(), vs, pdf
    alpha = b.roughness ** 2
    dv = _flip(vg, vg)
    wd, ws = _weights(b, vg)
    sw = wd + ws
    with np.errstate(divide="ignore", invalid="ignore"):
        take_diffuse = sw * u1 < wd
        # diffuse branch
        ld = cosine_sample_hemisphere(u0, np.where(take_diffuse, sw * u1 / wd, 0.5))
        md = (ld + dv) / np.linalg.norm(ld + dv, axis=-1, keepdims=True)
        lhd = np.minimum(_dot(ld, md), 1.0)
        specd = 1 / (4 * lhd) * ggx_pdf(alpha, dv, md)
        # specular branch
        ms, dms, mpdf = ggx_sample(alpha, dv, u0, np.where(take_diffuse, 0.5, (sw * u1 - wd) / ws))
        lhs = np.minimum(_dot(dv, ms), 1.0)
        ls = 2 * lhs[:, None] * ms - dv
        specs = 1 / (4 * lhs) * mpdf
        pick = take_diffuse[:, None]
        dl, m = np.where(pick, ld, ls), np.where(pick, md, ms)
        dot_lh = np.where(take_diffuse, lhd, lhs)
        d = np.where(take_diffuse, ggx_d(alpha, md), dms)
        spec_pdf = np.where(take_diffuse, specd, specs)
        val = _brdf_value(b, alpha, dl, dv, m, dot_lh, d)
        pdf = (dl[:, 2] / PI * wd + spec_pdf * ws) / sw
        thr = val * (dl[:, 2] / pdf)[:, None]
    dead = (sw == 0) | (~take_diffuse & (dl[:, 2] * dv[:, 2] <= 0))  # :565-568, :603-606
    thr = np.where(dead[:, None], 0.0, thr)
    pdf = np.where(dead, 0.0, pdf)
    return thr, _flip(vg, dl), pdf


def dh_reflectance_estimate(b: Bsdf, vg):  # Lambert :371-373, DiffuseAndSpecular :736-764 (the reference's ad-hoc estimate)
    vg = np.asarray(vg, np.float64)
    if b.type == 0:
        return np.broadcast_to(b.diffuse, (len(vg), 3)).copy()
    dz = np.abs(vg[:, 2])
    f_d90 = 0.5 * b.roughness + 2 * b.roughness * dz ** 2
    diff = b.diffuse[None, :] * (_lerp(1.0, f_d90, (1 - dz) ** 5) * _lerp(1.0, 1 / 1.51, b.roughness))[:, None]
    spec = _lerp(b.f0[None, :], 1.0, ((1 - dz) ** 5 * (1 - b.roughness))[:, None])
    return np.minimum(diff + spec, 1.0)


# ---- directional albedo -----------------------------------------------------------------------------------------------
def _gauss(n, a, b):
    x, w = np.polynomial.legendre.leggauss(n)
    return 0.5 * (b - a) * x + 0.5 * (b + a), 0.5 * (b - a) * w


def albedo(b: Bsdf, cos_o: float, n_xi=384, n_phi=384) -> np.ndarray:
    """rho(wo) = integral of evaluate(wo, wi) cos(theta_i) over the hemisphere of wo, in float64, per channel.

    The diffuse term is smooth: Gauss-Legendre in (cos^2 theta_i, phi_i), where cos(theta_i) dw = d(cos^2) dphi / 2.  The
    specular term is integrated over the half vector h instead of wi: dwi = 4 (v.h) dwh, and the GGX inverse CDF
    cos^2 theta_h = (1 - xi) / (1 + (alpha^2 - 1) xi) turns D(h) cos(theta_h) dwh into dxi dphi / (2 pi).  In (xi, phi) the
    integrand F G (v.h) / (cos_o cos theta_h) is bounded for every alpha, so the lobe is resolved at alpha = 1e-6 (smoothness
    0.999) as well as at alpha = 1; the xi panels are refined toward xi = 1, where wi crosses the horizon."""
    assert 0 < cos_o <= 1
    v = np.array([[np.sqrt(max(0.0, 1 - cos_o * cos_o)), 0.0, cos_o]])
    if b.type == 0:
        return b.diffuse.copy()
    alpha = b.roughness ** 2
    # diffuse part: the specular part of evaluate() is dropped by zeroing F0 and D through a Bsdf with only the diffuse term
    xs, wx = _gauss(96, 0.0, 1.0)
    ps, wp = _gauss(192, 0.0, 2 * PI)
    c2, ph = np.meshgrid(xs, ps, indexing="ij")
    ct = np.sqrt(c2).ravel()
    st = np.sqrt(1 - c2).ravel()
    l = np.stack([st * np.cos(ph.ravel()), st * np.sin(ph.ravel()), ct], -1)
    vv = np.broadcast_to(v, l.shape)
    m = (l + vv) / np.linalg.norm(l + vv, axis=-1, keepdims=True)
    dot_lh = _dot(l, m)
    f_d90 = 0.5 * b.roughness + 2 * b.roughness * dot_lh ** 2
    fd = _lerp(1.0, f_d90, (1 - cos_o) ** 5) * _lerp(1.0, f_d90, (1 - ct) ** 5) * _lerp(1.0, 1 / 1.51, b.roughness) / PI
    w2 = (wx[:, None] * wp[None, :]).ravel() / 2
    diffuse = b.diffuse * float(np.sum(fd * w2))
    # specular part over the half vector
    spec = np.zeros(3)
    edges = np.unique(np.concatenate([np.linspace(0, 1, 9), 1 - np.logspace(-2, -14, 7)]))
    ps, wp = _gauss(n_phi, 0.0, 2 * PI)
    for lo, hi in zip(edges[:-1], edges[1:]):
        xs, wx = _gauss(max(8, n_xi // 16), lo, hi)
        xi, ph = np.meshgrid(xs, ps, indexing="ij")
        xi, ph = xi.ravel(), ph.ravel()
        c2h = (1 - xi) / (1 + (alpha ** 2 - 1) * xi)
        ch = np.sqrt(np.clip(c2h, 0, 1))
        sh = np.sqrt(np.clip(1 - c2h, 0, 1))
        h = np.stack([sh * np.cos(ph), sh * np.sin(ph), ch], -1)
        vh = _dot(np.broadcast_to(v, h.shape), h)
        l = 2 * vh[:, None] * h - v
        ok = (l[:, 2] > 0) & (vh > 0)
        g = ggx_g2(alpha, np.where(ok[:, None], l, [0.0, 0.0, 1.0]), np.broadcast_to(v, h.shape), h)
        f = _lerp(b.f0[None, :], 1.0, ((1 - vh) ** 5)[:, None])
        with np.errstate(divide="ignore", invalid="ignore"):
            integrand = np.where(ok, g * vh / (cos_o * ch), 0.0)
        w = (wx[:, None] * wp[None, :]).ravel() / (2 * PI)
        spec += np.sum(f * (integrand * w)[:, None], 0)
    return diffuse + spec
