"""The three ways to run the shading layer's op table (gfxexp_b200/csrc/shading_debug.cuh) on arrays, and the input grid
the shading tests share.  TEST INFRASTRUCTURE.

  host    tests/cpp/shading_host.cpp: shading.cuh compiled for the CPU with g++ -ffp-contract=off
  oracle  orc_shading_debug of oracle/liboracle.so: the same table over oracle/shading.h
  device  gfx_shading_debug of the library, one thread per record on the GPU

Records are 8 float32 in and 8 out; a material is 9 float32 {bsdfType, p0[3], p1[3], p2, regularize}.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

(EVALUATE, EVALUATE_PDF, SAMPLE, DH_REFLECTANCE, CONCENTRIC_DISK, COSINE_HEMISPHERE, TO_POLAR, FROM_POLAR, ENCODE_VECTOR,
 DECODE_VECTOR, ENCODE_BARYCENTRIC, DECODE_BARYCENTRIC, ENCODE_TEXCOORDS, DECODE_TEXCOORDS, COORDINATE_SYSTEM,
 OFFSET_RAY_ORIGIN) = range(16)
BSDF_OPS = (EVALUATE, EVALUATE_PDF, SAMPLE, DH_REFLECTANCE)
STRIDE = 8


def material(bsdf_type, p0, p1=(0.0, 0.0, 0.0), p2=0.0, regularize=False) -> np.ndarray:
    return np.array([bsdf_type, *np.broadcast_to(p0, 3), *np.broadcast_to(p1, 3), p2, 1.0 if regularize else 0.0],
                    dtype=np.float32)


def records(*cols) -> np.ndarray:
    """packs columns ((N,) or (N, k) arrays) into (N, 8) float32 records"""
    n = len(cols[0])
    out = np.zeros((n, STRIDE), dtype=np.float32)
    k = 0
    for c in cols:
        c = np.asarray(c)
        c = c.reshape(n, -1)
        if c.dtype == np.uint32:
            c = c.view(np.float32)
        out[:, k:k + c.shape[1]] = c
        k += c.shape[1]
    return out


def build_host(out_dir):
    """compiles tests/cpp/shading_host.cpp into out_dir and returns run(op, material, records) -> (N, 8) float32"""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "shading_host.cpp")
    lib = os.path.join(str(out_dir), "shading_host.so")
    inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + inc, "-o", lib, src], check=True)
    L = C.CDLL(lib)
    L.shading_host.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    L.shading_host.restype = C.c_int

    def run(op, mat, rec):
        mat, rec = np.ascontiguousarray(mat, np.float32), np.ascontiguousarray(rec, np.float32)
        out = np.empty_like(rec)
        assert L.shading_host(op, mat.ctypes.data, rec.ctypes.data, len(rec), out.ctypes.data) == 0
        return out
    return run


def oracle_runner(oracle):
    L = oracle.lib()
    L.orc_shading_debug.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.orc_shading_debug.restype = C.c_int

    def run(op, mat, rec):
        mat, rec = np.ascontiguousarray(mat, np.float32), np.ascontiguousarray(rec, np.float32)
        out = np.empty_like(rec)
        assert L.orc_shading_debug(op, mat.ctypes.data, rec.ctypes.data, len(rec), out.ctypes.data) == 0
        return out
    return run


def device_runner(ctx):
    import torch

    def run(op, mat, rec):
        mat = np.ascontiguousarray(mat, np.float32)
        a = torch.from_numpy(np.ascontiguousarray(rec, np.float32)).cuda()
        out = torch.full_like(a, float("nan"))
        ctx._check(ctx.lib.gfx_shading_debug(ctx.h, None, op, mat.ctypes.data, a.data_ptr(), a.shape[0], out.data_ptr()),
                   "gfx_shading_debug")
        torch.cuda.synchronize()
        return out.cpu().numpy()
    return run


# ---- the grid ---------------------------------------------------------------------------------------------------------
SMOOTHNESS = (0.0, 0.3, 0.5, 0.78, 0.9, 0.99, 0.999, 1.0)
COLOURS = {"black": (0.0, 0.0, 0.0), "grey": (0.5, 0.5, 0.5), "white": (1.0, 1.0, 1.0)}
# diffuse / F0 pairs of DiffuseAndSpecular: every black / grey / white combination, and the issue's coloured pair
DS_PAIRS = [(d, f) for d in COLOURS for f in COLOURS] + [("(.5,.4,.3)", "F0 .04")]
_EXTRA = {"(.5,.4,.3)": (0.5, 0.4, 0.3), "F0 .04": (0.04, 0.04, 0.04)}
METALLIC = (0.0, 0.5, 1.0)
F32_ONE_MINUS_ULP = float(np.nextafter(np.float32(1), np.float32(0)))
COS_O = (1.0, F32_ONE_MINUS_ULP, 0.7, 0.2, 1e-3, 1e-6, 0.0, -0.0, -1e-6, -0.5)
PHI_O = 0.3  # azimuth of vGiven: off the axes, so that no component of it is exactly zero by accident


def _col(name):
    return COLOURS.get(name, _EXTRA.get(name))


def materials():
    """[(id, material record)] over the grid: Lambert, DiffuseAndSpecular and SimplePBR, REGULARIZE off and on"""
    out = []
    for reg in (False, True):
        r = "-reg" if reg else ""
        for c in ("black", "grey", "white"):
            out.append((f"lambert-{c}{r}", material(0, _col(c), regularize=reg)))
        for s in SMOOTHNESS:
            for d, f in DS_PAIRS:
                out.append((f"ds-s{s}-d{d}-f{f}{r}", material(1, _col(d), _col(f), s, reg)))
            for c in ("black", "grey", "white"):
                for mt in METALLIC:
                    out.append((f"pbr-s{s}-{c}-m{mt}{r}", material(2, _col(c), (1.0, 1.0 - s, mt), 0.0, reg)))
    return out


def view_dirs(cos_o=COS_O, phi=PHI_O):
    """vGiven at each cos(theta_o), computed in float64 and rounded once; +-0 keep their sign"""
    c = np.array(cos_o, dtype=np.float64)
    s = np.sqrt(np.maximum(0.0, 1 - c * c))
    v = np.stack([s * np.cos(phi), s * np.sin(phi), c], -1).astype(np.float32)
    v[:, 2] = np.array(cos_o, dtype=np.float32)
    return v


def pcg_floats(n, seed=0x853C49E6748FEA9B):
    """n draws of PCG32RNG::getFloat0cTo1o (common_shared.h:116-138): the lattice k 2^-23 the renderers draw from"""
    mask = (1 << 64) - 1
    state = seed & mask
    out = np.empty(n, dtype=np.uint32)
    for i in range(n):
        old = state
        state = (old * 6364136223846793005 + 1) & mask
        xs = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        out[i] = ((xs >> rot) | (xs << ((-rot) & 31))) & 0xFFFFFFFF
    return (((out >> 9) | 0x3F800000).view(np.float32) - np.float32(1)).astype(np.float32)


U_EDGES = np.array([0.0, 2.0 ** -23, 1 - 2.0 ** -24], dtype=np.float32)


def u_pairs(n_pcg=1024):
    """(u0, u1) pairs: PCG32 draws, plus every combination of 0, 2^-23, 1 - 2^-24 with each other and with 0.5"""
    p = pcg_floats(2 * n_pcg).reshape(-1, 2)
    e = np.concatenate([U_EDGES, [np.float32(0.5)]])
    ee = np.stack(np.meshgrid(e, e), -1).reshape(-1, 2).astype(np.float32)
    return np.concatenate([p, ee])


def stratified(n):
    """n x n stratified (u0, u1), cell centres rounded to float32"""
    g = (np.arange(n) + 0.5) / n
    u0, u1 = np.meshgrid(g, g, indexing="ij")
    return u0.ravel().astype(np.float32), u1.ravel().astype(np.float32)


def sphere_dirs(n, seed=5):
    """n float32 directions spread over the sphere, plus the axes and a few near-horizon ones"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    extra = np.array([[0, 0, 1], [0, 0, -1], [1, 0, 0], [0, 1, 0], [0.6, 0.8, 0], [0.6, 0.8, -0.0], [0.6, 0.8, 1e-6],
                      [0.6, 0.8, -1e-6]], dtype=np.float64)
    return np.concatenate([d, extra]).astype(np.float32)


def bsdf_inputs(host=None, mat=None):
    """{op: records} for the four BSDF ops over the grid's view directions.  With host and mat, evaluate / evaluatePDF also
    run at the directions sampleThroughput picked and at the mirror direction (the lobe's peak)."""
    vg = view_dirs()
    u = u_pairs()
    vv = np.repeat(vg, len(u), axis=0)
    uu = np.tile(u, (len(vg), 1))
    samp = records(vv, uu)
    ls = [sphere_dirs(512)]
    out = {SAMPLE: samp, DH_REFLECTANCE: records(vg)}
    pairs_v, pairs_l = [np.repeat(vg, len(ls[0]), axis=0)], [np.tile(ls[0], (len(vg), 1))]
    mirror = vg * np.array([-1, -1, 1], dtype=np.float32)
    pairs_v.append(vg)
    pairs_l.append(mirror)
    if host is not None:
        s = host(SAMPLE, mat, samp)
        pairs_v.append(vv)
        pairs_l.append(s[:, 3:6])
    ev = records(np.concatenate(pairs_v), np.concatenate(pairs_l))
    out[EVALUATE] = ev
    out[EVALUATE_PDF] = ev
    return out


def helper_inputs():
    """{op: records} for the warps, encoders, frames and offsetRayOrigin"""
    u = u_pairs()
    rng = np.random.default_rng(9)
    dirs = sphere_dirs(4096)
    codes = np.concatenate([rng.integers(0, 2 ** 32, 8192, dtype=np.uint64).astype(np.uint32),
                            np.array([0, 0xFFFF, 0xFFFF0000, 0xFFFFFFFF, 0x7FFF7FFF, 0x00010001], dtype=np.uint32)])
    phi = np.concatenate([rng.random(4096) * 2 * np.pi, [0, np.pi, 2 * np.pi, -1.0, 7.0]]).astype(np.float32)
    theta = np.concatenate([rng.random(4096) * np.pi, [0, np.pi / 2, np.pi, 0, 0]]).astype(np.float32)
    bc = np.concatenate([rng.random(4096), [0, 1, -1e-8, 1 + 1e-7, 2, -3, np.nan, np.inf, -np.inf, 0.5 / 65535,
                                            1 - 0.5 / 65535]]).astype(np.float32)
    tc = np.concatenate([rng.random((4096, 2)) * 8 - 4, [[0, 1], [-1e-8, 1 + 1e-7], [np.nan, 2.5], [-0.0, -1.0]]]).astype(np.float32)
    normals = np.concatenate([dirs, near_pole_normals()])
    p, n = offset_inputs()
    return {
        CONCENTRIC_DISK: records(u), COSINE_HEMISPHERE: records(u), TO_POLAR: records(dirs), FROM_POLAR: records(phi, theta),
        ENCODE_VECTOR: records(dirs), DECODE_VECTOR: records(codes), ENCODE_BARYCENTRIC: records(bc),
        DECODE_BARYCENTRIC: records(np.arange(65536, dtype=np.uint32)), ENCODE_TEXCOORDS: records(tc),
        DECODE_TEXCOORDS: records(codes), COORDINATE_SYSTEM: records(normals), OFFSET_RAY_ORIGIN: records(p, n),
    }


def near_pole_normals():
    """unit normals at and near +-z, including z = -0 on the equator"""
    out = [[0, 0, 1], [0, 0, -1], [1, 0, -0.0], [0, 1, -0.0], [0.6, 0.8, -0.0], [0.6, 0.8, 0.0]]
    for e in (1e-7, 1e-6, 1e-4, 1e-3, 1e-2):
        for sz in (1, -1):
            for ang in (0.1, 2.0, 4.0):
                x, y = e * np.cos(ang), e * np.sin(ang)
                out.append([x, y, sz * np.sqrt(1 - x * x - y * y)])
    v = np.array(out, dtype=np.float64)
    v[2:4, 2] = -0.0
    return v.astype(np.float32)


def offset_inputs(seed=13):
    """(p, n) pairs for offsetRayOrigin: |p| around 1/32 (both sides of the switch), +-0, denormals, up to 1e4"""
    rng = np.random.default_rng(seed)
    mags = np.array([0.0, 1e-40, 1e-38, 1e-6, 1 / 32 * (1 - 2 ** -23), 1 / 32, 1 / 32 * (1 + 2 ** -23), 0.03, 0.04, 1.0, 37.5,
                     1e3, 1e4], dtype=np.float64)
    p = []
    for m in mags:
        for s in (1, -1):
            p.append([s * m, -s * m, m])
    p = np.array(p, dtype=np.float32)
    p[0] = [0.0, -0.0, 0.0]
    p[1] = [-0.0, 0.0, -0.0]
    n = rng.normal(size=(len(p) * 16, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    pp = np.repeat(p, 16, axis=0)
    n[::16] = [0, 0, 1]
    n[1::16] = [0, 0, -1]
    return pp, n.astype(np.float32)
