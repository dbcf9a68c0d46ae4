"""Seeded ray families at the edges of BVH traversal, shared by the host-compiled traversal check (tests/test_traverse_host.py),
the oracle's walks (tests/test_oracle_bvh.py) and the GPU kernels (tests/test_gpu_trace_edges.py).

Each family takes the exported TriangleStorage array of a scene (abi.TRI_DTYPE) and returns abi.RAY_DTYPE rays.  They aim
where a slab test with too little slack drops a box together with the hit in it: at triangle edges and vertices (which lie
on child-box faces), along axes (zero and tiny direction components, origins on box and triangle planes), at the two ends
of the ray interval, and down deep trees (stacks past the shared-memory part)."""
import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi, scenes
from tests import bvh_scenes as B

F32 = np.float32
FLT_MAX = F32(3.402823466e+38)
GUARD = F32(2.0 ** -80)  # traverseInit's smallest direction component (traverse.cuh)


def _corners(tris):
    return [np.asarray(tris[k], np.float64) for k in ("pA", "pB", "pC")]


def _unit(rng, n):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _ulp_steps(x, outward, k):
    """x (float32) moved |k| ulps per coordinate, along `outward` for k > 0 and against it for k < 0"""
    x = x.astype(F32)
    toward = np.where((outward >= 0) == (k[:, None] >= 0), F32(np.inf), F32(-np.inf)).astype(F32)
    for done in range(2):
        x = np.where(np.abs(k)[:, None] > done, np.nextafter(x, toward), x)
    return x


def _rays(org, dirs, tmin=0.0, tmax=FLT_MAX):
    rays = np.zeros(len(org), dtype=abi.RAY_DTYPE)
    rays["org"] = np.asarray(org, F32)
    rays["dir"] = np.asarray(dirs, F32)
    rays["tmin"] = tmin
    rays["tmax"] = tmax
    return rays


def _edge_targets(tris, n, rng):
    """points on random edges (a quarter exactly at a vertex), moved 0, ±1, ±2 ulps or a relative 1e-8..1e-3 of their
    distance to the centroid, towards it (inside) or away from it (outside)"""
    a, b, c = _corners(tris)
    i = rng.integers(0, len(tris), n)
    e = rng.integers(0, 3, n)
    p = np.stack([a[i], b[i], c[i]], axis=1)
    p0 = p[np.arange(n), e]
    p1 = p[np.arange(n), (e + 1) % 3]
    lam = np.where(rng.uniform(size=n) < 0.25, 0.0, rng.uniform(size=n))[:, None]
    target = p0 + lam * (p1 - p0)
    out = target - p.mean(axis=1)
    kind = rng.integers(0, 2, n)
    rel = 10.0 ** rng.uniform(-8, -3, n) * rng.choice([-1.0, 1.0], n)
    moved = target + (rel[:, None] * out)
    ulp = _ulp_steps(target.astype(F32), out, rng.integers(-2, 3, n)).astype(np.float64)
    return np.where(kind[:, None] == 0, ulp, moved), i


def edge_rays(tris, n, seed):
    """Rays through edge and vertex targets.  Half start at log-uniform distances 1e-3..10 in a random direction; the
    other half start on a random point of another triangle with tmin 0, like a bounce ray."""
    rng = np.random.default_rng(seed)
    target, src = _edge_targets(tris, n, rng)
    half = n // 2
    d = _unit(rng, n)
    dist = 10.0 ** rng.uniform(-3, 1, n)
    org = target - dist[:, None] * d
    a, b, c = _corners(tris)
    j = rng.integers(0, len(tris), n - half)
    j = np.where(j == src[half:], (j + 1) % len(tris), j)
    u, v = rng.uniform(size=(2, n - half))
    flip = u + v > 1
    u, v = np.where(flip, 1 - u, u), np.where(flip, 1 - v, v)
    org[half:] = (a[j] + u[:, None] * (b[j] - a[j]) + v[:, None] * (c[j] - a[j])).astype(F32)
    to = target[half:] - org[half:]
    d[half:] = to / np.maximum(np.linalg.norm(to, axis=1, keepdims=True), 1e-30)
    return _rays(org, d)


def axis_rays(tris, n, seed):
    """Rays with one or two direction components exactly ±0, at traverseInit's 2^-80 guard ±1 ulp, or denormal, through
    points on (and at edges of) triangles.  A third of the origins is moved onto the plane of a vertex coordinate, another
    third onto the nearest integer plane (the faces of lattice_scene's cubes)."""
    rng = np.random.default_rng(seed)
    a, b, c = _corners(tris)
    i = rng.integers(0, len(tris), n)
    u, v = rng.uniform(size=(2, n))
    u = np.where(rng.uniform(size=n) < 0.3, 0.0, u)  # on edge CA
    flip = u + v > 1
    u, v = np.where(flip, 1 - u, u), np.where(flip, 1 - v, v)
    target = a[i] + u[:, None] * (b[i] - a[i]) + v[:, None] * (c[i] - a[i])
    d = _unit(rng, n)
    special = np.array([0.0, 0.0, GUARD, np.nextafter(GUARD, F32(0)), np.nextafter(GUARD, F32(1)), 1e-40, 1.4e-45],
                       dtype=F32)
    nsmall = rng.integers(1, 3, n)
    for k in range(n):
        axes = rng.permutation(3)[:nsmall[k]]
        d[k, axes] = special[rng.integers(0, len(special), len(axes))] * rng.choice([-1.0, 1.0], len(axes))
        rest = np.setdiff1d(np.arange(3), axes)
        d[k, rest] /= np.linalg.norm(d[k, rest])
    d = d.astype(F32)
    dist = 10.0 ** rng.uniform(-3, 1, n)
    org = (target - dist[:, None] * d.astype(np.float64)).astype(F32)
    # the small components leave those coordinates at the target's (float32) value: origins on the triangle's box faces
    plane = rng.integers(0, 3, n)
    axis = rng.integers(0, 3, n)
    vert = np.stack([a, b, c], axis=1)[rng.integers(0, len(tris), n), rng.integers(0, 3, n)]
    rows = np.arange(n)
    org[rows, axis] = np.where(plane == 0, vert[rows, axis].astype(F32),
                               np.where(plane == 1, np.round(org[rows, axis]), org[rows, axis]))
    return _rays(org, d)


def interval_rays(rays, hits):
    """The rays that hit at distance t, retraced with tmax and tmin set to t and to nextafter(t, ±inf): the triangle test is
    strict at both ends, so tmax = t must miss that triangle and tmin = t must too"""
    hit = (hits["primIndex"] != 0xFFFFFFFF) & np.isfinite(hits["dist"]) & (hits["dist"] > 0)
    base, t = rays[hit], hits["dist"][hit].astype(F32)
    out = []
    for end in ("tmax", "tmin"):
        for v in (t, np.nextafter(t, F32(np.inf)), np.nextafter(t, F32(-np.inf))):
            r = base.copy()
            r[end] = v
            if end == "tmin":
                r["tmax"] = FLT_MAX
            out.append(r)
    return np.concatenate(out) if out else rays[:0]


def corridor_rays(length, half_width, n, seed):
    """rays along the corridor axis (corridor_scene) in both directions, from beyond either end and from inside, exactly
    axis-parallel or tilted by at most 1e-4, at lateral offsets that hit some of the triangles and miss others"""
    rng = np.random.default_rng(seed)
    sign = rng.choice([-1.0, 1.0], n)
    start = np.where(rng.uniform(size=n) < 0.7, np.where(sign > 0, -1.0, length + 1.0), rng.uniform(0, length, n))
    org = np.stack([start, *rng.uniform(-1.2 * half_width, 1.2 * half_width, (2, n))], axis=1)
    tilt = np.where(rng.uniform(size=n) < 0.5, 0.0, 1e-4)[:, None] * _unit(rng, n)
    d = np.stack([sign, np.zeros(n), np.zeros(n)], axis=1) + tilt
    return _rays(org, d / np.linalg.norm(d, axis=1, keepdims=True))


def families(tris, n, seed, closest, corridor=None):
    """{family: rays}, about n rays each: edge and axis rays, the interval-end retrace of their hits (`closest(rays)` gives
    the reference hits), and the corridor rays when `corridor` = (length, half width) names a corridor_scene"""
    fam = {"edge": edge_rays(tris, n, seed), "axis": axis_rays(tris, n, seed + 1)}
    base = np.concatenate([fam["edge"], fam["axis"]])
    ends = interval_rays(base, closest(base))
    fam["interval"] = ends[np.random.default_rng(seed + 2).permutation(len(ends))[:n]]
    if corridor is not None:
        fam["corridor"] = corridor_rays(corridor[0], corridor[1], n, seed + 3)
    return fam


def leaf_tris(refs, tris):
    """the traversal's leaf-ordered triangle copy (k_leafTris, bvh_build.cu): TriangleStorage of every primitive reference
    with the reference word in the padding field, as [numPrimRefs, 12] uint32"""
    out = tris.view(np.uint32).reshape(-1, 12)[refs & 0x7FFFFFFF].copy()
    out[:, 11] = refs
    return out


def wrong_per_family(fam, got, want, any_hit=False, instances=True):
    """{family: number of rays whose answer differs}; `got` / `want` are hit records in the order of fam's rays.  Closest
    hits compare bit for bit (bvh_scenes.hit_mismatch; instances=False leaves out the instance id, which the traversal
    itself does not produce), any-hit answers by occlusion."""
    out, at = {}, 0
    for name, rays in fam.items():
        g, w = got[at:at + len(rays)].copy(), want[at:at + len(rays)].copy()
        at += len(rays)
        if not instances:
            g["instIndex"] = w["instIndex"] = 0
        if any_hit:
            out[name] = int(np.count_nonzero((g["primIndex"] != 0xFFFFFFFF) != (w["primIndex"] != 0xFFFFFFFF)))
        else:
            out[name] = len(B.hit_mismatch(g, w))
    return out


SCENES = {
    "lattice": lambda: B.lattice_scene(10, 10, 10),
    "tiny_city": scenes.tiny_city_scene,
    "teapot": B.teapot_scene,
    "flat": lambda: B.flat_scene(60),
    "city+1e5": lambda: B.translated(scenes.tiny_city_scene(), 1e5),
    "corridor": B.corridor_scene,
}
RAYS_PER_FAMILY = 3000


def gpu_style_case(oracle, name, flags, n=RAYS_PER_FAMILY, seed=11):
    """(oracle scene holding the restated GPU tree of gfx_bvh_build(flags), or the reference's SBVH for flags None,
    the exported tree, {family: rays}, all rays in family order)"""
    scene = SCENES[name]()
    o = oracle.OracleScene(scene, build_bvh=flags is None)
    if flags is not None:
        o.build_gpu_style(flags)
    nodes, refs, tris = o.export_bvh()
    corridor = (scene.num_triangles - 1, B.CORRIDOR_HALF_WIDTH) if name == "corridor" else None
    fam = families(tris, n, seed, lambda r: o.trace(r, oracle.TRACE_BRUTE_FORCE), corridor)
    return o, (nodes, refs, tris), fam, np.concatenate(list(fam.values()))


def build_host_traversal(out_dir):
    """Compiles tests/cpp/traverse_host.cpp (traverse.cuh for the CPU, -ffp-contract=off like nvcc's -fmad=false) into
    out_dir and returns trace(nodes, refs, tris, rays, mode) -> (hits, deepest stack, overflowed); mode 0 closest hit, 1 any
    hit, 2 any hit with postponed leaf tests."""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "traverse_host.cpp")
    lib = os.path.join(str(out_dir), "traverse_host.so")
    inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + inc, "-o", lib, src],
                   check=True)
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.trace_host.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.trace_host.restype = C.c_int

    def trace(nodes, refs, tris, rays, mode):
        leaves = leaf_tris(refs, tris)
        nodes, rays = np.ascontiguousarray(nodes), np.ascontiguousarray(rays)
        hits = np.zeros(len(rays), dtype=abi.HIT_DTYPE)
        depth, overflow = C.c_int(0), C.c_int(0)
        assert L.trace_host(nodes.ctypes.data, len(nodes), leaves.ctypes.data, rays.ctypes.data, len(rays), hits.ctypes.data,
                            mode, C.byref(depth), C.byref(overflow)) == 0
        return hits, depth.value, bool(overflow.value)
    return trace
