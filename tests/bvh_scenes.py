"""Synthetic scenes at the edges of the GPU BVH builders (gfxexp_b200/csrc/bvh_build.cu), shared by the CPU tests of the
builder restatement (tests/test_oracle_bvh.py) and the GPU tree comparisons (tests/test_gpu_bvh_trees.py).

The sizes follow the builder's thresholds: nodes above SAH_BIG_NODE triangles are split by one 1024-thread block, nodes
above SAH_HUGE_NODE by many blocks of SAH_HUGE_CHUNK triangles each."""
import os

import numpy as np

from gfxexp_b200 import abi, scenes

SAH_BIG_NODE = 4096
SAH_HUGE_NODE = 131072
SAH_HUGE_CHUNK = 8192
BVH_BUILD_FAST = 0x100  # GFX_BVH_BUILD_FAST: Karras LBVH; 0 is the binned-SAH hierarchy
BVH_BUILD_PLOC = 0x200

F32 = np.float32


def _materials():
    mats = np.zeros(1, dtype=scenes.MATERIAL_DTYPE)
    mats[0]["bsdfType"] = scenes.BSDF_LAMBERT
    mats[0]["p0"] = 0.5
    return mats


def scene_of(meshes, instances, name):
    """a scene of the given meshes / instances with one Lambert material and a camera looking down -z"""
    return scenes.Scene(meshes, _materials(), instances, np.array([0.0, 0.0, 10.0], F32), np.eye(3, dtype=F32), 1.0, name)


def mesh(verts, faces):
    return scenes.mesh_from_triangles(np.asarray(verts, F32), np.asarray(faces, np.uint32), 0)


def soup_mesh(n, seed, size=1.0, tri=0.02):
    """n independent small triangles with random corners in a cube of edge `size`"""
    rng = np.random.default_rng(seed)
    base = rng.uniform(0.0, size, size=(n, 1, 3))
    verts = (base + rng.uniform(-tri, tri, size=(n, 3, 3))).reshape(-1, 3)
    return mesh(verts, np.arange(3 * n, dtype=np.uint32).reshape(n, 3))


def soup_scene(n, seed=1):
    """n random triangles: one instance of one mesh"""
    return scene_of([soup_mesh(n, seed)], [scenes.make_instance([0])], f"soup{n}")


def clusters_scene():
    """Two well-separated instances of one 200 k-triangle mesh, with a 20 k-triangle cluster beyond the second and a 3 k one
    beside the first: SAH level 1 holds two huge nodes (the multi-block kernels walk a node list longer than one, and the
    second node's blocks do not start at block 0), level 2 holds huge, big and small nodes at once."""
    big = soup_mesh(200000, 2, size=10.0)
    mid = soup_mesh(20000, 3, size=3.0)
    small = soup_mesh(3000, 4, size=1.0)
    inst = [scenes.make_instance([0], (0.0, 0.0, 0.0)), scenes.make_instance([0], (1000.0, 0.0, 0.0)),
            scenes.make_instance([1], (1.0e4, 0.0, 0.0)), scenes.make_instance([2], (0.0, 0.0, 300.0))]
    return scene_of([big, mid, small], inst, "clusters")


def coincident_scene(n=SAH_HUGE_NODE + 5000):
    """n copies of one triangle: every centroid and every Morton key coincide, so every SAH split is the num / 2 fallback"""
    faces = np.zeros((n, 3), np.uint32)
    faces[:, 1], faces[:, 2] = 1, 2
    return scene_of([mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0]], faces)], [scenes.make_instance([0])], "coincident")


def flat_scene(tess=300):
    """a plane of 2 tess^2 triangles at y = 0: zero extent on one axis (bin scale 0, quantisation exponent 0)"""
    return scene_of([scenes.make_plane(tess, 50.0, 0)], [scenes.make_instance([0])], "flat")


def lattice_scene(nx=24, ny=24, nz=21):
    """identical axis-aligned unit cubes (12 triangles each) on a lattice of pitch 2, in one mesh: plane costs, axis costs
    and child areas tie exactly, so the first-minimum / first-maximum rules of the SAH and the collapse decide the tree"""
    cube = scenes.make_box(1, (1.0, 1.0, 1.0), 0)
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), axis=-1).reshape(-1, 3) * 2.0
    verts = (cube.positions[None, :, :] + g[:, None, :]).reshape(-1, 3)
    faces = (cube.triangles[None, :, :] + (np.arange(len(g)) * len(cube.positions))[:, None, None]).reshape(-1, 3)
    return scene_of([mesh(verts, faces)], [scenes.make_instance([0])], "lattice")


def mirror_tie_scene():
    """Three identical cube lattices (46 k triangles each) at x = -1000, 0 and 1000: at the huge root the planes
    {left} | {middle, right} and {left, middle} | {right} cost exactly the same (the same two terms, added in swapped order),
    and only the first-cheapest-plane rule picks between them."""
    return scene_of([lattice_scene(16, 16, 15).meshes[0]],
                    [scenes.make_instance([0], (x, 0.0, 0.0)) for x in (-1000.0, 0.0, 1000.0)], "mirror_tie")


def last_bin_scene(seed=6):
    """A 140 k-triangle slab whose centroids all fall into the last of the 16 bins, and 100-triangle clusters in bins 0
    and 14: the huge root's best plane is the last one, 15."""
    rng = np.random.default_rng(seed)

    def slab(n, x0, sx):
        base = rng.uniform(0.0, 1.0, size=(n, 1, 3)) * np.array([sx, 1.0, 1.0]) + np.array([x0, 0.0, 0.0])
        return (base + rng.uniform(-0.005, 0.005, size=(n, 3, 3))).reshape(-1, 3)
    verts = np.concatenate([slab(140000, 15.9, 0.1), slab(100, 0.0, 0.05), slab(100, 14.5, 0.05)])
    n = len(verts) // 3
    return scene_of([mesh(verts, np.arange(3 * n, dtype=np.uint32).reshape(n, 3))], [scenes.make_instance([0])], "last_bin")


def translated(scene, offset):
    """the scene moved by `offset` along every axis (coordinates far from the origin: the exponent search and the child-box
    fix-up loops of the quantisation)"""
    for inst in scene.instances:
        inst.transform = inst.transform.copy()
        inst.transform[:, 3] += F32(offset)
    scene.name = f"{scene.name}+{offset:g}"
    return scene


def signed_zero_scene(n=SAH_HUGE_NODE + 9000, seed=5):
    """Triangles whose x coordinates are often -0.0 or +0.0, both in world space: box bounds and centroids of either sign
    of zero meet in every node.  The instance transform is the identity with -0.0 off the diagonal and in the translation,
    which keeps the sign of a zero x (and y, z >= 0 unchanged)."""
    rng = np.random.default_rng(seed)
    verts = rng.uniform(0.0, 1.0, size=(3 * n, 3)).astype(F32)
    x = rng.uniform(-1.0, 1.0, size=3 * n).astype(F32)
    pick = rng.integers(0, 4, size=3 * n)
    x[pick == 0] = F32(-0.0)
    x[pick == 1] = F32(0.0)
    verts[:, 0] = x
    inst = scenes.make_instance([0])
    m = np.full((3, 4), F32(-0.0), F32)
    m[0, 0] = m[1, 1] = m[2, 2] = 1.0
    inst.transform = m
    return scene_of([mesh(verts, np.arange(3 * n, dtype=np.uint32).reshape(n, 3))], [inst], "signed_zero")


CORRIDOR_HALF_WIDTH = 0.05


def corridor_scene(n=5000):
    """n small triangles strung along x (one at every integer x, in the plane perpendicular to it, each turned by the golden
    angle against the previous one): built with maxLeaf 1, a ray along x meets every level of a deep tree and pushes up to
    seven siblings per level"""
    k = np.arange(n)
    ang = k[:, None] * 2.39996323 + np.array([0.0, 2.1, 4.2])[None, :]
    r = np.array([1.0, 0.6, 0.9]) * CORRIDOR_HALF_WIDTH
    verts = np.stack([np.broadcast_to(k[:, None], (n, 3)), r * np.cos(ang), r * np.sin(ang)], axis=-1).reshape(-1, 3)
    return scene_of([mesh(verts, np.arange(3 * n, dtype=np.uint32).reshape(n, 3))], [scenes.make_instance([0])], "corridor")


def teapot_scene():
    return scenes.teapot_like_scene(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "teapot.obj.gz"))


def random_rays(lo, hi, n, seed):
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    rays = np.zeros(n, dtype=abi.RAY_DTYPE)
    rays["org"] = (lo + (hi - lo) * rng.uniform(-0.2, 1.2, size=(n, 3))).astype(F32)
    d = rng.normal(size=(n, 3))
    rays["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)
    rays["tmax"] = F32(3.402823466e+38)
    return rays


def hit_mismatch(a, b):
    """indices of rays whose closest hits differ in distance, ids or barycentrics (bit for bit)"""
    hit = a["primIndex"] != 0xFFFFFFFF
    return np.nonzero((a["dist"].view(np.uint32) != b["dist"].view(np.uint32)) | (a["primIndex"] != b["primIndex"])
                      | (a["geomIndex"] != b["geomIndex"]) | (a["instIndex"] != b["instIndex"])
                      | ((a["bcB"].view(np.uint32) != b["bcB"].view(np.uint32)) & hit)
                      | ((a["bcC"].view(np.uint32) != b["bcC"].view(np.uint32)) & hit))[0]
