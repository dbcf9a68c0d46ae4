"""Every traversal kernel against the exhaustive brute force on the ray families of tests/trace_rays.py (rays at triangle
edges and vertices, axis-parallel rays, rays whose interval ends at their hit, rays down a deep tree).

Kernels: gfx_trace (the wavefront kernel, also with GFX_TRACE_STATS, whose hits must equal the plain ones) and the three
kernels of gfx_trace_debug - the wavefront kernel, the wavefront kernel with postponed leaf tests (ReSTIR visibility
queue) and the fused one-ray-per-thread traversal (G-buffer, lighting any-hit).  Trees: the SAH, LBVH and PLOC builders at
maxLeaf 1 and the default, and the reference's SBVH through gfx_bvh_import.  Closest hits must equal the brute force bit for
bit, any-hit answers "a brute-force hit exists in (tmin, tmax)", and every answer must equal what the same traversal code
gives when compiled for the CPU (tests/cpp/traverse_host.cpp)."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import bvh_scenes as B
from tests import trace_rays as R

pytestmark = pytest.mark.gpu

RAYS_PER_FAMILY = 2000  # brute force: about 6 x 2000 rays x (at most 15 706 triangles) < 2e8 ray-triangle tests per scene
TREES = {"sah_leaf1": 1, "sah": 0, "lbvh_leaf1": B.BVH_BUILD_FAST | 1, "lbvh": B.BVH_BUILD_FAST,
         "ploc_leaf1": B.BVH_BUILD_PLOC | 1, "ploc": B.BVH_BUILD_PLOC, "sbvh": None}


@pytest.fixture(scope="module")
def host_trace(tmp_path_factory):
    return R.build_host_traversal(tmp_path_factory.mktemp("traverse_host"))


_CASES = {}


def _scene_case(oracle, name):
    """per scene, once: the scene, an oracle scene holding its SBVH, the ray families and their brute-force closest hits"""
    if name not in _CASES:
        scene = R.SCENES[name]()
        o = oracle.OracleScene(scene)
        _, _, tris = o.export_bvh()
        corridor = (scene.num_triangles - 1, B.CORRIDOR_HALF_WIDTH) if name == "corridor" else None
        fam = R.families(tris, RAYS_PER_FAMILY, 29, lambda r: o.trace(r, oracle.TRACE_BRUTE_FORCE), corridor)
        rays = np.ascontiguousarray(np.concatenate(list(fam.values())))
        _CASES.clear()  # one scene at a time (the parametrisation keeps a scene's trees together)
        _CASES[name] = (scene, o, fam, rays, o.trace(rays, oracle.TRACE_BRUTE_FORCE))
    return _CASES[name]


def _debug_trace(ctx, rays, mode, kernel):
    import torch
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_hits = torch.zeros(len(rays) * abi.HIT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    ctx.trace_debug(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), mode, kernel)
    ctx.synchronize()
    return d_hits.cpu().numpy().view(abi.HIT_DTYPE)


@pytest.mark.parametrize("tree", list(TREES))
@pytest.mark.parametrize("name", list(R.SCENES))
def test_kernels_equal_brute_force(gfx_ctx, oracle, host_trace, name, tree):
    scene, o, fam, rays, brute = _scene_case(oracle, name)
    gfx_ctx.upload_scene(scene)
    if TREES[tree] is None:
        gfx_ctx.import_bvh(*o.export_bvh())
    else:
        gfx_ctx.build_bvh(TREES[tree])
    nodes, refs, tris = gfx_ctx.export_bvh()
    wrong = {}
    closest = {"gfx_trace": gfx_ctx.trace(rays, abi.TRACE_CLOSEST),
               "gfx_trace stats": gfx_ctx.trace(rays, abi.TRACE_CLOSEST | abi.TRACE_STATS),
               "kernel 0": _debug_trace(gfx_ctx, rays, abi.TRACE_CLOSEST, 0),
               "kernel 2": _debug_trace(gfx_ctx, rays, abi.TRACE_CLOSEST, 2)}
    host = host_trace(nodes, refs, tris, rays, 0)[0]
    for kernel, got in closest.items():
        wrong[f"closest, {kernel}"] = R.wrong_per_family(fam, got, brute)
        wrong[f"closest, {kernel} vs host"] = R.wrong_per_family(fam, got, host, instances=False)
    anyhit = {"gfx_trace": gfx_ctx.trace(rays, abi.TRACE_ANY),
              "gfx_trace stats": gfx_ctx.trace(rays, abi.TRACE_ANY | abi.TRACE_STATS),
              "kernel 0": _debug_trace(gfx_ctx, rays, abi.TRACE_ANY, 0),
              "kernel 1": _debug_trace(gfx_ctx, rays, abi.TRACE_ANY, 1),
              "kernel 2": _debug_trace(gfx_ctx, rays, abi.TRACE_ANY, 2)}
    host_any = host_trace(nodes, refs, tris, rays, 1)[0]
    for kernel, got in anyhit.items():
        wrong[f"any hit, {kernel}"] = R.wrong_per_family(fam, got, brute, any_hit=True)
        same = (got["dist"].view(np.uint32) == host_any["dist"].view(np.uint32)) & (got["primIndex"] == host_any["primIndex"])
        wrong[f"any hit, {kernel} vs host"] = {"all": int(np.count_nonzero(~same))}
    bad = {k: v for k, v in wrong.items() if sum(v.values())}
    assert not bad, f"{name}, {tree}: wrong rays per family (of {RAYS_PER_FAMILY} each): {bad}"


def test_trace_debug_rejects_unknown_kernels_and_modes(gfx_ctx):
    gfx_ctx.upload_scene(scenes.tiny_city_scene())
    gfx_ctx.build_bvh(0)
    rays = B.random_rays([0, 0, 0], [1, 1, 1], 4, 1)
    for mode, kernel in ((abi.TRACE_CLOSEST, 3), (abi.TRACE_CLOSEST, -1), (abi.TRACE_CLOSEST, 1),
                         (abi.TRACE_ANY | abi.TRACE_STATS, 1), (4, 0), (4, 2)):
        with pytest.raises(engine.GfxError, match="status -1: gfx_trace_debug: kernel 0"):
            _debug_trace(gfx_ctx, rays, mode, kernel)


def test_stack_overflow_is_reported_once_and_cleared():
    """A traversal whose stack overflows (the coincident scene: 17 levels of ties) makes the next gfx_synchronize fail with
    the overflow named; that report clears it, and so do gfx_bvh_build and gfx_bvh_import: the context then traces a sound
    tree normally."""
    import torch
    ctx = engine.Context(0)
    try:
        ctx.upload_scene(B.coincident_scene())
        ctx.build_bvh(0)
        rays = np.zeros(64, dtype=abi.RAY_DTYPE)
        rays["org"] = np.column_stack([np.linspace(0.05, 0.4, 64), np.full(64, 0.2), np.full(64, 1.0)]).astype(np.float32)
        rays["dir"] = (0.0, 0.0, -1.0)
        rays["tmax"] = R.FLT_MAX
        with pytest.raises(engine.GfxError, match="overflow"):
            ctx.trace(rays, abi.TRACE_CLOSEST)
        ctx.synchronize()  # reported once
        # set it again without a synchronize, then build a sound scene: the build clears it
        d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
        d_hits = torch.zeros(len(rays) * 32, dtype=torch.uint8, device="cuda")
        ctx.trace_device(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), abi.TRACE_CLOSEST)
        torch.cuda.synchronize()
        city = scenes.tiny_city_scene()
        ctx.upload_scene(city)
        ctx.build_bvh(0)
        ctx.synchronize()
        city_tree = ctx.export_bvh()
        # and once more, then import the city's tree without a build: the import clears it
        ctx.upload_scene(B.coincident_scene())
        ctx.build_bvh(0)
        ctx.trace_device(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), abi.TRACE_CLOSEST)
        torch.cuda.synchronize()
        ctx.upload_scene(city)
        ctx.import_bvh(*city_tree)
        ctx.synchronize()
        from tests import oracle_lib
        o = oracle_lib.OracleScene(city, build_bvh=False)
        o.import_bvh(*ctx.export_bvh())
        info = ctx.bvh_info()
        city_rays = B.random_rays(info.sceneMin, info.sceneMax, 2000, 3)
        bad = B.hit_mismatch(ctx.trace(city_rays, abi.TRACE_CLOSEST), o.trace(city_rays, oracle_lib.TRACE_BRUTE_FORCE))
        assert len(bad) == 0
    finally:
        ctx.close()
