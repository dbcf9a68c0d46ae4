"""GPU BVH builders against their CPU restatement (oracle/gpu_bvh.cpp): the binned-SAH and LBVH trees gfx_bvh_build exports
must be the restated trees node for node (orc_bvh_same_tree: every node field but the two base indices, every leaf's
references in order).  Closest hits cannot see a wrong split plane, an unstable partition or a badly collapsed node -
they do not depend on the tree - so this is the check of the builders themselves.  The scenes sit at the builder's edges:
the 4096 / 131072 node-size thresholds, several huge nodes in one level, mixed levels, coincident centroids, a flat scene,
exact plane, axis and area ties, a best plane in the last bin, coordinates far from the origin, both signs of zero, and
rebuilds that reuse or reallocate the scratch."""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import bvh_scenes as B

pytestmark = pytest.mark.gpu


def _check(gfx_ctx, oracle, scene, flags, num_rays=2000, uploaded=False):
    if not uploaded:
        gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh(flags)
    nodes, refs, tris = gfx_ctx.export_bvh()
    want = oracle.OracleScene(scene, build_bvh=False)
    want.build_gpu_style(flags)
    _, _, otris = want.export_bvh()
    assert np.array_equal(tris.view(np.uint8), otris.view(np.uint8)), "TriangleStorage differs from the oracle's"
    got = oracle.OracleScene(scene, build_bvh=False)
    got.import_bvh(nodes, refs, tris)
    assert got.validate() == ""
    diff = want.same_tree(got)
    assert diff == "", f"{scene.name}, flags {flags:#x}: GPU tree differs from the restatement at {diff}"
    if num_rays:
        info = want.info()
        rays = B.random_rays(info.sceneMin, info.sceneMax, num_rays, 23)
        # brute force where it is affordable; the restated tree's canonical walk equals it (tests/test_oracle_bvh.py)
        mode = oracle.TRACE_BRUTE_FORCE if num_rays * scene.num_triangles <= 200_000_000 else oracle.TRACE_CANONICAL
        bad = B.hit_mismatch(gfx_ctx.trace(rays, abi.TRACE_CLOSEST), want.trace(rays, mode))
        assert len(bad) == 0, f"{len(bad)} of {num_rays} rays differ"


@pytest.mark.parametrize("max_leaf", [0, 1, 4, 8, 31, 200])
@pytest.mark.parametrize("builder", [0, B.BVH_BUILD_FAST], ids=["sah", "lbvh"])
@pytest.mark.parametrize("scene_fn", [scenes.tiny_city_scene, scenes.small_city_scene, B.teapot_scene],
                         ids=["tiny_city", "small_city", "teapot"])
def test_existing_scenes_every_leaf_size(gfx_ctx, oracle, scene_fn, builder, max_leaf):
    """maxLeaf 0 means 2, 200 is clamped to 31"""
    _check(gfx_ctx, oracle, scene_fn(), builder | max_leaf)


@pytest.mark.parametrize("builder", [0, B.BVH_BUILD_FAST], ids=["sah", "lbvh"])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 4096, 4097, 131072, 131073])
def test_triangle_counts_at_the_thresholds(gfx_ctx, oracle, n, builder):
    """n < 3 takes the LBVH path whatever the flag; 4097 makes a big root, 131073 a huge one whose last chunk holds one
    triangle"""
    _check(gfx_ctx, oracle, B.soup_scene(n), builder)


_EDGE_SCENES = {
    "clusters": B.clusters_scene,
    "coincident": B.coincident_scene,
    "flat": B.flat_scene,
    "lattice": B.lattice_scene,
    "mirror_tie": B.mirror_tie_scene,
    "last_bin": B.last_bin_scene,
    "city+1e5": lambda: B.translated(scenes.tiny_city_scene(), 1e5),
    "city+1e6": lambda: B.translated(scenes.tiny_city_scene(), 1e6),
    "signed_zero": B.signed_zero_scene,
}


@pytest.mark.parametrize("builder", [0, B.BVH_BUILD_FAST], ids=["sah", "lbvh"])
@pytest.mark.parametrize("name", list(_EDGE_SCENES))
def test_edge_scenes(gfx_ctx, oracle, name, builder):
    # No rays for the coincident scene: every ray that meets the triangle ties with all 136 k copies, and with every child
    # area equal the collapse opens the first child each time, so the 8-wide tree is as deep as the binary one (17 levels)
    # and the GPU traverser's fixed stack (kStackSize) reports an overflow.  The tree itself is compared.
    _check(gfx_ctx, oracle, _EDGE_SCENES[name](), builder, num_rays=0 if name == "coincident" else 2000)


@pytest.mark.parametrize("builder", [0, B.BVH_BUILD_FAST], ids=["sah", "lbvh"])
def test_rebuild_with_moved_instances(gfx_ctx, oracle, builder):
    """same triangle count, new transforms: the scratch arena is reused and the tree equals a fresh build's"""
    scene = scenes.tiny_city_scene()
    _check(gfx_ctx, oracle, scene, builder)
    for step in range(1, 3):
        scene.instances = [scenes.move_instance(inst, tuple(inst.transform[:, 3] + np.float32(0.7 * step * (k % 3 - 1))),
                                                yaw_deg=5.0 * step * (k % 2)) for k, inst in enumerate(scene.instances)]
        gfx_ctx.update_instances(abi.make_instance_descs(scene.instances))
        _check(gfx_ctx, oracle, scene, builder, uploaded=True)


def test_rebuild_big_small_big(gfx_ctx, oracle):
    """changing the triangle count reallocates the scratch: big -> small -> big, both builders, equal to fresh builds"""
    for scene in (B.clusters_scene(), scenes.tiny_city_scene(), B.soup_scene(131073)):
        for builder in (0, B.BVH_BUILD_FAST):
            _check(gfx_ctx, oracle, scene, builder, num_rays=500)
