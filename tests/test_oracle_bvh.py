"""The CPU oracle pinned against reference-independent ground truth (no GPU needed):
 * struct sizes of the reference node formats,
 * the restated SBVH builder produces a valid BVH within the reference's budget,
 * bvh::traverse (first-found and canonical tie-break) equals the exhaustive brute-force closest hit,
 * any-hit equals "brute-force closest hit exists in range".
"""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import bvh_scenes as B
from tests import trace_rays as R


@pytest.fixture(scope="module")
def tiny(oracle):
    scene = scenes.tiny_city_scene()
    return scene, oracle.OracleScene(scene)


def _rays(oracle, scene, oscene, n=6000, seed=3):
    info = oscene.info()
    rng = np.random.default_rng(seed)
    lo, hi = np.array(info.sceneMin), np.array(info.sceneMax)
    rays = np.zeros(n, dtype=abi.RAY_DTYPE)
    rays["org"] = (lo + (hi - lo) * rng.uniform(-0.2, 1.2, size=(n, 3))).astype(np.float32)
    d = rng.normal(size=(n, 3))
    rays["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["tmax"] = np.float32(3.402823466e+38)
    p = abi.default_frame_params(scene, 64, 40)
    return np.concatenate([rays, oracle.primary_rays(p, 64, 40)])


def test_sbvh_build_invariants(tiny):
    scene, oscene = tiny
    info = oscene.info()
    assert info.numTriangles == scene.num_triangles
    # splittingBudget 0.3 (nrtdsm_sandbox.cpp:3177-3184): at most floor(1.3 N) references
    assert info.numTriangles <= info.numPrimRefs <= int(1.3 * info.numTriangles)
    assert oscene.validate() == ""
    nodes, refs, tris = oscene.export_bvh()
    # root is node 0, internal children are contiguous blocks (intNodeChildBaseIndex)
    assert nodes["intNodeChildBaseIndex"][0] == 1
    # every leaf chain ends with isLeafEnd
    assert (refs >> 31).sum() > 0 and (refs[-1] >> 31) == 1


def test_traverse_equals_brute_force(oracle, tiny):
    scene, oscene = tiny
    rays = _rays(oracle, scene, oscene)
    brute = oscene.trace(rays, oracle.TRACE_BRUTE_FORCE)
    canon = oscene.trace(rays, oracle.TRACE_CANONICAL)
    first, stats = oscene.trace(rays, oracle.TRACE_FIRST_FOUND, want_stats=True)
    for name, got in (("canonical", canon), ("first-found", first)):
        same = (got["dist"].view(np.uint32) == brute["dist"].view(np.uint32)) & (got["primIndex"] == brute["primIndex"]) \
            & (got["geomIndex"] == brute["geomIndex"])
        if name == "first-found":
            # ties in distance may resolve to another triangle; the distance itself must still match
            assert np.array_equal(got["dist"].view(np.uint32), brute["dist"].view(np.uint32))
        else:
            assert same.all(), f"{name}: {np.count_nonzero(~same)} rays differ from brute force"
    assert stats.numHits == np.count_nonzero(brute["primIndex"] != 0xFFFFFFFF)
    assert stats.numIntNodes > 0 and stats.maxStackDepth < 32


def test_any_hit_equals_brute_force(oracle, tiny):
    scene, oscene = tiny
    rays = _rays(oracle, scene, oscene, seed=9)
    rays["tmax"] = np.random.default_rng(2).uniform(0.5, 25.0, size=len(rays)).astype(np.float32)
    brute = oscene.trace(rays, oracle.TRACE_BRUTE_FORCE)
    anyhit = oscene.trace(rays, oracle.TRACE_ANY)
    assert np.array_equal(anyhit["primIndex"] != 0xFFFFFFFF, brute["primIndex"] != 0xFFFFFFFF)


@pytest.mark.parametrize("seed", [11, 4])
@pytest.mark.parametrize("tree", ["sbvh", "sah", "lbvh", "sah_leaf1", "lbvh_leaf1"])
@pytest.mark.parametrize("name", list(R.SCENES))
def test_walks_equal_brute_force_on_edge_rays(oracle, name, tree, seed):
    """The canonical and any-hit walks (the parity modes) on the ray families of tests/trace_rays.py - edges, vertices, axis-
    parallel directions, interval ends, the deep corridor - on the reference's SBVH and the restated GPU trees, at the rays of
    the host-compiled traversal check (seed 11) and at another seed: closest hits equal the brute force bit for bit, any-hit
    answers are "a brute-force hit exists in (tmin, tmax)"."""
    flags = {"sbvh": None, "sah": 0, "lbvh": B.BVH_BUILD_FAST, "sah_leaf1": 1, "lbvh_leaf1": B.BVH_BUILD_FAST | 1}[tree]
    o, _, fam, rays = R.gpu_style_case(oracle, name, flags, seed=seed)
    brute = o.trace(rays, oracle.TRACE_BRUTE_FORCE)
    wrong = R.wrong_per_family(fam, o.trace(rays, oracle.TRACE_CANONICAL), brute)
    assert sum(wrong.values()) == 0, f"canonical: wrong rays per family {wrong} of {R.RAYS_PER_FAMILY} each"
    wrong = R.wrong_per_family(fam, o.trace(rays, oracle.TRACE_ANY), brute, any_hit=True)
    assert sum(wrong.values()) == 0, f"any hit: wrong rays per family {wrong} of {R.RAYS_PER_FAMILY} each"


def test_node_codec_is_conservative(tiny):
    """setChildAabb (common_shared.h:839-851): decoded child boxes contain the exact ones (checked by
    orc_bvh_validate for un-split references) and quantised coordinates stay within 8 bits."""
    _, oscene = tiny
    nodes, _, _ = oscene.export_bvh()
    valid = (nodes["childQMin"][:, 0, :] != 255) | (nodes["childQMax"][:, 0, :] != 0)
    assert (nodes["childQMin"][:, :, :].transpose(0, 2, 1)[valid] <= nodes["childQMax"].transpose(0, 2, 1)[valid]).all()


def test_teapot_config1_build(oracle):
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "teapot.obj.gz")  # the reference's data/teapot.obj
    scene = scenes.teapot_like_scene(path)
    oscene = oracle.OracleScene(scene)
    info = oscene.info()
    assert info.numTriangles == 15704 + 2  # SURVEY.md §0: 15 704 faces + the rectangle light
    assert oscene.validate() == ""


# ---- the restatement of the GPU builders (oracle/gpu_bvh.cpp) --------------------------------------------------------------
_GPU_STYLE_SCENES = {
    "tiny_city": scenes.tiny_city_scene,
    "teapot": B.teapot_scene,
    **{f"soup{n}": (lambda n=n: B.soup_scene(n)) for n in (1, 2, 3, 4, 4096, 4097, 131072, 131073)},
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


@pytest.mark.parametrize("flags", [0, B.BVH_BUILD_FAST], ids=["sah", "lbvh"])
@pytest.mark.parametrize("name", list(_GPU_STYLE_SCENES))
def test_gpu_style_build_is_valid_deterministic_and_exact(oracle, name, flags):
    """The restated SAH / LBVH tree is a valid reference-format BVH, two builds give the same tree, and closest hits through it
    equal the exhaustive brute force."""
    scene = _GPU_STYLE_SCENES[name]()
    a = oracle.OracleScene(scene, build_bvh=False)
    a.build_gpu_style(flags)
    assert a.validate() == ""
    info = a.info()
    assert info.numTriangles == info.numPrimRefs == scene.num_triangles
    b = oracle.OracleScene(scene, build_bvh=False)
    b.build_gpu_style(flags)
    assert a.same_tree(b) == ""
    num_rays = max(64, min(3000, 60_000_000 // scene.num_triangles))
    rays = B.random_rays(info.sceneMin, info.sceneMax, num_rays, 17)
    bad = B.hit_mismatch(a.trace(rays, oracle.TRACE_CANONICAL), a.trace(rays, oracle.TRACE_BRUTE_FORCE))
    assert len(bad) == 0, f"{len(bad)} of {num_rays} rays differ from brute force"


def _levels(oracle, scene, flags=0):
    return oracle.OracleScene(scene, build_bvh=False).build_gpu_style(flags)


@pytest.mark.parametrize("n,root", [(3, 0), (4096, 0), (4097, 1), (131072, 1), (131073, 2)])
def test_sah_size_thresholds(oracle, n, root):
    """a root of n triangles is a small (<= 4096), big (<= 131072) or huge node"""
    levels = _levels(oracle, B.soup_scene(n))
    assert levels[0].tolist() == [1 if k == root else 0 for k in range(3)]


def test_sah_scenes_reach_their_paths(oracle):
    levels = _levels(oracle, B.clusters_scene())
    assert levels[1].tolist() == [0, 0, 2], levels[:3]  # two huge nodes in one level
    assert (levels > 0).all(axis=1).any(), levels[:4]   # huge, big and small nodes in one level
    for scene in (B.coincident_scene(), B.flat_scene(), B.lattice_scene(), B.signed_zero_scene(), B.mirror_tie_scene(),
                  B.last_bin_scene()):
        assert _levels(oracle, scene)[0].tolist() == [0, 0, 1], scene.name
    # the tied root planes: the first one cuts off the left lattice (46 k triangles, big) from the other two (big)
    assert _levels(oracle, B.mirror_tie_scene())[1].tolist() == [0, 2, 0]
    # the last plane cuts the two 100-triangle clusters (small) off the slab (huge)
    assert _levels(oracle, B.last_bin_scene())[1].tolist() == [1, 0, 1]
    # coincident centroids: no plane exists, every node is cut in the middle of its slice (a balanced tree); every binary
    # internal node is listed in exactly one level
    scene = B.coincident_scene()
    levels = _levels(oracle, scene)
    assert levels.sum() == scene.num_triangles - 1
    assert levels[1].tolist() == [0, 2, 0] and len(levels) == int(np.ceil(np.log2(scene.num_triangles)))
    assert _levels(oracle, B.soup_scene(4096), B.BVH_BUILD_FAST).shape[0] == 0  # no SAH levels for the LBVH


def test_signed_zero_scene_has_both_zeros(oracle):
    """the ±0 scene really puts both signs of zero into world-space coordinates, node origins included"""
    o = oracle.OracleScene(B.signed_zero_scene(), build_bvh=False)
    o.build_gpu_style(0)
    nodes, _, tris = o.export_bvh()
    x = np.concatenate([tris["pA"][:, 0], tris["pB"][:, 0], tris["pC"][:, 0]])
    assert ((x == 0) & np.signbit(x)).sum() > 1000 and ((x == 0) & ~np.signbit(x)).sum() > 1000
    ox = nodes["quantBoxOrigin"][:, 0]
    assert ((ox == 0) & np.signbit(ox)).any()


def test_gpu_style_flags(oracle):
    """maxLeaf 0 means 2 and values above 31 are clamped to 31; fewer than 3 triangles take the LBVH path whatever the flag;
    PLOC has no restatement"""
    scene = scenes.tiny_city_scene()

    def tree(flags, sc=scene):
        o = oracle.OracleScene(sc, build_bvh=False)
        o.build_gpu_style(flags)
        return o
    assert tree(0).same_tree(tree(2)) == ""
    assert tree(B.BVH_BUILD_FAST).same_tree(tree(B.BVH_BUILD_FAST | 2)) == ""
    assert tree(31).same_tree(tree(200)) == ""
    assert tree(4).same_tree(tree(2)) != ""
    assert tree(0).same_tree(tree(B.BVH_BUILD_FAST)) != ""
    for n in (1, 2):
        sc = B.soup_scene(n)
        assert tree(0, sc).same_tree(tree(B.BVH_BUILD_FAST, sc)) == ""
    with pytest.raises(AssertionError):
        tree(B.BVH_BUILD_PLOC)


def test_same_tree_reports_the_first_difference(oracle):
    """orc_bvh_same_tree sees a changed quantised byte and two swapped references"""
    scene = scenes.tiny_city_scene()
    ref = oracle.OracleScene(scene, build_bvh=False)
    ref.build_gpu_style(0)
    nodes, refs, tris = ref.export_bvh()
    other = oracle.OracleScene(scene, build_bvh=False)
    other.import_bvh(nodes, refs, tris)
    assert ref.same_tree(other) == ""
    leaf_node = int(np.nonzero(nodes["internalMask"] != 0xFF)[0][-1])
    bad = nodes.copy()
    bad["childQMax"][leaf_node, 1, 0] ^= 1
    other.import_bvh(bad, refs, tris)
    assert "childQMax" in ref.same_tree(other)
    bad_refs = refs.copy()
    bad_refs[[0, 1]] = ((refs[1] & 0x7FFFFFFF) | (refs[0] & 0x80000000), (refs[0] & 0x7FFFFFFF) | (refs[1] & 0x80000000))
    other.import_bvh(nodes, bad_refs, tris)
    assert "reference" in ref.same_tree(other)
