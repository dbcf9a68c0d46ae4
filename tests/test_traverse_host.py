"""The CUDA traversal (gfxexp_b200/csrc/traverse.cuh), compiled for the CPU by tests/cpp/traverse_host.cpp, against the
exhaustive brute force on the ray families of tests/trace_rays.py: closest hits bit for bit, any-hit answers (immediate
and postponed leaf tests) by occlusion.  The trees are the CPU restatements of the GPU builders (oracle/gpu_bvh.cpp), SAH
and LBVH at maxLeaf 1 and the default, and the reference's SBVH.  No GPU is needed: the host build rounds every float
operation like sm_90a."""
import pytest

from tests import bvh_scenes as B
from tests import trace_rays as R
from tests.trace_rays import RAYS_PER_FAMILY, SCENES, gpu_style_case


@pytest.fixture(scope="module")
def host_trace(tmp_path_factory):
    return R.build_host_traversal(tmp_path_factory.mktemp("traverse_host"))


@pytest.mark.parametrize("tree", ["sah_leaf1", "sah", "lbvh_leaf1", "lbvh", "sbvh"])
@pytest.mark.parametrize("name", list(SCENES))
def test_host_traversal_equals_brute_force(oracle, host_trace, name, tree):
    """the restated GPU trees, and the reference's SBVH (imported through gfx_bvh_import on the GPU), whose boxes contain
    their triangles only as decoded in float (corner + q * 2^e rounded)"""
    flags = {"sah_leaf1": 1, "sah": 0, "lbvh_leaf1": B.BVH_BUILD_FAST | 1, "lbvh": B.BVH_BUILD_FAST, "sbvh": None}[tree]
    o, tree, fam, rays = gpu_style_case(oracle, name, flags)
    brute = o.trace(rays, oracle.TRACE_BRUTE_FORCE)
    closest, depth, overflow = host_trace(*tree, rays, 0)
    assert not overflow
    wrong = R.wrong_per_family(fam, closest, brute, instances=False)
    assert sum(wrong.values()) == 0, f"closest hit: wrong rays per family {wrong} of {RAYS_PER_FAMILY} each"
    # any hit: occluded iff a brute-force hit lies in (tmin, tmax); the interval rays keep their ends
    for mode, what in ((1, "any hit"), (2, "any hit, postponed leaves")):
        got, _, _ = host_trace(*tree, rays, mode)
        wrong = R.wrong_per_family(fam, got, brute, any_hit=True)
        assert sum(wrong.values()) == 0, f"{what}: wrong rays per family {wrong}"


def test_corridor_stack_passes_shared_memory_part(oracle, host_trace):
    """The corridor's maxLeaf-1 trees push more than the 16 shared-memory entries of the wavefront kernels' stack (kSmemStack,
    traverse.cuh) and stay below the 64 entries of kStackSize, so the tests on it reach the local-memory part."""
    for builder in (0, B.BVH_BUILD_FAST):
        o, tree, fam, rays = gpu_style_case(oracle, "corridor", builder | 1, n=500)
        _, depth, overflow = host_trace(*tree, fam["corridor"], 0)
        assert 16 < depth < 64 and not overflow, (builder, depth)
