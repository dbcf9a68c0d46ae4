"""The GPU-built traversal copy of the nodes (k_travNodes) against the host function it shares with the CPU build of the
traversal (octantOrderNode through tests/cpp/trav_nodes_host.cpp), at config 2's size: a ray's walk is a deterministic
function of the copy, so the per-ray internal-node and triangle counts of gfx_trace(CLOSEST | STATS) on the primary rays
must equal those the host build counts on the copy it makes from the exported tree, for closest-hit rays (sorted walk) and
any-hit rays (octant order)."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import trav_nodes_host

pytestmark = pytest.mark.gpu

W, H = 1920, 1080


def test_gpu_traversal_copy_walks_like_the_host_one(gfx_ctx, tmp_path):
    scene = scenes.bistro_class_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh(0)
    p = abi.default_frame_params(scene, W, H)
    rays = np.ascontiguousarray(engine.primary_rays(p, W, H)[::7])
    _, counts = trav_nodes_host.build(tmp_path)
    tree = gfx_ctx.export_bvh()
    for mode, any_hit in ((abi.TRACE_CLOSEST, False), (abi.TRACE_ANY, True)):
        packed = gfx_ctx.trace(rays, mode | abi.TRACE_STATS)["instUserData"]
        visited, tested = counts(*tree, rays, any_hit)
        assert visited.min() >= 1
        node_diff = np.flatnonzero((packed & 0xFFFF) != np.minimum(visited, 0xFFFF))
        tri_diff = np.flatnonzero((packed >> 16) != np.minimum(tested, 0xFFFF))
        assert len(node_diff) == 0 and len(tri_diff) == 0, \
            f"any hit {any_hit}: {len(node_diff)} rays visit other node counts, {len(tri_diff)} test other triangle counts " \
            f"(of {len(rays)})"
