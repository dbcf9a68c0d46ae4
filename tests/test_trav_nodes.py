"""The traversal copy of the BVH nodes (octantOrderNode, gfxexp_b200/csrc/traverse.cuh; built by k_travNodes in finishBvh),
made on the CPU by the same function through tests/cpp/trav_nodes_host.cpp from the restated GPU trees (SAH, LBVH at maxLeaf 1
and the default) and the reference's SBVH on the scenes of tests/trace_rays.py.  The copy is the same tree in the reference
format with every node's child slots permuted: walked in step with the original from the root, every node holds the same
children with the same boxes (internal children found at childBase + popc(internalMask below the slot) in both, leaves by
their triangle offset), every node of the copy is reached once, empty slots stay empty, and a child sits off its octant's slot
only where the greedy matching gave that slot to a child that fits it at least as well."""
import numpy as np
import pytest

from tests import bvh_scenes as B
from tests import trace_rays as R
from tests import trav_nodes_host

TREES = {"sah_leaf1": 1, "sah": 0, "lbvh_leaf1": B.BVH_BUILD_FAST | 1, "lbvh": B.BVH_BUILD_FAST, "sbvh": None}


@pytest.fixture(scope="module")
def trav_nodes(tmp_path_factory):
    return trav_nodes_host.build(tmp_path_factory.mktemp("trav_nodes"))[0]


def _children(words):
    """per node: internal [N, 8], meta bytes [N, 8], qmin / qmax bytes [N, 3 axes, 8 slots], empty slots [N, 8], rank of each
    internal child in its node's child block [N, 8]"""
    b = words.view(np.uint8).reshape(len(words), 80)
    internal = ((words[:, 3] >> 24)[:, None] >> np.arange(8)) & 1 != 0
    metas = b[:, 24:32].astype(np.int64)
    qmin = b[:, 32:56].reshape(-1, 3, 8).astype(np.int64)
    qmax = b[:, 56:80].reshape(-1, 3, 8).astype(np.int64)
    empty = (qmin[:, 0] == 255) & (qmax[:, 0] == 0) & ~internal
    rank = np.cumsum(internal, axis=1) - internal
    return internal, metas, qmin, qmax, empty, rank


@pytest.mark.parametrize("tree", list(TREES))
@pytest.mark.parametrize("name", [n for n in R.SCENES if n != "corridor"])
def test_traversal_copy_permutes_children_into_octant_slots(oracle, trav_nodes, name, tree):
    o = oracle.OracleScene(R.SCENES[name](), build_bvh=TREES[tree] is None)
    if TREES[tree] is not None:
        o.build_gpu_style(TREES[tree])
    nodes, _, _ = o.export_bvh()
    ref = np.ascontiguousarray(nodes).view(np.uint32).reshape(len(nodes), 20)
    trav = trav_nodes(nodes)

    rint, rmeta, rqmin, rqmax, rempty, rrank = _children(ref)
    tint, tmeta, tqmin, tqmax, tempty, trank = _children(trav)
    # empty slots: (qmin, qmax) = (255, 0) on every axis, meta 0 (how many: checked per node in the walk)
    assert np.all(tqmin.transpose(0, 2, 1)[tempty] == 255) and np.all(tqmax.transpose(0, 2, 1)[tempty] == 0)
    assert np.all(tmeta[tempty] == 0)

    # walk both trees from the root: copy node j stands for reference node of[j]
    frame = [0, 1, 2, 4, 5]  # corner, child block, triangle base; word 3 below the internal mask holds the exponents

    def key(words, internal, meta, qmin, qmax, rank, i, k):
        """what slot k of node i holds: box, meta, and for an internal child its node's frame (unique: a node has a
        child block or a triangle base of its own)"""
        box = tuple(qmin[i, :, k]) + tuple(qmax[i, :, k]) + (int(meta[i, k]),)
        if not internal[i, k]:
            return ("leaf",) + box, None
        c = int(words[i, 4]) + int(rank[i, k])
        return ("node",) + box + tuple(int(x) for x in words[c, frame]) + (int(words[c, 3]) & 0xFFFFFF,), c

    of = np.full(len(trav), -1, np.int64)
    of[0] = 0
    todo = [0]
    while todo:
        j = todo.pop()
        i = int(of[j])
        assert np.array_equal(ref[i, frame], trav[j, frame]) and (ref[i, 3] & 0xFFFFFF) == (trav[j, 3] & 0xFFFFFF), (i, j)
        want = dict(key(ref, rint, rmeta, rqmin, rqmax, rrank, i, k) for k in np.flatnonzero(~rempty[i]))
        got = dict(key(trav, tint, tmeta, tqmin, tqmax, trank, j, s) for s in np.flatnonzero(~tempty[j]))
        assert len(want) == (~rempty[i]).sum() == len(got) == (~tempty[j]).sum() and set(want) == set(got), \
            f"node {i}: the copy holds other children"
        for k, c in got.items():
            if c is not None:
                assert of[c] == -1, f"copy node {c} is reached twice"
                of[c] = want[k]
                todo.append(c)

        # octant slots: cost(child, slot) = -<2 (box centre - node centre), slot's octant direction>
        centre = tqmin[j] + tqmax[j] - 255                      # [axis, slot]
        sign = np.where((np.arange(8)[:, None] >> np.arange(3)) & 1, -1, 1)  # [octant slot, axis]
        cost = sign @ centre                                    # [octant slot, child slot]
        for s in np.flatnonzero(~tempty[j]):
            own = int(((centre[:, s] > 0) * (1 << np.arange(3))).sum())  # the slot of its octant: a cheapest one
            if cost[s, s] == cost[own, s]:
                continue
            # the greedy matching gave `own` to another child, one that fits it at least as well
            assert not tempty[j, own] and cost[own, own] <= cost[own, s], (j, s, own)
    assert np.all(of >= 0) and len(np.unique(of)) == len(of), "the copy is not the same tree"
