"""Builds tests/cpp/trav_nodes_host.cpp: the traversal copy of a BVH (octantOrderNode, gfxexp_b200/csrc/traverse.cuh) and the
per-ray counts of the closest-hit STATS walk on it, computed on the CPU by the code the GPU runs."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests import trace_rays as R


def build(out_dir):
    """returns (trav_nodes(nodes) -> [N, 20] uint32 copy, counts(nodes, refs, tris, rays, any_hit) -> (nodes visited, triangles tested))"""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "trav_nodes_host.cpp")
    lib = os.path.join(str(out_dir), "trav_nodes_host.so")
    inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + inc, "-o", lib, src],
                   check=True)
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.trav_nodes_host.argtypes = [vp, C.c_uint32, vp]
    L.trav_nodes_host.restype = None
    L.trace_host_counts.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_int, vp, vp]
    L.trace_host_counts.restype = None

    def trav_nodes(nodes):
        nodes = np.ascontiguousarray(nodes)
        out = np.zeros((len(nodes), 20), np.uint32)
        L.trav_nodes_host(nodes.ctypes.data, len(nodes), out.ctypes.data)
        return out

    def counts(nodes, refs, tris, rays, any_hit):
        nodes, rays = np.ascontiguousarray(nodes), np.ascontiguousarray(rays)
        leaves = R.leaf_tris(refs, tris)
        visited = np.zeros(len(rays), np.uint32)
        tested = np.zeros(len(rays), np.uint32)
        L.trace_host_counts(nodes.ctypes.data, len(nodes), leaves.ctypes.data, rays.ctypes.data, len(rays), int(any_hit),
                            visited.ctypes.data, tested.ctypes.data)
        return visited, tested
    return trav_nodes, counts
