// trav_nodes_host.cpp — the traversal copy of a BVH (octantOrderNode, gfxexp_b200/csrc/traverse.cuh) built on the CPU by the
// same function k_travNodes runs, and the walks of the STATS trace variants on that copy, for the tests of the copy.
// Built like tests/cpp/traverse_host.cpp (-ffp-contract=off, shims for the device intrinsics the header uses):
//   trav_nodes_host     reference-format nodes -> traversal copy
//   trace_host_counts   per ray: internal nodes visited and triangles tested by traverseStep<anyHit, STATS> (immediate leaf
//                       tests, as gfx_trace) on the copy made from `nodes` (with the leaf-ordered triangle copy k_leafTris makes)
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>

static inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }
static inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }

#include "../../gfxexp_b200/csrc/traverse.cuh"

using namespace gfx;

namespace {

std::vector<uint4> travNodes(const void* nodes, uint32_t numNodes) {
    std::vector<uint4> out(5 * (size_t)numNodes);
    for (uint32_t i = 0; i < numNodes; ++i)
        octantOrderNode(static_cast<const uint4*>(nodes), i, out.data());
    return out;
}

} // namespace

extern "C" void trav_nodes_host(const void* nodes, uint32_t numNodes, void* out) {
    const std::vector<uint4> t = travNodes(nodes, numNodes);
    std::memcpy(out, t.data(), t.size() * sizeof(uint4));
}

extern "C" void trace_host_counts(const void* nodes, uint32_t numNodes, const void* leafTris, const float* rays,
                                  uint32_t numRays, int anyHit, uint32_t* nodesVisited, uint32_t* trisTested) {
    const std::vector<uint4> trav = travNodes(nodes, numNodes);
    uint32_t flag = 0;
    DevBvh bvh{};
    bvh.nodes = trav.data();
    bvh.leafTris = static_cast<const float4*>(leafTris);
    bvh.numNodes = numNodes;
    bvh.overflowFlag = &flag;
    TraversalState st;
    for (uint32_t r = 0; r < numRays; ++r) {
        const float* ray = rays + 8 * (size_t)r;
        traverseInit(st, f3(ray[0], ray[1], ray[2]), f3(ray[4], ray[5], ray[6]), ray[3], ray[7]);
        if (numNodes) {
            traverseSlack(st, bvh);
            if (anyHit)
                while (traverseStep<true, true>(bvh, st)) {
                }
            else
                while (traverseStep<false, true>(bvh, st)) {
                }
        }
        nodesVisited[r] = st.best.statNodes;
        trisTested[r] = st.best.statTris;
    }
}
