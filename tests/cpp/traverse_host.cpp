// traverse_host.cpp — the device traversal of gfxexp_b200/csrc/traverse.cuh, compiled for the CPU without changes.
//
// Shims stand in for the five device intrinsics the header uses and for the device's unsigned min / max; with
// -ffp-contract=off (the host counterpart of nvcc's -fmad=false) every float operation rounds as on sm_90a, so a ray gets the
// bits the GPU gives it.  The entry point walks an exported tree (nodes + the leaf-ordered triangle copy k_leafTris makes) ray by ray:
//   mode 0  closest hit, immediate leaf tests (k_traceWavefront<false>, traverseBvh<false>)
//   mode 1  any hit, immediate leaf tests (k_traceWavefront<true>, traverseBvh<true>)
//   mode 2  any hit, postponed leaf tests (k_traceWavefrontDeferred<true>): the pending list is flushed when it is full
//           or the walk has ended, one of the flush points the warp-level kernel may choose
// Hits are written as GfxHitObject records without instance ids (instIndex = 0xFFFFFFFF); any-hit records follow
// HitWriter.  maxDepth receives the deepest stack of the batch, overflow whether a push was dropped.
#include <cmath>
#include <cstdint>
#include <cstring>

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

struct HitRecord { // GfxHitObject
    float dist;
    uint32_t instIndex, instUserData, geomIndex, primIndex;
    float bcA, bcB, bcC;
};

HitRecord record(const TraversalState &st, bool anyHit) {
    const Hit &h = st.best;
    const bool isHit = h.storageIndex != 0xFFFFFFFFu;
    const float qnan = __uint_as_float(0x7FC00000u);
    if (anyHit)
        return { isHit ? 0.0f : st.tmax, 0xFFFFFFFFu, 0u, 0xFFFFFFFFu, isHit ? 0u : 0xFFFFFFFFu, qnan, qnan, qnan };
    if (!isHit)
        return { h.dist, 0xFFFFFFFFu, 0u, h.geomIndex, 0xFFFFFFFFu, qnan, qnan, qnan };
    return { h.dist, 0xFFFFFFFFu, 0u, h.geomIndex, h.primIndex, 1.0f - (h.bcB + h.bcC), h.bcB, h.bcC };
}

} // namespace

extern "C" int trace_host(const void* nodes, uint32_t numNodes, const void* leafTris, const float* rays, uint32_t numRays,
                          void* hitsOut, int mode, int* maxDepth, int* overflow) {
    if (mode < 0 || mode > 2)
        return 1;
    uint32_t flag = 0;
    DevBvh bvh{};
    bvh.nodes = static_cast<const uint4*>(nodes);
    bvh.leafTris = static_cast<const float4*>(leafTris);
    bvh.numNodes = numNodes;
    bvh.overflowFlag = &flag;
    HitRecord* hits = static_cast<HitRecord*>(hitsOut);
    int deepest = 0;
    TraversalState st;
    for (uint32_t r = 0; r < numRays; ++r) {
        const float* ray = rays + 8 * (size_t)r;
        traverseInit(st, f3(ray[0], ray[1], ray[2]), f3(ray[4], ray[5], ray[6]), ray[3], ray[7]);
        if (numNodes == 0) {
            hits[r] = record(st, mode != 0);
            continue;
        }
        traverseSlack(st, bvh);
        if (mode == 2) {
            PendingLeaves pend;
            pend.n = 0;
            bool running = true, occluded = false;
            while (running && !occluded) {
                running = traverseStep<true, false, true>(bvh, st, &pend);
                deepest = st.sp > deepest ? st.sp : deepest;
                if (!running || pend.n > kPendingLeaves - 8)
                    while (pend.n > 0 && !occluded)
                        occluded = testPendingTriangle<true, false>(bvh, st, pend);
            }
        } else if (mode == 1) {
            while (traverseStep<true, false>(bvh, st))
                deepest = st.sp > deepest ? st.sp : deepest;
        } else {
            while (traverseStep<false, false>(bvh, st))
                deepest = st.sp > deepest ? st.sp : deepest;
        }
        hits[r] = record(st, mode != 0);
    }
    *maxDepth = deepest;
    *overflow = flag != 0;
    return 0;
}
