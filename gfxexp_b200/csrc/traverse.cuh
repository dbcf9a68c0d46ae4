// traverse.cuh — per-thread stack traversal of the reference's 8-wide quantised BVH on sm_90a.
//
// Replaces optixTrace (utils/optix_util.h:575-584) for closest-hit and visibility rays, with the
// semantics of the only BVH traverser in the reference tree, bvh::traverse<8>
// (common/bvh_builder.cpp:1272-1649): the leaf children of a node are tested before its internal children are descended,
// both groups near to far - closest-hit rays by the same key (entry distance, isInternal<<31), any-hit rays by the octant
// order of the traversal copy of the nodes (octantOrderNode), without sorting; the ray/triangle test is bit-for-bit
// testRayVsTriangle (common/bvh_builder.cpp:1251-1270) on the explicit-FMA vector kernels of
// vec.cuh / oracle/vecmath.h.
//
// Differences by design (documented in DESIGN.md):
//  * ties in hit distance resolve to the smaller TriangleStorage index instead of "first found"
//    (makes the result independent of BVH topology, so a Morton LBVH and the reference SBVH give
//    identical hits);
//  * the slab test works on t = q * (scale/dir) + (origin-org)/dir with explicit FMAs, a 1e-5 relative slack
//    and a per-ray absolute slack that bounds the rounding error of t (derived at traverseSlack), i.e. it is
//    conservative w.r.t. AABB::intersect (common/basic_types.h:3450-3465); it only decides which nodes are
//    visited, never the hit itself (tests/test_traverse_host.py compiles this file for the CPU and checks that
//    against brute force on rays aimed at edges, along axes and at the ends of the ray interval).
//
// The traversal is exposed as a resumable state machine (TraversalState + traverseStep = one internal
// node incl. its leaf children) so that the wavefront kernel of trace.cu can refill finished lanes
// with new rays (persistent threads) while the fused kernels simply loop traverseStep to completion.
#pragma once
#include "scene.cuh"

namespace gfx {

struct Hit {
    float dist;
    uint32_t storageIndex; // 0xFFFFFFFF = miss
    uint32_t geomIndex;
    uint32_t primIndex;
    float bcB, bcC;
    uint32_t statNodes, statTris; // only maintained by the STATS instantiation
};

GFX_D bool testRayVsTriangle( // common/bvh_builder.cpp:1251-1270
    const f3 &rayOrg, const f3 &rayDir, const float distMin, const float distMax,
    const f3 &pA, const f3 &pB, const f3 &pC,
    float* hitDist, float* bcB, float* bcC) {
    const f3 eAB = pB - pA;
    const f3 eCA = pA - pC;
    const f3 hitNormal = cross(eCA, eAB);
    const f3 e = (1.0f / dot(hitNormal, rayDir)) * (pA - rayOrg);
    const f3 i = cross(rayDir, e);
    *bcB = dot(i, eCA);
    *bcC = dot(i, eAB);
    *hitDist = dot(hitNormal, e);
    return ((*hitDist < distMax) && (*hitDist > distMin) &&
            (*bcB >= 0.0f) && (*bcC >= 0.0f) && (*bcB + *bcC <= 1));
}

// The traversal copy of the tree (DevBvh::nodes, built by finishBvh): the reference format, byte for byte in meaning, with
// the child slots of every node permuted so that bit d of a slot index says on which side of the node centre the child lies
// along axis d (1 = positive).  Visiting slot ^ octant(ray) in ascending order is then near to far without sorting (Ylitie,
// Karras and Laine, HPG 2017).  The slots are assigned by a greedy matching on the integer quantised boxes: repeatedly the
// (child, free slot) pair whose centre offset agrees best with the slot's octant, ties to the smaller child index, then the
// smaller slot index.  An internal child is found as in the reference, at childBase + popc(internalMask below its slot), so
// the nodes of each child block move with their parent's permutation; the traversal reads either tree.

// newSlot[k] = the slot child k of `node` moves to, -1 for an empty slot ((qmin, qmax) = (255, 0) on x, not internal)
GFX_HD void octantSlots(const uint4* node, int newSlot[8]) {
    const uint4 n0 = node[0], n2 = node[2], n3 = node[3], n4 = node[4];
    const uint32_t qmin[3][2] = { { n2.x, n2.y }, { n2.z, n2.w }, { n3.x, n3.y } };
    const uint32_t qmax[3][2] = { { n3.z, n3.w }, { n4.x, n4.y }, { n4.z, n4.w } };
    int centre[8][3]; // child box centre - node centre, in half quantisation steps
    bool placed[8], taken[8];
    for (int k = 0; k < 8; ++k) {
        const int w = k >> 2, sh = 8 * (k & 3);
        for (int d = 0; d < 3; ++d)
            centre[k][d] = (int)((qmin[d][w] >> sh) & 0xFFu) + (int)((qmax[d][w] >> sh) & 0xFFu) - 255;
        const bool empty = ((qmin[0][w] >> sh) & 0xFFu) == 255u && ((qmax[0][w] >> sh) & 0xFFu) == 0u &&
                           !((n0.w >> (24 + k)) & 1u);
        newSlot[k] = -1;
        placed[k] = empty;
        taken[k] = false;
    }
    for (int round = 0; round < 8; ++round) {
        int bestCost = 1 << 30, bestChild = -1, bestSlot = -1;
        for (int k = 0; k < 8; ++k) {
            if (placed[k])
                continue;
            for (int s = 0; s < 8; ++s) {
                if (taken[s])
                    continue;
                int cost = 0;
                for (int d = 0; d < 3; ++d)
                    cost += ((s >> d) & 1) ? -centre[k][d] : centre[k][d];
                if (cost < bestCost) {
                    bestCost = cost;
                    bestChild = k;
                    bestSlot = s;
                }
            }
        }
        if (bestChild < 0)
            break;
        newSlot[bestChild] = bestSlot;
        placed[bestChild] = taken[bestSlot] = true;
    }
}

// `in` with child k moved to slot newSlot[k]: its plane bytes, meta byte and internal bit; empty slots (255, 0), meta 0
GFX_HD void permuteSlots(const uint4* in, const int newSlot[8], uint4* out) {
    const uint4 n0 = in[0], n1 = in[1], n2 = in[2], n3 = in[3], n4 = in[4];
    const uint32_t q[7][2] = { { n1.z, n1.w }, { n2.x, n2.y }, { n2.z, n2.w }, { n3.x, n3.y },
                               { n3.z, n3.w }, { n4.x, n4.y }, { n4.z, n4.w } }; // metas, qmin xyz, qmax xyz
    uint32_t o[7][2] = { { 0, 0 }, { ~0u, ~0u }, { ~0u, ~0u }, { ~0u, ~0u }, { 0, 0 }, { 0, 0 }, { 0, 0 } };
    uint32_t mask = 0;
    for (int k = 0; k < 8; ++k) {
        const int s = newSlot[k];
        if (s < 0)
            continue;
        const int w = k >> 2, sh = 8 * (k & 3), ws = s >> 2, shs = 8 * (s & 3);
        for (int a = 0; a < 7; ++a)
            o[a][ws] = (o[a][ws] & ~(0xFFu << shs)) | (((q[a][w] >> sh) & 0xFFu) << shs);
        mask |= ((n0.w >> (24 + k)) & 1u) << s;
    }
    out[0] = make_uint4(n0.x, n0.y, n0.z, (n0.w & 0xFFFFFFu) | (mask << 24));
    out[1] = make_uint4(n1.x, n1.y, o[0][0], o[0][1]);
    out[2] = make_uint4(o[1][0], o[1][1], o[2][0], o[2][1]);
    out[3] = make_uint4(o[3][0], o[3][1], o[4][0], o[4][1]);
    out[4] = make_uint4(o[5][0], o[5][1], o[6][0], o[6][1]);
}

// The part of the traversal copy that node i of `nodes` decides: its internal children, each permuted, at their ranks in i's
// permuted slot order (and for the root, the root itself).  Running it for every node writes every node of `out` once.
GFX_HD void octantOrderNode(const uint4* nodes, uint32_t i, uint4* out) {
    const uint4* node = nodes + 5 * (size_t)i;
    int slots[8], childSlots[8];
    octantSlots(node, slots);
    if (i == 0)
        permuteSlots(node, slots, out);
    const uint32_t internalMask = node[0].w >> 24, childBase = node[1].x;
    uint32_t oldRank = 0;
    for (int k = 0; k < 8; ++k) {
        if (!((internalMask >> k) & 1u))
            continue;
        uint32_t newRank = 0;
        for (int j = 0; j < 8; ++j)
            newRank += ((internalMask >> j) & 1u) && slots[j] < slots[k] ? 1u : 0u;
        const uint4* child = nodes + 5 * (size_t)(childBase + oldRank++);
        octantSlots(child, childSlots);
        permuteSlots(child, childSlots, out + 5 * (size_t)(childBase + newRank));
    }
}

// lowest / highest set bit of m != 0, and __byte_perm with selector nibbles 0..7, on the device and in the host build
GFX_HD uint32_t lowestBit(uint32_t m) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__ffs(m) - 1u;
#else
    return (uint32_t)__builtin_ctz(m);
#endif
}
GFX_HD uint32_t highestBit(uint32_t m) {
#ifdef __CUDA_ARCH__
    return 31u - (uint32_t)__clz(m);
#else
    return 31u - (uint32_t)__builtin_clz(m);
#endif
}
GFX_HD uint32_t bytePerm(uint32_t x, uint32_t y, uint32_t s) {
#ifdef __CUDA_ARCH__
    return __byte_perm(x, y, s);
#else
    const uint64_t v = (uint64_t)y << 32 | x;
    uint32_t r = 0;
    for (int b = 0; b < 4; ++b)
        r |= (uint32_t)((v >> (8 * ((s >> (4 * b)) & 7u))) & 0xFFu) << (8 * b);
    return r;
#endif
}

// Relative slack of the slab test's far bound and of the culls against the closest hit so far: the distances of a box and of a
// triangle are computed along different paths (1 / dir here, 1 / dot(normal, dir) in testRayVsTriangle).
constexpr float kRelSlack = 1.00001f;

constexpr int kStackSize = 64;
// The wavefront kernels keep the first kSmemStack entries of every lane's stack in shared memory, laid out [entry][thread] so
// that a warp's pushes and pops are conflict-free whatever the lanes' depths (a per-thread local-memory stack makes every push a
// divergent store, and the push / pop section dominates the trace kernel's stalls); deeper entries - rare with
// an 8-wide tree - spill to the local array.
constexpr int kSmemStack = 16;
constexpr int kSmemStackThreads = 128; // block size of the wavefront kernels

struct TraversalState {
    f3 org, dir, idir;
    f3 slack; // per-axis absolute slack of the slab distances (traverseSlack)
    float tmin, tmax;
    Hit best;
    uint32_t nodeIdx;
    int sp;
    uint2 stack[kStackSize]; // (node index, truncated entry distance bits); unused with a split stack
};
// The wavefront kernels' stack is split: `sstack` is this thread's column of the shared-memory part, `spill` a local array of
// the kStackSize - kSmemStack deeper entries.  Both are passed along rather than kept in TraversalState.  A state whose
// stack is indexed dynamically lives in local memory: every node step would reload the ray and the traversal position from
// there, and a pointer loaded from there is a generic one, so every push and pop would be a generic store / load instead of
// STS / LDS.  Without the stack the state stays in registers.
template <int SMEM_STRIDE> // threads per block of the shared-memory stack, 0 = st.stack only
GFX_D void stackStore(TraversalState &st, uint2* sstack, uint2* spill, int at, const uint2 &v) {
    if (SMEM_STRIDE == 0)
        st.stack[at] = v;
    else if (at < kSmemStack)
        sstack[at * SMEM_STRIDE] = v;
    else
        spill[at - kSmemStack] = v;
}
template <int SMEM_STRIDE>
GFX_D uint2 stackLoad(const TraversalState &st, const uint2* sstack, const uint2* spill, int at) {
    if (SMEM_STRIDE == 0)
        return st.stack[at];
    if (at < kSmemStack)
        return sstack[at * SMEM_STRIDE];
    return spill[at - kSmemStack];
}

GFX_D void traverseInit(TraversalState &st, const f3 &org, const f3 &dir, float tmin, float tmax) {
    st.org = org;
    st.dir = dir;
    st.tmin = tmin;
    st.tmax = tmax;
    st.best.dist = tmax;
    st.best.storageIndex = 0xFFFFFFFFu;
    st.best.geomIndex = 0xFFFFFFFFu;
    st.best.primIndex = 0xFFFFFFFFu;
    st.best.bcB = 0.0f;
    st.best.bcC = 0.0f;
    st.best.statNodes = 0;
    st.best.statTris = 0;
    // guarded reciprocal direction for the slab test only
    const float ooeps = 8.271806e-25f; // 2^-80
    const f3 sd(fabsf(dir.x) > ooeps ? dir.x : copysignf(ooeps, dir.x),
                fabsf(dir.y) > ooeps ? dir.y : copysignf(ooeps, dir.y),
                fabsf(dir.z) > ooeps ? dir.z : copysignf(ooeps, dir.z));
    st.idir = f3(1.0f / sd.x, 1.0f / sd.y, 1.0f / sd.z);
    st.nodeIdx = 0;
    st.sp = 0;
}

// Absolute slack s of the slab distances, per axis (u = 2^-24).  traverseStep computes a slab distance as t = fmaf(q, a, b)
// with a = 2^e * idir (exact) and b = fl(fl(corner - org) * idir) -+ s: the distance to the exact plane corner + q 2^e of a
// node, lowered by s for the near planes and raised by s for the far ones.  The box a builder made to contain a child,
// though, is the decoded one, fl(corner + q 2^e) (getChildAabb; the imported reference trees rely on it).  Along one axis the
// computed t differs from that box's plane, before the shift by s, by at most
//   the subtraction and the product that make b       2u |b|
//   b -+ s                                            u (|b| + s)
//   the FMA                                           u (255 |a| + |b| + s)
//   the decoded plane: u (|corner| + 255 2^e) away    u (|corner * idir| + 255 |a|)
// i.e. by u (510 |a| + 4 |b| + |corner * idir| + 2s) <= 4u |idir| (255 2^e + 2 |corner| + |org|) + 2u s, as
// |b| <= |idir| (|corner| + |org|).  Every node's box lies in the root's quantisation box [c, c + 255 2^E] and has
// 255 2^e <= 2 * extent, so 255 2^e + 2 |corner| <= B = 2 |c| + 1024 2^E and the error is below 4u M + 2u s with
// M = |idir| (B + |org|): s = 8u M = 2^-21 M per ray keeps every near plane in front of the decoded box's and every far plane
// behind it, with room for the rounding of s itself and for the reference SBVH's split references, whose part boxes (clipped
// in float) contain their part only to a fraction of an ulp of the coordinates, <= 2u |idir| |plane| <= 2u M more.
// Without it a ray that starts near a box but far from its parent's corner (bounce and shadow rays), or meets a box far
// from the origin, loses the box at its edges.  Per axis, so that a nearly parallel axis (huge |idir|, huge t) widens only
// its own slab.
GFX_D void traverseSlack(TraversalState &st, const DevBvh &bvh) {
    const uint4 root = __ldg(bvh.nodes);
    const f3 bound(fmaf(1024.0f, __uint_as_float((root.w & 0xFFu) << 23), 2.0f * fabsf(__uint_as_float(root.x))),
                   fmaf(1024.0f, __uint_as_float(((root.w >> 8) & 0xFFu) << 23), 2.0f * fabsf(__uint_as_float(root.y))),
                   fmaf(1024.0f, __uint_as_float(((root.w >> 16) & 0xFFu) << 23), 2.0f * fabsf(__uint_as_float(root.z))));
    st.slack = f3(4.76837158e-7f * fabsf(st.idir.x) * (bound.x + fabsf(st.org.x)),
                  4.76837158e-7f * fabsf(st.idir.y) * (bound.y + fabsf(st.org.y)),
                  4.76837158e-7f * fabsf(st.idir.z) * (bound.z + fabsf(st.org.z)));
}

// Leaf children whose triangle tests have been postponed (wavefront kernel, any-hit rays only): the start of each triangle
// chain.  A node step appends at most 8.  An any-hit ray ends at its first hit, so no entry distance is kept to cull against.
constexpr int kPendingLeaves = 12;
struct PendingLeaves {
    uint32_t idx[kPendingLeaves];
    int n;
    GFX_HD uint32_t &at(int i) { return idx[i]; }
};
// The same list in the wavefront kernel: `col` is this thread's column of a [kPendingLeaves][kSmemStackThreads] shared array,
// laid out like the stack, so that the dynamically indexed entries cause no local-memory traffic.
struct SmemPendingLeaves {
    uint32_t* col;
    int n;
    GFX_HD uint32_t &at(int i) { return col[i * kSmemStackThreads]; }
};

// One triangle of a leaf chain (leaf-ordered storage).  Returns true when an any-hit ray has found its occluder.
template <bool ANY_HIT, bool STATS>
GFX_D bool testLeafTriangle(const DevBvh &bvh, TraversalState &st, uint32_t idx, bool* endOfChain) {
    const float4* tp = bvh.leafTris + 3 * (size_t)idx;
    const float4 t0 = __ldg(tp + 0);
    const float4 t1 = __ldg(tp + 1);
    const float4 t2 = __ldg(tp + 2);
    const uint32_t pr = __float_as_uint(t2.w); // PrimitiveReference word: storage index | end-of-leaf << 31
    const uint32_t si = pr & 0x7FFFFFFFu;
    *endOfChain = (pr >> 31) != 0;
    float hitDist, bcB, bcC;
    if (STATS)
        ++st.best.statTris;
    const bool hit = testRayVsTriangle(st.org, st.dir, st.tmin, st.tmax,
                                       f3(t0.x, t0.y, t0.z), f3(t0.w, t1.x, t1.y), f3(t1.z, t1.w, t2.x),
                                       &hitDist, &bcB, &bcC);
    if (hit && (hitDist < st.best.dist || (hitDist == st.best.dist && si < st.best.storageIndex))) {
        st.best.dist = hitDist;
        st.best.storageIndex = si;
        st.best.geomIndex = __float_as_uint(t2.y);
        st.best.primIndex = __float_as_uint(t2.z);
        st.best.bcB = bcB;
        st.best.bcC = bcC;
        if (ANY_HIT)
            return true;
    }
    return false;
}

// Advances the newest postponed leaf of this lane by one triangle.  Returns true when an any-hit ray is occluded.
template <bool ANY_HIT, bool STATS, typename Pending>
GFX_D bool testPendingTriangle(const DevBvh &bvh, TraversalState &st, Pending &pend) {
    static_assert(ANY_HIT, "postponed leaf tests are for any-hit rays");
    const int top = pend.n - 1;
    const uint32_t idx = pend.at(top);
    bool end;
    if (testLeafTriangle<ANY_HIT, STATS>(bvh, st, idx, &end))
        return true;
    if (end)
        pend.n = top;
    else
        pend.at(top) = idx + 1;
    return false;
}

// Bit p of the result = bit p ^ o of m (8 bits): a node's slot mask in the visiting order of a ray of octant o.
GFX_D uint32_t octantOrderBits(uint32_t m, uint32_t o) {
    if (o & 1u)
        m = ((m & 0x55u) << 1) | ((m >> 1) & 0x55u);
    if (o & 2u)
        m = ((m & 0x33u) << 2) | ((m >> 2) & 0x33u);
    if (o & 4u)
        m = ((m & 0x0Fu) << 4) | ((m >> 4) & 0x0Fu);
    return m;
}
#define GFX_CSWAP(a, b) { const uint32_t lo_ = min(a, b); const uint32_t hi_ = max(a, b); a = lo_; b = hi_; }

// Processes node st.nodeIdx of the traversal copy (octantOrderNode): slab-tests its children, intersects the triangle
// chains of the leaf children that are hit (or, with `pend`, postpones them), selects the next internal node.  Returns false
// when the traversal is finished.  With SMEM_STRIDE > 0, the stack is split into `sstack` and `spill` (stackStore).
template <bool ANY_HIT, bool STATS, bool DEFER = false, int SMEM_STRIDE = 0, typename Pending = PendingLeaves>
GFX_D bool traverseStep(const DevBvh &bvh, TraversalState &st, Pending* pend = nullptr, uint2* sstack = nullptr,
                        uint2* spill = nullptr) {
    static_assert(ANY_HIT || !DEFER, "postponed leaf tests are for any-hit rays");
    const uint4* np = bvh.nodes + 5 * (size_t)st.nodeIdx;
    const uint4 n0 = __ldg(np + 0);
    const uint4 n1 = __ldg(np + 1);
    const uint4 n2 = __ldg(np + 2);
    const uint4 n3 = __ldg(np + 3);
    const uint4 n4 = __ldg(np + 4);
    if (STATS)
        ++st.best.statNodes;

    const uint32_t internalMask = n0.w >> 24;
    const float ax = __uint_as_float((n0.w & 0xFFu) << 23) * st.idir.x;
    const float ay = __uint_as_float(((n0.w >> 8) & 0xFFu) << 23) * st.idir.y;
    const float az = __uint_as_float(((n0.w >> 16) & 0xFFu) << 23) * st.idir.z;
    const float bx = (__uint_as_float(n0.x) - st.org.x) * st.idir.x;
    const float by = (__uint_as_float(n0.y) - st.org.y) * st.idir.y;
    const float bz = (__uint_as_float(n0.z) - st.org.z) * st.idir.z;
    // near planes lowered, far planes raised by the slack (traverseSlack): the entry distance, also the one kept for the
    // culls against the closest hit, is a lower bound, the exit distance an upper bound
    const float bnx = bx - st.slack.x, bfx = bx + st.slack.x;
    const float bny = by - st.slack.y, bfy = by + st.slack.y;
    const float bnz = bz - st.slack.z, bfz = bz + st.slack.z;

    // The sign of the ray direction decides which quantised plane of each axis is entered first, once per node and
    // axis instead of a min/max pair per child (same t values as min(tlo, thi) / max(tlo, thi)).
    const bool sx = st.idir.x < 0.0f, sy = st.idir.y < 0.0f, sz = st.idir.z < 0.0f;
    // Any hit: position p holds slot p ^ octant(ray), so ascending positions go near to far (octantOrderNode); a byte permute
    // puts the plane and meta bytes of the 8 slots (two words each) in that order.  Closest hit: position = slot, the
    // children are sorted by entry distance below.
    const uint32_t order = ANY_HIT ? (sx ? 1u : 0u) | (sy ? 2u : 0u) | (sz ? 4u : 0u) : 0u;
    const uint32_t sel0 = 0x3210u ^ (order * 0x1111u), sel1 = sel0 ^ 0x4444u;
#define GFX_IN_ORDER(name, lo, hi) \
    const uint32_t name[2] = { ANY_HIT ? bytePerm(lo, hi, sel0) : (lo), ANY_HIT ? bytePerm(lo, hi, sel1) : (hi) }
    GFX_IN_ORDER(nearX, sx ? n3.z : n2.x, sx ? n3.w : n2.y); GFX_IN_ORDER(farX, sx ? n2.x : n3.z, sx ? n2.y : n3.w);
    GFX_IN_ORDER(nearY, sy ? n4.x : n2.z, sy ? n4.y : n2.w); GFX_IN_ORDER(farY, sy ? n2.z : n4.x, sy ? n2.w : n4.y);
    GFX_IN_ORDER(nearZ, sz ? n4.z : n3.x, sz ? n4.w : n3.y); GFX_IN_ORDER(farZ, sz ? n3.x : n4.z, sz ? n3.y : n4.w);
    GFX_IN_ORDER(metas, n1.z, n1.w);
#undef GFX_IN_ORDER
    const uint32_t internalAt = octantOrderBits(internalMask, order);
    const float invalidNearX = sx ? 0.0f : 255.0f, invalidFarX = sx ? 255.0f : 0.0f; // (qminx, qmaxx) = (255, 0) marks an empty slot

    uint32_t hits = 0;  // any hit: by position
    uint32_t keys[8];   // closest hit: (isInternal, entry distance, slot) of the children hit, ~0 for the others
#pragma unroll
    for (int p = 0; p < 8; ++p) {
        const int sh = 8 * (p & 3), w = p >> 2;
        const float qnx = (float)((nearX[w] >> sh) & 0xFFu), qfx = (float)((farX[w] >> sh) & 0xFFu);
        const float qny = (float)((nearY[w] >> sh) & 0xFFu), qfy = (float)((farY[w] >> sh) & 0xFFu);
        const float qnz = (float)((nearZ[w] >> sh) & 0xFFu), qfz = (float)((farZ[w] >> sh) & 0xFFu);
        const bool valid = (qnx != invalidNearX) || (qfx != invalidFarX);
        const float tnx = __fmaf_rn(qnx, ax, bnx), tfx = __fmaf_rn(qfx, ax, bfx);
        const float tny = __fmaf_rn(qny, ay, bny), tfy = __fmaf_rn(qfy, ay, bfy);
        const float tnz = __fmaf_rn(qnz, az, bnz), tfz = __fmaf_rn(qfz, az, bfz);
        const float tn = fmaxf(fmaxf(tnx, tny), fmaxf(tnz, st.tmin));
        const float tf = fminf(fminf(tfx, tfy), fminf(tfz, st.best.dist));
        const bool hit = valid && (tn <= tf * kRelSlack);
        if (ANY_HIT)
            hits |= hit ? 1u << p : 0u;
        else
            keys[p] = hit ? (((internalAt >> p) & 1u) << 31) | ((__float_as_uint(tn) >> 1) & 0x7FFFFFF8u) | (uint32_t)p
                          : 0xFFFFFFFFu;
    }
    // meta byte at position p: the triangle offset of a leaf
#define GFX_META_AT(p) ((((p) & 4u ? metas[1] : metas[0]) >> (8 * ((p) & 3u))) & 0xFFu)
    const uint32_t leafBase = n1.y, childBase = n1.x;
    uint32_t next = 0xFFFFFFFFu, nextT = 0u;
    if (ANY_HIT) {
        // An any-hit ray that is not occluded visits every node it meets whatever the order, and best.dist stays tmax until
        // it ends, so nothing is culled and no entry distance is kept.  Leaf children first, near to far.
        for (uint32_t leaves = hits & ~internalAt; leaves != 0; leaves &= leaves - 1u) {
            uint32_t idx = leafBase + GFX_META_AT(lowestBit(leaves));
            if (DEFER) {
                pend->at(pend->n++) = idx;
                continue;
            }
            while (true) {
                bool end;
                if (testLeafTriangle<ANY_HIT, STATS>(bvh, st, idx, &end))
                    return false;
                if (end)
                    break;
                ++idx;
            }
        }
        // internal children: the first in octant order becomes the next node, the others are pushed far -> near
        for (uint32_t internals = hits & internalAt; internals != 0;) {
            const uint32_t p = highestBit(internals);
            internals ^= 1u << p;
            if (next != 0xFFFFFFFFu) {
                if (st.sp < kStackSize)
                    stackStore<SMEM_STRIDE>(st, sstack, spill, st.sp++, make_uint2(next, 0u));
                else if (bvh.overflowFlag)
                    *bvh.overflowFlag = 1u;
            }
            next = childBase + __popc(internalMask & ((1u << (p ^ order)) - 1u));
        }
    } else {
        // Closest hit: the nearest leaves shrink best.dist before the farther ones and the internal children are culled
        // against it, so the order is exact.  19-comparator network, ascending: leaf hits (near..far), internal hits
        // (near..far), misses.
        GFX_CSWAP(keys[0], keys[2]); GFX_CSWAP(keys[1], keys[3]); GFX_CSWAP(keys[4], keys[6]); GFX_CSWAP(keys[5], keys[7]);
        GFX_CSWAP(keys[0], keys[4]); GFX_CSWAP(keys[1], keys[5]); GFX_CSWAP(keys[2], keys[6]); GFX_CSWAP(keys[3], keys[7]);
        GFX_CSWAP(keys[0], keys[1]); GFX_CSWAP(keys[2], keys[3]); GFX_CSWAP(keys[4], keys[5]); GFX_CSWAP(keys[6], keys[7]);
        GFX_CSWAP(keys[2], keys[4]); GFX_CSWAP(keys[3], keys[5]);
        GFX_CSWAP(keys[1], keys[4]); GFX_CSWAP(keys[3], keys[6]);
        GFX_CSWAP(keys[1], keys[2]); GFX_CSWAP(keys[3], keys[4]); GFX_CSWAP(keys[5], keys[6]);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t key = keys[k];
            if (key >= 0x80000000u)
                break;
            if (__uint_as_float((key & 0x7FFFFFF8u) << 1) > st.best.dist * kRelSlack)
                continue;
            uint32_t idx = leafBase + GFX_META_AT(key & 7u);
            while (true) {
                bool end;
                if (testLeafTriangle<ANY_HIT, STATS>(bvh, st, idx, &end))
                    return false;
                if (end)
                    break;
                ++idx;
            }
        }
        // internal children: nearest becomes the next node, the others are pushed far -> near
#pragma unroll
        for (int k = 7; k >= 0; --k) {
            const uint32_t key = keys[k];
            if (key == 0xFFFFFFFFu || key < 0x80000000u)
                continue;
            const uint32_t tnBits = (key & 0x7FFFFFF8u) << 1; // truncated entry distance (<= true tn)
            if (__uint_as_float(tnBits) > st.best.dist * kRelSlack)
                continue;
            if (next != 0xFFFFFFFFu) {
                if (st.sp < kStackSize)
                    stackStore<SMEM_STRIDE>(st, sstack, spill, st.sp++, make_uint2(next, nextT));
                else if (bvh.overflowFlag)
                    *bvh.overflowFlag = 1u;
            }
            next = childBase + __popc(internalMask & ((1u << (key & 7u)) - 1u));
            nextT = tnBits;
        }
    }
#undef GFX_META_AT
    if (next != 0xFFFFFFFFu) {
        st.nodeIdx = next;
        return true;
    }
    while (st.sp > 0) {
        const uint2 e = stackLoad<SMEM_STRIDE>(st, sstack, spill, --st.sp);
        if (ANY_HIT || __uint_as_float(e.y) <= st.best.dist * kRelSlack) {
            st.nodeIdx = e.x;
            return true;
        }
    }
    return false;
}

template <bool ANY_HIT, bool STATS = false>
GFX_D Hit traverseBvh(const DevBvh &bvh, const f3 &org, const f3 &dir, const float tmin, const float tmax) {
    TraversalState st;
    traverseInit(st, org, dir, tmin, tmax);
    if (bvh.numNodes == 0)
        return st.best;
    traverseSlack(st, bvh);
    while (traverseStep<ANY_HIT, STATS>(bvh, st)) {
    }
    return st.best;
}

} // namespace gfx
