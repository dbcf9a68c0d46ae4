// oracle/gpu_bvh.cpp — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// CPU restatement of the two deterministic hierarchies of gfxexp_b200/csrc/bvh_build.cu and of its 8-wide collapse, so that
// the exported GPU tree can be pinned node for node (orc_bvh_same_tree):
//   triangle boxes     k_flatten             bvh_build.cu:50-93
//   Morton keys        k_morton              :96-123, then a stable sort by key (cub::DeviceRadixSort, :1209)
//   LBVH               k_hierarchy, k_refit  :126-207 (also every scene of fewer than 3 triangles, :1213)
//   binned SAH         k_sahSplit            :543-770, and the multi-block k_sahHuge* (:777-1101), restated once: they
//                      compute the same split, which is what the tests check
//   collapse           k_collapse            :234-393, level by level from buildBvh :1328-1359
//   flags              maxLeaf default and clamp, buildBvh :1127-1129
// Box bounds are minima / maxima in the order of the ordered-integer images (-0 < +0), as on the GPU (:41-47).  Node and
// reference numbering on the GPU comes from atomics; the restatement numbers breadth-first.  The numbering does not change the
// tree, and orc_bvh_same_tree ignores it.
#include "oracle.h"
#include "bvh.h"
#include "../gfxexp_b200/csrc/detmath.h"
#include <algorithm>
#include <cstdio>
#include <numeric>

namespace orc {

namespace {

constexpr uint32_t kSahBins = 16;        // bvh_build.cu:500-505
constexpr uint32_t kSahBigNode = 4096;
constexpr uint32_t kSahHugeNode = 131072;
constexpr uint32_t kLeafBit = 0x80000000u;

inline uint32_t ordered(float f) { return floatToOrderedUInt(f); }
inline float fromOrdered(uint32_t u) { return u2f(u ^ (u >= 0x80000000u ? 0x80000000u : 0xFFFFFFFFu)); }
inline float minOrdered(float a, float b) { return ordered(b) < ordered(a) ? b : a; }
inline float maxOrdered(float a, float b) { return ordered(b) > ordered(a) ? b : a; }

struct Box { float lo[3], hi[3]; };

// the binary tree every hierarchy hands to the collapse: internal node i -> childL/R[i], count[i], box[i];
// leaf j (position j of `order`) -> box[(n - 1) + j]; references carry kLeafBit for leaves
struct BinaryTree {
    uint32_t n = 0;
    std::vector<uint32_t> order, childL, childR, count;
    std::vector<Box> box;
    uint32_t root = 0;
    uint32_t refCount(uint32_t ref) const { return (ref & kLeafBit) ? 1u : count[ref]; }
    const Box &refBox(uint32_t ref) const { return box[(ref & kLeafBit) ? (n - 1) + (ref & 0x7FFFFFFFu) : ref]; }
};

// ---- k_morton (:96-123) -------------------------------------------------------------------------------------------------
uint64_t expandBits21(uint64_t v) {
    v &= 0x1FFFFFull;
    v = (v | v << 32) & 0x1F00000000FFFFull;
    v = (v | v << 16) & 0x1F0000FF0000FFull;
    v = (v | v << 8) & 0x100F00F00F00F00Full;
    v = (v | v << 4) & 0x10C30C30C30C30C3ull;
    v = (v | v << 2) & 0x1249249249249249ull;
    return v;
}
uint64_t quantiseMorton(float c, float smin, float s) { // (uint64_t)fminf(fmaxf((c - smin) * s, 0), 2097151): NaN -> 0
    return (uint64_t)std::fmin(std::fmax((c - smin) * s, 0.0f), 2097151.0f);
}

// ---- k_hierarchy (:126-172) ---------------------------------------------------------------------------------------------
int deltaKey(const std::vector<uint64_t> &keys, int n, int i, int j) {
    if (j < 0 || j >= n)
        return -1;
    const uint64_t a = keys[i], b = keys[j];
    if (a == b)
        return 64 + __builtin_clz((uint32_t)i ^ (uint32_t)j); // i != j here
    return __builtin_clzll(a ^ b);
}

void buildKarras(const std::vector<uint64_t> &keys, const std::vector<Box> &triBox, BinaryTree* T) {
    const int n = (int)T->n;
    T->childL.assign(n > 1 ? n - 1 : 0, 0);
    T->childR.assign(n > 1 ? n - 1 : 0, 0);
    T->count.assign(n > 1 ? n - 1 : 0, 0);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n - 1; ++i) {
        const int d = (deltaKey(keys, n, i, i + 1) - deltaKey(keys, n, i, i - 1)) >= 0 ? 1 : -1;
        const int deltaMin = deltaKey(keys, n, i, i - d);
        int lmax = 2;
        while (deltaKey(keys, n, i, i + lmax * d) > deltaMin)
            lmax *= 2;
        int l = 0;
        for (int t = lmax / 2; t >= 1; t /= 2)
            if (deltaKey(keys, n, i, i + (l + t) * d) > deltaMin)
                l += t;
        const int j = i + l * d;
        const int deltaNode = deltaKey(keys, n, i, j);
        int s = 0;
        for (int t = (l + 1) / 2;; t = (t + 1) / 2) {
            if (deltaKey(keys, n, i, i + (s + t) * d) > deltaNode)
                s += t;
            if (t == 1)
                break;
        }
        const int gamma = i + s * d + std::min(d, 0);
        const int first = std::min(i, j), last = std::max(i, j);
        const uint32_t left = (first == gamma) ? ((uint32_t)gamma | kLeafBit) : (uint32_t)gamma;
        const uint32_t right = (last == gamma + 1) ? ((uint32_t)(gamma + 1) | kLeafBit) : (uint32_t)(gamma + 1);
        T->childL[i] = left;
        T->childR[i] = right;
        T->count[i] = (uint32_t)(last - first + 1);
    }
    // k_refit (:176-207): leaf boxes, then every internal box as the ordered min / max of its children's, which does not
    // depend on the order the GPU threads arrive in; bottom-up here by the count (a parent covers more triangles)
    T->box.assign(n > 1 ? 2 * n - 1 : 1, Box());
    for (int j = 0; j < n; ++j)
        T->box[(n - 1) + j] = triBox[T->order[j]];
    std::vector<uint32_t> byCount(n > 1 ? n - 1 : 0);
    std::iota(byCount.begin(), byCount.end(), 0u);
    std::stable_sort(byCount.begin(), byCount.end(), [&](uint32_t a, uint32_t b) { return T->count[a] < T->count[b]; });
    for (uint32_t p : byCount) {
        const Box &a = T->refBox(T->childL[p]), &b = T->refBox(T->childR[p]);
        Box &r = T->box[p];
        for (int d = 0; d < 3; ++d) {
            r.lo[d] = minOrdered(a.lo[d], b.lo[d]);
            r.hi[d] = maxOrdered(a.hi[d], b.hi[d]);
        }
    }
    T->root = n == 1 ? kLeafBit : 0u;
}

// ---- k_sahSplit / k_sahHuge* (:543-1101) ---------------------------------------------------------------------------------
struct SahTask { uint32_t node, start, end; };

struct SahSplitter {
    const std::vector<Box>* triBox;
    BinaryTree* T;

    static uint32_t binOf(float c, float cLo, float binScale) { // binOf (:616-620, SahBinning::binOf :865-869)
        const float f = (c - cLo) * binScale;
        const uint32_t b = dm_f2uint(std::fmax(f, 0.0f)); // CUDA's saturating float -> uint conversion
        return b < kSahBins - 1 ? b : kSahBins - 1;
    }
    static float centroid(const Box &b, int d) { return 0.5f * b.lo[d] + 0.5f * b.hi[d]; }

    // one node: its box, and the number of its triangles that go left (0: no plane, the slice is cut in the middle as it is)
    void split(const SahTask &task, std::vector<uint32_t> &scratch, uint32_t* numLeftOut) {
        const std::vector<Box> &tb = *triBox;
        uint32_t* order = T->order.data();
        const uint32_t start = task.start, end = task.end, num = end - start;
        // 1. bounds, ordered images (:572-602, :821-853)
        uint32_t lo[3] = { 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu }, hi[3] = { 0, 0, 0 };
        uint32_t clo[3] = { 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu }, chi[3] = { 0, 0, 0 };
        for (uint32_t i = start; i < end; ++i) {
            const Box &b = tb[order[i]];
            for (int d = 0; d < 3; ++d) {
                const uint32_t c = ordered(centroid(b, d));
                lo[d] = std::min(lo[d], ordered(b.lo[d]));
                hi[d] = std::max(hi[d], ordered(b.hi[d]));
                clo[d] = std::min(clo[d], c);
                chi[d] = std::max(chi[d], c);
            }
        }
        float cLo[3], binScale[3];
        for (int d = 0; d < 3; ++d) {
            cLo[d] = fromOrdered(clo[d]);
            const float ext = fromOrdered(chi[d]) - cLo[d];
            binScale[d] = ext > 0.0f ? (float)kSahBins / ext : 0.0f;
        }
        Box &nb = T->box[task.node];
        for (int d = 0; d < 3; ++d) {
            nb.lo[d] = fromOrdered(lo[d]);
            nb.hi[d] = fromOrdered(hi[d]);
        }
        T->count[task.node] = num;

        // 2. binning (:626-661, :871-925): per axis and bin, ordered min / max of the triangle boxes and a count
        uint32_t binLo[3][kSahBins][3], binHi[3][kSahBins][3], binCount[3][kSahBins];
        for (int d = 0; d < 3; ++d)
            for (uint32_t b = 0; b < kSahBins; ++b) {
                binCount[d][b] = 0;
                for (int e = 0; e < 3; ++e) {
                    binLo[d][b][e] = 0xFFFFFFFFu;
                    binHi[d][b][e] = 0u;
                }
            }
        for (uint32_t i = start; i < end; ++i) {
            const Box &bx = tb[order[i]];
            for (int d = 0; d < 3; ++d) {
                const uint32_t b = binOf(centroid(bx, d), cLo[d], binScale[d]);
                ++binCount[d][b];
                for (int e = 0; e < 3; ++e) {
                    binLo[d][b][e] = std::min(binLo[d][b][e], ordered(bx.lo[e]));
                    binHi[d][b][e] = std::max(binHi[d][b][e], ordered(bx.hi[e]));
                }
            }
        }

        // 3. plane evaluation (:663-707, k_sahHugeEval :927-977): first cheapest plane per axis (strict <)
        float axisCost[3];
        uint32_t axisPlane[3], axisLeft[3];
        for (int d = 0; d < 3; ++d) {
            float rightArea[kSahBins];
            uint32_t rightCount[kSahBins];
            float l[3] = { INFINITY, INFINITY, INFINITY }, h[3] = { -INFINITY, -INFINITY, -INFINITY };
            uint32_t cnt = 0;
            for (int b = (int)kSahBins - 1; b >= 1; --b) {
                if (binCount[d][b]) {
                    for (int e = 0; e < 3; ++e) {
                        l[e] = std::fmin(l[e], fromOrdered(binLo[d][b][e]));
                        h[e] = std::fmax(h[e], fromOrdered(binHi[d][b][e]));
                    }
                    cnt += binCount[d][b];
                }
                const float ex = h[0] - l[0], ey = h[1] - l[1], ez = h[2] - l[2];
                rightArea[b] = cnt ? ex * ey + ey * ez + ez * ex : 0.0f;
                rightCount[b] = cnt;
            }
            for (int e = 0; e < 3; ++e) { l[e] = INFINITY; h[e] = -INFINITY; }
            cnt = 0;
            float bestCost = INFINITY;
            uint32_t bestPlane = 0, bestLeft = 0;
            for (int b = 0; b < (int)kSahBins - 1; ++b) {
                if (binCount[d][b]) {
                    for (int e = 0; e < 3; ++e) {
                        l[e] = std::fmin(l[e], fromOrdered(binLo[d][b][e]));
                        h[e] = std::fmax(h[e], fromOrdered(binHi[d][b][e]));
                    }
                    cnt += binCount[d][b];
                }
                if (cnt == 0 || rightCount[b + 1] == 0)
                    continue;
                const float ex = h[0] - l[0], ey = h[1] - l[1], ez = h[2] - l[2];
                const float cost = (ex * ey + ey * ez + ez * ex) * (float)cnt + rightArea[b + 1] * (float)rightCount[b + 1];
                if (cost < bestCost) {
                    bestCost = cost;
                    bestPlane = (uint32_t)b + 1;
                    bestLeft = cnt;
                }
            }
            axisCost[d] = bestCost;
            axisPlane[d] = bestPlane;
            axisLeft[d] = bestLeft;
        }
        // first cheapest axis (:709-716)
        uint32_t axis = 0;
        if (axisCost[1] < axisCost[axis]) axis = 1;
        if (axisCost[2] < axisCost[axis]) axis = 2;
        const uint32_t plane = axisPlane[axis];
        const uint32_t numLeft = plane ? axisLeft[axis] : num / 2;

        // 4. stable partition (:722-763, k_sahHugeCount / Offsets / Scatter :997-1101)
        if (plane) {
            uint32_t offL = 0, offR = 0;
            for (uint32_t i = start; i < end; ++i) {
                const uint32_t t = order[i];
                if (binOf(centroid(tb[t], (int)axis), cLo[axis], binScale[axis]) < plane)
                    scratch[start + offL++] = t;
                else
                    scratch[start + numLeft + offR++] = t;
            }
            std::copy(scratch.begin() + start, scratch.begin() + end, T->order.begin() + start);
        }
        *numLeftOut = numLeft;
    }
};

void buildSah(const std::vector<Box> &triBox, BinaryTree* T, std::vector<uint32_t>* levels) {
    const uint32_t n = T->n;
    T->childL.assign(n - 1, 0);
    T->childR.assign(n - 1, 0);
    T->count.assign(n - 1, 0);
    T->box.assign(2 * n - 1, Box());
    std::vector<uint32_t> scratch(n);
    SahSplitter sp{ &triBox, T };
    std::vector<SahTask> level = { { 0u, 0u, n } }, next;
    uint32_t numNodes = 1;
    while (!level.empty()) {
        uint32_t sizes[3] = { 0, 0, 0 }; // small, big, huge (sahEmitChild :527-540)
        for (const SahTask &t : level) {
            const uint32_t num = t.end - t.start;
            ++sizes[num > kSahHugeNode ? 2 : num > kSahBigNode ? 1 : 0];
        }
        levels->insert(levels->end(), sizes, sizes + 3);
        std::vector<uint32_t> numLeft(level.size());
#pragma omp parallel for schedule(dynamic, 1)
        for (size_t k = 0; k < level.size(); ++k)
            sp.split(level[k], scratch, &numLeft[k]);
        next.clear();
        auto emit = [&](uint32_t first, uint32_t last) -> uint32_t {
            if (last - first == 1)
                return kLeafBit | first;
            next.push_back({ numNodes, first, last });
            return numNodes++;
        };
        for (size_t k = 0; k < level.size(); ++k) {
            const SahTask &t = level[k];
            T->childL[t.node] = emit(t.start, t.start + numLeft[k]);
            T->childR[t.node] = emit(t.start + numLeft[k], t.end);
        }
        level.swap(next);
    }
    for (uint32_t j = 0; j < n; ++j) // k_sahLeafBoxes (:1104-1112)
        T->box[(n - 1) + j] = triBox[T->order[j]];
    T->root = 0u;
}

// ---- k_collapse (:234-393) ----------------------------------------------------------------------------------------------
struct Collapser {
    const BinaryTree* T;
    uint32_t maxLeaf;
    std::vector<InternalNode8>* nodes;
    std::vector<uint32_t>* primRefs;

    static float area(const Box &b) {
        const float dx = b.hi[0] - b.lo[0], dy = b.hi[1] - b.lo[1], dz = b.hi[2] - b.lo[2];
        return dx * dy + dy * dz + dz * dx;
    }

    // writes wide node `wide` for binary subtree `root`; appends its internal children to `queue`
    void collapse(uint32_t wide, uint32_t root, std::vector<std::pair<uint32_t, uint32_t>>* queue) {
        uint32_t ch[8];
        float ar[8];
        bool leafSized[8];
        int nc = 0;
        auto pushChild = [&](uint32_t ref) {
            ch[nc] = ref;
            leafSized[nc] = T->refCount(ref) <= maxLeaf;
            ar[nc] = area(T->refBox(ref));
            ++nc;
        };
        auto openChild = [&](int k) { // child k becomes its left half in place, the right half is appended
            const uint32_t ref = ch[k];
            const int saved = nc;
            nc = k;
            pushChild(T->childL[ref]);
            nc = saved;
            pushChild(T->childR[ref]);
        };
        if (T->refCount(root) <= maxLeaf && (root & kLeafBit)) {
            pushChild(root);
        }
        else {
            pushChild(T->childL[root]);
            pushChild(T->childR[root]);
            while (nc < 8) { // phase 1: the first largest-area child too big for a leaf
                int best = -1;
                float bestArea = -1.0f;
                for (int k = 0; k < nc; ++k)
                    if (!leafSized[k] && ar[k] > bestArea) {
                        bestArea = ar[k];
                        best = k;
                    }
                if (best < 0)
                    break;
                openChild(best);
            }
            while (nc < 8) { // phase 2: the first largest-area multi-triangle leaf
                int best = -1;
                float bestArea = -1.0f;
                for (int k = 0; k < nc; ++k)
                    if (leafSized[k] && !(ch[k] & kLeafBit) && ar[k] > bestArea) {
                        bestArea = ar[k];
                        best = k;
                    }
                if (best < 0)
                    break;
                openChild(best);
            }
        }

        uint32_t numInt = 0, numLeafPrims = 0;
        for (int k = 0; k < nc; ++k) {
            if (!leafSized[k]) ++numInt;
            else numLeafPrims += T->refCount(ch[k]);
        }
        const uint32_t nodeBase = numInt ? (uint32_t)nodes->size() : 0xFFFFFFFFu;
        const uint32_t primBase = numLeafPrims ? (uint32_t)primRefs->size() : 0xFFFFFFFFu;
        nodes->resize(nodes->size() + numInt);
        primRefs->resize(primRefs->size() + numLeafPrims);

        // quantisation frame with the exponent search (:309-326)
        const Box &nb = T->refBox(root);
        float scale[3], recScale[3];
        uint32_t expo[3];
        for (int d = 0; d < 3; ++d) {
            const float dd = (nb.hi[d] - nb.lo[d]) * (1.0f / 255.0f);
            const uint32_t us = f2u(dd);
            uint32_t e = (us >> 23) + ((us & 0x7FFFFFu) ? 1u : 0u);
            while (e < 254u && nb.lo[d] + 255.0f * u2f(e << 23) < nb.hi[d])
                ++e;
            expo[d] = e;
            scale[d] = u2f(e << 23);
            recScale[d] = scale[d] != 0.0f ? 1.0f / scale[d] : 0.0f;
        }
        uint32_t qmin[3][2] = { { 0, 0 }, { 0, 0 }, { 0, 0 } }, qmax[3][2] = { { 0, 0 }, { 0, 0 }, { 0, 0 } };
        uint32_t metas[2] = { 0, 0 };
        uint32_t internalMask = 0, nthInt = 0, leafOffset = 0;
        for (int k = 0; k < 8; ++k) {
            const int w = k >> 2, sh = 8 * (k & 3);
            if (k >= nc) {
                for (int d = 0; d < 3; ++d)
                    qmin[d][w] |= 255u << sh;
                continue;
            }
            const uint32_t ref = ch[k];
            const Box &cb = T->refBox(ref);
            for (int d = 0; d < 3; ++d) { // setChildAabb + the fix-up loops (:346-357)
                const float org = nb.lo[d];
                int q0 = (int)dm_f2uint((cb.lo[d] - org) * recScale[d]);
                q0 = std::min(q0, 255);
                while (q0 > 0 && org + (float)q0 * scale[d] > cb.lo[d])
                    --q0;
                int q1 = (int)std::min(dm_f2uint((cb.hi[d] - org) * recScale[d]) + 1u, 255u);
                while (q1 < 255 && org + (float)q1 * scale[d] < cb.hi[d])
                    ++q1;
                qmin[d][w] |= (uint32_t)q0 << sh;
                qmax[d][w] |= (uint32_t)q1 << sh;
            }
            if (!leafSized[k]) {
                internalMask |= 1u << k;
                queue->push_back({ nodeBase + nthInt, ref });
                ++nthInt;
            }
            else { // the subtree's triangles left to right, end-of-leaf bit on the last (:363-382)
                metas[w] |= leafOffset << sh;
                const uint32_t total = T->refCount(ref);
                uint32_t stack[32];
                int sp = 0;
                uint32_t written = 0;
                stack[sp++] = ref;
                while (sp > 0) {
                    const uint32_t r = stack[--sp];
                    if (r & kLeafBit) {
                        (*primRefs)[primBase + leafOffset + written] = T->order[r & 0x7FFFFFFFu] | (written + 1 == total ? kLeafBit : 0u);
                        ++written;
                    }
                    else {
                        stack[sp++] = T->childR[r];
                        stack[sp++] = T->childL[r];
                    }
                }
                leafOffset += total;
            }
        }
        const uint32_t words[20] = {
            f2u(nb.lo[0]), f2u(nb.lo[1]), f2u(nb.lo[2]), expo[0] | (expo[1] << 8) | (expo[2] << 16) | (internalMask << 24),
            nodeBase, primBase, metas[0], metas[1],
            qmin[0][0], qmin[0][1], qmin[1][0], qmin[1][1],
            qmin[2][0], qmin[2][1], qmax[0][0], qmax[0][1],
            qmax[1][0], qmax[1][1], qmax[2][0], qmax[2][1] };
        std::memcpy(&(*nodes)[wide], words, sizeof(words));
    }
};

} // namespace

std::vector<TriangleStorage> flattenTriangles(const Geometry* geoms, uint32_t numGeoms) {
    std::vector<TriangleStorage> out;
    for (uint32_t g = 0; g < numGeoms; ++g) {
        const Geometry &geom = geoms[g];
        for (uint32_t p = 0; p < geom.numTriangles; ++p) {
            const uint32_t* tri = geom.triangles + 3 * (size_t)p;
            float3 ps[3];
            for (int i = 0; i < 3; ++i) {
                const float* v = reinterpret_cast<const float*>(geom.vertices + (size_t)geom.vertexStride * tri[i]);
                ps[i] = geom.preTransform.point(float3(v[0], v[1], v[2]));
            }
            TriangleStorage ts;
            std::memset(&ts, 0, sizeof(ts));
            for (int i = 0; i < 3; ++i) {
                ts.pA[i] = ps[0][i];
                ts.pB[i] = ps[1][i];
                ts.pC[i] = ps[2][i];
            }
            ts.geomIndex = g;
            ts.primIndex = p;
            out.push_back(ts);
        }
    }
    return out;
}

int buildGpuStyleBVH(const Geometry* geoms, uint32_t numGeoms, uint32_t flags, GeometryBVH* bvh, std::vector<uint32_t>* sahLevels) {
    if (flags & GFX_BVH_BUILD_PLOC)
        return -1;
    uint32_t maxLeaf = flags & 0xFFu; // buildBvh :1127-1129
    if (maxLeaf == 0) maxLeaf = 2;
    if (maxLeaf > 31) maxLeaf = 31;
    sahLevels->clear();

    *bvh = GeometryBVH();
    bvh->triStorages = flattenTriangles(geoms, numGeoms);
    bvh->numGeoms = numGeoms;
    const uint32_t n = (uint32_t)bvh->triStorages.size();
    bvh->totalNumPrims = n;
    if (n == 0)
        return 0;

    // k_flatten: triangle boxes
    std::vector<Box> triBox(n);
    float smin[3] = { INFINITY, INFINITY, INFINITY }, smax[3] = { -INFINITY, -INFINITY, -INFINITY };
    for (uint32_t t = 0; t < n; ++t) {
        const TriangleStorage &ts = bvh->triStorages[t];
        for (int d = 0; d < 3; ++d) {
            triBox[t].lo[d] = minOrdered(minOrdered(ts.pA[d], ts.pB[d]), ts.pC[d]);
            triBox[t].hi[d] = maxOrdered(maxOrdered(ts.pA[d], ts.pB[d]), ts.pC[d]);
            smin[d] = minOrdered(smin[d], triBox[t].lo[d]);
            smax[d] = maxOrdered(smax[d], triBox[t].hi[d]);
        }
    }
    // k_morton + stable sort by key
    std::vector<uint64_t> keys(n);
    {
        float s[3];
        for (int d = 0; d < 3; ++d) {
            const float ext = smax[d] - smin[d];
            s[d] = ext > 0 ? 2097151.0f / ext : 0.0f;
        }
        for (uint32_t t = 0; t < n; ++t) {
            const Box &b = triBox[t];
            const float c[3] = { 0.5f * (b.lo[0] + b.hi[0]), 0.5f * (b.lo[1] + b.hi[1]), 0.5f * (b.lo[2] + b.hi[2]) };
            keys[t] = (expandBits21(quantiseMorton(c[0], smin[0], s[0])) << 2) | (expandBits21(quantiseMorton(c[1], smin[1], s[1])) << 1) |
                      expandBits21(quantiseMorton(c[2], smin[2], s[2]));
        }
    }
    BinaryTree T;
    T.n = n;
    T.order.resize(n);
    std::iota(T.order.begin(), T.order.end(), 0u);
    std::stable_sort(T.order.begin(), T.order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });

    if ((flags & GFX_BVH_BUILD_FAST) || n < 3) {
        std::vector<uint64_t> sortedKeys(n);
        for (uint32_t j = 0; j < n; ++j)
            sortedKeys[j] = keys[T.order[j]];
        buildKarras(sortedKeys, triBox, &T);
    }
    else {
        buildSah(triBox, &T, sahLevels);
    }

    // collapse, breadth-first
    Collapser c{ &T, maxLeaf, &bvh->intNodes, &bvh->primRefs };
    bvh->intNodes.resize(1);
    std::vector<std::pair<uint32_t, uint32_t>> queue = { { 0u, T.root } }, next;
    while (!queue.empty()) {
        next.clear();
        for (const auto &item : queue)
            c.collapse(item.first, item.second, &next);
        queue.swap(next);
    }
    return 0;
}

// ---- structural comparison ------------------------------------------------------------------------------------------------
std::string sameTree(const GeometryBVH &a, const GeometryBVH &b) {
    char buf[512];
    if (a.intNodes.size() != b.intNodes.size() || a.primRefs.size() != b.primRefs.size()) {
        snprintf(buf, sizeof(buf), "sizes differ: %zu / %zu nodes, %zu / %zu references", a.intNodes.size(), b.intNodes.size(),
                 a.primRefs.size(), b.primRefs.size());
        return buf;
    }
    if (a.intNodes.empty())
        return "";
    struct Item { uint32_t na, nb; std::string path; };
    std::vector<Item> stack = { { 0u, 0u, "root" } };
    size_t visited = 0;
    const size_t numNodes = a.intNodes.size();
    while (!stack.empty()) {
        const Item it = stack.back();
        stack.pop_back();
        if (it.na >= numNodes || it.nb >= numNodes || ++visited > numNodes)
            return it.path + ": node index out of range or visited twice";
        const InternalNode8 &x = a.intNodes[it.na], &y = b.intNodes[it.nb];
        const uint8_t* px = reinterpret_cast<const uint8_t*>(&x);
        const uint8_t* py = reinterpret_cast<const uint8_t*>(&y);
        // every field but intNodeChildBaseIndex / leafBaseIndex (bytes 16..23)
        static const struct { const char* name; int begin, end; } fields[] = {
            { "quantBoxOrigin", 0, 12 }, { "quantBoxExpScale", 12, 15 }, { "internalMask", 15, 16 }, { "childMetas", 24, 32 },
            { "childQMin", 32, 56 }, { "childQMax", 56, 80 } };
        for (const auto &f : fields) {
            if (std::memcmp(px + f.begin, py + f.begin, f.end - f.begin) != 0) {
                std::string hx, hy;
                for (int i = f.begin; i < f.end; ++i) {
                    char h[4];
                    snprintf(h, sizeof(h), "%02x", px[i]); hx += h;
                    snprintf(h, sizeof(h), "%02x", py[i]); hy += h;
                }
                return it.path + ": " + f.name + " differs (" + hx + " vs " + hy + ")";
            }
        }
        std::vector<Item> children;
        for (uint32_t slot = 0; slot < kArity; ++slot) {
            if (!nodeChildIsValid(x, slot))
                break;
            const std::string path = it.path + "/" + std::to_string(slot);
            if ((x.internalMask >> slot) & 1) {
                const uint32_t below = popcnt(x.internalMask & ((1u << slot) - 1));
                children.push_back({ x.intNodeChildBaseIndex + below, y.intNodeChildBaseIndex + below, path });
                continue;
            }
            uint32_t ia = x.leafBaseIndex + x.childMetas[slot], ib = y.leafBaseIndex + y.childMetas[slot];
            for (uint32_t k = 0;; ++k, ++ia, ++ib) {
                if (ia >= a.primRefs.size() || ib >= b.primRefs.size() || k > 64)
                    return path + ": leaf runs out of range";
                if (a.primRefs[ia] != b.primRefs[ib]) {
                    snprintf(buf, sizeof(buf), ": reference %u differs (%08x vs %08x)", k, a.primRefs[ia], b.primRefs[ib]);
                    return path + buf;
                }
                if (a.primRefs[ia] >> 31)
                    break;
            }
        }
        for (size_t k = children.size(); k-- > 0;) // slot order: the last pushed is visited first
            stack.push_back(children[k]);
    }
    return "";
}

} // namespace orc
