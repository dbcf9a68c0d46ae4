// oracle/bvh.cpp — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
// CPU restatement of common/bvh_builder.cpp (builder :213-652, :656-1125; traverser :1227-1649)
// and of the node codec in common/common_shared.h:757-917.  See bvh.h for the parity status.
#include "bvh.h"
#include <omp.h>
#include <cassert>
#include <cstdio>

namespace orc {

// ---------------------------------------------------------------------------------------
// node codec — common_shared.h:795-866
// ---------------------------------------------------------------------------------------
static inline float3 decodeQuantBoxScale(const InternalNode8 &n) { // :795-801
    return float3(u2f((uint32_t)n.quantBoxExpScaleX << 23),
                  u2f((uint32_t)n.quantBoxExpScaleY << 23),
                  u2f((uint32_t)n.quantBoxExpScaleZ << 23));
}
bool nodeChildIsValid(const InternalNode8 &n, uint32_t slot) { // :868-870
    return n.childQMinXs[slot] != 255 || n.childQMaxXs[slot] != 0;
}
AABB nodeChildAabb(const InternalNode8 &n, uint32_t slot) { // :802-812, :871-875
    const float3 d = decodeQuantBoxScale(n);
    const float3 o(n.quantBoxOrigin[0], n.quantBoxOrigin[1], n.quantBoxOrigin[2]);
    const float3 qMin((float)n.childQMinXs[slot], (float)n.childQMinYs[slot], (float)n.childQMinZs[slot]);
    const float3 qMax((float)n.childQMaxXs[slot], (float)n.childQMaxYs[slot], (float)n.childQMaxZs[slot]);
    return AABB(o + qMin * d, o + qMax * d);
}
void nodeSetQuantizationAabb(InternalNode8 &n, const AABB &box) { // :814-830
    n.quantBoxOrigin[0] = box.minP.x;
    n.quantBoxOrigin[1] = box.minP.y;
    n.quantBoxOrigin[2] = box.minP.z;
    const float3 d = (box.maxP - box.minP) / 255.0f;
    auto calcExpScale = [](float s) {
        const uint32_t us = f2u(s);
        return (uint8_t)((us >> 23) + ((us & 0x7FFFFFu) ? 1 : 0));
    };
    n.quantBoxExpScaleX = calcExpScale(d.x);
    n.quantBoxExpScaleY = calcExpScale(d.y);
    n.quantBoxExpScaleZ = calcExpScale(d.z);
}
static inline uint32_t f2uint_sat(float f) { // CUDA float->uint semantics (negative/NaN -> 0)
    if (!(f > 0.0f)) return 0u;
    if (f >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)f;
}
void nodeSetChildAabb(InternalNode8 &n, uint32_t slot, const AABB &box) { // :839-851
    const float3 recD = safeDivide(float3(1.0f), decodeQuantBoxScale(n));
    const float3 o(n.quantBoxOrigin[0], n.quantBoxOrigin[1], n.quantBoxOrigin[2]);
    const float3 qMinPf = (box.minP - o) * recD;
    const float3 qMaxPf = (box.maxP - o) * recD;
    const uint32_t qMin[3] = { f2uint_sat(qMinPf.x), f2uint_sat(qMinPf.y), f2uint_sat(qMinPf.z) };
    const uint32_t qMax[3] = {
        std::min(f2uint_sat(qMaxPf.x) + 1, 255u),
        std::min(f2uint_sat(qMaxPf.y) + 1, 255u),
        std::min(f2uint_sat(qMaxPf.z) + 1, 255u) };
    n.childQMinXs[slot] = (uint8_t)qMin[0];
    n.childQMinYs[slot] = (uint8_t)qMin[1];
    n.childQMinZs[slot] = (uint8_t)qMin[2];
    n.childQMaxXs[slot] = (uint8_t)qMax[0];
    n.childQMaxYs[slot] = (uint8_t)qMax[1];
    n.childQMaxZs[slot] = (uint8_t)qMax[2];
}
void nodeSetInvalidChildBox(InternalNode8 &n, uint32_t slot) { // :852-860
    n.childQMinXs[slot] = 255; n.childQMinYs[slot] = 255; n.childQMinZs[slot] = 255;
    n.childQMaxXs[slot] = 0; n.childQMaxYs[slot] = 0; n.childQMaxZs[slot] = 0;
}

// ---------------------------------------------------------------------------------------
// builder — bvh_builder.cpp:48-58 constants
// ---------------------------------------------------------------------------------------
static constexpr int32_t numObjBins = 16;
static constexpr int32_t numObjPlanes = 15;
static constexpr int32_t numSpaBins = 32;
static constexpr int32_t numSpaPlanes = 31;

struct BuildPrimRef { // :60-74
    AABB box;
    uint32_t geomIndex = 0;
    uint32_t primIndex = 0;
};
struct PrimSplitInfo { // :76-141 (a union in the reference: object-bin indices, or the isRight flag)
    uint8_t binIdx[3];
    uint8_t isRight;
};
struct SplitTask { // :143-152 — spans replaced by (offset, reserved) into the global arrays
    AABB geomAabb;
    AABB centAabb;
    uint32_t offset = 0;
    uint32_t numReserved = 0;
    uint32_t numActualElems = 0;
    uint32_t parentIndex = 0;
    uint32_t slotInParent = 0;
    bool isSplittable = false;
};
struct SplitInfo { // :154-163
    uint32_t leftPrimCount, rightPrimCount;
    AABB leftAabb, rightAabb;
    float cost;
    uint32_t dim;
    uint32_t planeIndex;
    bool isSpecialSplit;
};
struct TempInternalNode { // :165-172
    struct Child { AABB aabb; uint32_t index; uint32_t numLeaves; } children[kArity];
};

struct Builder {
    const Geometry* geoms;
    uint32_t numGeoms;
    BuildConfig cfg;
    std::vector<uint32_t> inputPrimOffsets;
    std::vector<BuildPrimRef> primRefs;
    std::vector<PrimSplitInfo> primSplitInfos;

    void calcTriangleVertices(uint32_t geomIdx, uint32_t primIdx, float3* pA, float3* pB, float3* pC) const { // :176-209
        const Geometry &g = geoms[geomIdx];
        const uint32_t* tri = g.triangles + 3 * (size_t)primIdx;
        float3 ps[3];
        for (int i = 0; i < 3; ++i) {
            const float* v = reinterpret_cast<const float*>(g.vertices + (size_t)g.vertexStride * tri[i]);
            ps[i] = float3(v[0], v[1], v[2]);
        }
        *pA = g.preTransform.point(ps[0]);
        *pB = g.preTransform.point(ps[1]);
        *pC = g.preTransform.point(ps[2]);
    }

    void extractGeomAndPrimIndex(uint32_t inputPrimIdx, uint32_t* geomIdx, uint32_t* primIdx) const { // :680-692
        *geomIdx = 0;
        for (int d = (int)(nextPowerOf2(numGeoms) >> 1); d >= 1; d >>= 1) {
            if (*geomIdx + d >= numGeoms)
                continue;
            if (inputPrimOffsets[*geomIdx + d] <= inputPrimIdx)
                *geomIdx += d;
        }
        *primIdx = inputPrimIdx - inputPrimOffsets[*geomIdx];
    }

    static inline uint32_t binOf(float np, int32_t numBins) { // min(make_uint3(numBins * np), numBins - 1)
        return std::min(f2uint_sat((float)numBins * np), (uint32_t)(numBins - 1));
    }

    void findBestObjectSplit(const SplitTask &task, SplitInfo* splitInfo) { // :213-311
        AABB binAabbs[numObjBins][3];
        uint32_t binPrimCounts[numObjBins][3];
        for (int b = 0; b < numObjBins; ++b)
            for (int d = 0; d < 3; ++d)
                binPrimCounts[b][d] = 0;

        for (uint32_t i = 0; i < task.numActualElems; ++i) {
            const BuildPrimRef &pr = primRefs[task.offset + i];
            PrimSplitInfo &psi = primSplitInfos[task.offset + i];
            const float3 np = task.centAabb.normalize(pr.box.getCenter());
            for (int d = 0; d < 3; ++d) {
                const uint32_t binIdx = binOf(np[d], numObjBins);
                binAabbs[binIdx][d].unify(pr.box);
                ++binPrimCounts[binIdx][d];
                psi.binIdx[d] = (uint8_t)binIdx;
            }
        }

        AABB rightAabbs[numObjPlanes][3];
        uint32_t rightPrimCounts[numObjPlanes][3];
        {
            AABB acc[3];
            uint32_t accCounts[3] = { 0, 0, 0 };
            for (int planeIdx = numObjPlanes - 1; planeIdx >= 0; --planeIdx) {
                const int binIdx = planeIdx + 1;
                for (int d = 0; d < 3; ++d) {
                    acc[d].unify(binAabbs[binIdx][d]);
                    accCounts[d] += binPrimCounts[binIdx][d];
                    rightAabbs[planeIdx][d] = acc[d];
                    rightPrimCounts[planeIdx][d] = accCounts[d];
                }
            }
        }

        int32_t bestPlaneIndices[3] = { -1, -1, -1 };
        float bestCosts[3] = { INFINITY, INFINITY, INFINITY };
        uint32_t bestLeftPrimCounts[3] = { 0, 0, 0 };
        uint32_t bestRightPrimCounts[3] = { 0, 0, 0 };
        AABB bestLeftAabbs[3], bestRightAabbs[3];
        {
            AABB accLeft[3];
            uint32_t accLeftCounts[3] = { 0, 0, 0 };
            for (int planeIdx = 0; planeIdx < numObjPlanes; ++planeIdx) {
                const int binIdx = planeIdx;
                for (int d = 0; d < 3; ++d) {
                    accLeft[d].unify(binAabbs[binIdx][d]);
                    accLeftCounts[d] += binPrimCounts[binIdx][d];
                    const float leftArea = accLeft[d].calcHalfSurfaceArea();
                    const uint32_t leftPrimCount = accLeftCounts[d];
                    const AABB &rightAabb = rightAabbs[planeIdx][d];
                    const float rightArea = rightAabb.calcHalfSurfaceArea();
                    const uint32_t rightPrimCount = rightPrimCounts[planeIdx][d];
                    const float cost = leftArea * leftPrimCount + rightArea * rightPrimCount;
                    if (cost < bestCosts[d]) {
                        bestPlaneIndices[d] = planeIdx;
                        bestCosts[d] = cost;
                        bestLeftPrimCounts[d] = leftPrimCount;
                        bestRightPrimCounts[d] = rightPrimCount;
                        bestLeftAabbs[d] = accLeft[d];
                        bestRightAabbs[d] = rightAabb;
                    }
                }
            }
        }

        const uint32_t bestDim = (uint32_t)std::distance(bestCosts, std::min_element(bestCosts, bestCosts + 3));
        splitInfo->dim = bestDim;
        splitInfo->planeIndex = (uint32_t)bestPlaneIndices[bestDim];
        splitInfo->cost = bestCosts[bestDim];
        splitInfo->leftPrimCount = bestLeftPrimCounts[bestDim];
        splitInfo->rightPrimCount = bestRightPrimCounts[bestDim];
        splitInfo->leftAabb = bestLeftAabbs[bestDim];
        splitInfo->rightAabb = bestRightAabbs[bestDim];
        splitInfo->isSpecialSplit = false;
    }

    void findBestSpatialSplit(const SplitTask &task, SplitInfo* splitInfo) { // :313-415
        const AABB &geomAabb = task.geomAabb;
        AABB binAabbs[numSpaBins][3];
        uint32_t binEntry[numSpaBins][3];
        uint32_t binExit[numSpaBins][3];
        const float3 planePosCoeff = (geomAabb.maxP - geomAabb.minP) / (float)numSpaBins;
        for (int b = 0; b < numSpaBins; ++b)
            for (int d = 0; d < 3; ++d) {
                binEntry[b][d] = 0;
                binExit[b][d] = 0;
            }

        for (uint32_t i = 0; i < task.numActualElems; ++i) {
            const BuildPrimRef &pr = primRefs[task.offset + i];
            const float3 entryNp = geomAabb.normalize(pr.box.minP);
            const float3 exitNp = geomAabb.normalize(pr.box.maxP);
            for (int d = 0; d < 3; ++d) {
                const uint32_t entryBinIdx = binOf(entryNp[d], numSpaBins);
                const uint32_t exitBinIdx = binOf(exitNp[d], numSpaBins);
                for (int32_t b = (int32_t)entryBinIdx; b <= (int32_t)exitBinIdx; ++b)
                    binAabbs[b][d].unify(pr.box);
                ++binEntry[entryBinIdx][d];
                ++binExit[exitBinIdx][d];
            }
        }

        AABB rightAabbs[numSpaPlanes][3];
        uint32_t rightPrimCounts[numSpaPlanes][3];
        {
            AABB acc[3];
            uint32_t accCounts[3] = { 0, 0, 0 };
            for (int planeIdx = numSpaPlanes - 1; planeIdx >= 0; --planeIdx) {
                const int binIdx = planeIdx + 1;
                for (int d = 0; d < 3; ++d) {
                    acc[d].unify(binAabbs[binIdx][d]);
                    accCounts[d] += binExit[binIdx][d];
                    AABB rightAabb = acc[d];
                    rightAabb.minP[d] = geomAabb.minP[d] + (float)(planeIdx + 1) * planePosCoeff[d];
                    rightAabbs[planeIdx][d] = rightAabb;
                    rightPrimCounts[planeIdx][d] = accCounts[d];
                }
            }
        }

        int32_t bestPlaneIndices[3] = { -1, -1, -1 };
        float bestCosts[3] = { INFINITY, INFINITY, INFINITY };
        uint32_t bestLeftPrimCounts[3] = { 0, 0, 0 };
        uint32_t bestRightPrimCounts[3] = { 0, 0, 0 };
        AABB bestLeftAabbs[3], bestRightAabbs[3];
        {
            AABB accLeft[3];
            uint32_t accLeftCounts[3] = { 0, 0, 0 };
            for (int planeIdx = 0; planeIdx < numSpaPlanes; ++planeIdx) {
                const int binIdx = planeIdx;
                for (int d = 0; d < 3; ++d) {
                    accLeft[d].unify(binAabbs[binIdx][d]);
                    accLeftCounts[d] += binEntry[binIdx][d];
                    AABB leftAabb = accLeft[d];
                    leftAabb.maxP[d] = geomAabb.minP[d] + (float)(planeIdx + 1) * planePosCoeff[d];
                    const float leftArea = leftAabb.calcHalfSurfaceArea();
                    const uint32_t leftPrimCount = accLeftCounts[d];
                    const AABB &rightAabb = rightAabbs[planeIdx][d];
                    const float rightArea = rightAabb.calcHalfSurfaceArea();
                    const uint32_t rightPrimCount = rightPrimCounts[planeIdx][d];
                    const float cost = leftArea * leftPrimCount + rightArea * rightPrimCount;
                    if (cost < bestCosts[d]) {
                        bestPlaneIndices[d] = planeIdx;
                        bestCosts[d] = cost;
                        bestLeftPrimCounts[d] = leftPrimCount;
                        bestRightPrimCounts[d] = rightPrimCount;
                        bestLeftAabbs[d] = leftAabb;
                        bestRightAabbs[d] = rightAabb;
                    }
                }
            }
        }

        const uint32_t bestDim = (uint32_t)std::distance(bestCosts, std::min_element(bestCosts, bestCosts + 3));
        splitInfo->dim = bestDim;
        splitInfo->planeIndex = (uint32_t)bestPlaneIndices[bestDim];
        splitInfo->cost = bestCosts[bestDim];
        splitInfo->leftPrimCount = bestLeftPrimCounts[bestDim];
        splitInfo->rightPrimCount = bestRightPrimCounts[bestDim];
        splitInfo->leftAabb = bestLeftAabbs[bestDim];
        splitInfo->rightAabb = bestRightAabbs[bestDim];
        splitInfo->isSpecialSplit = true;
    }

    template <typename Pred>
    void performPartition(const SplitTask &task, const Pred &pred, uint32_t minNumPrimsPerLeaf,
                          uint32_t leftPrimCount, uint32_t rightPrimCount,
                          SplitTask* leftTask, SplitTask* rightTask) { // :419-486
        *leftTask = SplitTask();
        *rightTask = SplitTask();
        BuildPrimRef* refs = primRefs.data() + task.offset;
        PrimSplitInfo* infos = primSplitInfos.data() + task.offset;

        const uint32_t numActualElems = leftPrimCount + rightPrimCount;
        uint32_t leftIdx = 0;
        uint32_t rightIdx = numActualElems - 1;
        while (leftIdx < rightIdx) {
            while (leftIdx < rightIdx && pred(leftIdx)) {
                const BuildPrimRef &pr = refs[leftIdx];
                leftTask->geomAabb.unify(pr.box);
                leftTask->centAabb.unify(pr.box.getCenter());
                ++leftIdx;
            }
            while (leftIdx < rightIdx && !pred(rightIdx)) {
                const BuildPrimRef &pr = refs[rightIdx];
                rightTask->geomAabb.unify(pr.box);
                rightTask->centAabb.unify(pr.box.getCenter());
                --rightIdx;
            }
            if (leftIdx < rightIdx) {
                std::swap(refs[leftIdx], refs[rightIdx]);
                std::swap(infos[leftIdx], infos[rightIdx]);
            }
            else {
                const BuildPrimRef &pr = refs[rightIdx];
                rightTask->geomAabb.unify(pr.box);
                rightTask->centAabb.unify(pr.box.getCenter());
            }
        }

        const uint32_t numPrimsReserved = task.numReserved;
        const uint32_t numLeftPrimsReserved = std::max(
            (uint32_t)((float)numPrimsReserved * (float)leftPrimCount / (float)(leftPrimCount + rightPrimCount)),
            leftPrimCount);
        const uint32_t numRightPrimsReserved = numPrimsReserved - numLeftPrimsReserved;

        if (leftPrimCount < numLeftPrimsReserved) {
            std::copy_backward(refs + leftPrimCount, refs + numActualElems,
                               refs + numLeftPrimsReserved + rightPrimCount);
            for (uint32_t i = leftPrimCount; i < numLeftPrimsReserved; ++i)
                refs[i] = BuildPrimRef();
        }

        leftTask->offset = task.offset;
        leftTask->numReserved = numLeftPrimsReserved;
        leftTask->numActualElems = leftPrimCount;
        leftTask->isSplittable = leftPrimCount > minNumPrimsPerLeaf;

        rightTask->offset = task.offset + numLeftPrimsReserved;
        rightTask->numReserved = numRightPrimsReserved;
        rightTask->numActualElems = rightPrimCount;
        rightTask->isSplittable = rightPrimCount > minNumPrimsPerLeaf;
    }

    static void splitTriangle(float3 pA, float3 pB, float3 pC, float splitPlane, uint32_t splitAxis,
                              AABB* bbA, AABB* bbB) { // :506-545
        uint32_t mask =
            (((pC[splitAxis] >= splitPlane) ? 1u : 0u) << 2) |
            (((pB[splitAxis] >= splitPlane) ? 1u : 0u) << 1) |
            (((pA[splitAxis] >= splitPlane) ? 1u : 0u) << 0);
        bool lrSwap = false;
        if (pA[splitAxis] >= splitPlane) {
            mask = ~mask & 0b111u;
            lrSwap = true;
        }
        if (popcnt(mask) == 1) {
            const float3 temp = pA;
            if (mask == 0b010u) {
                pA = pB;
                pB = temp;
            }
            else {
                pA = pC;
                pC = temp;
            }
            lrSwap ^= true;
        }
        const float tAB = (splitPlane - pA[splitAxis]) / (pB[splitAxis] - pA[splitAxis]);
        const float3 pAB = pA + tAB * (pB - pA);
        const float tAC = (splitPlane - pA[splitAxis]) / (pC[splitAxis] - pA[splitAxis]);
        const float3 pAC = pA + tAC * (pC - pA);

        AABB aabb;
        aabb.unify(pAB).unify(pAC);
        *bbA = unify(aabb, pA);
        *bbB = unify(aabb, pB).unify(pC);
        if (lrSwap)
            std::swap(*bbA, *bbB);
    }

    void performSpatialSplit(const SplitTask &task, const SplitInfo &splitInfo,
                             SplitTask* leftTask, SplitTask* rightTask) { // :547-652
        const uint32_t splitDim = splitInfo.dim;
        const uint32_t splitPlaneIdx = splitInfo.planeIndex;
        const float binCoeff = (task.geomAabb.maxP[splitDim] - task.geomAabb.minP[splitDim]) / (float)numSpaBins;
        const float splitPlane = task.geomAabb.minP[splitDim] + (float)(splitPlaneIdx + 1) * binCoeff;

        const float addToLeftPartialCost =
            splitInfo.rightAabb.calcHalfSurfaceArea() * (float)(splitInfo.rightPrimCount - 1);
        const float addToRightPartialCost =
            splitInfo.leftAabb.calcHalfSurfaceArea() * (float)(splitInfo.leftPrimCount - 1);

        BuildPrimRef* refs = primRefs.data() + task.offset;
        PrimSplitInfo* infos = primSplitInfos.data() + task.offset;
        const uint32_t numPrimsReserved = task.numReserved;
        uint32_t leftPrimCount = 0;
        uint32_t rightPrimCount = 0;
        uint32_t curNumPrims = task.numActualElems;
        for (uint32_t i = 0; i < task.numActualElems; ++i) {
            BuildPrimRef &pr = refs[i];
            PrimSplitInfo &psi = infos[i];

            const float fEntryBinIdx = (pr.box.minP[splitDim] - task.geomAabb.minP[splitDim]) / binCoeff;
            const uint32_t entryBinIdx = std::min(f2uint_sat(fEntryBinIdx), (uint32_t)(numSpaBins - 1));
            const float fExitBinIdx = (pr.box.maxP[splitDim] - task.geomAabb.minP[splitDim]) / binCoeff;
            const uint32_t exitBinIdx = std::min(f2uint_sat(fExitBinIdx), (uint32_t)(numSpaBins - 1));

            if (entryBinIdx <= splitPlaneIdx && exitBinIdx > splitPlaneIdx) {
                const float splitCost = splitInfo.cost;
                const float addToLeftCost =
                    unify(splitInfo.leftAabb, pr.box).calcHalfSurfaceArea() * (float)splitInfo.leftPrimCount +
                    addToLeftPartialCost;
                const float addToRightCost =
                    addToRightPartialCost +
                    unify(splitInfo.rightAabb, pr.box).calcHalfSurfaceArea() * (float)splitInfo.rightPrimCount;
                if (splitCost < addToLeftCost && splitCost < addToRightCost && curNumPrims < numPrimsReserved) {
                    psi.isRight = 0;
                    float3 pA, pB, pC;
                    calcTriangleVertices(pr.geomIndex, pr.primIndex, &pA, &pB, &pC);
                    BuildPrimRef &newPr = refs[curNumPrims];
                    PrimSplitInfo &newPsi = infos[curNumPrims];
                    AABB leftAabb, rightAabb;
                    splitTriangle(pA, pB, pC, splitPlane, splitDim, &leftAabb, &rightAabb);
                    leftAabb.intersect(pr.box);
                    rightAabb.intersect(pr.box);
                    pr.box = leftAabb;
                    newPr.box = rightAabb;
                    newPr.geomIndex = pr.geomIndex;
                    newPr.primIndex = pr.primIndex;
                    newPsi.isRight = 1;
                    ++leftPrimCount;
                    ++rightPrimCount;
                    ++curNumPrims;
                }
                else if (addToLeftCost < addToRightCost) {
                    psi.isRight = 0;
                    ++leftPrimCount;
                }
                else {
                    psi.isRight = 1;
                    ++rightPrimCount;
                }
            }
            else {
                if (entryBinIdx <= splitPlaneIdx) {
                    psi.isRight = 0;
                    ++leftPrimCount;
                }
                else {
                    psi.isRight = 1;
                    ++rightPrimCount;
                }
            }
        }

        const PrimSplitInfo* cinfos = infos;
        auto pred = [cinfos](uint32_t idx) { return !cinfos[idx].isRight; };
        performPartition(task, pred, cfg.minNumPrimsPerLeaf, leftPrimCount, rightPrimCount, leftTask, rightTask);
    }

    void build(GeometryBVH* bvh) { // :656-1125
        uint32_t numInputPrimitives = 0;
        inputPrimOffsets.resize(numGeoms);
        for (uint32_t g = 0; g < numGeoms; ++g) {
            inputPrimOffsets[g] = numInputPrimitives;
            numInputPrimitives += geoms[g].numTriangles;
        }
        const uint32_t minNumPrimsPerLeaf = cfg.minNumPrimsPerLeaf;
        const uint32_t maxNumPrimsPerLeaf = cfg.maxNumPrimsPerLeaf;
        const uint32_t numPrimRefsAllocated = std::max(
            numInputPrimitives, (uint32_t)((1.0f + cfg.splittingBudget) * (float)numInputPrimitives));
        const float intTravCost = cfg.intNodeTravCost;
        const float primIsectCost = cfg.primIntersectCost;

        primRefs.assign(numPrimRefsAllocated, BuildPrimRef());
        primSplitInfos.assign(numPrimRefsAllocated, PrimSplitInfo());
        for (uint32_t i = 0; i < numInputPrimitives; ++i) {
            uint32_t geomIdx, primIdx;
            extractGeomAndPrimIndex(i, &geomIdx, &primIdx);
            float3 pA, pB, pC;
            calcTriangleVertices(geomIdx, primIdx, &pA, &pB, &pC);
            BuildPrimRef pr;
            pr.box.unify(pA).unify(pB).unify(pC);
            pr.geomIndex = geomIdx;
            pr.primIndex = primIdx;
            primRefs[i] = pr;
        }

        std::vector<SplitTask> stack;
        {
            SplitTask rootTask;
            for (uint32_t i = 0; i < numInputPrimitives; ++i) {
                rootTask.geomAabb.unify(primRefs[i].box);
                rootTask.centAabb.unify(primRefs[i].box.getCenter());
            }
            rootTask.offset = 0;
            rootTask.numReserved = numPrimRefsAllocated;
            rootTask.numActualElems = numInputPrimitives;
            rootTask.parentIndex = UINT32_MAX;
            rootTask.slotInParent = 0;
            rootTask.isSplittable = numInputPrimitives > 1;
            stack.push_back(rootTask);
        }

        const bool allowPrimRefIncrease = numPrimRefsAllocated > numInputPrimitives;
        const float rootSA = stack.back().geomAabb.calcHalfSurfaceArea();
        std::vector<TempInternalNode> tempIntNodes;

        while (!stack.empty()) {
            const SplitTask task = stack.back();
            stack.pop_back();

            SplitTask children[kArity];
            children[0] = task;
            uint32_t numChildren = 1;
            while (numChildren < kArity) {
                float maxArea = -INFINITY;
                uint32_t slotToSplit = UINT32_MAX;
                for (uint32_t slot = 0; slot < numChildren; ++slot) {
                    const SplitTask &child = children[slot];
                    if (!child.isSplittable)
                        continue;
                    const float area = child.geomAabb.calcHalfSurfaceArea();
                    if (area > maxArea) {
                        maxArea = area;
                        slotToSplit = slot;
                    }
                }
                if (slotToSplit == UINT32_MAX)
                    break;

                const SplitTask taskToSplit = children[slotToSplit];
                const uint32_t numPrimRefsInSubSeg = taskToSplit.numActualElems;
                const float geomSA = taskToSplit.geomAabb.calcHalfSurfaceArea();
                const float leafCost = geomSA * (float)numPrimRefsInSubSeg * primIsectCost;

                SplitInfo splitInfo;
                findBestObjectSplit(taskToSplit, &splitInfo);
                float splitCost = geomSA * intTravCost + splitInfo.cost * primIsectCost;
                const bool objSplitSuccess = !std::isinf(splitInfo.cost);

                if (allowPrimRefIncrease && objSplitSuccess && numPrimRefsInSubSeg < taskToSplit.numReserved) {
                    const AABB overlappedAabb = intersect(splitInfo.leftAabb, splitInfo.rightAabb);
                    const float overlappedSA = overlappedAabb.isValid() ? overlappedAabb.calcHalfSurfaceArea() : 0.0f;
                    constexpr float splittingThreshold = 1e-5f;
                    if (overlappedSA / rootSA > splittingThreshold) {
                        SplitInfo spaSplitInfo;
                        findBestSpatialSplit(taskToSplit, &spaSplitInfo);
                        const float spaSplitCost = geomSA * intTravCost + spaSplitInfo.cost * primIsectCost;
                        if (spaSplitCost < splitCost) {
                            splitInfo = spaSplitInfo;
                            splitCost = spaSplitCost;
                        }
                    }
                }

                if (leafCost < splitCost && numPrimRefsInSubSeg <= maxNumPrimsPerLeaf) {
                    children[slotToSplit].isSplittable = false;
                    continue;
                }

                SplitTask leftTask, rightTask;
                if (objSplitSuccess) {
                    if (splitInfo.isSpecialSplit) {
                        performSpatialSplit(taskToSplit, splitInfo, &leftTask, &rightTask);
                    }
                    else {
                        const uint32_t splitDim = splitInfo.dim;
                        const uint32_t planeIndex = splitInfo.planeIndex;
                        const PrimSplitInfo* infos = primSplitInfos.data() + taskToSplit.offset;
                        auto pred = [infos, splitDim, planeIndex](uint32_t idx) { // :488-504
                            return infos[idx].binIdx[splitDim] <= planeIndex;
                        };
                        performPartition(taskToSplit, pred, minNumPrimsPerLeaf,
                                         splitInfo.leftPrimCount, splitInfo.rightPrimCount, &leftTask, &rightTask);
                    }
                }
                else {
                    const uint32_t leftPrimCount = numPrimRefsInSubSeg / 2;
                    const uint32_t rightPrimCount = numPrimRefsInSubSeg - leftPrimCount;
                    auto pred = [leftPrimCount](uint32_t idx) { return idx < leftPrimCount; };
                    performPartition(taskToSplit, pred, minNumPrimsPerLeaf, leftPrimCount, rightPrimCount,
                                     &leftTask, &rightTask);
                }
                children[slotToSplit] = leftTask;
                children[numChildren] = rightTask;
                ++numChildren;
            }

            if (numChildren == 1 && task.parentIndex != UINT32_MAX) { // :896-903
                TempInternalNode::Child &selfSlot = tempIntNodes[task.parentIndex].children[task.slotInParent];
                selfSlot.index = task.offset;
                selfSlot.numLeaves = task.numActualElems;
                continue;
            }

            std::stable_sort(children, children + numChildren,
                             [](const SplitTask &a, const SplitTask &b) { return a.numActualElems > b.numActualElems; });

            const uint32_t intNodeIdx = (uint32_t)tempIntNodes.size();
            if (task.parentIndex != UINT32_MAX)
                tempIntNodes[task.parentIndex].children[task.slotInParent].index = intNodeIdx;
            tempIntNodes.resize(tempIntNodes.size() + 1);

            TempInternalNode &intNode = tempIntNodes[intNodeIdx];
            for (uint32_t slot = 0; slot < numChildren; ++slot) {
                SplitTask &childTask = children[slot];
                TempInternalNode::Child &child = intNode.children[slot];
                child.aabb = childTask.geomAabb;
                if (childTask.isSplittable) {
                    childTask.parentIndex = intNodeIdx;
                    childTask.slotInParent = slot;
                    stack.push_back(childTask);
                    child.index = 0; // filled when the child task is processed
                    child.numLeaves = 0;
                }
                else {
                    child.index = childTask.offset;
                    child.numLeaves = childTask.numActualElems;
                }
            }
            for (uint32_t slot = numChildren; slot < kArity; ++slot) {
                TempInternalNode::Child &child = intNode.children[slot];
                child.aabb = AABB();
                child.index = UINT32_MAX;
                child.numLeaves = 0;
            }
        }

        // ---- flatten (:943-1079)
        std::vector<TriangleStorage> triStorages(numInputPrimitives);
        for (uint32_t i = 0; i < numInputPrimitives; ++i) {
            uint32_t geomIdx, primIdx;
            extractGeomAndPrimIndex(i, &geomIdx, &primIdx);
            float3 pA, pB, pC;
            calcTriangleVertices(geomIdx, primIdx, &pA, &pB, &pC);
            TriangleStorage &ts = triStorages[i];
            std::memset(&ts, 0, sizeof(ts));
            ts.pA[0] = pA.x; ts.pA[1] = pA.y; ts.pA[2] = pA.z;
            ts.pB[0] = pB.x; ts.pB[1] = pB.y; ts.pB[2] = pB.z;
            ts.pC[0] = pC.x; ts.pC[1] = pC.y; ts.pC[2] = pC.z;
            ts.geomIndex = geomIdx;
            ts.primIndex = primIdx;
        }

        const uint32_t numIntNodes = (uint32_t)tempIntNodes.size();
        std::vector<uint32_t> dstIntNodeIndices(numIntNodes);
        std::vector<uint32_t> leafChildBlockIndices(numIntNodes);
        if (numIntNodes > 0)
            dstIntNodeIndices[0] = 0;
        uint32_t intChildBlockIdx = 1;
        uint32_t leafChildBlockIdx = 0;
        for (uint32_t n = 0; n < numIntNodes; ++n) {
            const TempInternalNode &intNode = tempIntNodes[n];
            leafChildBlockIndices[n] = leafChildBlockIdx;
            uint32_t intChildCount = 0;
            for (uint32_t slot = 0; slot < kArity; ++slot) {
                const TempInternalNode::Child &child = intNode.children[slot];
                if (child.index == UINT32_MAX)
                    break;
                if (child.numLeaves > 0) {
                    leafChildBlockIdx += child.numLeaves;
                }
                else {
                    dstIntNodeIndices[child.index] = intChildBlockIdx + intChildCount;
                    ++intChildCount;
                }
            }
            intChildBlockIdx += intChildCount;
        }

        const uint32_t numFinalPrimRefs = leafChildBlockIdx;
        std::vector<InternalNode8> dstIntNodes(numIntNodes);
        std::vector<uint32_t> dstPrimRefs(numFinalPrimRefs);
        std::vector<uint32_t> parentPointers(numIntNodes);
        if (numIntNodes > 0)
            parentPointers[0] = 0xFFFFFFFFu;
        for (uint32_t srcIdx = 0; srcIdx < numIntNodes; ++srcIdx) {
            const uint32_t dstIdx = dstIntNodeIndices[srcIdx];
            const TempInternalNode &src = tempIntNodes[srcIdx];
            InternalNode8 &dst = dstIntNodes[dstIdx];
            std::memset(&dst, 0, sizeof(dst));

            AABB quantAabb;
            uint32_t internalMask = 0;
            uint32_t firstIntChildSlot = UINT32_MAX;
            uint32_t primRefOffset = leafChildBlockIndices[srcIdx];
            uint32_t numValidChildren = 0;
            for (uint32_t slot = 0; slot < kArity; ++slot) {
                const TempInternalNode::Child &sc = src.children[slot];
                if (sc.index == UINT32_MAX)
                    break;
                ++numValidChildren;
                quantAabb.unify(sc.aabb);
                if (sc.numLeaves > 0) {
                    for (uint32_t i = 0; i < sc.numLeaves; ++i) {
                        const BuildPrimRef &spr = primRefs[sc.index + i];
                        const uint32_t storageIndex = inputPrimOffsets[spr.geomIndex] + spr.primIndex;
                        const uint32_t isLeafEnd = (i == sc.numLeaves - 1) ? 1u : 0u;
                        dstPrimRefs[primRefOffset + i] = (storageIndex & 0x7FFFFFFFu) | (isLeafEnd << 31);
                    }
                    primRefOffset += sc.numLeaves;
                }
                else {
                    internalMask |= 1u << slot;
                    if (firstIntChildSlot == UINT32_MAX)
                        firstIntChildSlot = slot;
                }
            }

            nodeSetQuantizationAabb(dst, quantAabb);
            dst.internalMask = (uint8_t)internalMask;
            dst.intNodeChildBaseIndex = firstIntChildSlot != UINT32_MAX ?
                dstIntNodeIndices[src.children[firstIntChildSlot].index] : UINT32_MAX;
            dst.leafBaseIndex = (~internalMask & ((1u << numValidChildren) - 1)) ?
                leafChildBlockIndices[srcIdx] : UINT32_MAX;

            uint32_t leafOffset = 0;
            for (uint32_t slot = 0; slot < kArity; ++slot) {
                const TempInternalNode::Child &sc = src.children[slot];
                if (sc.index != UINT32_MAX) {
                    nodeSetChildAabb(dst, slot, sc.aabb);
                    uint8_t meta = 0;
                    if (sc.numLeaves > 0) {
                        meta = (uint8_t)leafOffset;
                        leafOffset += sc.numLeaves;
                    }
                    else {
                        parentPointers[dstIntNodeIndices[sc.index]] = (dstIdx & 0x1FFFFFFFu) | (slot << 29);
                    }
                    dst.childMetas[slot] = meta;
                }
                else {
                    nodeSetInvalidChildBox(dst, slot);
                }
            }
        }

        bvh->intNodes = std::move(dstIntNodes);
        bvh->primRefs = std::move(dstPrimRefs);
        bvh->triStorages = std::move(triStorages);
        bvh->parentPointers = std::move(parentPointers);
        bvh->numGeoms = numGeoms;
        bvh->totalNumPrims = numInputPrimitives;
    }
};

void buildGeometryBVH(const Geometry* geoms, uint32_t numGeoms, const BuildConfig &cfg, GeometryBVH* bvh) { // :1129-1143
    Builder b;
    b.geoms = geoms;
    b.numGeoms = numGeoms;
    b.cfg = cfg;
    b.build(bvh);
}

// ---------------------------------------------------------------------------------------
// traverser — bvh_builder.cpp:1227-1270, 1272-1649
// ---------------------------------------------------------------------------------------
bool testRayVsTriangle(
    const float3 &rayOrg, const float3 &rayDir, float distMin, float distMax,
    const float3 &pA, const float3 &pB, const float3 &pC,
    float* hitDist, float3* hitNormal, float* bcB, float* bcC) { // :1251-1270
    const float3 eAB = pB - pA;
    const float3 eCA = pA - pC;
    *hitNormal = cross(eCA, eAB);

    const float3 e = (1.0f / dot(*hitNormal, rayDir)) * (pA - rayOrg);
    const float3 i = cross(rayDir, e);

    *bcB = dot(i, eCA);
    *bcC = dot(i, eAB);
    *hitDist = dot(*hitNormal, e);

    return ((*hitDist < distMax) && (*hitDist > distMin) &&
            (*bcB >= 0.0f) && (*bcC >= 0.0f) && (*bcB + *bcC <= 1));
}

#define SWAP_ORDER(A, B, W) \
    if (keys[A] > keys[B]) { \
        std::swap(keys[A], keys[B]); \
        const uint32_t mask = (1u << W) - 1; \
        const uint32_t offsetA = A * W; \
        const uint32_t offsetB = B * W; \
        const uint32_t vA = (*values >> offsetA) & mask; \
        const uint32_t vB = (*values >> offsetB) & mask; \
        *values &= ~(mask << offsetA); \
        *values |= (vB << offsetA); \
        *values &= ~(mask << offsetB); \
        *values |= (vA << offsetB); \
    }
static inline void sortOrder(uint32_t (&keys)[8], uint32_t* const values) { // :1240-1247
    SWAP_ORDER(0, 2, 3); SWAP_ORDER(1, 3, 3); SWAP_ORDER(4, 6, 3); SWAP_ORDER(5, 7, 3);
    SWAP_ORDER(0, 4, 3); SWAP_ORDER(1, 5, 3); SWAP_ORDER(2, 6, 3); SWAP_ORDER(3, 7, 3);
    SWAP_ORDER(0, 1, 3); SWAP_ORDER(2, 3, 3); SWAP_ORDER(4, 5, 3); SWAP_ORDER(6, 7, 3);
    SWAP_ORDER(2, 4, 3); SWAP_ORDER(3, 5, 3);
    SWAP_ORDER(1, 4, 3); SWAP_ORDER(3, 6, 3);
    SWAP_ORDER(1, 2, 3); SWAP_ORDER(3, 4, 3); SWAP_ORDER(5, 6, 3);
}
#undef SWAP_ORDER

static inline float3 f3(const float* p) { return float3(p[0], p[1], p[2]); }

enum class HitMode { FirstFound, Canonical, Any };

// The slab test of the parity modes (canonical, any hit).  AABB::intersectRay (:1393) is exact about neither end: a zero
// direction component gives 0 * inf = NaN on a box face through the origin, and the computed distances of a ray passing a box
// edge can cross.  Per axis (u = 2^-24), t = fl(fl(plane - org) * idir) errs by u |plane - org| |idir| + u |t|, at most
// 2u |idir| (|plane| + |org|); and the boxes themselves contain their triangles only to the precision of the coordinates: the
// SBVH clips split references in float, so the box of a part can miss a point of the part by a fraction of an ulp
// (<= 2u |plane|).  Together at most 4u |idir| (|plane| + |org|) per plane, a term in the size of the coordinates, not of t:
// a ray with a short hit far from the origin needs it.  So each axis gets s = 2^-21 |idir| (|min| + |max| + |org|), twice that
// bound, the near distances are lowered and the far ones raised by it, and the far bound is widened by 1e-5 relative for the
// culls against the closest hit.  The reciprocal is guarded like the CUDA traverser's (components below 2^-80 become +-2^-80),
// so a nearly parallel axis widens only its own slab.  The test decides which boxes are visited, never a hit, so a box it
// keeps too many only costs time.
static inline bool intersectBoxConservative(const AABB &box, const float3 &org, const float3 &idir, float distMin,
                                            float distMax, float* hitDistMin, float* hitDistMax) {
    float tn = distMin, tf = distMax * 1.00001f;
    for (int a = 0; a < 3; ++a) {
        const float t0 = (box.minP[a] - org[a]) * idir[a];
        const float t1 = (box.maxP[a] - org[a]) * idir[a];
        const float slack = 4.76837158e-7f * std::fabs(idir[a]) *
                            (std::fabs(box.minP[a]) + std::fabs(box.maxP[a]) + std::fabs(org[a]));
        tn = std::fmax(tn, std::fmin(t0, t1) - slack);
        tf = std::fmin(tf, std::fmax(t0, t1) + slack);
    }
    *hitDistMin = tn;
    *hitDistMax = tf;
    return tn <= tf;
}
static inline float3 guardedReciprocal(const float3 &dir) {
    const float ooeps = 8.271806e-25f; // 2^-80
    auto g = [&](float d) { return 1.0f / (std::fabs(d) > ooeps ? d : std::copysign(ooeps, d)); };
    return float3(g(dir.x), g(dir.y), g(dir.z));
}

template <HitMode mode>
static inline HitObject traverseImpl(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                                     const float distMin, const float distMax, TraversalStatistics* stats) {
    HitObject ret = {};
    ret.dist = distMax;
    ret.instIndex = UINT32_MAX;
    ret.instUserData = 0;
    ret.geomIndex = UINT32_MAX;
    ret.primIndex = UINT32_MAX;
    ret.bcA = NAN;
    ret.bcB = NAN;
    ret.bcC = NAN;
    uint32_t bestStorageIndex = UINT32_MAX;

    if (stats) {
        stats->numAabbTests = 0;
        stats->numTriTests = 0;
        stats->numIntNodes = 0;
        stats->maxStackDepth = -1;
    }
    if (bvh.intNodes.empty())
        return ret;

    constexpr uint32_t orderBitWidth = 3;
    constexpr uint32_t orderMask = 7;
    struct Entry { // :1307-1315
        uint32_t baseIndex;  // 31 bits
        uint32_t isLeafGroup;
        uint32_t orderInfo;  // 28 bits
        uint32_t numItems;   // 4 bits
    };
    Entry stack[64];
    uint8_t leafOffsets[kArity] = {};
    const float3 invDir = guardedReciprocal(rayDir);
    int32_t stackIdx = 0;
    Entry curGroup = { 0, 0, 0, 1 };

    while (true) {
        if (curGroup.numItems == 0) {
            if (stackIdx == 0)
                break;
            curGroup = stack[--stackIdx];
        }

        Entry curTriGroup = {};
        if (curGroup.isLeafGroup) {
            curTriGroup = curGroup;
            curGroup.numItems = 0;
        }
        else {
            const uint32_t nodeIdx = curGroup.baseIndex + (curGroup.orderInfo & orderMask);
            curGroup.orderInfo >>= orderBitWidth;
            --curGroup.numItems;
            const InternalNode8 &intNode = bvh.intNodes[nodeIdx];
            if (stats)
                ++stats->numIntNodes;

            uint32_t keys[kArity];
            uint32_t orderInfo = 0;
            uint32_t numIntHits = 0;
            uint32_t numLeafHits = 0;
            for (uint32_t slot = 0; slot < kArity; ++slot) {
                if (!nodeChildIsValid(intNode, slot)) {
                    for (; slot < kArity; ++slot)
                        keys[slot] = floatToOrderedUInt(INFINITY);
                    break;
                }
                if (stats)
                    ++stats->numAabbTests;
                const AABB aabb = nodeChildAabb(intNode, slot);
                float hitDistMin, hitDistMax;
                // The reference culls a child box against the current closest distance exactly (:1393); a triangle whose
                // computed distance is an ulp inside a box whose computed entry is an ulp outside is then lost, and which
                // of two near-equal hits survives depends on the tree.  The canonical / any-hit modes (the parity modes)
                // use the conservative test above, so that they equal the brute-force answer.
                const bool boxHit = mode == HitMode::FirstFound
                    ? aabb.intersectRay(rayOrg, rayDir, distMin, ret.dist, &hitDistMin, &hitDistMax)
                    : intersectBoxConservative(aabb, rayOrg, invDir, distMin, ret.dist, &hitDistMin, &hitDistMax);
                if (boxHit) {
                    const bool isLeaf = ((intNode.internalMask >> slot) & 1) == 0;
                    const float dist = 0.5f * (hitDistMin + hitDistMax);
                    keys[slot] = (floatToOrderedUInt(dist) >> 1) | ((isLeaf ? 0u : 1u) << 31);
                    if (isLeaf) {
                        orderInfo |= (slot << (orderBitWidth * slot));
                        ++numLeafHits;
                    }
                    else {
                        const uint32_t nthIntChild = popcnt(intNode.internalMask & ((1u << slot) - 1));
                        orderInfo |= (nthIntChild << (orderBitWidth * slot));
                        ++numIntHits;
                    }
                }
                else {
                    keys[slot] = floatToOrderedUInt(INFINITY);
                }
            }

            if (numIntHits + numLeafHits > 0)
                sortOrder(keys, &orderInfo);

            if (numLeafHits > 0) {
                curTriGroup.numItems = numLeafHits;
                curTriGroup.baseIndex = intNode.leafBaseIndex;
                curTriGroup.isLeafGroup = 1;
                curTriGroup.orderInfo = orderInfo;
                for (uint32_t slot = 0; slot < kArity; ++slot)
                    leafOffsets[slot] = intNode.childMetas[slot];
            }

            if (numIntHits > 0) {
                if (curGroup.numItems > 0) {
                    if (stats)
                        stats->maxStackDepth = std::max(stackIdx, stats->maxStackDepth);
                    stack[stackIdx++] = curGroup;
                }
                curGroup.numItems = numIntHits;
                curGroup.baseIndex = intNode.intNodeChildBaseIndex;
                curGroup.isLeafGroup = 0;
                curGroup.orderInfo = orderInfo >> (orderBitWidth * numLeafHits);
            }
        }

        if (curTriGroup.numItems > 0) {
            const uint32_t slot = curTriGroup.orderInfo & orderMask;
            const uint32_t primRefIdx = curTriGroup.baseIndex + leafOffsets[slot]++;
            if (stats)
                ++stats->numTriTests;
            const uint32_t primRef = bvh.primRefs[primRefIdx];
            const uint32_t storageIndex = primRef & 0x7FFFFFFFu;
            const TriangleStorage &ts = bvh.triStorages[storageIndex];
            float hitDist, hitBcB, hitBcC;
            float3 hitNormal;
            bool hit;
            if (mode == HitMode::Canonical) {
                hit = testRayVsTriangle(rayOrg, rayDir, distMin, distMax, f3(ts.pA), f3(ts.pB), f3(ts.pC),
                                        &hitDist, &hitNormal, &hitBcB, &hitBcC);
                hit = hit && (hitDist < ret.dist || (hitDist == ret.dist && storageIndex < bestStorageIndex));
            }
            else {
                hit = testRayVsTriangle(rayOrg, rayDir, distMin, ret.dist, f3(ts.pA), f3(ts.pB), f3(ts.pC),
                                        &hitDist, &hitNormal, &hitBcB, &hitBcC);
            }
            if (hit) {
                ret.dist = hitDist;
                ret.geomIndex = ts.geomIndex;
                ret.primIndex = ts.primIndex;
                ret.bcA = 1.0f - (hitBcB + hitBcC);
                ret.bcB = hitBcB;
                ret.bcC = hitBcC;
                bestStorageIndex = storageIndex;
                if (mode == HitMode::Any)
                    return ret;
            }
            if (primRef >> 31) {
                curTriGroup.orderInfo >>= orderBitWidth;
                --curTriGroup.numItems;
            }
            if (curTriGroup.numItems > 0) {
                if (curGroup.numItems > 0) {
                    if (stats)
                        stats->maxStackDepth = std::max(stackIdx, stats->maxStackDepth);
                    stack[stackIdx++] = curGroup;
                }
                curGroup = curTriGroup;
            }
        }
    }
    return ret;
}

HitObject traverse(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                   float distMin, float distMax, TraversalStatistics* stats) {
    return traverseImpl<HitMode::FirstFound>(bvh, rayOrg, rayDir, distMin, distMax, stats);
}
// rays traced through the two wrappers below (bench.py's reference arm counts its own rays): one padded counter per thread
namespace { struct alignas(64) RayCounter { unsigned long long n = 0; }; RayCounter g_rayCounters[1024]; }
static inline void countRay() { ++g_rayCounters[omp_get_thread_num() & 1023].n; }
extern "C" unsigned long long orc_rays_traced(int reset) {
    unsigned long long total = 0;
    for (RayCounter &c : g_rayCounters) {
        total += c.n;
        if (reset)
            c.n = 0;
    }
    return total;
}

HitObject traverseCanonical(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                            float distMin, float distMax) {
    countRay();
    return traverseImpl<HitMode::Canonical>(bvh, rayOrg, rayDir, distMin, distMax, nullptr);
}
bool traverseAny(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                 float distMin, float distMax) {
    countRay();
    const HitObject h = traverseImpl<HitMode::Any>(bvh, rayOrg, rayDir, distMin, distMax, nullptr);
    return h.primIndex != UINT32_MAX;
}

HitObject bruteForceClosest(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                            float distMin, float distMax) {
    HitObject ret = {};
    ret.dist = distMax;
    ret.instIndex = UINT32_MAX;
    ret.geomIndex = UINT32_MAX;
    ret.primIndex = UINT32_MAX;
    ret.bcA = ret.bcB = ret.bcC = NAN;
    const uint32_t n = (uint32_t)bvh.triStorages.size();
    for (uint32_t i = 0; i < n; ++i) {
        const TriangleStorage &ts = bvh.triStorages[i];
        float hitDist, hitBcB, hitBcC;
        float3 hitNormal;
        // strict '<' + ascending index == "equal distance -> smaller storage index wins"
        if (testRayVsTriangle(rayOrg, rayDir, distMin, ret.dist, f3(ts.pA), f3(ts.pB), f3(ts.pC),
                              &hitDist, &hitNormal, &hitBcB, &hitBcC)) {
            ret.dist = hitDist;
            ret.geomIndex = ts.geomIndex;
            ret.primIndex = ts.primIndex;
            ret.bcA = 1.0f - (hitBcB + hitBcC);
            ret.bcB = hitBcB;
            ret.bcC = hitBcC;
        }
    }
    return ret;
}

} // namespace orc
