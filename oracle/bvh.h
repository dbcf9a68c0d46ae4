// oracle/bvh.h — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// CPU restatement of the reference's wide-BVH node codec, SBVH builder and scalar traverser:
//   node codec : common/common_shared.h:757-917 (CompressedInternalNode_T<8>, 80 B)
//   storages   : common/common_shared.h:1012-1078 (PrimitiveReference, TriangleStorage, HitObject)
//   builder    : common/bvh_builder.cpp:213-652, 656-1125
//   traverser  : common/bvh_builder.cpp:1227-1270, 1272-1649
// Parity status: the reference ships no golden vectors for this path and cannot be compiled
// here (OptiX SDK + MSVC-only headers), so the BVH oracle is pinned by (i) the struct-size
// static_asserts of the reference (80/48/4/32 B, checked below), and (ii) an exhaustive
// brute-force closest-hit over all triangles (BVH-independent definition of the answer).
#pragma once
#include "vecmath.h"
#include <string>
#include <vector>

namespace orc {

constexpr uint32_t kArity = 8;

#pragma pack(push, 1)
struct InternalNode8 { // common_shared.h:757-806
    float quantBoxOrigin[3];
    uint8_t quantBoxExpScaleX, quantBoxExpScaleY, quantBoxExpScaleZ;
    uint8_t internalMask;
    uint32_t intNodeChildBaseIndex;
    uint32_t leafBaseIndex;
    uint8_t childMetas[8]; // leafOffset
    uint8_t childQMinXs[8], childQMinYs[8], childQMinZs[8];
    uint8_t childQMaxXs[8], childQMaxYs[8], childQMaxZs[8];
};
struct TriangleStorage { // common_shared.h:1017-1025
    float pA[3], pB[3], pC[3];
    uint32_t geomIndex, primIndex, padding;
};
struct HitObject { // common_shared.h:1065-1078
    float dist;
    uint32_t instIndex, instUserData, geomIndex, primIndex;
    float bcA, bcB, bcC;
};
#pragma pack(pop)
static_assert(sizeof(InternalNode8) == 80, "common_shared.h:917");
static_assert(sizeof(TriangleStorage) == 48, "common_shared.h:1025");
static_assert(sizeof(HitObject) == 32, "HitObject");

struct TraversalStatistics { // bvh_builder.h:79-86 (subset that is data, not config)
    uint32_t numAabbTests;
    uint32_t numTriTests;
    uint32_t numIntNodes; // internal nodes popped (not in the reference struct; = AABB-test batches)
    int32_t maxStackDepth;
};

struct Geometry { // bvh_builder.h:26-36
    const uint8_t* vertices;
    uint32_t vertexStride;
    uint32_t numVertices;
    const uint32_t* triangles; // UI32x3, stride 12
    uint32_t numTriangles;
    Affine preTransform;
};

struct BuildConfig { // bvh_builder.h:38-44
    float splittingBudget;
    float intNodeTravCost;
    float primIntersectCost;
    uint32_t minNumPrimsPerLeaf;
    uint32_t maxNumPrimsPerLeaf;
};

struct GeometryBVH { // bvh_builder.h:7-15
    std::vector<InternalNode8> intNodes;
    std::vector<TriangleStorage> triStorages;
    std::vector<uint32_t> primRefs; // storageIndex:31 | isLeafEnd:1 (bit 31)
    std::vector<uint32_t> parentPointers; // index:29 | slot:3
    uint32_t numGeoms = 0;
    uint32_t totalNumPrims = 0;
};

// node codec helpers (common_shared.h:795-866)
AABB nodeChildAabb(const InternalNode8 &n, uint32_t slot);
bool nodeChildIsValid(const InternalNode8 &n, uint32_t slot);
void nodeSetQuantizationAabb(InternalNode8 &n, const AABB &box);
void nodeSetChildAabb(InternalNode8 &n, uint32_t slot, const AABB &box);
void nodeSetInvalidChildBox(InternalNode8 &n, uint32_t slot);

void buildGeometryBVH(const Geometry* geoms, uint32_t numGeoms, const BuildConfig &cfg, GeometryBVH* bvh);

// gpu_bvh.cpp: the world-space TriangleStorage of the geometries in order (calcTriangleVertices), and the tree the CUDA
// builder (gfxexp_b200/csrc/bvh_build.cu) emits for gfx_bvh_build flags `flags` (binned SAH, or LBVH with
// GFX_BVH_BUILD_FAST; PLOC is refused with -1).  sahLevels receives { small, big, huge } node counts per SAH level.
std::vector<TriangleStorage> flattenTriangles(const Geometry* geoms, uint32_t numGeoms);
int buildGpuStyleBVH(const Geometry* geoms, uint32_t numGeoms, uint32_t flags, GeometryBVH* bvh, std::vector<uint32_t>* sahLevels);
// "" if both trees have the same shape, node fields (all but the two base indices) and leaf references, else the first
// difference as a slot path from the root
std::string sameTree(const GeometryBVH &a, const GeometryBVH &b);

bool testRayVsTriangle(
    const float3 &rayOrg, const float3 &rayDir, float distMin, float distMax,
    const float3 &pA, const float3 &pB, const float3 &pC,
    float* hitDist, float3* hitNormal, float* bcB, float* bcC);

HitObject traverse(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                   float distMin, float distMax, TraversalStatistics* stats);

// any-hit in (distMin, distMax): true if something is hit (OptiX visibility ray semantics,
// restir_di_shared.h:559-582 + the AH program optix_restir_di_kernels.cu:5-8).
bool traverseAny(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                 float distMin, float distMax);

// BVH-independent definition of the closest hit: loop over every TriangleStorage, keep the
// smallest hitDist; ties broken towards the smaller storage index.
HitObject bruteForceClosest(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                            float distMin, float distMax);

// Closest hit through the BVH but with the canonical tie-break of bruteForceClosest
// (equal hitDist -> smaller storage index) instead of "first found wins".
HitObject traverseCanonical(const GeometryBVH &bvh, const float3 &rayOrg, const float3 &rayDir,
                            float distMin, float distMax);

} // namespace orc
