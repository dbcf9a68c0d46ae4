// scene.cuh — device-side scene tables, BVH views and frame buffers (all plain pointers into HBM).
//
// Layout decisions (see DESIGN.md "Data layout in HBM"):
//  * vertices: AoS of three float4 per vertex (pos+u | normal+v | tangent) = 48 B, so a gather of one
//    vertex is three aligned 16-byte loads from two 32-byte sectors (the reference's shared::Vertex
//    is 44 B and straddles sectors; common_shared.h:1109-1114);
//  * triangles: uint4 {i0,i1,i2,-} per mesh triangle (aligned 16-byte load);
//  * BVH: the reference's own formats (CompressedInternalNode_T<8> 80 B = five 16-byte loads,
//    TriangleStorage 48 B = three 16-byte loads, PrimitiveReference 4 B), world-space triangles of
//    ALL instances flattened into one single-level BVH (80 GB of HBM makes the IAS/GAS split of the
//    reference unnecessary and saves the per-instance ray transform);
//  * per-pixel frame state: SoA planes of float4/uint4 (one 16-byte load per thread, fully coalesced
//    along x), reservoirs as three float4 planes.
#pragma once
#include "vec.cuh"
#include <cstddef>
#include "../../include/gfxb200.h"

namespace gfx {

constexpr uint32_t kInstGuideSize = 2048;
constexpr uint32_t kPrimGuideSize = 128;

struct DevMesh {
    uint32_t vertexBase;   // into vertices (units of vertices)
    uint32_t triBase;      // into triangles / primWeights / primCdf
    uint32_t numTriangles;
    uint32_t materialSlot;
    float primIntegral;    // emitterPrimDist.integral()
    uint32_t pad[3];
};

// Light records (lights.cu): one 128-byte, 128-byte-aligned record per triangle of every emissive geometry = ONE cache line per
// RIS candidate, read 32 bytes at a time (two 128-bit loads, lighting.cuh ldg256) in the
// order sampleLightUnlessDark (lighting.cuh) needs them - in the candidate kernel every load of the sampling chain is a
// divergent gather, i.e. one L1 wavefront per lane per instruction, so the number of load INSTRUCTIONS per candidate is what the
// L1 data pipe charges for:
//   H0 = q0 (centre.xyz, radius) q1 (density, instance slot, -, -)   cull sphere of the world-space triangle (radius < 0 = never
//        cull: degenerate area, or the selection density lightProb * recArea is not a positive finite number) and the area
//        density lightProb * recArea; a copy of H0 sits in the pick guide, so only the 6 % impure buckets read it from here
//   H1 = q2 (pA.xyz, pB.x) q3 (pB.yz, pC.xy)     H2 = q4 (pC.z, nA.xyz) q5 (nB.xyz, nC.x)      -> sample position
//   H3 = q6 (nC.yz, E.rg) q7 (E.b, radius before the density switch, density, instance slot)   -> light normal, emittance
//        (the second copy of density / instance slot serves callers that kept only the key of a pick, see classifyLight)
// Positions, normals, emittance are produced by the very expressions of sampleLight (restir_di_shared.h:417-425, 485-511),
// the density by the products of DiscreteDistribution1D::sample's probabilities (:356-409) times 2 / |cross| (:496), so reading
// them is bit-identical to recomputing them.
constexpr uint32_t kLightTriStride = 8u; // float4 per light record
// normal matrices of the instances, 64-byte stride (m0..m7 | m8, -, -, -): one 256-bit + one 32-bit load
constexpr uint32_t kNormalMatStride = 4u; // float4 per instance

// Flattened light pick (lights.cu, k_pick*): sampleLight's three nested DiscreteDistribution1D::sample calls (instance ->
// geometry instance -> primitive, each a CDF search plus a remap of u) are a pure, monotone, piecewise-constant function of
// the one random number ul.  Its pieces are found once per light-distribution change by evaluating the exact chain
// (chainPickLightTriangle, lighting.cuh) at interval end points and refining every interval whose ends disagree, down to adjacent
// floats; a candidate then costs one guide-table read (+ a short scan of the piece starts in the 6 % of buckets that hold a
// boundary) instead of ~25 dependent loads.  Exact by construction for every float ul in [0, 1).  A guide entry is 32 bytes:
// (key or piece index, centre.xyz | radius, density, instance slot, -) - for a pure bucket the light's H0 rides along, so the
// one 256-bit read also answers the bounding-sphere test.
constexpr uint32_t kPickGuideBits = 17;
constexpr uint32_t kPickGuideSize = 1u << kPickGuideBits;
constexpr uint32_t kPickPure = 0x80000000u;      // guide entry: bit 31 set = the whole bucket maps to key (low 31 bits)
constexpr uint32_t kPickNone = 0x40000000u;      // key: bit 30 set = sampleLight's probability-0 early out (no light)
constexpr uint32_t kPickMaxUlBits = 0x3F7FFFFFu; // largest float below 1

struct DevInstance {
    float transform[12];
    float curToPrevTransform[12];
    float normalMatrix[9];
    float uniformScale;
    uint32_t firstMeshSlot;
    uint32_t numMeshSlots;
    float geomIntegral;    // lightGeomInstDist.integral()
    uint32_t geomBase;     // index of this instance's first flattened geometry (instance order)
    uint32_t pad[2];
};
static_assert(offsetof(DevInstance, normalMatrix) % 16 == 0, "the normal matrix is read with two 128-bit loads + one scalar");
static_assert(sizeof(DevInstance) % 16 == 0, "DevInstance must stay 16-byte aligned");

struct DevBvh {
    const uint4* nodes;     // 5 x uint4 per node: the traversal copy (octantOrderNode), not the reference-format tree
    const uint32_t* primRefs;
    const float4* tris;     // 3 x float4 per triangle (reference layout, indexed by TriangleStorage index)
    const float4* leafTris; // 3 x float4 per primitive reference, leaf order; .w of the third = primRef word
    uint32_t numNodes;
    uint32_t* overflowFlag; // set to 1 if a traversal stack overflowed (checked by the host)
};

// Environment light: Scene::envLightTexture + envLightImportanceMap (restir_di_shared.h:221-222) and the per-frame
// envLightPowerCoeff / envLightRotation / enableEnvLight (:249-250,269).  texels: W x H RGBA, clamped on upload; pdf / cdf: the H row
// distributions (W and W + 1 values each), topPdf / topCdf: the distribution over rows (RegularConstantContinuousDistribution2D,
// common_shared.h:283-386; built on the host like common_host.cpp:292-357).  enabled = the scene has a map and the frame wants it.
struct DevEnvLight {
    const float4* texels;
    const float* pdf;
    const float* cdf;
    const float* topPdf;
    const float* topCdf;
    uint32_t W, H;
    uint32_t enabled;
    float powerCoeff, rotation;
};
constexpr float kProbToSampleEnvLight = 0.25f; // restir_di_shared.h:6 (and the other apps' *_shared.h:6)

struct DevScene {
    const float4* vertices;          // 3 per vertex
    const uint4* triangles;
    const DevMesh* meshes;
    const GfxMaterialDesc* materials;
    const DevInstance* instances;
    const uint32_t* instanceMeshSlots;
    const uint2* geomToInstMesh;     // flattened geometry -> (instance, mesh slot)
    const float* primWeights;        // per mesh triangle
    const float* primCdf;
    const float* geomWeights;        // per (instance, mesh slot)
    const float* geomCdf;
    const float* instWeights;        // per instance
    const float* instCdf;
    const float* instIntegral;       // device scalar (rebuilt every frame on the GPU)
    // pre-divided selection probabilities weights[i] / integral (same IEEE division the sampler did)
    const float* primProb;
    const float* geomProb;
    const float* instProb;
    // light records of the triangles of every emissive geometry (layout above); lightTriBase[g] = first record of flattened
    // geometry g or 0xFFFFFFFF
    const float4* lightTris;
    const uint32_t* lightTriBase;
    uint32_t numLightTris;
    // flattened light pick: guide[b] (2 x float4) for ul in [b, b + 1) / kPickGuideSize: .x of the first = kPickPure | key, or
    // the index of the piece that holds the bucket's first float; pieces = (first float bit pattern, key) sorted by start,
    // terminated by 0xFFFFFFFF starts
    const float4* pickGuide;
    const uint2* pickPieces;
    const float4* normalMats;        // kNormalMatStride float4 per instance
    // guide tables for the CDF searches: guide[b] = search(cdf, fl(b / G * integral)), b = 0..G, so the
    // answer for u = fl(ul * integral) with ul in [b/G, (b+1)/G) lies in [guide[b], guide[b+1]]
    // (rounding is monotone) and a short scan finishes the exact search.
    const uint32_t* instGuide;       // kInstGuideSize + 1 entries
    const uint32_t* primGuide;       // per mesh: kPrimGuideSize + 1 entries
    uint32_t numInstances;
    unsigned long long* rayCounter;  // frame statistics: rays traced (primary + visibility)
    DevBvh bvh;
    DevEnvLight env;
    // image textures of the materials: texTable[t] = (first texel in texPool, width, height, -); materialTextures[m] = the
    // textures of p0 / p1 / p2 / emittance or 0xFFFFFFFF; nullptr when no material is textured
    const float4* texPool;
    const uint4* texTable;
    const uint4* materialTextures;
    // bump maps: bumpTable[m] = (first texel in bumpTexels, width, height, GfxBumpMapType) of material m's map, or of the default
    // 1x1 texel for a material without one (lights.cu uploadTextures, ensureBumpTable); only read by the BUMP variants of the
    // kernels, which the host launches for frames with GfxFrameParams::enableBumpMapping
    const uint4* bumpTable;
    const float4* bumpTexels;
};

struct DevFrame {
    uint32_t W, H;
    uint4* gb0[2];
    float2* gb1[2];
    float4* gb2[2];
    uint4* gb3[2];
    unsigned long long* rng;
    float4* reservoir[2];       // 3 planes of W*H float4
    float2* reservoirInfo[2];
    float4* beauty;
    float4* albedo;
    float4* normal;
    const float2* neighborDeltas; // 1024 entries
    unsigned long long* stats;    // [0] rays traced (primary + visibility)
    float4* rayQueue;             // wavefront visibility queue, see context.h
    uint32_t* rayPixel;
    uint32_t* rayCounters;
    uint8_t* visibility;
};

struct DevCamera {
    float aspect, fovY;
    f3 position;
    float orientation[9];
    float invOrientation[9];
    float vh, vw;
};

struct DevFrameParams {
    DevCamera camera, prevCamera;
    uint32_t numAccumFrames, frameIndex, bufferIndex;
    float spatialNeighborRadius;
    uint32_t log2NumCandidateSamples, numSpatialNeighbors;
    uint32_t useLowDiscrepancyNeighbors, reuseVisibility, enableTemporalReuse, enableSpatialReuse;
    uint32_t useUnbiasedEstimator, resetFlowBuffer, enableJittering;
    uint32_t currentReservoirIndex, spatialNeighborBaseIndex;
    uint32_t y0, y1; // rows owned by this rank
    uint32_t maxPathLength;
    f3 sceneAabbMin, sceneAabbMax;
    float radianceScale;
    uint32_t reuseVisibilityForTemporal, reuseVisibilityForSpatiotemporal;
    float radiusThresholdForSpatialVisReuse;
    float envLightRotation; // also without a map: the miss program of the G-buffer pass encodes (u, v) with it
};

} // namespace gfx
