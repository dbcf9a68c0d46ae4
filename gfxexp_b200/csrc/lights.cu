// lights.cu — light importance, CDFs, selection probabilities and the emissive-triangle table.
//
// Replaces common/gpu_kernels/compute_light_probs.cu (computeTriangleProbBuffer :68-82,
// computeGeomInstProbBuffer :115-129, computeInstProbBuffer :162-174, finalizeDiscreteDistribution1D
// :206-212) and the ext/cubd ExclusiveSum calls in Scene::setupLightGeomDistributions /
// setupLightInstDistribution (common/common_host.h:1102-1359).
//
// CUB's scan order is unspecified, which makes CDF entries irreproducible at the ULP level; here
// every CDF is a *sequential* fp32 exclusive scan (the order the oracle uses), so CDFs are
// bit-identical.  The triangle- and geometry-level distributions are static and built once; the
// instance-level one is rebuilt per frame by ONE single-block kernel (importance in parallel ->
// sequential scan out of shared memory -> probabilities in parallel), as the reference rebuilds it
// every frame (restir_di_main.cpp:2303-2309).
//
// Two derived tables make the 32-candidate RIS loop cheap without changing a single bit:
//  * prob[i] = weights[i] / integral — the very division DiscreteDistribution1D::sample performs
//    (common_shared.h:243), hoisted out of the per-candidate path;
//  * lightTris — for every triangle of every emissive geometry the world-space vertices
//    (inst.transform * v.position), recArea = 2 / |cross|, the object-space vertex normals and the
//    material emittance, i.e. the operands sampleLight (restir_di_shared.h:417-425,485-511) would
//    recompute for each of the 66 M candidates per frame.
#include "pathtrace.cuh"
#include "shading_debug.cuh"
#include "context.h"
#include <cmath>
#include <algorithm>
#include <cub/device/device_radix_sort.cuh>

namespace gfx {

// DiscreteDistribution1DTemplate::sample's stepping search (common_shared.h:226-232): last index with cdf <= u
GFX_D uint32_t steppingSearch(const float* cdf, uint32_t numValues, float u) {
    int idx = 0;
    uint32_t p2 = numValues <= 1 ? numValues : 1u << (32 - __clz(numValues - 1));
    for (int d = (int)(p2 >> 1); d >= 1; d >>= 1) {
        if (idx + d >= (int)numValues)
            continue;
        if (cdf[idx + d] <= u)
            idx += d;
    }
    return (uint32_t)idx;
}

// per-mesh guide table for the primitive-level search
__global__ void k_primGuide(DevScene scene, uint32_t numMeshes) {
    const uint32_t mesh = blockIdx.x;
    if (mesh >= numMeshes)
        return;
    const DevMesh m = scene.meshes[mesh];
    uint32_t* guide = const_cast<uint32_t*>(scene.primGuide) + (size_t)mesh * (kPrimGuideSize + 1);
    for (uint32_t b = threadIdx.x; b <= kPrimGuideSize; b += blockDim.x) {
        const float u = ((float)b / (float)kPrimGuideSize) * m.primIntegral;
        guide[b] = m.numTriangles ? steppingSearch(scene.primCdf + m.triBase, m.numTriangles, u) : 0u;
    }
}

// computeTriangleImportance (compute_light_probs.cu:22-46)
__global__ void k_triangleImportance(DevScene scene, uint32_t numMeshes) {
    const uint32_t mesh = blockIdx.y;
    if (mesh >= numMeshes)
        return;
    const DevMesh m = scene.meshes[mesh];
    const GfxMaterialDesc mat = scene.materials[m.materialSlot];
    float* w = const_cast<float*>(scene.primWeights);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < m.numTriangles; t += gridDim.x * blockDim.x) {
        const uint4 tri = scene.triangles[m.triBase + t];
        const float4 a = scene.vertices[3 * (size_t)(m.vertexBase + tri.x)];
        const float4 b = scene.vertices[3 * (size_t)(m.vertexBase + tri.y)];
        const float4 c = scene.vertices[3 * (size_t)(m.vertexBase + tri.z)];
        const f3 p0(a.x, a.y, a.z), p1(b.x, b.y, b.z), p2(c.x, c.y, c.z);
        const f3 normal = cross(p1 - p0, p2 - p0);
        const float area = 0.5f * length(normal);
        const f3 e = mat.hasEmittance ? f3(mat.emittance[0], mat.emittance[1], mat.emittance[2]) : f3(0.0f);
        f3 emittanceEstimate(0.0f);
        emittanceEstimate += e;
        emittanceEstimate += e;
        emittanceEstimate += e;
        emittanceEstimate /= 3;
        w[m.triBase + t] = sRGB_calcLuminance(emittanceEstimate) * area;
    }
}

// one thread per distribution: sequential exclusive scan + finalize (common_shared.h:268-271)
__global__ void k_scanMeshes(DevScene scene, uint32_t numMeshes) {
    const uint32_t mesh = blockIdx.x * blockDim.x + threadIdx.x;
    if (mesh >= numMeshes)
        return;
    DevMesh* m = const_cast<DevMesh*>(scene.meshes) + mesh;
    const float* w = scene.primWeights + m->triBase;
    float* cdf = const_cast<float*>(scene.primCdf) + m->triBase;
    float sum = 0.0f;
    float last = 0.0f, lastCdf = 0.0f;
    for (uint32_t t = 0; t < m->numTriangles; ++t) {
        cdf[t] = sum;
        lastCdf = sum;
        last = w[t];
        sum = sum + last;
    }
    m->primIntegral = m->numTriangles ? lastCdf + last : 0.0f;
}

__global__ void k_primProb(DevScene scene, uint32_t numMeshes) {
    const uint32_t mesh = blockIdx.y;
    if (mesh >= numMeshes)
        return;
    const DevMesh m = scene.meshes[mesh];
    float* prob = const_cast<float*>(scene.primProb);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < m.numTriangles; t += gridDim.x * blockDim.x)
        prob[m.triBase + t] = scene.primWeights[m.triBase + t] / m.primIntegral;
}

__global__ void k_scanInstanceGeoms(DevScene scene, uint32_t numInstances) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numInstances)
        return;
    DevInstance* inst = const_cast<DevInstance*>(scene.instances) + i;
    float* w = const_cast<float*>(scene.geomWeights) + inst->firstMeshSlot;
    float* cdf = const_cast<float*>(scene.geomCdf) + inst->firstMeshSlot;
    float* prob = const_cast<float*>(scene.geomProb) + inst->firstMeshSlot;
    float sum = 0.0f, last = 0.0f, lastCdf = 0.0f;
    for (uint32_t k = 0; k < inst->numMeshSlots; ++k) {
        // computeGeomInstImportance (compute_light_probs.cu:68-82)
        const float imp = scene.meshes[scene.instanceMeshSlots[inst->firstMeshSlot + k]].primIntegral;
        w[k] = imp;
        cdf[k] = sum;
        lastCdf = sum;
        last = imp;
        sum = sum + imp;
    }
    const float integral = inst->numMeshSlots ? lastCdf + last : 0.0f;
    inst->geomIntegral = integral;
    for (uint32_t k = 0; k < inst->numMeshSlots; ++k)
        prob[k] = w[k] / integral;
}

// emissive-triangle table: one block per emissive flattened geometry
__global__ void k_lightTris(DevScene scene, const uint32_t* __restrict__ emissiveGeoms, uint32_t numEmissiveGeoms) {
    if (blockIdx.x >= numEmissiveGeoms)
        return;
    const uint32_t g = emissiveGeoms[blockIdx.x];
    const uint2 im = scene.geomToInstMesh[g];
    const DevInstance* inst = scene.instances + im.x;
    const DevMesh mesh = scene.meshes[im.y];
    const GfxMaterialDesc* mat = scene.materials + mesh.materialSlot;
    float4* out = const_cast<float4*>(scene.lightTris) + kLightTriStride * (size_t)scene.lightTriBase[g];
    for (uint32_t prim = threadIdx.x; prim < mesh.numTriangles; prim += blockDim.x) {
        const uint4 tri = scene.triangles[mesh.triBase + prim];
        const float4* vA = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.x);
        const float4* vB = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.y);
        const float4* vC = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.z);
        const float4 a0 = vA[0], a1 = vA[1], b0 = vB[0], b1 = vB[1], c0 = vC[0], c1 = vC[1];
        // restir_di_shared.h:417-425
        const f3 pA = xfmPoint(inst->transform, f3(a0.x, a0.y, a0.z));
        const f3 pB = xfmPoint(inst->transform, f3(b0.x, b0.y, b0.z));
        const f3 pC = xfmPoint(inst->transform, f3(c0.x, c0.y, c0.z));
        const f3 geomNormal = cross(pB - pA, pC - pA);
        const float recArea = 2.0f / length(geomNormal); // :496
        f3 emittance(0.0f);
        if (mat->hasEmittance) { // :505-511 with a 1x1 emittance texture
            emittance = f3(1.0f, 1.0f, 1.0f);
            emittance *= f3(mat->emittance[0], mat->emittance[1], mat->emittance[2]);
        }
        float4* o = out + kLightTriStride * (size_t)prim;
        // bounding sphere of the world-space triangle, slightly inflated; negative radius = never cull (degenerate area)
        const f3 c = (pA + pB + pC) * (1.0f / 3.0f);
        const float r2 = fmaxf(fmaxf(sqLength(pA - c), sqLength(pB - c)), sqLength(pC - c));
        const bool usable = recArea > 0.0f && isfinite(recArea) && isfinite(r2);
        const float radius = usable ? sqrtf(r2) * 1.0001f + 1e-30f : -1.0f;
        o[0] = make_float4(c.x, c.y, c.z, -1.0f);   // k_pickLightProbs switches the cull on once the density is known
        o[1] = make_float4(0.0f, __uint_as_float(im.x), recArea, 0.0f); // density: k_pickLightProbs; recArea parked in .z for it
        o[2] = make_float4(pA.x, pA.y, pA.z, pB.x);
        o[3] = make_float4(pB.y, pB.z, pC.x, pC.y);
        o[4] = make_float4(pC.z, a1.x, a1.y, a1.z);
        o[5] = make_float4(b1.x, b1.y, b1.z, c1.x);
        o[6] = make_float4(c1.y, c1.z, emittance.x, emittance.y);
        o[7] = make_float4(emittance.z, radius, 0.0f, __uint_as_float(im.x)); // .z: density, k_pickLightProbs
    }
}

// ---- flattened light pick (scene.cuh) -------------------------------------------------------------------------------------
// Every float ul in [0, 1) is a bit pattern in [0, kPickMaxUlBits]; positive floats order like their bit patterns.  The chain
// (chainPickLightTriangle) is monotone in ul - u = ul * integral, the CDF search and the remap (u - l) / (r - l) are each
// monotone, so the (instance, geometry, primitive) triple grows lexicographically - hence equal keys at two bit patterns
// mean one key in between, and all boundaries are found by refining only the intervals whose end keys differ.

GFX_D uint32_t pickBucketStart(uint32_t j) { // bit pattern of j / kPickGuideSize; the end of the domain for j = kPickGuideSize
    return j < kPickGuideSize ? __float_as_uint((float)j * (1.0f / (float)kPickGuideSize)) : kPickMaxUlBits;
}
GFX_D uint32_t chainKey(const DevScene &s, uint32_t ulBits) {
    float unusedProb;
    return chainPickLightTriangle(s, __uint_as_float(ulBits), &unusedProb);
}

__global__ void k_pickBucketKeys(DevScene scene, uint32_t* __restrict__ keyAt) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j <= kPickGuideSize)
        keyAt[j] = chainKey(scene, pickBucketStart(j));
}

struct PickWork {
    uint4* queue[2];        // (a, b, key(a), key(b)): key changes somewhere in (a, b]
    uint32_t* counters;     // [0], [1] queue lengths, [2] number of boundaries, [3] error flags
    uint2* boundaries;      // (first bit pattern of a piece, key), unsorted
    uint32_t capacity;
};
GFX_D void pickEmitBoundary(const PickWork &w, uint32_t x, uint32_t key) {
    const uint32_t at = atomicAdd(w.counters + 2, 1u);
    if (at < w.capacity)
        w.boundaries[at] = make_uint2(x, key);
    else
        atomicOr(w.counters + 3, 1u);
}
GFX_D void pickPushInterval(const PickWork &w, int q, uint32_t a, uint32_t b, uint32_t ka, uint32_t kb) {
    const uint32_t at = atomicAdd(w.counters + q, 1u);
    if (at < w.capacity)
        w.queue[q][at] = make_uint4(a, b, ka, kb);
    else
        atomicOr(w.counters + 3, 1u);
}

__global__ void k_pickSeed(const uint32_t* __restrict__ keyAt, PickWork w) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= kPickGuideSize)
        return;
    if (j == 0)
        pickEmitBoundary(w, 0u, keyAt[0]);
    const uint32_t ka = keyAt[j], kb = keyAt[j + 1];
    if (ka != kb)
        pickPushInterval(w, 0, pickBucketStart(j), pickBucketStart(j + 1), ka, kb);
}

// one warp per interval (a, b]: 32 sub-intervals, the chain evaluated at their upper ends; intervals of at most 32 floats are
// resolved float by float
__global__ void __launch_bounds__(256) k_pickRefine(DevScene scene, PickWork w, int qin) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warpsPerGrid = gridDim.x * (blockDim.x >> 5);
    const uint32_t numItems = min(w.counters[qin], w.capacity);
    for (uint32_t item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < numItems; item += warpsPerGrid) {
        const uint4 it = w.queue[qin][item];
        const uint32_t a = it.x, n = it.y - it.x;
        uint32_t lo, hi;
        if (n <= 32) {
            lo = a + min(lane, n);
            hi = a + min(lane + 1, n);
        }
        else { // every sub-interval holds at least one float
            lo = a + (uint32_t)(((uint64_t)n * lane) >> 5);
            hi = a + (uint32_t)(((uint64_t)n * (lane + 1)) >> 5);
        }
        const bool live = hi > lo;
        const uint32_t khi = hi == it.y ? it.w : (live ? chainKey(scene, hi) : it.w);
        uint32_t klo = __shfl_up_sync(0xFFFFFFFFu, khi, 1); // live sub-intervals are contiguous from lane 0
        if (lane == 0)
            klo = it.z;
        if (live && khi != klo) {
            if (hi == lo + 1)
                pickEmitBoundary(w, hi, khi);
            else
                pickPushInterval(w, qin ^ 1, lo, hi, klo, khi);
        }
    }
}

__global__ void k_pickResetQueue(PickWork w, int q, int last) {
    if (last && w.counters[q ^ 1] != 0)
        atomicOr(w.counters + 3, 2u); // intervals left after the last level
    w.counters[q] = 0;
}

// guide entry of bucket j from the sorted pieces (after k_pickLightProbs: a pure bucket copies its light's H0)
__global__ void k_pickGuide(DevScene scene, const uint2* __restrict__ pieces, const uint32_t* __restrict__ counters, uint32_t capacity,
                            float4* __restrict__ guide) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= kPickGuideSize)
        return;
    const uint32_t numPieces = min(counters[2], capacity);
    const uint32_t first = pickBucketStart(j);
    const uint32_t last = j + 1 < kPickGuideSize ? pickBucketStart(j + 1) - 1 : kPickMaxUlBits;
    uint32_t lo = 0, hi = numPieces; // last piece with start <= first (piece 0 starts at 0)
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (pieces[mid].x <= first)
            lo = mid;
        else
            hi = mid;
    }
    const bool pure = lo + 1 >= numPieces || pieces[lo + 1].x > last;
    float4 g0 = make_float4(__uint_as_float(lo), 0.0f, 0.0f, 0.0f), g1 = make_float4(-1.0f, 0.0f, 0.0f, 0.0f);
    if (pure) {
        const uint32_t key = pieces[lo].y;
        g0.x = __uint_as_float(kPickPure | key);
        if (!(key & kPickNone)) {
            const float4* rec = scene.lightTris + kLightTriStride * (size_t)key;
            const float4 q0 = rec[0], q1 = rec[1];
            g0.y = q0.x; g0.z = q0.y; g0.w = q0.z;
            g1 = make_float4(q0.w, q1.x, q1.y, 0.0f);
        }
    }
    guide[2 * (size_t)j] = g0;
    guide[2 * (size_t)j + 1] = g1;
}

// compact normal-matrix table (scene.cuh)
__global__ void k_normalMats(DevScene scene, uint32_t numInstances) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numInstances)
        return;
    const float* m = scene.instances[i].normalMatrix;
    float4* o = const_cast<float4*>(scene.normalMats) + (size_t)kNormalMatStride * i;
    o[0] = make_float4(m[0], m[1], m[2], m[3]);
    o[1] = make_float4(m[4], m[5], m[6], m[7]);
    o[2] = make_float4(m[8], 0.0f, 0.0f, 0.0f);
    o[3] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// selection probability of every reachable light (the chain's own product, taken at the first float of its piece) and the
// switch of its bounding-sphere cull
__global__ void k_pickLightProbs(DevScene scene, const uint2* __restrict__ pieces, const uint32_t* __restrict__ counters,
                                 uint32_t capacity) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(counters[2], capacity))
        return;
    const uint2 piece = pieces[i];
    if (piece.y & kPickNone)
        return;
    float lightProb = 0.0f;
    const uint32_t key = chainPickLightTriangle(scene, __uint_as_float(piece.x), &lightProb);
    if (key != piece.y || key >= scene.numLightTris) { // cannot happen: the piece start was produced by this very evaluation
        atomicOr(const_cast<uint32_t*>(counters) + 3, 4u);
        return;
    }
    float4* rec = const_cast<float4*>(scene.lightTris) + kLightTriStride * (size_t)key;
    const float recArea = rec[1].z;
    const float density = lightProb * recArea; // sampleLight's areaPDensity (restir_di_shared.h:409,496), the one product
    rec[1].x = density;
    rec[7].z = density;
    rec[0].w = (density > 0.0f && isfinite(density)) ? rec[7].y : -1.0f;
}

// debug / test entry: flattened and chain pick of arbitrary ul values side by side
__global__ void k_pickDebug(DevScene scene, const float* __restrict__ ul, uint32_t n, uint32_t* __restrict__ flat,
                            uint32_t* __restrict__ chain) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    float unusedProb;
    flat[i] = pickLightTriangle(scene, ul[i]);
    chain[i] = chainPickLightTriangle(scene, ul[i], &unusedProb);
}

// per frame: computeInstImportance (compute_light_probs.cu:115-129) + exclusive scan + finalize +
// selection probabilities, one block, weights staged in shared memory
__global__ void __launch_bounds__(1024) k_instanceDist(DevScene scene, uint32_t numInstances) {
    extern __shared__ float smem[]; // weights[n], cdf[n]
    float* sw = smem;
    float* sc = smem + numInstances;
    __shared__ float sIntegral;
    for (uint32_t i = threadIdx.x; i < numInstances; i += blockDim.x) {
        const DevInstance* inst = scene.instances + i;
        sw[i] = pow2f(inst->uniformScale) * inst->geomIntegral;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float sum = 0.0f, last = 0.0f, lastCdf = 0.0f;
        for (uint32_t i = 0; i < numInstances; ++i) {
            sc[i] = sum;
            lastCdf = sum;
            last = sw[i];
            sum = sum + last;
        }
        sIntegral = numInstances ? lastCdf + last : 0.0f;
        *const_cast<float*>(scene.instIntegral) = sIntegral;
    }
    __syncthreads();
    const float integral = sIntegral;
    for (uint32_t i = threadIdx.x; i < numInstances; i += blockDim.x) {
        const_cast<float*>(scene.instWeights)[i] = sw[i];
        const_cast<float*>(scene.instCdf)[i] = sc[i];
        const_cast<float*>(scene.instProb)[i] = sw[i] / integral;
    }
    for (uint32_t b = threadIdx.x; b <= kInstGuideSize; b += blockDim.x) {
        const float u = ((float)b / (float)kInstGuideSize) * integral;
        const_cast<uint32_t*>(scene.instGuide)[b] = steppingSearch(sc, numInstances, u);
    }
}

int buildLightPick(gfx_ctx* ctx, cudaStream_t stream);

int buildLightDistributions(gfx_ctx* ctx, cudaStream_t stream, uint32_t /*bufferIndex*/) {
    SceneState &S = ctx->scene;
    const DevScene dev = ctx->devScene();
    if (!S.staticLightDistsBuilt) {
        if (S.numMeshes) {
            k_triangleImportance<<<dim3(64, S.numMeshes), 128, 0, stream>>>(dev, S.numMeshes); ctx->launches++;
            k_scanMeshes<<<(S.numMeshes + 31) / 32, 32, 0, stream>>>(dev, S.numMeshes); ctx->launches++;
            k_primProb<<<dim3(64, S.numMeshes), 128, 0, stream>>>(dev, S.numMeshes); ctx->launches++;
            k_primGuide<<<S.numMeshes, 128, 0, stream>>>(dev, S.numMeshes); ctx->launches++;
        }
        if (S.numInstances) {
            k_scanInstanceGeoms<<<(S.numInstances + 63) / 64, 64, 0, stream>>>(dev, S.numInstances); ctx->launches++;
        }
        S.staticLightDistsBuilt = true;
        S.lightTrisDirty = true;
    }
    if (S.lightTrisDirty)
        S.pickDirty = true; // the records are rewritten (and the instance importances may have changed)
    if (S.lightTrisDirty && S.numEmissiveGeoms) {
        // world-space light triangles follow the instance transforms (gfx_scene_update_instances marks them dirty)
        k_lightTris<<<S.numEmissiveGeoms, 128, 0, stream>>>(dev, S.emissiveGeoms, S.numEmissiveGeoms); ctx->launches++;
    }
    S.lightTrisDirty = false;
    if (S.numInstances) {
        if (S.numInstances > 28000) {
            ctx->setError("gfx_light_dist_build: more than 28 000 instances (shared-memory scan limit)");
            return GFX_ERR_UNSUPPORTED;
        }
        const size_t smem = (size_t)S.numInstances * 8;
        if (smem > 48 * 1024)
            GFX_CUDA(ctx, cudaFuncSetAttribute(k_instanceDist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_instanceDist<<<1, 1024, smem, stream>>>(dev, S.numInstances); ctx->launches++;
    }
    if (S.pickDirty && S.numInstances) {
        const int rc = buildLightPick(ctx, stream);
        if (rc != GFX_OK)
            return rc;
    }
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

// Rebuilds the flattened light pick from the distributions just built (stream-ordered; see the notes above k_pickBucketKeys).
int buildLightPick(gfx_ctx* ctx, cudaStream_t stream) {
    SceneState &S = ctx->scene;
    const DevScene dev = ctx->devScene();
    if (S.pickFlagsPending) { // error flags of the previous (asynchronously checked) rebuild
        GFX_CUDA(ctx, cudaEventSynchronize(S.pickFlagsEvent));
        S.pickFlagsPending = false;
        if (*S.pickFlagsHost) {
            ctx->setError("gfx_light_dist_build: the flattened light pick overflowed its tables (flags " + std::to_string(*S.pickFlagsHost) + ")");
            return GFX_ERR_UNSUPPORTED;
        }
    }
    PickWork w;
    w.queue[0] = S.pickQueue[0];
    w.queue[1] = S.pickQueue[1];
    w.counters = S.pickCounters;
    w.boundaries = S.pickBoundaries;
    w.capacity = S.pickCapacity;
    GFX_CUDA(ctx, cudaMemsetAsync(S.pickCounters, 0, 16, stream));
    GFX_CUDA(ctx, cudaMemsetAsync(S.pickBoundaries, 0xFF, (size_t)S.pickCapacity * 8, stream));
    k_pickBucketKeys<<<(kPickGuideSize + 256) / 256, 256, 0, stream>>>(dev, S.pickKeyAt); ctx->launches++;
    k_pickSeed<<<kPickGuideSize / 256, 256, 0, stream>>>(S.pickKeyAt, w); ctx->launches++;
    // an interval holds at most 2^30 floats (bucket 0: all floats below 2^-17) and shrinks 32-fold per level
    const int numLevels = 8;
    for (int level = 0; level < numLevels; ++level) {
        const int qin = level & 1;
        k_pickRefine<<<296, 256, 0, stream>>>(dev, w, qin); ctx->launches++;
        k_pickResetQueue<<<1, 1, 0, stream>>>(w, qin, level == numLevels - 1); ctx->launches++;
    }
    // pieces = boundaries sorted by their first bit pattern; the unused tail (0xFFFFFFFF starts) terminates the scans
    GFX_CUDA(ctx, cudaMemcpy2DAsync(S.pickSortKeys[0], 4, &S.pickBoundaries[0].x, 8, 4, S.pickCapacity, cudaMemcpyDeviceToDevice, stream));
    GFX_CUDA(ctx, cudaMemcpy2DAsync(S.pickSortVals[0], 4, &S.pickBoundaries[0].y, 8, 4, S.pickCapacity, cudaMemcpyDeviceToDevice, stream));
    size_t tempBytes = S.pickSortTempBytes;
    GFX_CUDA(ctx, cub::DeviceRadixSort::SortPairs(S.pickSortTemp, tempBytes, S.pickSortKeys[0], S.pickSortKeys[1], S.pickSortVals[0],
                                                  S.pickSortVals[1], (int)S.pickCapacity, 0, 32, stream));
    ctx->launches += 3;
    GFX_CUDA(ctx, cudaMemcpy2DAsync(&S.pickPieces[0].x, 8, S.pickSortKeys[1], 4, 4, S.pickCapacity, cudaMemcpyDeviceToDevice, stream));
    GFX_CUDA(ctx, cudaMemcpy2DAsync(&S.pickPieces[0].y, 8, S.pickSortVals[1], 4, 4, S.pickCapacity, cudaMemcpyDeviceToDevice, stream));
    k_pickLightProbs<<<(S.pickCapacity + 255) / 256, 256, 0, stream>>>(dev, S.pickPieces, S.pickCounters, S.pickCapacity); ctx->launches++;
    k_pickGuide<<<kPickGuideSize / 256, 256, 0, stream>>>(dev, S.pickPieces, S.pickCounters, S.pickCapacity, S.pickGuide); ctx->launches++;
    k_normalMats<<<(S.numInstances + 127) / 128, 128, 0, stream>>>(dev, S.numInstances); ctx->launches++;
    GFX_CUDA(ctx, cudaMemcpyAsync(S.pickFlagsHost, S.pickCounters + 3, 4, cudaMemcpyDeviceToHost, stream));
    GFX_CUDA(ctx, cudaEventRecord(S.pickFlagsEvent, stream));
    S.pickFlagsPending = true;
    if (!S.pickBuiltOnce) { // the first build is checked at once (scene set-up is not on the per-frame path)
        GFX_CUDA(ctx, cudaEventSynchronize(S.pickFlagsEvent));
        S.pickFlagsPending = false;
        if (*S.pickFlagsHost) {
            ctx->setError("gfx_light_dist_build: the flattened light pick overflowed its tables (flags " + std::to_string(*S.pickFlagsHost) + ")");
            return GFX_ERR_UNSUPPORTED;
        }
        S.pickBuiltOnce = true;
    }
    S.pickDirty = false;
    return GFX_OK;
}

size_t lightPickSortTempBytes(uint32_t capacity) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)capacity, 0, 32, (cudaStream_t)0);
    return bytes ? bytes : 16;
}

int debugLightPick(gfx_ctx* ctx, cudaStream_t stream, const float* dUl, uint32_t n, uint32_t* dFlat, uint32_t* dChain) {
    if (n)
        k_pickDebug<<<(n + 255) / 256, 256, 0, stream>>>(ctx->devScene(), dUl, n, dFlat, dChain);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Environment light: what loadEnvironmentalTexture (common/common_host.cpp:2658-2711) leaves on the device.  Host work, like the
// reference: clamp the texels to [0, 65504], importance = luminance x sin(theta of the texel centre), then one piecewise-constant
// distribution per row and one over the row integrals (RegularConstantContinuousDistribution1D/2D::initialize, :292-357: the CDF
// is a compensated running sum of PDF[i] / N, both normalised by the integral).
namespace {
struct KahanSum { // CompensatedSum_T<float>, basic_types.h:5427-5452
    float result = 0.0f, comp = 0.0f;
    void operator+=(float value) {
        const float cInput = value - comp;
        const float sumTemp = result + cInput;
        comp = (sumTemp - result) - cInput;
        result = sumTemp;
    }
};
// Integral 0 (a black row, or a black map): the reference's lines divide 0 by 0 and leave NaN in every pdf and CDF entry, which
// reaches the miss programs' MIS weights; here such a distribution gets pdf 0 and the uniform CDF i / n instead (DESIGN.md,
// "Environment maps with black rows").  Every other distribution is the reference's, bit for bit.
float regularDistribution(const float* values, uint32_t n, float* pdf, float* cdf) {
    KahanSum sum;
    for (uint32_t i = 0; i < n; ++i) {
        cdf[i] = sum.result;
        sum += values[i] / n;
    }
    const float integral = sum.result;
    for (uint32_t i = 0; i < n; ++i) {
        if (integral > 0.0f) {
            pdf[i] = values[i] / integral;
            cdf[i] /= integral;
        }
        else {
            pdf[i] = 0.0f;
            cdf[i] = (float)i / (float)n;
        }
    }
    cdf[n] = 1.0f;
    return integral;
}
} // namespace

int uploadEnvLight(gfx_ctx* ctx, const float* rgba, uint32_t width, uint32_t height) {
    SceneState &S = ctx->scene;
    if (!rgba || !width || !height)
        return GFX_OK;
    const size_t n = (size_t)width * height;
    std::vector<float4> texels(n);
    std::vector<float> importance(n), pdf(n), cdf((size_t)(width + 1) * height), rowIntegral(height), topPdf(height), topCdf(height + 1);
    for (uint32_t y = 0; y < height; ++y) {
        const float theta = 3.14159265358979323846f * (y + 0.5f) / height;
        const float sinTheta = std::sin(theta);
        for (uint32_t x = 0; x < width; ++x) {
            const float* src = rgba + 4 * ((size_t)y * width + x);
            if (std::isnan(src[0]) || std::isnan(src[1]) || std::isnan(src[2])) { // the clamp below would pass it into every pdf
                ctx->setError("gfx_scene_upload: NaN texel in the environment map");
                return GFX_ERR_INVALID_ARGUMENT;
            }
            float4 t;
            t.x = std::min(std::max(src[0], 0.0f), 65504.0f);
            t.y = std::min(std::max(src[1], 0.0f), 65504.0f);
            t.z = std::min(std::max(src[2], 0.0f), 65504.0f);
            t.w = src[3];
            texels[(size_t)y * width + x] = t;
            importance[(size_t)y * width + x] = (0.2126729f * t.x + 0.7151522f * t.y + 0.0721750f * t.z) * sinTheta;
        }
    }
    for (uint32_t y = 0; y < height; ++y)
        rowIntegral[y] = regularDistribution(importance.data() + (size_t)y * width, width, pdf.data() + (size_t)y * width,
                                             cdf.data() + (size_t)y * (width + 1));
    const float integral = regularDistribution(rowIntegral.data(), height, topPdf.data(), topCdf.data());
    auto upload = [&](void** dst, const void* src, size_t bytes) {
        cudaError_t e = cudaMalloc(dst, bytes);
        if (e == cudaSuccess)
            e = cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice);
        return e;
    };
    GFX_CUDA(ctx, upload((void**)&S.envTexels, texels.data(), n * 16));
    GFX_CUDA(ctx, upload((void**)&S.envPdf, pdf.data(), n * 4));
    GFX_CUDA(ctx, upload((void**)&S.envCdf, cdf.data(), cdf.size() * 4));
    GFX_CUDA(ctx, upload((void**)&S.envTopPdf, topPdf.data(), topPdf.size() * 4));
    GFX_CUDA(ctx, upload((void**)&S.envTopCdf, topCdf.data(), topCdf.size() * 4));
    S.envW = width;
    S.envH = height;
    S.envIntegral = integral;
    return GFX_OK;
}

// createNormalTexture without a file (common_host.cpp:1396-1412): createImmTexture's UNORM8 of (0.5, 0.5, 1), i.e. 127, 127, 255
static const float4 kDefaultBumpTexel = make_float4(127.0f / 255.0f, 127.0f / 255.0f, 1.0f, 1.0f);

// image textures of the materials: one pool of texels, a table of (offset, width, height) and the per-material indices.  With
// bump maps also their table (offset, width, height, type) per material, whose default entry is a 1x1 texel at the end of the
// pool; a scene without bump maps allocates exactly what it did before they existed (ensureBumpTable adds the table when a
// frame first asks for bump mapping).
int uploadTextures(gfx_ctx* ctx, const GfxSceneDesc* sd) {
    SceneState &S = ctx->scene;
    const bool colourMaps = sd->materialTextures && sd->numTextures;
    const uint32_t numTextures = (colourMaps || sd->bumpMaps) ? sd->numTextures : 0u;
    if (!colourMaps && !sd->bumpMaps)
        return GFX_OK;
    if (numTextures && !sd->textures)
        return GFX_ERR_INVALID_ARGUMENT;
    std::vector<uint4> table(numTextures);
    size_t total = 0;
    for (uint32_t t = 0; t < numTextures; ++t) {
        const GfxTextureDesc &d = sd->textures[t];
        if (!d.texels || !d.width || !d.height || total + (size_t)d.width * d.height > 0xFFFFFFFFull) {
            ctx->setError("gfx_scene_upload: empty or oversized texture");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        table[t] = make_uint4((uint32_t)total, d.width, d.height, 0u);
        total += (size_t)d.width * d.height;
    }
    std::vector<uint4> perMaterial(colourMaps ? sd->numMaterials : 0u);
    for (uint32_t m = 0; m < perMaterial.size(); ++m) {
        const uint32_t* k = sd->materialTextures + 4 * (size_t)m;
        for (int c = 0; c < 4; ++c)
            if (k[c] != 0xFFFFFFFFu && k[c] >= sd->numTextures) {
                ctx->setError("gfx_scene_upload: material texture index out of range");
                return GFX_ERR_INVALID_ARGUMENT;
            }
        if (k[3] != 0xFFFFFFFFu) {
            ctx->setError("gfx_scene_upload: textured emittance is not supported (light sampling reads constant emittances)");
            return GFX_ERR_UNSUPPORTED;
        }
        perMaterial[m] = make_uint4(k[0], k[1], k[2], k[3]);
    }
    const uint32_t defaultTexel = (uint32_t)total;
    std::vector<uint4> bump(sd->numMaterials ? sd->numMaterials : 1u, make_uint4(defaultTexel, 1u, 1u, GFX_BUMP_NORMAL_MAP));
    for (uint32_t m = 0; sd->bumpMaps && m < sd->numMaterials; ++m) {
        const uint32_t idx = sd->bumpMaps[2 * (size_t)m], type = sd->bumpMaps[2 * (size_t)m + 1];
        if ((idx != 0xFFFFFFFFu && idx >= numTextures) || (type != GFX_BUMP_NORMAL_MAP && type != GFX_BUMP_HEIGHT_MAP)) {
            ctx->setError("gfx_scene_upload: bump map index out of range or unknown GfxBumpMapType");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        if (idx != 0xFFFFFFFFu)
            bump[m] = make_uint4(table[idx].x, table[idx].y, table[idx].z, type);
    }
    GFX_CUDA(ctx, cudaMalloc((void**)&S.texPool, (total + (sd->bumpMaps ? 1 : 0)) * 16));
    for (uint32_t t = 0; t < numTextures; ++t)
        GFX_CUDA(ctx, cudaMemcpy(S.texPool + table[t].x, sd->textures[t].texels, (size_t)table[t].y * table[t].z * 16, cudaMemcpyHostToDevice));
    if (sd->bumpMaps) {
        GFX_CUDA(ctx, cudaMemcpy(S.texPool + defaultTexel, &kDefaultBumpTexel, 16, cudaMemcpyHostToDevice));
        GFX_CUDA(ctx, cudaMalloc((void**)&S.bumpTable, bump.size() * 16));
        GFX_CUDA(ctx, cudaMemcpy(S.bumpTable, bump.data(), bump.size() * 16, cudaMemcpyHostToDevice));
        S.bumpTexels = S.texPool;
    }
    if (!colourMaps)
        return GFX_OK;
    GFX_CUDA(ctx, cudaMalloc((void**)&S.texTable, table.size() * 16));
    GFX_CUDA(ctx, cudaMemcpy(S.texTable, table.data(), table.size() * 16, cudaMemcpyHostToDevice));
    GFX_CUDA(ctx, cudaMalloc((void**)&S.materialTextures, perMaterial.size() * 16));
    GFX_CUDA(ctx, cudaMemcpy(S.materialTextures, perMaterial.data(), perMaterial.size() * 16, cudaMemcpyHostToDevice));
    return GFX_OK;
}

// test hook (gfx_env_light_debug): the device-side importance-map sampler, its density and the software texture fetch
__global__ void k_envDebug(DevEnvLight env, int op, const float2* in, uint32_t n, float* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const float2 ab = in[i];
    float* o = out + 3 * (size_t)i;
    if (op == 0) {
        envSample(env, ab.x, ab.y, &o[0], &o[1], &o[2]);
    }
    else if (op == 1) {
        o[0] = envEvaluatePDF(env, ab.x, ab.y);
        o[1] = o[2] = 0.0f;
    }
    else {
        const f3 c = envFetch(env, ab.x, ab.y);
        o[0] = c.x; o[1] = c.y; o[2] = c.z;
    }
}
int debugEnvLight(gfx_ctx* ctx, cudaStream_t stream, int op, const float* dIn, uint32_t n, float* dOut) {
    const DevScene s = ctx->devScene();
    if (!s.env.W) {
        ctx->setError("gfx_env_light_debug: the scene has no environment map");
        return GFX_ERR_NOT_READY;
    }
    if (n)
        k_envDebug<<<(n + 127) / 128, 128, 0, stream>>>(s.env, op, reinterpret_cast<const float2*>(dIn), n, dOut);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

// test hook (gfx_light_sample_debug): light sampling as the renderers call it, one record of kLightSampleDebugStride floats in and
// out per op (include/gfxb200.h lists the layouts); integers travel as their bits
constexpr int kLightSampleDebugStride = 16;
__global__ void k_lightSampleDebug(DevScene s, int op, const float* __restrict__ in, uint32_t n, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const float* a = in + kLightSampleDebugStride * (size_t)i;
    float o[kLightSampleDebugStride];
    for (int k = 0; k < kLightSampleDebugStride; ++k)
        o[k] = 0.0f;
    if (op <= 2) {
        const float ul = a[0], u0 = a[1], u1 = a[2];
        const f3 shadingPoint(a[3], a[4], a[5]), shadingNormal(a[6], a[7], a[8]);
        const float vOutLocalZ = a[9];
        LightSample ls = emptyLightSample();
        float density = 0.0f, lightProb = 0.0f;
        bool dark = false;
        if (op == 0) {
            sampleLight(s, ul, u0, u1, &ls, &density);
        }
        else if (op == 1) {
            dark = sampleLightUnlessDark(s, ul, u0, u1, shadingPoint, shadingNormal, vOutLocalZ, &ls, &density);
        }
        else {
            const uint32_t code = classifyLight(s, ul, pickGuideFetch(s, ul), shadingPoint, shadingNormal, vOutLocalZ);
            dark = code == kLightDark || finishLightSample(s, code, u0, u1, shadingPoint, shadingNormal, vOutLocalZ, &ls, &density);
        }
        o[0] = __uint_as_float(pickLightTriangle(s, ul));
        chainPickLightTriangle(s, ul, &lightProb);
        o[1] = ls.position.x; o[2] = ls.position.y; o[3] = ls.position.z;
        o[4] = ls.normal.x; o[5] = ls.normal.y; o[6] = ls.normal.z;
        o[7] = ls.emittance.x; o[8] = ls.emittance.y; o[9] = ls.emittance.z;
        o[10] = density;
        o[11] = lightProb;
        o[12] = dark ? 1.0f : 0.0f;
    }
    else if (op == 3) {
        LightSample ls = emptyLightSample();
        float density = 0.0f;
        sampleEnvLight(s, a[0], a[1], &ls, &density);
        o[0] = ls.position.x; o[1] = ls.position.y; o[2] = ls.position.z;
        o[3] = density;
        o[4] = ls.emittance.x; o[5] = ls.emittance.y; o[6] = ls.emittance.z;
    }
    else if (op == 4) {
        float tu, tv, theta;
        envMissCoordinates(s.env, f3(a[0], a[1], a[2]), &tu, &tv, &theta);
        o[0] = envMissHypAreaPDensity(s.env, tu, tv, theta);
        o[1] = envMissMisWeight(o[0], a[3], a[4]);
        o[2] = tu; o[3] = tv;
    }
    else if (op == 5) {
        const uint32_t instSlot = __float_as_uint(a[0]), geomInInst = __float_as_uint(a[1]), primIndex = __float_as_uint(a[2]);
        if (instSlot < s.numInstances && geomInInst < s.instances[instSlot].numMeshSlots) {
            const DevInstance* inst = s.instances + instSlot;
            const DevMesh mesh = s.meshes[s.instanceMeshSlots[inst->firstMeshSlot + geomInInst]];
            if (primIndex < mesh.numTriangles) {
                SurfacePoint sp;
                computeSurfacePointAtHit(s, inst, mesh, primIndex, a[3], a[4], &sp);
                o[0] = sp.hypAreaPDensity;
            }
        }
    }
    else {
        float ul = op == 6 ? a[2] : a[0], prob = 0.0f;
        const bool env = op == 6 ? chooseEnvForCandidate(s, __float_as_uint(a[0]), __float_as_uint(a[1]), &ul, &prob)
                                 : chooseEnvForNee(s, &ul, &prob);
        o[0] = env ? 1.0f : 0.0f; o[1] = ul; o[2] = prob;
    }
    for (int k = 0; k < kLightSampleDebugStride; ++k)
        out[kLightSampleDebugStride * (size_t)i + k] = o[k];
}
int debugLightSample(gfx_ctx* ctx, cudaStream_t stream, int op, const float* params, const float* dIn, uint32_t n, float* dOut) {
    GfxFrameParams p;
    memset(&p, 0, sizeof(p));
    p.envLightRotation = params[0];
    p.envLightPowerCoeff = params[1];
    p.enableEnvLight = params[2] != 0.0f ? 1u : 0u;
    const DevScene s = ctx->devScene(&p);
    if ((op == 3 || op == 4) && !s.env.W) {
        ctx->setError("gfx_light_sample_debug: the scene has no environment map");
        return GFX_ERR_NOT_READY;
    }
    if (n)
        k_lightSampleDebug<<<(n + 127) / 128, 128, 0, stream>>>(s, op, dIn, n, dOut);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

// test hook (gfx_shading_debug): one op of the shading layer's table (shading_debug.cuh) per record; needs no scene
static_assert(kShadingDebugNumOps == 16, "gfx_shading_debug accepts ops 0..15");
struct ShadingDebugMaterial {
    float m[9];
};
__global__ void k_shadingDebug(int op, ShadingDebugMaterial mat, const float* in, uint32_t n, float* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    float a[kShadingDebugStride], o[kShadingDebugStride];
    for (int k = 0; k < kShadingDebugStride; ++k)
        a[k] = in[kShadingDebugStride * (size_t)i + k];
    shadingDebugOp(op, mat.m, a, o);
    for (int k = 0; k < kShadingDebugStride; ++k)
        out[kShadingDebugStride * (size_t)i + k] = o[k];
}
int debugShading(gfx_ctx* ctx, cudaStream_t stream, int op, const float* material, const float* dIn, uint32_t n, float* dOut) {
    ShadingDebugMaterial mat;
    for (int k = 0; k < 9; ++k)
        mat.m[k] = material[k];
    if (n)
        k_shadingDebug<<<(n + 127) / 128, 128, 0, stream>>>(op, mat, dIn, n, dOut);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

// a scene uploaded without bump maps: every material reads the default texel, from a table made the first time a frame enables
// bump mapping (allocated then, so that the switch-off frames keep the memory layout of a build without bump mapping)
int ensureBumpTable(gfx_ctx* ctx) {
    SceneState &S = ctx->scene;
    if (S.bumpTable)
        return GFX_OK;
    const std::vector<uint4> bump(S.numMaterials ? S.numMaterials : 1u, make_uint4(0u, 1u, 1u, GFX_BUMP_NORMAL_MAP));
    GFX_CUDA(ctx, cudaMalloc((void**)&S.bumpDefaultTexel, 16));
    GFX_CUDA(ctx, cudaMemcpy(S.bumpDefaultTexel, &kDefaultBumpTexel, 16, cudaMemcpyHostToDevice));
    GFX_CUDA(ctx, cudaMalloc((void**)&S.bumpTable, bump.size() * 16));
    GFX_CUDA(ctx, cudaMemcpy(S.bumpTable, bump.data(), bump.size() * 16, cudaMemcpyHostToDevice));
    S.bumpTexels = S.bumpDefaultTexel;
    return GFX_OK;
}

// test hook (gfx_bump_debug): readModifiedNormal, applyBumpMapping, and the software gather next to the texture unit's
__global__ void k_bumpDebug(DevScene s, int op, uint4 bump, cudaTextureObject_t hwTex, const float* in, uint32_t n, float* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    if (op == 1) {
        const float* a = in + 12 * (size_t)i;
        ReferenceFrame frame;
        frame.tangent = f3(a[3], a[4], a[5]);
        frame.bitangent = f3(a[6], a[7], a[8]);
        frame.normal = f3(a[9], a[10], a[11]);
        const ReferenceFrame r = applyBumpMapping(f3(a[0], a[1], a[2]), frame);
        float* o = out + 9 * (size_t)i;
        o[0] = r.tangent.x; o[1] = r.tangent.y; o[2] = r.tangent.z;
        o[3] = r.bitangent.x; o[4] = r.bitangent.y; o[5] = r.bitangent.z;
        o[6] = r.normal.x; o[7] = r.normal.y; o[8] = r.normal.z;
        return;
    }
    const float u = in[2 * (size_t)i], v = in[2 * (size_t)i + 1];
    if (op == 0) {
        const f3 m = readModifiedNormal(s.bumpTexels + bump.x, bump.y, bump.z, bump.w, u, v);
        float* o = out + 3 * (size_t)i;
        o[0] = m.x; o[1] = m.y; o[2] = m.z;
        return;
    }
    const float4 sw = textureGatherRepeat(s.bumpTexels + bump.x, bump.y, bump.z, u, v);
    const float4 hw = tex2Dgather<float4>(hwTex, u, v, 0);
    float* o = out + 8 * (size_t)i;
    o[0] = sw.x; o[1] = sw.y; o[2] = sw.z; o[3] = sw.w;
    o[4] = hw.x; o[5] = hw.y; o[6] = hw.z; o[7] = hw.w;
}
int debugBump(gfx_ctx* ctx, cudaStream_t stream, int op, uint32_t matSlot, const float* dIn, uint32_t n, float* dOut) {
    const int rc = ensureBumpTable(ctx);
    if (rc != GFX_OK)
        return rc;
    const DevScene s = ctx->devScene();
    uint4 bump = make_uint4(0, 0, 0, 0);
    if (op != 1)
        GFX_CUDA(ctx, cudaMemcpy(&bump, s.bumpTable + matSlot, 16, cudaMemcpyDeviceToHost));
    cudaArray_t array = nullptr;
    cudaTextureObject_t tex = 0;
    auto release = [&]() {
        if (tex)
            cudaDestroyTextureObject(tex);
        if (array)
            cudaFreeArray(array);
    };
    if (op == 2) {
        // the map as the reference holds it: UNORM8 RGBA in a cudaArray read through a texture object with sampler_normFloat
        // (common_host.cpp:1476-1481: normalised float, linear filter, repeat addressing, normalised coordinates)
        std::vector<float4> texels((size_t)bump.y * bump.z);
        GFX_CUDA(ctx, cudaMemcpy(texels.data(), s.bumpTexels + bump.x, texels.size() * 16, cudaMemcpyDeviceToHost));
        std::vector<uchar4> q(texels.size());
        auto unorm8 = [](float x) { return (unsigned char)std::lround(std::fmin(std::fmax(x, 0.0f), 1.0f) * 255.0f); };
        for (size_t k = 0; k < texels.size(); ++k)
            q[k] = make_uchar4(unorm8(texels[k].x), unorm8(texels[k].y), unorm8(texels[k].z), unorm8(texels[k].w));
        const cudaChannelFormatDesc fmt = cudaCreateChannelDesc<uchar4>();
        cudaError_t e = cudaMallocArray(&array, &fmt, bump.y, bump.z);
        if (e == cudaSuccess)
            e = cudaMemcpy2DToArray(array, 0, 0, q.data(), (size_t)bump.y * 4, (size_t)bump.y * 4, bump.z, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            cudaResourceDesc res = {};
            res.resType = cudaResourceTypeArray;
            res.res.array.array = array;
            cudaTextureDesc td = {};
            td.addressMode[0] = td.addressMode[1] = cudaAddressModeWrap;
            td.filterMode = cudaFilterModeLinear;
            td.readMode = cudaReadModeNormalizedFloat;
            td.normalizedCoords = 1;
            e = cudaCreateTextureObject(&tex, &res, &td, nullptr);
        }
        if (e != cudaSuccess) {
            release();
            GFX_CUDA(ctx, e);
        }
    }
    if (n)
        k_bumpDebug<<<(n + 127) / 128, 128, 0, stream>>>(s, op, bump, tex, dIn, n, dOut);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && op == 2)
        e = cudaStreamSynchronize(stream); // the texture object must outlive the kernel
    release();
    GFX_CUDA(ctx, e);
    return GFX_OK;
}

} // namespace gfx