// api.cu — the extern "C" entry points of include/gfxb200.h: context, scene upload, BVH
// import/export, frame buffers.  Kernels live in bvh_build.cu / trace.cu / lights.cu /
// gbuffer.cu / restir.cu / svgf.cu / nrc.cu.
#include "context.h"
#include <random>
#include <cmath>

using namespace gfx;

namespace gfx {

void SceneState::release() {
    cudaFree(vertices); cudaFree(triangles); cudaFree(meshes); cudaFree(materials); cudaFree(instances);
    cudaFree(instanceMeshSlots); cudaFree(geomToInstMesh); cudaFree(geomTriOffsets);
    cudaFree(primWeights); cudaFree(primCdf); cudaFree(geomWeights); cudaFree(geomCdf);
    cudaFree(instWeights); cudaFree(instCdf); cudaFree(instIntegral);
    cudaFree(primProb); cudaFree(geomProb); cudaFree(instProb); cudaFree(lightTris); cudaFree(lightTriBase); cudaFree(emissiveGeoms); cudaFree(instGuide); cudaFree(primGuide);
    cudaFree(texPool); cudaFree(texTable); cudaFree(materialTextures); cudaFree(bumpTable); cudaFree(bumpDefaultTexel);
    cudaFree(envTexels); cudaFree(envPdf); cudaFree(envCdf); cudaFree(envTopPdf); cudaFree(envTopCdf);
    cudaFree(pickGuide); cudaFree(normalMats); cudaFree(pickPieces); cudaFree(pickKeyAt); cudaFree(pickBoundaries); cudaFree(pickCounters); cudaFree(pickSortTemp);
    if (pickFlagsHost) cudaFreeHost(pickFlagsHost);
    if (pickFlagsEvent) cudaEventDestroy(pickFlagsEvent);
    for (int i = 0; i < 2; ++i) {
        cudaFree(pickQueue[i]); cudaFree(pickSortKeys[i]); cudaFree(pickSortVals[i]);
        if (pinnedInstances[i]) cudaFreeHost(pinnedInstances[i]);
        if (pinnedInstancesFree[i]) cudaEventDestroy(pinnedInstancesFree[i]);
    }
    *this = SceneState();
}
void BvhState::release() {
    cudaFree(nodes); cudaFree(primRefs); cudaFree(tris); cudaFree(leafTris); cudaFree(travNodes); cudaFree(sceneBounds);
    uint32_t* keepFlag = overflowFlag;
    void* keepScratch = scratch;
    const size_t keepScratchBytes = scratchBytes;
    *this = BvhState();
    overflowFlag = keepFlag;
    scratch = keepScratch;
    scratchBytes = keepScratchBytes;
}
void FrameState::release() {
    for (int i = 0; i < 2; ++i) {
        cudaFree(gb0[i]); cudaFree(gb1[i]); cudaFree(gb2[i]); cudaFree(gb3[i]);
        cudaFree(reservoir[i]); cudaFree(reservoirInfo[i]);
        cudaFree(svgfLighting[i]); cudaFree(svgfMoments[i]); cudaFree(svgfFinal[i]); cudaFree(svgfDepth[i]);
        cudaFree(ptExtRays[i]); cudaFree(ptExtPixel[i]);
    }
    cudaFree(rayQueue); cudaFree(rayPixel); cudaFree(rayCounters); cudaFree(visibility);
    cudaFree(presentRgba8);
    cudaFree(stats); cudaFree(rng); cudaFree(beauty); cudaFree(albedo); cudaFree(normal); cudaFree(neighborDeltas);
    cudaFree(svgfPrevLighting); cudaFree(svgfAlbedo); cudaFree(svgfPrevScreenPos); cudaFree(svgfNormal); cudaFree(svgfDebugVisualize);
    cudaFree(ptAlphaPdf); cudaFree(ptRadiance); cudaFree(ptExtHits); cudaFree(ptShadowPending); cudaFree(ptCounters);
    cudaFree(rearch.preSampledLights); cudaFree(rearch.rngs); cudaFree(rearch.sampleVis[0]); cudaFree(rearch.sampleVis[1]);
    cudaFree(rearch.rays); cudaFree(rearch.rayPixel); cudaFree(rearch.rayMask); cudaFree(rearch.counters);
    cudaFree(regir.slots[0]); cudaFree(regir.slots[1]); cudaFree(regir.slotRngs); cudaFree(regir.perCellNumAccesses);
    cudaFree(regir.lastAccessFrameIndices); cudaFree(regir.numActiveCells);
    cudaFree(nrc.inferenceQuery); cudaFree(nrc.terminalInfo); cudaFree(nrc.inferredRadiance); cudaFree(nrc.frameContribution);
    for (int i = 0; i < 2; ++i) {
        cudaFree(nrc.trainQuery[i]); cudaFree(nrc.trainTarget[i]);
    }
    cudaFree(nrc.trainVertexInfo); cudaFree(nrc.suffixTerminal); cudaFree(nrc.shufflers); cudaFree(nrc.state);
    cudaFree(nrc.pathA); cudaFree(nrc.pathB); cudaFree(nrc.shadowPending2); cudaFree(nrc.tilePrev); cudaFree(nrc.tileSuffixEnded);
    cudaFree(nrc.stagedFlags); cudaFree(nrc.stagedIndex); cudaFree(nrc.stagedQuery); cudaFree(nrc.stagedThroughput); cudaFree(nrc.stagedNEE); cudaFree(nrc.shardCounts);
    *this = FrameState();
}

DevFrameParams makeDevParams(const gfx_ctx* ctx, const GfxFrameParams* p) {
    auto cam = [](const GfxCamera &c) {
        DevCamera d;
        d.aspect = c.aspect;
        d.fovY = c.fovY;
        d.position = f3(c.position[0], c.position[1], c.position[2]);
        memcpy(d.orientation, c.orientation, 36);
        // Matrix3x3::invert (common/basic_types.h:4150-4158): adjugate * (1/det), on the host
        const float* m = c.orientation;
        const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
        const float det = m00 * m11 * m22 + m01 * m12 * m20 + m02 * m10 * m21
            - m02 * m11 * m20 - m01 * m10 * m22 - m00 * m12 * m21;
        const float rdet = 1 / det;
        d.invOrientation[0] = (m11 * m22 - m12 * m21) * rdet;
        d.invOrientation[1] = -(m01 * m22 - m02 * m21) * rdet;
        d.invOrientation[2] = (m01 * m12 - m02 * m11) * rdet;
        d.invOrientation[3] = -(m10 * m22 - m12 * m20) * rdet;
        d.invOrientation[4] = (m00 * m22 - m02 * m20) * rdet;
        d.invOrientation[5] = -(m00 * m12 - m02 * m10) * rdet;
        d.invOrientation[6] = (m10 * m21 - m11 * m20) * rdet;
        d.invOrientation[7] = -(m00 * m21 - m01 * m20) * rdet;
        d.invOrientation[8] = (m00 * m11 - m01 * m10) * rdet;
        // vh = 2 tan(fovY/2) is evaluated once on the host (optix_gbuffer_kernels.cu:23-24 does it per pixel)
        d.vh = 2 * std::tan(c.fovY * 0.5f);
        d.vw = c.aspect * d.vh;
        return d;
    };
    DevFrameParams d;
    d.camera = cam(p->camera);
    d.prevCamera = cam(p->prevCamera);
    d.numAccumFrames = p->numAccumFrames;
    d.frameIndex = p->frameIndex;
    d.bufferIndex = p->bufferIndex & 1;
    d.spatialNeighborRadius = p->spatialNeighborRadius;
    d.log2NumCandidateSamples = p->log2NumCandidateSamples;
    d.numSpatialNeighbors = p->numSpatialNeighbors;
    d.useLowDiscrepancyNeighbors = p->useLowDiscrepancyNeighbors;
    d.reuseVisibility = p->reuseVisibility;
    d.enableTemporalReuse = p->enableTemporalReuse;
    d.enableSpatialReuse = p->enableSpatialReuse;
    d.useUnbiasedEstimator = p->useUnbiasedEstimator;
    d.resetFlowBuffer = p->resetFlowBuffer;
    d.enableJittering = p->enableJittering;
    d.currentReservoirIndex = p->currentReservoirIndex & 1;
    d.spatialNeighborBaseIndex = p->spatialNeighborBaseIndex;
    d.y0 = p->tileOriginY;
    d.y1 = p->tileRows ? min(ctx->frame.H, p->tileOriginY + p->tileRows) : ctx->frame.H;
    d.maxPathLength = p->maxPathLength;
    d.sceneAabbMin = f3(p->sceneAabbMin[0], p->sceneAabbMin[1], p->sceneAabbMin[2]);
    d.sceneAabbMax = f3(p->sceneAabbMax[0], p->sceneAabbMax[1], p->sceneAabbMax[2]);
    d.radianceScale = p->radianceScale;
    d.reuseVisibilityForTemporal = p->reuseVisibilityForTemporal;
    d.reuseVisibilityForSpatiotemporal = p->reuseVisibilityForSpatiotemporal;
    d.radiusThresholdForSpatialVisReuse = p->radiusThresholdForSpatialVisReuse;
    d.envLightRotation = p->envLightRotation;
    return d;
}

int svgfSubPixelSample(gfx_ctx* ctx, const GfxFrameParams* p, bool* jitter, float2* sample) {
    *jitter = false;
    *sample = make_float2(0.5f, 0.5f);
    if (!(p->svgfFlags & GFX_SVGF_SUBPIXEL_JITTER))
        return GFX_OK;
    if (p->enableJittering) {
        ctx->setError("GFX_SVGF_SUBPIXEL_JITTER and enableJittering both move the primary ray's sample: set one of them");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    if (!(p->svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_AA)) // svgf_main.cpp:2005-2007: the pixel centre without TAA
        return GFX_OK;
    // subPixelOffsets[frameIndex % taaHistoryLength] (svgf_main.cpp:1422-1424, 2007)
    const uint32_t taaHistoryLength = p->taaHistoryLength ? p->taaHistoryLength : 16;
    const uint32_t i = p->frameIndex % taaHistoryLength;
    const float ox = dm_halton(2, i), oy = dm_halton(3, i);
    // The app rasterises the G-buffer with addOffset(matV2C, ox, oy) (svgf_main.cpp:2015-2028): clip x gains
    // (2 ox - 1) / W times view z, so after the divide by w = -z the fragment at GL pixel centre X + 0.5 shows the point whose
    // unjittered projection lies at X + ox; likewise Y + oy in y.  The qRotateY(pi) of matW2V makes GL's x run the way this
    // library's x does, and GL counts rows from the bottom: GL row Y is row y = H - 1 - Y here, so the sample lies at
    // H - (Y + oy) = y + 1 - oy.  fillBackground (svgf.cu:406-408) writes the same position.
    *jitter = true;
    *sample = make_float2(ox, 1.0f - oy);
    return GFX_OK;
}

} // namespace gfx

DevScene gfx_ctx::devScene() const {
    DevScene d;
    d.vertices = scene.vertices;
    d.triangles = scene.triangles;
    d.meshes = scene.meshes;
    d.materials = scene.materials;
    d.instances = scene.instances;
    d.instanceMeshSlots = scene.instanceMeshSlots;
    d.geomToInstMesh = scene.geomToInstMesh;
    d.primWeights = scene.primWeights;
    d.primCdf = scene.primCdf;
    d.geomWeights = scene.geomWeights;
    d.geomCdf = scene.geomCdf;
    d.instWeights = scene.instWeights;
    d.instCdf = scene.instCdf;
    d.instIntegral = scene.instIntegral;
    d.primProb = scene.primProb;
    d.geomProb = scene.geomProb;
    d.instProb = scene.instProb;
    d.lightTris = scene.lightTris;
    d.lightTriBase = scene.lightTriBase;
    d.numLightTris = scene.numLightTris;
    d.pickGuide = scene.pickGuide;
    d.pickPieces = scene.pickPieces;
    d.normalMats = scene.normalMats;
    d.instGuide = scene.instGuide;
    d.primGuide = scene.primGuide;
    d.numInstances = scene.numInstances;
    d.rayCounter = frame.stats;
    d.bvh.nodes = bvh.travNodes;
    d.bvh.primRefs = bvh.primRefs;
    d.bvh.tris = bvh.tris;
    d.bvh.leafTris = bvh.leafTris;
    d.bvh.numNodes = bvh.numNodes;
    d.bvh.overflowFlag = bvh.overflowFlag;
    d.texPool = scene.texPool;
    d.texTable = scene.texTable;
    d.materialTextures = scene.materialTextures;
    d.bumpTable = scene.bumpTable;
    d.bumpTexels = scene.bumpTexels;
    d.env.texels = scene.envTexels;
    d.env.pdf = scene.envPdf;
    d.env.cdf = scene.envCdf;
    d.env.topPdf = scene.envTopPdf;
    d.env.topCdf = scene.envTopCdf;
    d.env.W = scene.envW;
    d.env.H = scene.envH;
    d.env.enabled = 0;
    d.env.powerCoeff = 0.0f;
    d.env.rotation = 0.0f;
    return d;
}
DevScene gfx_ctx::devScene(const GfxFrameParams* p) const {
    DevScene d = devScene();
    // plp.s->envLightTexture && plp.f->enableEnvLight; a map that is black everywhere has nothing to sample (its importance map has
    // integral 0, so every density would be 0) and is treated as no environment light (DESIGN.md, "Environment maps with black rows")
    d.env.enabled = scene.envW != 0 && scene.envIntegral > 0.0f && p->enableEnvLight ? 1u : 0u;
    d.env.powerCoeff = p->envLightPowerCoeff;
    d.env.rotation = p->envLightRotation;
    return d;
}
DevFrame gfx_ctx::devFrame() const {
    DevFrame d;
    d.W = frame.W;
    d.H = frame.H;
    for (int i = 0; i < 2; ++i) {
        d.gb0[i] = frame.gb0[i];
        d.gb1[i] = frame.gb1[i];
        d.gb2[i] = frame.gb2[i];
        d.gb3[i] = frame.gb3[i];
        d.reservoir[i] = frame.reservoir[i];
        d.reservoirInfo[i] = frame.reservoirInfo[i];
    }
    d.rng = frame.rng;
    d.beauty = frame.beauty;
    d.albedo = frame.albedo;
    d.normal = frame.normal;
    d.neighborDeltas = frame.neighborDeltas;
    d.stats = frame.stats;
    d.rayQueue = frame.rayQueue;
    d.rayPixel = frame.rayPixel;
    d.rayCounters = frame.rayCounters;
    d.visibility = frame.visibility;
    return d;
}

#define CHECK_CTX(ctx) do { if (!(ctx)) return GFX_ERR_INVALID_ARGUMENT; } while (0)

extern "C" {

int gfx_ctx_create(int device, gfx_ctx** out) {
    if (!out)
        return GFX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return GFX_ERR_NO_DEVICE; // no CPU fallback by design
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess)
        return GFX_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0)
        return GFX_ERR_NO_DEVICE; // the fat binary only carries sm_90a code, which loads on compute capability 9.0 alone
    if (cudaSetDevice(device) != cudaSuccess)
        return GFX_ERR_CUDA;
    gfx_ctx* ctx = new gfx_ctx();
    ctx->device = device;
    if (cudaMalloc(&ctx->bvh.overflowFlag, 4) != cudaSuccess) {
        delete ctx;
        return GFX_ERR_OUT_OF_MEMORY;
    }
    cudaMemset(ctx->bvh.overflowFlag, 0, 4);
    if (cudaMalloc(&ctx->traceFetchCounter, 4) != cudaSuccess) {
        delete ctx;
        return GFX_ERR_OUT_OF_MEMORY;
    }
    *out = ctx;
    return GFX_OK;
}

void gfx_ctx_destroy(gfx_ctx* ctx) {
    if (!ctx)
        return;
    gfx_peer_close(ctx);
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ctx->frame.release();
    ctx->bvh.release();
    cudaFree(ctx->bvh.scratch);
    cudaFree(ctx->bvh.overflowFlag);
    cudaFree(ctx->traceFetchCounter);
    ctx->scene.release();
    delete ctx;
}

const char* gfx_last_error_string(gfx_ctx* ctx) { return ctx ? ctx->lastError.c_str() : "null context"; }

int gfx_synchronize(gfx_ctx* ctx, void* stream) {
    CHECK_CTX(ctx);
    GFX_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    uint32_t flag = 0;
    GFX_CUDA(ctx, cudaMemcpy(&flag, ctx->bvh.overflowFlag, 4, cudaMemcpyDeviceToHost));
    if (flag) {
        // reported once: the next traces on this context start clean
        GFX_CUDA(ctx, cudaMemset(ctx->bvh.overflowFlag, 0, 4));
        ctx->setError("traversal stack overflow (kStackSize too small for this BVH)");
        return GFX_ERR_CUDA;
    }
    return GFX_OK;
}

uint64_t gfx_kernel_launch_count(gfx_ctx* ctx) { return ctx ? ctx->launches : 0; }

int gfx_scene_upload(gfx_ctx* ctx, const GfxSceneDesc* sd) {
    CHECK_CTX(ctx);
    if (!sd || (sd->numMeshes && !sd->meshes) || (sd->numInstances && !sd->instances))
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    SceneState &S = ctx->scene;
    S.release();
    ctx->bvh.release();

    // meshes: concatenate vertex / triangle tables
    std::vector<DevMesh> meshes(sd->numMeshes);
    size_t numVerts = 0, numTris = 0;
    for (uint32_t i = 0; i < sd->numMeshes; ++i) {
        const GfxMeshDesc &m = sd->meshes[i];
        if (m.materialSlot >= sd->numMaterials) {
            ctx->setError("gfx_scene_upload: material slot out of range");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        meshes[i].vertexBase = (uint32_t)numVerts;
        meshes[i].triBase = (uint32_t)numTris;
        meshes[i].numTriangles = m.numTriangles;
        meshes[i].materialSlot = m.materialSlot;
        meshes[i].primIntegral = 0.0f;
        numVerts += m.numVertices;
        numTris += m.numTriangles;
    }
    std::vector<float4> verts(3 * numVerts);
    std::vector<uint4> tris(numTris);
    for (uint32_t i = 0; i < sd->numMeshes; ++i) {
        const GfxMeshDesc &m = sd->meshes[i];
        for (uint32_t v = 0; v < m.numVertices; ++v) {
            float4* o = &verts[3 * (size_t)(meshes[i].vertexBase + v)];
            o[0] = make_float4(m.positions[3 * v], m.positions[3 * v + 1], m.positions[3 * v + 2], m.texcoords[2 * v]);
            o[1] = make_float4(m.normals[3 * v], m.normals[3 * v + 1], m.normals[3 * v + 2], m.texcoords[2 * v + 1]);
            o[2] = make_float4(m.tangents[3 * v], m.tangents[3 * v + 1], m.tangents[3 * v + 2], 0.0f);
        }
        for (uint32_t t = 0; t < m.numTriangles; ++t) {
            const uint32_t* idx = m.triangles + 3 * (size_t)t;
            if (idx[0] >= m.numVertices || idx[1] >= m.numVertices || idx[2] >= m.numVertices) {
                ctx->setError("gfx_scene_upload: vertex index out of range");
                return GFX_ERR_INVALID_ARGUMENT;
            }
            tris[meshes[i].triBase + t] = make_uint4(idx[0], idx[1], idx[2], 0u);
        }
    }
    // instances + flattened geometry table (instance order, then mesh slot order)
    std::vector<DevInstance> insts(sd->numInstances);
    std::vector<uint2> geomToInstMesh;
    std::vector<uint32_t> geomTriOffsets;
    uint32_t flatTris = 0;
    for (uint32_t i = 0; i < sd->numInstances; ++i) {
        const GfxInstanceDesc &in = sd->instances[i];
        if ((size_t)in.firstMeshSlot + in.numMeshSlots > sd->numInstanceMeshSlots) {
            ctx->setError("gfx_scene_upload: instance mesh-slot range out of bounds");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        DevInstance &d = insts[i];
        memset(&d, 0, sizeof(d));
        memcpy(d.transform, in.transform, 48);
        memcpy(d.curToPrevTransform, in.curToPrevTransform, 48);
        memcpy(d.normalMatrix, in.normalMatrix, 36);
        d.uniformScale = in.uniformScale;
        d.firstMeshSlot = in.firstMeshSlot;
        d.numMeshSlots = in.numMeshSlots;
        d.geomBase = (uint32_t)geomToInstMesh.size();
        for (uint32_t k = 0; k < in.numMeshSlots; ++k) {
            const uint32_t slot = sd->instanceMeshSlots[in.firstMeshSlot + k];
            if (slot >= sd->numMeshes) {
                ctx->setError("gfx_scene_upload: mesh slot out of range");
                return GFX_ERR_INVALID_ARGUMENT;
            }
            geomToInstMesh.push_back(make_uint2(i, slot));
            geomTriOffsets.push_back(flatTris);
            flatTris += meshes[slot].numTriangles;
        }
    }
    geomTriOffsets.push_back(flatTris);
    // light-triangle table layout: every triangle of every geometry whose material is an emitter
    std::vector<uint32_t> lightTriBase(geomToInstMesh.size(), 0xFFFFFFFFu), emissiveGeoms;
    uint32_t numLightTris = 0;
    for (size_t g = 0; g < geomToInstMesh.size(); ++g) {
        const DevMesh &m = meshes[geomToInstMesh[g].y];
        if (sd->materials[m.materialSlot].hasEmittance) {
            lightTriBase[g] = numLightTris;
            emissiveGeoms.push_back((uint32_t)g);
            numLightTris += m.numTriangles;
        }
    }

    auto upload = [&](auto** dst, const void* src, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc((void**)dst, bytes ? bytes : 16);
        if (e != cudaSuccess) return e;
        return bytes ? cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice) : cudaSuccess;
    };
    GFX_CUDA(ctx, upload(&S.vertices, verts.data(), verts.size() * 16));
    GFX_CUDA(ctx, upload(&S.triangles, tris.data(), tris.size() * 16));
    GFX_CUDA(ctx, upload(&S.meshes, meshes.data(), meshes.size() * sizeof(DevMesh)));
    GFX_CUDA(ctx, upload(&S.materials, sd->materials, sd->numMaterials * sizeof(GfxMaterialDesc)));
    GFX_CUDA(ctx, upload(&S.instances, insts.data(), insts.size() * sizeof(DevInstance)));
    GFX_CUDA(ctx, upload(&S.instanceMeshSlots, sd->instanceMeshSlots, sd->numInstanceMeshSlots * 4));
    GFX_CUDA(ctx, upload(&S.geomToInstMesh, geomToInstMesh.data(), geomToInstMesh.size() * 8));
    GFX_CUDA(ctx, upload(&S.geomTriOffsets, geomTriOffsets.data(), geomTriOffsets.size() * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.primWeights, (numTris ? numTris : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.primCdf, (numTris ? numTris : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.geomWeights, (sd->numInstanceMeshSlots ? sd->numInstanceMeshSlots : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.geomCdf, (sd->numInstanceMeshSlots ? sd->numInstanceMeshSlots : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.instWeights, (sd->numInstances ? sd->numInstances : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.instCdf, (sd->numInstances ? sd->numInstances : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.instIntegral, 16));
    GFX_CUDA(ctx, cudaMalloc(&S.primProb, (numTris ? numTris : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.geomProb, (sd->numInstanceMeshSlots ? sd->numInstanceMeshSlots : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.instProb, (sd->numInstances ? sd->numInstances : 4) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.lightTris, (size_t)(numLightTris ? numLightTris : 1) * 16 * kLightTriStride));
    GFX_CUDA(ctx, upload(&S.lightTriBase, lightTriBase.data(), lightTriBase.size() * 4));
    GFX_CUDA(ctx, upload(&S.emissiveGeoms, emissiveGeoms.data(), emissiveGeoms.size() * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.instGuide, (kInstGuideSize + 1) * 4));
    GFX_CUDA(ctx, cudaMemset(S.instGuide, 0, (kInstGuideSize + 1) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.primGuide, (size_t)(sd->numMeshes ? sd->numMeshes : 1) * (kPrimGuideSize + 1) * 4));
    // flattened light pick: every reachable (instance, geometry, primitive) position is one piece at most
    S.pickCapacity = numLightTris + sd->numInstanceMeshSlots + sd->numInstances + 64;
    GFX_CUDA(ctx, cudaMalloc(&S.pickGuide, (size_t)kPickGuideSize * 32));
    GFX_CUDA(ctx, cudaMemset(S.pickGuide, 0xC0, (size_t)kPickGuideSize * 32)); // kPickPure | kPickNone until the first build
    GFX_CUDA(ctx, cudaMalloc(&S.normalMats, (size_t)(sd->numInstances ? sd->numInstances : 1) * kNormalMatStride * 16));
    GFX_CUDA(ctx, cudaMalloc(&S.pickPieces, ((size_t)S.pickCapacity + 2) * 8));
    GFX_CUDA(ctx, cudaMemset(S.pickPieces, 0xFF, ((size_t)S.pickCapacity + 2) * 8));
    GFX_CUDA(ctx, cudaMalloc(&S.pickKeyAt, ((size_t)kPickGuideSize + 1) * 4));
    GFX_CUDA(ctx, cudaMalloc(&S.pickBoundaries, (size_t)S.pickCapacity * 8));
    GFX_CUDA(ctx, cudaMalloc(&S.pickCounters, 16));
    for (int i = 0; i < 2; ++i) {
        GFX_CUDA(ctx, cudaMalloc(&S.pickQueue[i], (size_t)S.pickCapacity * 16));
        GFX_CUDA(ctx, cudaMalloc(&S.pickSortKeys[i], (size_t)S.pickCapacity * 4));
        GFX_CUDA(ctx, cudaMalloc(&S.pickSortVals[i], (size_t)S.pickCapacity * 4));
    }
    S.pickSortTempBytes = lightPickSortTempBytes(S.pickCapacity);
    GFX_CUDA(ctx, cudaMalloc(&S.pickSortTemp, S.pickSortTempBytes));
    GFX_CUDA(ctx, cudaMallocHost(&S.pickFlagsHost, 4));
    *S.pickFlagsHost = 0;
    GFX_CUDA(ctx, cudaEventCreateWithFlags(&S.pickFlagsEvent, cudaEventDisableTiming));
    S.numEmissiveGeoms = (uint32_t)emissiveGeoms.size();
    S.numLightTris = numLightTris;
    GFX_CUDA(ctx, cudaMemset(S.instIntegral, 0, 16));
    S.numMeshes = sd->numMeshes;
    S.numMaterials = sd->numMaterials;
    S.numInstances = sd->numInstances;
    S.numInstanceMeshSlots = sd->numInstanceMeshSlots;
    S.numGeoms = (uint32_t)geomToInstMesh.size();
    S.numFlatTris = flatTris;
    S.numMeshTris = (uint32_t)numTris;
    S.numVertices = (uint32_t)numVerts;
    S.hostMeshes = meshes;
    S.hostInstances = insts;
    const int envRc = uploadEnvLight(ctx, sd->envTexels, sd->envWidth, sd->envHeight);
    if (envRc != GFX_OK)
        return envRc;
    const int texRc = uploadTextures(ctx, sd);
    if (texRc != GFX_OK)
        return texRc;
    S.uploaded = true;
    return GFX_OK;
}

int gfx_scene_update_instances(gfx_ctx* ctx, void* stream, const GfxInstanceDesc* instances, uint32_t numInstances) {
    CHECK_CTX(ctx);
    SceneState &S = ctx->scene;
    if (!S.uploaded)
        return GFX_ERR_NOT_READY;
    if (!instances || numInstances != S.numInstances)
        return GFX_ERR_INVALID_ARGUMENT;
    bool moved = false; // light records, importances and the flattened pick follow transform / normal matrix / scale only
    for (uint32_t i = 0; i < numInstances; ++i) {
        DevInstance &d = S.hostInstances[i];
        moved = moved || memcmp(d.transform, instances[i].transform, 48) != 0 || memcmp(d.normalMatrix, instances[i].normalMatrix, 36) != 0 ||
                memcmp(&d.uniformScale, &instances[i].uniformScale, 4) != 0;
        memcpy(d.transform, instances[i].transform, 48);
        memcpy(d.curToPrevTransform, instances[i].curToPrevTransform, 48);
        memcpy(d.normalMatrix, instances[i].normalMatrix, 36);
        d.uniformScale = instances[i].uniformScale;
    }
    if (moved)
        S.lightTrisDirty = true;
    // geomIntegral lives on the device copy only: patch the transform part of every record with ONE strided copy
    // out of pinned memory (double-buffered so that the host may run a frame ahead of the device)
    const size_t bytes = (size_t)numInstances * sizeof(DevInstance);
    if (!S.pinnedInstances[0]) {
        for (int i = 0; i < 2; ++i) {
            GFX_CUDA(ctx, cudaMallocHost(&S.pinnedInstances[i], bytes));
            GFX_CUDA(ctx, cudaEventCreateWithFlags(&S.pinnedInstancesFree[i], cudaEventDisableTiming));
        }
    }
    const uint32_t slot = S.pinnedInstancesNext++ & 1u;
    GFX_CUDA(ctx, cudaEventSynchronize(S.pinnedInstancesFree[slot]));
    memcpy(S.pinnedInstances[slot], S.hostInstances.data(), bytes);
    GFX_CUDA(ctx, cudaMemcpy2DAsync(S.instances, sizeof(DevInstance), S.pinnedInstances[slot], sizeof(DevInstance),
                                    offsetof(DevInstance, firstMeshSlot), numInstances, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    GFX_CUDA(ctx, cudaEventRecord(S.pinnedInstancesFree[slot], (cudaStream_t)stream));
    return GFX_OK;
}

int gfx_bvh_build(gfx_ctx* ctx, void* stream, uint32_t flags) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded) {
        ctx->setError("gfx_bvh_build: no scene uploaded");
        return GFX_ERR_NOT_READY;
    }
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    // an overflow reported against the previous tree says nothing about this one
    GFX_CUDA(ctx, cudaMemsetAsync(ctx->bvh.overflowFlag, 0, 4, (cudaStream_t)stream));
    int rc = buildBvh(ctx, (cudaStream_t)stream, flags);
    if (rc == GFX_OK)
        rc = finishBvh(ctx, (cudaStream_t)stream);
    if (rc == GFX_OK)
        ctx->bvh.ready = true;
    return rc;
}

int gfx_bvh_info(gfx_ctx* ctx, GfxBvhInfo* info) {
    CHECK_CTX(ctx);
    if (!info)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->bvh.ready)
        return GFX_ERR_NOT_READY;
    info->numNodes = ctx->bvh.numNodes;
    info->numPrimRefs = ctx->bvh.numPrimRefs;
    info->numTriangles = ctx->bvh.numTris;
    info->numGeoms = ctx->scene.numGeoms;
    for (int i = 0; i < 3; ++i) {
        info->sceneMin[i] = ctx->bvh.sceneMin[i];
        info->sceneMax[i] = ctx->bvh.sceneMax[i];
    }
    return GFX_OK;
}

int gfx_bvh_export(gfx_ctx* ctx, GfxBvhNode8* nodes, uint32_t* primRefs, GfxTriangleStorage* tris) {
    CHECK_CTX(ctx);
    if (!ctx->bvh.ready)
        return GFX_ERR_NOT_READY;
    static_assert(sizeof(GfxBvhNode8) == 80 && sizeof(GfxTriangleStorage) == 48 && sizeof(GfxHitObject) == 32, "reference layouts");
    if (nodes) GFX_CUDA(ctx, cudaMemcpy(nodes, ctx->bvh.nodes, (size_t)ctx->bvh.numNodes * 80, cudaMemcpyDeviceToHost));
    if (primRefs) GFX_CUDA(ctx, cudaMemcpy(primRefs, ctx->bvh.primRefs, (size_t)ctx->bvh.numPrimRefs * 4, cudaMemcpyDeviceToHost));
    if (tris) GFX_CUDA(ctx, cudaMemcpy(tris, ctx->bvh.tris, (size_t)ctx->bvh.numTris * 48, cudaMemcpyDeviceToHost));
    return GFX_OK;
}

int gfx_bvh_import(gfx_ctx* ctx, const GfxBvhNode8* nodes, uint32_t numNodes, const uint32_t* primRefs,
                   uint32_t numPrimRefs, const GfxTriangleStorage* tris, uint32_t numTris) {
    CHECK_CTX(ctx);
    if (!nodes || !primRefs || !tris)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    BvhState &B = ctx->bvh;
    B.release();
    GFX_CUDA(ctx, cudaMemset(B.overflowFlag, 0, 4));
    GFX_CUDA(ctx, cudaMalloc(&B.nodes, (size_t)max(numNodes, 1u) * 80));
    GFX_CUDA(ctx, cudaMalloc(&B.primRefs, (size_t)max(numPrimRefs, 1u) * 4));
    GFX_CUDA(ctx, cudaMalloc(&B.tris, (size_t)max(numTris, 1u) * 48));
    GFX_CUDA(ctx, cudaMemcpy(B.nodes, nodes, (size_t)numNodes * 80, cudaMemcpyHostToDevice));
    GFX_CUDA(ctx, cudaMemcpy(B.primRefs, primRefs, (size_t)numPrimRefs * 4, cudaMemcpyHostToDevice));
    GFX_CUDA(ctx, cudaMemcpy(B.tris, tris, (size_t)numTris * 48, cudaMemcpyHostToDevice));
    B.numNodes = numNodes;
    B.numPrimRefs = numPrimRefs;
    B.numTris = numTris;
    if (int rc = finishBvh(ctx, nullptr))
        return rc;
    GFX_CUDA(ctx, cudaStreamSynchronize(nullptr));
    B.ready = true;
    return GFX_OK;
}

int gfx_trace_device(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays, GfxHitObject* hits, int mode) {
    CHECK_CTX(ctx);
    if (!ctx->bvh.ready) {
        ctx->setError("gfx_trace: BVH not built");
        return GFX_ERR_NOT_READY;
    }
    if ((!rays || !hits) && numRays)
        return GFX_ERR_INVALID_ARGUMENT;
    return traceRays(ctx, (cudaStream_t)stream, rays, numRays, hits, mode);
}

int gfx_trace_debug(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays, GfxHitObject* hits, int mode, int kernel) {
    CHECK_CTX(ctx);
    if (!ctx->bvh.ready) {
        ctx->setError("gfx_trace_debug: BVH not built");
        return GFX_ERR_NOT_READY;
    }
    if ((!rays || !hits) && numRays)
        return GFX_ERR_INVALID_ARGUMENT;
    return traceRaysDebug(ctx, (cudaStream_t)stream, rays, numRays, hits, mode, kernel);
}

int gfx_trace(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays, GfxHitObject* hits, int mode) {
    CHECK_CTX(ctx);
    if (!ctx->bvh.ready) {
        ctx->setError("gfx_trace: BVH not built");
        return GFX_ERR_NOT_READY;
    }
    if (numRays == 0)
        return GFX_OK;
    if (!rays || !hits)
        return GFX_ERR_INVALID_ARGUMENT;
    GfxRay* dRays = nullptr;
    GfxHitObject* dHits = nullptr;
    GFX_CUDA(ctx, cudaMalloc(&dRays, (size_t)numRays * sizeof(GfxRay)));
    GFX_CUDA(ctx, cudaMalloc(&dHits, (size_t)numRays * sizeof(GfxHitObject)));
    GFX_CUDA(ctx, cudaMemcpyAsync(dRays, rays, (size_t)numRays * sizeof(GfxRay), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    const int rc = traceRays(ctx, (cudaStream_t)stream, dRays, numRays, dHits, mode);
    if (rc == GFX_OK) {
        GFX_CUDA(ctx, cudaMemcpyAsync(hits, dHits, (size_t)numRays * sizeof(GfxHitObject), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
        GFX_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    }
    cudaFree(dRays);
    cudaFree(dHits);
    return rc;
}

int gfx_light_dist_build(gfx_ctx* ctx, void* stream, uint32_t bufferIndex) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded)
        return GFX_ERR_NOT_READY;
    return buildLightDistributions(ctx, (cudaStream_t)stream, bufferIndex);
}

int gfx_launch_batch(gfx_ctx* ctx, void* stream, const GfxBatchOp* ops, uint32_t numOps) {
    CHECK_CTX(ctx);
    if (!ops && numOps)
        return GFX_ERR_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < numOps; ++i) {
        const GfxBatchOp &o = ops[i];
        int rc = GFX_ERR_INVALID_ARGUMENT;
        switch (o.op) {
        case GFX_OP_LIGHT_DIST: rc = gfx_light_dist_build(ctx, stream, o.a); break;
        case GFX_OP_GBUFFER: rc = gfx_gbuffer_launch(ctx, stream, &o.params); break;
        case GFX_OP_RESTIR: rc = gfx_restir_launch(ctx, stream, &o.params, (int)o.a); break;
        case GFX_OP_PEER_PUSH_ROWS: rc = gfx_peer_push_rows(ctx, stream, o.a, (int)o.b, o.c, o.d, o.e); break;
        case GFX_OP_PEER_SIGNAL: rc = gfx_peer_signal(ctx, stream, o.a, o.b, o.c); break;
        case GFX_OP_PEER_WAIT: rc = gfx_peer_wait(ctx, stream, o.a, o.b); break;
        default: ctx->setError("gfx_launch_batch: unknown op"); break;
        }
        if (rc != GFX_OK)
            return rc;
    }
    return GFX_OK;
}

int gfx_restir_strip_frame(gfx_ctx* ctx, void* stream, GfxFrameParams* p, GfxStripFrame* st) {
    CHECK_CTX(ctx);
    if (!p || !st || st->y1 <= st->y0 || st->y1 > ctx->frame.H || st->world == 0 || st->rank >= st->world)
        return GFX_ERR_INVALID_ARGUMENT;
    const uint32_t H = ctx->frame.H, f = st->frameIndex, nsp = st->numSpatialPasses;
    const bool up = st->rank > 0, down = st->rank + 1 < st->world;
    int rc = GFX_OK;
#define STRIP_CALL(expr) do { rc = (expr); if (rc != GFX_OK) return rc; } while (0)
    // seam rows of the given reservoir buffer pair: push to both neighbours, raise their flags, wait for mine (peer.cu)
    auto exchange = [&](uint32_t reservoirIndex) -> int {
        if (st->world == 1 || !st->usePeer)
            return GFX_OK;
        const uint32_t seq = ++st->peerSeq;
        const int bufs[2] = { GFX_BUF_RESERVOIR, GFX_BUF_RESERVOIR_INFO };
        for (int b : bufs) {
            if (up)
                STRIP_CALL(gfx_peer_push_rows(ctx, stream, 0, b, reservoirIndex, st->y0, st->y0 + st->halo < st->y1 ? st->y0 + st->halo : st->y1));
            if (down)
                STRIP_CALL(gfx_peer_push_rows(ctx, stream, 1, b, reservoirIndex, st->y1 > st->y0 + st->halo ? st->y1 - st->halo : st->y0, st->y1));
        }
        if (up)
            STRIP_CALL(gfx_peer_signal(ctx, stream, 0, 1, seq)); // I am the upper neighbour's lower neighbour: its flag word 1
        if (down)
            STRIP_CALL(gfx_peer_signal(ctx, stream, 1, 0, seq));
        if (up)
            STRIP_CALL(gfx_peer_wait(ctx, stream, 0, seq));
        if (down)
            STRIP_CALL(gfx_peer_wait(ctx, stream, 1, seq));
        return GFX_OK;
    };
    auto tile = [&](uint32_t lo, uint32_t hi) { p->tileOriginY = lo; p->tileRows = hi - lo; };

    STRIP_CALL(gfx_light_dist_build(ctx, stream, f % 2));
    // the launch list of restir_di_main.cpp:2321-2421 (gfxexp_b200/engine.py restir_frame_passes is the same list)
    p->frameIndex = f;
    p->bufferIndex = f % 2;
    p->useUnbiasedEstimator = st->unbiased ? 1 : 0;
    p->enableTemporalReuse = st->temporal ? 1 : 0;
    p->enableSpatialReuse = nsp > 0 ? 1 : 0;
    const bool newSequence = f == 0;
    p->resetFlowBuffer = newSequence ? 1 : 0;
    tile(st->y0 > st->halo ? st->y0 - st->halo : 0, st->y1 + st->halo < H ? st->y1 + st->halo : H);
    if (st->world == 1)
        tile(0, H);
    STRIP_CALL(gfx_gbuffer_launch(ctx, stream, p));
    const uint32_t base = (uint32_t)(((uint64_t)f * (1 + nsp)) % 2);
    p->currentReservoirIndex = base;
    tile(st->y0, st->y1);
    const int initialPass = (p->enableTemporalReuse && !newSequence)
        ? (st->unbiased ? GFX_RESTIR_INITIAL_AND_TEMPORAL_UNBIASED : GFX_RESTIR_INITIAL_AND_TEMPORAL_BIASED) : GFX_RESTIR_INITIAL_RIS;
    STRIP_CALL(gfx_restir_launch(ctx, stream, p, initialPass));
    if (nsp > 0)
        STRIP_CALL(exchange(p->currentReservoirIndex));
    uint32_t cur = base;
    for (uint32_t s = 0; s < nsp; ++s) {
        p->currentReservoirIndex = cur;
        const uint32_t k = p->numSpatialNeighbors > 1 ? p->numSpatialNeighbors : 1;
        p->spatialNeighborBaseIndex = (uint32_t)(((uint64_t)f * nsp * k + (uint64_t)s * p->numSpatialNeighbors) % 1024);
        STRIP_CALL(gfx_restir_launch(ctx, stream, p, st->unbiased ? GFX_RESTIR_SPATIAL_UNBIASED : GFX_RESTIR_SPATIAL_BIASED));
        if (s + 1 < nsp)
            STRIP_CALL(exchange((cur + 1) % 2));
        cur = (cur + 1) % 2;
    }
    p->currentReservoirIndex = cur;
    STRIP_CALL(gfx_restir_launch(ctx, stream, p, GFX_RESTIR_SHADING));
    // final reservoirs of the seam rows: next frame's temporal reuse may look across the seam
    STRIP_CALL(exchange(cur));
    tile(0, 0);
    p->tileRows = 0;
#undef STRIP_CALL
    return GFX_OK;
}

int gfx_light_pick_debug(gfx_ctx* ctx, void* stream, const float* ul, uint32_t n, uint32_t* keysFlat, uint32_t* keysChain) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded || ctx->scene.pickDirty)
        return GFX_ERR_NOT_READY;
    if (!ul || !keysFlat || !keysChain)
        return GFX_ERR_INVALID_ARGUMENT;
    return debugLightPick(ctx, (cudaStream_t)stream, ul, n, keysFlat, keysChain);
}

int gfx_env_light_debug(gfx_ctx* ctx, void* stream, int op, const float* in, uint32_t n, float* out) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded)
        return GFX_ERR_NOT_READY;
    if ((n && (!in || !out)) || op < 0 || op > 2)
        return GFX_ERR_INVALID_ARGUMENT;
    return debugEnvLight(ctx, (cudaStream_t)stream, op, in, n, out);
}

int gfx_light_sample_debug(gfx_ctx* ctx, void* stream, int op, const float* params, const float* in, uint32_t n, float* out) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded || ctx->scene.pickDirty || ctx->scene.lightTrisDirty)
        return GFX_ERR_NOT_READY;
    if (!params || (n && (!in || !out)) || op < 0 || op > 7)
        return GFX_ERR_INVALID_ARGUMENT;
    return debugLightSample(ctx, (cudaStream_t)stream, op, params, in, n, out);
}

int gfx_shading_debug(gfx_ctx* ctx, void* stream, int op, const float* material, const float* in, uint32_t n, float* out) {
    CHECK_CTX(ctx);
    if (!material || (n && (!in || !out)) || op < 0 || op > 15)
        return GFX_ERR_INVALID_ARGUMENT;
    return debugShading(ctx, (cudaStream_t)stream, op, material, in, n, out);
}

int gfx_bump_debug(gfx_ctx* ctx, void* stream, int op, uint32_t matSlot, const float* in, uint32_t n, float* out) {
    CHECK_CTX(ctx);
    if (!ctx->scene.uploaded)
        return GFX_ERR_NOT_READY;
    if ((n && (!in || !out)) || op < 0 || op > 2 || (op != 1 && matSlot >= ctx->scene.numMaterials))
        return GFX_ERR_INVALID_ARGUMENT;
    return debugBump(ctx, (cudaStream_t)stream, op, matSlot, in, n, out);
}

int gfx_light_dist_export(gfx_ctx* ctx, float* instWeights, float* instCdf, float* integral) {
    CHECK_CTX(ctx);
    const SceneState &S = ctx->scene;
    if (!S.uploaded)
        return GFX_ERR_NOT_READY;
    GFX_CUDA(ctx, cudaDeviceSynchronize());
    if (instWeights) GFX_CUDA(ctx, cudaMemcpy(instWeights, S.instWeights, (size_t)S.numInstances * 4, cudaMemcpyDeviceToHost));
    if (instCdf) GFX_CUDA(ctx, cudaMemcpy(instCdf, S.instCdf, (size_t)S.numInstances * 4, cudaMemcpyDeviceToHost));
    if (integral) GFX_CUDA(ctx, cudaMemcpy(integral, S.instIntegral, 4, cudaMemcpyDeviceToHost));
    return GFX_OK;
}

int gfx_frame_create(gfx_ctx* ctx, uint32_t W, uint32_t H) {
    CHECK_CTX(ctx);
    if (W == 0 || H == 0)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    FrameState &F = ctx->frame;
    F.release();
    const size_t n = (size_t)W * H;
    for (int i = 0; i < 2; ++i) {
        GFX_CUDA(ctx, cudaMalloc(&F.gb0[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.gb1[i], n * 8));
        GFX_CUDA(ctx, cudaMalloc(&F.gb2[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.gb3[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.reservoir[i], n * 48));
        GFX_CUDA(ctx, cudaMalloc(&F.reservoirInfo[i], n * 8));
        GFX_CUDA(ctx, cudaMemset(F.gb0[i], 0xFF, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.gb1[i], 0, n * 8));
        GFX_CUDA(ctx, cudaMemset(F.gb2[i], 0, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.gb3[i], 0, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.reservoir[i], 0, n * 48));
        GFX_CUDA(ctx, cudaMemset(F.reservoirInfo[i], 0, n * 8));
        GFX_CUDA(ctx, cudaMalloc(&F.svgfLighting[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.svgfMoments[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.svgfFinal[i], n * 16));
        GFX_CUDA(ctx, cudaMalloc(&F.svgfDepth[i], n * 4));
        GFX_CUDA(ctx, cudaMemset(F.svgfLighting[i], 0, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.svgfMoments[i], 0, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.svgfFinal[i], 0, n * 16));
        GFX_CUDA(ctx, cudaMemset(F.svgfDepth[i], 0, n * 4));
    }
    GFX_CUDA(ctx, cudaMalloc(&F.svgfPrevLighting, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.svgfPrevLighting, 0, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.svgfNormal, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.svgfNormal, 0, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.svgfAlbedo, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.svgfAlbedo, 0, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.svgfPrevScreenPos, n * 8));
    GFX_CUDA(ctx, cudaMemset(F.svgfPrevScreenPos, 0, n * 8));
    GFX_CUDA(ctx, cudaMalloc(&F.rng, n * 8));
    GFX_CUDA(ctx, cudaMalloc(&F.beauty, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.albedo, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.normal, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.neighborDeltas, 1024 * 8));
    GFX_CUDA(ctx, cudaMalloc(&F.stats, 4 * 8));
    GFX_CUDA(ctx, cudaMalloc(&F.rayQueue, n * 32));
    GFX_CUDA(ctx, cudaMalloc(&F.rayPixel, n * 4));
    GFX_CUDA(ctx, cudaMalloc(&F.rayCounters, 16));
    GFX_CUDA(ctx, cudaMemset(F.rayCounters, 0, 16));
    GFX_CUDA(ctx, cudaMalloc(&F.visibility, n));
    GFX_CUDA(ctx, cudaMemset(F.visibility, 0, n));
    GFX_CUDA(ctx, cudaMemset(F.stats, 0, 4 * 8));
    GFX_CUDA(ctx, cudaMemset(F.rng, 0, n * 8));
    GFX_CUDA(ctx, cudaMemset(F.beauty, 0, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.albedo, 0, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.normal, 0, n * 16));
    GFX_CUDA(ctx, cudaMemset(F.neighborDeltas, 0, 1024 * 8));
    F.W = W;
    F.H = H;
    F.created = true;
    return GFX_OK;
}

int gfx_rng_seed(gfx_ctx* ctx, uint64_t seed) {
    CHECK_CTX(ctx);
    FrameState &F = ctx->frame;
    if (!F.created)
        return GFX_ERR_NOT_READY;
    // restir_di_main.cpp:1309-1321: one std::mt19937_64 draw per pixel, row-major
    std::vector<unsigned long long> states((size_t)F.W * F.H);
    std::mt19937_64 rngSeed(seed);
    for (size_t i = 0; i < states.size(); ++i)
        states[i] = rngSeed();
    GFX_CUDA(ctx, cudaMemcpy(F.rng, states.data(), states.size() * 8, cudaMemcpyHostToDevice));
    return GFX_OK;
}

int gfx_restir_setup_neighbor_table(gfx_ctx* ctx) {
    CHECK_CTX(ctx);
    FrameState &F = ctx->frame;
    if (!F.created)
        return GFX_ERR_NOT_READY;
    // restir_di_main.cpp:1489-1542: Halton(2,3) mapped through the concentric disk map
    auto halton = [](uint32_t base, uint32_t idx) {
        const float recBase = 1.0f / base;
        float ret = 0.0f;
        float scale = 1.0f;
        while (idx) {
            scale *= recBase;
            ret += (idx % base) * scale;
            idx /= base;
        }
        return ret;
    };
    std::vector<float2> deltas(1024);
    const float pi = 3.14159265358979323846f;
    for (uint32_t i = 0; i < 1024; ++i) {
        const float u0 = halton(2, i), u1 = halton(3, i);
        const float sx = 2 * u0 - 1;
        const float sy = 2 * u1 - 1;
        float2 d = make_float2(0.0f, 0.0f);
        if (!(sx == 0 && sy == 0)) {
            float r, theta;
            if (sx >= -sy) {
                if (sx > sy) { r = sx; theta = sy / sx; }
                else { r = sy; theta = 2 - sx / sy; }
            }
            else {
                if (sx > sy) { r = -sy; theta = 6 + sx / sy; }
                else { r = -sx; theta = 4 + sy / sx; }
            }
            theta *= pi / 4;
            d.x = (float)(r * std::cos((double)theta));
            d.y = (float)(r * std::sin((double)theta));
        }
        deltas[i] = d;
    }
    GFX_CUDA(ctx, cudaMemcpy(F.neighborDeltas, deltas.data(), 1024 * 8, cudaMemcpyHostToDevice));
    return GFX_OK;
}

int gfx_stats_read(gfx_ctx* ctx, void* stream, uint64_t* out4, int reset) {
    CHECK_CTX(ctx);
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    if (!out4)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaMemcpyAsync(out4, ctx->frame.stats, 32, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GFX_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    if (reset)
        GFX_CUDA(ctx, cudaMemsetAsync(ctx->frame.stats, 0, 32, (cudaStream_t)stream));
    return GFX_OK;
}

static void* bufferPtr(gfx_ctx* ctx, int id, uint32_t index, size_t* bytes) {
    FrameState &F = ctx->frame;
    const size_t n = (size_t)F.W * F.H;
    const uint32_t i = index & 1;
    void* p = nullptr;
    size_t b = 0;
    switch (id) {
    case GFX_BUF_GBUFFER0: p = F.gb0[i]; b = n * 16; break;
    case GFX_BUF_GBUFFER1: p = F.gb1[i]; b = n * 8; break;
    case GFX_BUF_GBUFFER2: p = F.gb2[i]; b = n * 16; break;
    case GFX_BUF_GBUFFER3: p = F.gb3[i]; b = n * 16; break;
    case GFX_BUF_RNG: p = F.rng; b = n * 8; break;
    case GFX_BUF_RESERVOIR: p = F.reservoir[i]; b = n * 48; break;
    case GFX_BUF_RESERVOIR_INFO: p = F.reservoirInfo[i]; b = n * 8; break;
    case GFX_BUF_BEAUTY_ACCUM: p = F.beauty; b = n * 16; break;
    case GFX_BUF_PRESENT_RGBA8: p = F.presentRgba8; b = F.presentRgba8 ? n * 4 : 0; break;
    case GFX_BUF_ALBEDO_ACCUM: p = F.albedo; b = n * 16; break;
    case GFX_BUF_NORMAL_ACCUM: p = F.normal; b = n * 16; break;
    case GFX_BUF_SVGF_LIGHTING_VARIANCE: p = F.svgfLighting[i]; b = n * 16; break;
    case GFX_BUF_SVGF_FINAL: p = F.svgfFinal[i]; b = n * 16; break;
    case GFX_BUF_SVGF_MOMENTS: p = F.svgfMoments[i]; b = n * 16; break;
    case GFX_BUF_SVGF_PREV_LIGHTING: p = F.svgfPrevLighting; b = n * 16; break;
    case GFX_BUF_SVGF_ALBEDO: p = F.svgfAlbedo; b = n * 16; break;
    case GFX_BUF_SVGF_DEPTH: p = F.svgfDepth[i]; b = n * 4; break;
    case GFX_BUF_SVGF_DEBUG_VISUALIZE: p = F.svgfDebugVisualize; b = F.svgfDebugVisualize ? n * 16 : 0; break;
    default: break;
    }
    if (id >= GFX_BUF_NRC_INFERENCE_QUERY && id <= GFX_BUF_NRC_STATE) {
        if (ensureNrcFrame(ctx) != GFX_OK) {
            if (bytes) *bytes = 0;
            return nullptr;
        }
        const FrameState::Nrc &N = F.nrc;
        switch (id) {
        case GFX_BUF_NRC_INFERENCE_QUERY: p = N.inferenceQuery; b = (size_t)N.queryCapacity * 56; break;
        case GFX_BUF_NRC_TERMINAL_INFO: p = N.terminalInfo; b = n * 16; break;
        case GFX_BUF_NRC_INFERRED_RADIANCE: p = N.inferredRadiance; b = (size_t)N.queryCapacity * 12; break;
        case GFX_BUF_NRC_FRAME_CONTRIBUTION: p = N.frameContribution; b = n * 12; break;
        case GFX_BUF_NRC_TRAIN_QUERY: p = N.trainQuery[i]; b = (size_t)131072 * 56; break;
        case GFX_BUF_NRC_TRAIN_TARGET: p = N.trainTarget[i]; b = (size_t)131072 * 12; break;
        case GFX_BUF_NRC_TRAIN_VERTEX_INFO: p = N.trainVertexInfo; b = (size_t)131072 * 16; break;
        case GFX_BUF_NRC_TRAIN_SUFFIX_TERMINAL: p = N.suffixTerminal; b = (size_t)N.numSuffixes * 4; break;
        case GFX_BUF_NRC_STATE: p = N.state; b = 32 * 4; break;
        default: break;
        }
    }
    if (id >= GFX_BUF_SAMPLE_VISIBILITY && id <= GFX_BUF_PRESAMPLE_RNG) {
        if (ensureRearch(ctx, 0) != GFX_OK) {
            if (bytes) *bytes = 0;
            return nullptr;
        }
        const FrameState::Rearch &R = F.rearch;
        switch (id) {
        case GFX_BUF_SAMPLE_VISIBILITY: p = R.sampleVis[i]; b = n * 4; break;
        case GFX_BUF_PRESAMPLED_LIGHTS: p = R.preSampledLights; b = (size_t)131072 * 48; break;
        case GFX_BUF_PRESAMPLE_RNG: p = R.rngs; b = (size_t)131072 * 8; break;
        default: break;
        }
    }
    if (id >= GFX_BUF_REGIR_SLOTS && id <= GFX_BUF_REGIR_NUM_ACTIVE_CELLS && F.regir.created) {
        const FrameState::Regir &R = F.regir;
        switch (id) {
        case GFX_BUF_REGIR_SLOTS: p = R.slots[i]; b = (size_t)R.numSlots * 64; break;
        case GFX_BUF_REGIR_SLOT_RNG: p = R.slotRngs; b = (size_t)R.numSlots * 8; break;
        case GFX_BUF_REGIR_CELL_ACCESSES: p = R.perCellNumAccesses; b = (size_t)R.numCells * 4; break;
        case GFX_BUF_REGIR_LAST_ACCESS: p = R.lastAccessFrameIndices; b = (size_t)R.numCells * 4; break;
        case GFX_BUF_REGIR_NUM_ACTIVE_CELLS: p = R.numActiveCells; b = 8; break;
        default: break;
        }
    }
    if (bytes) *bytes = b;
    return p;
}

void* gfx_buffer_device_ptr(gfx_ctx* ctx, int bufferId, uint32_t index, size_t* bytes) {
    if (!ctx || !ctx->frame.created) {
        if (bytes) *bytes = 0;
        return nullptr;
    }
    return bufferPtr(ctx, bufferId, index, bytes);
}

int gfx_buffer_download(gfx_ctx* ctx, void* stream, int bufferId, uint32_t index, void* host, size_t bytes) {
    CHECK_CTX(ctx);
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    size_t have = 0;
    void* p = bufferPtr(ctx, bufferId, index, &have);
    if (!p || !host || bytes > have)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaMemcpyAsync(host, p, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GFX_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return GFX_OK;
}

int gfx_buffer_upload(gfx_ctx* ctx, void* stream, int bufferId, uint32_t index, const void* host, size_t bytes) {
    CHECK_CTX(ctx);
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    size_t have = 0;
    void* p = bufferPtr(ctx, bufferId, index, &have);
    if (!p || !host || bytes > have)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaMemcpyAsync(p, host, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    GFX_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)stream));
    return GFX_OK;
}

int gfx_gbuffer_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->bvh.ready || !ctx->frame.created) {
        ctx->setError("gfx_gbuffer_launch: BVH or frame buffers missing");
        return GFX_ERR_NOT_READY;
    }
    return launchGBuffer(ctx, (cudaStream_t)stream, params);
}

int gfx_restir_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int pass) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->bvh.ready || !ctx->frame.created) {
        ctx->setError("gfx_restir_launch: BVH or frame buffers missing");
        return GFX_ERR_NOT_READY;
    }
    if (pass >= GFX_RESTIR_PRESAMPLE_LIGHTS)
        return launchReSTIRRearch(ctx, (cudaStream_t)stream, params, pass);
    return launchReSTIR(ctx, (cudaStream_t)stream, params, pass);
}

int gfx_present_launch(gfx_ctx* ctx, void* stream, const GfxPresentParams* params) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    return launchPresent(ctx, (cudaStream_t)stream, params);
}

int gfx_svgf_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int pass, uint32_t stage) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchSVGF(ctx, (cudaStream_t)stream, params, pass, stage);
}

int gfx_svgf_debug_visualize(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int view, float motionVectorOffset,
                             float motionVectorScale, uint32_t numFilteringStages) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchSVGFDebugVisualize(ctx, (cudaStream_t)stream, params, view, motionVectorOffset, motionVectorScale,
                                    numFilteringStages);
}

int gfx_pathtrace_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int variant) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created || !ctx->bvh.ready)
        return GFX_ERR_NOT_READY;
    return launchPathTrace(ctx, (cudaStream_t)stream, params, variant);
}

int gfx_timing_enable(gfx_ctx* ctx, int enable) {
    CHECK_CTX(ctx);
    ctx->timer.enabled = enable != 0;
    return GFX_OK;
}

int gfx_timing_read(gfx_ctx* ctx, GfxKernelTiming* out, uint32_t capacity, uint32_t* numWritten) {
    CHECK_CTX(ctx);
    if (!out || !numWritten)
        return GFX_ERR_INVALID_ARGUMENT;
    GFX_CUDA(ctx, cudaDeviceSynchronize());
    uint32_t n = 0;
    for (const KernelTimer::Rec &r : ctx->timer.recs) {
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, r.start, r.stop);
        uint32_t k = 0;
        while (k < n && strncmp(out[k].label, r.label, sizeof(out[k].label) - 1) != 0)
            ++k;
        if (k == n) {
            if (n == capacity)
                continue;
            memset(&out[n], 0, sizeof(out[n]));
            strncpy(out[n].label, r.label, sizeof(out[n].label) - 1);
            ++n;
        }
        out[k].totalMs += ms;
        out[k].launches += 1;
        ctx->timer.pool.push_back(r.start);
        ctx->timer.pool.push_back(r.stop);
    }
    ctx->timer.recs.clear();
    *numWritten = n;
    return GFX_OK;
}

int gfx_regir_build_cells(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t frameIndex, int useTemporalReuse) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchRegirBuildCells(ctx, (cudaStream_t)stream, params, frameIndex, useTemporalReuse);
}

int gfx_regir_update_access(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t frameIndex) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchRegirUpdateAccess(ctx, (cudaStream_t)stream, params, frameIndex);
}

int gfx_nrc_preprocess(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t offsetToSelectUnbiasedTile,
                       uint32_t offsetToSelectTrainingPath, int isNewSequence) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchNrcPreprocess(ctx, (cudaStream_t)stream, params, offsetToSelectUnbiasedTile, offsetToSelectTrainingPath, isNewSequence);
}

static int nrcPass(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int pass) {
    CHECK_CTX(ctx);
    if (!params)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    return launchNrcPass(ctx, (cudaStream_t)stream, params, pass);
}
int gfx_nrc_shard(gfx_ctx* ctx, void* ncclComm, int rank, int world) {
    CHECK_CTX(ctx);
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    if (ncclComm && (world < 1 || world > 64 || rank < 0 || rank >= world))
        return GFX_ERR_INVALID_ARGUMENT;
    const int rc = ensureNrcFrame(ctx);
    if (rc != GFX_OK)
        return rc;
    FrameState::Nrc &N = ctx->frame.nrc;
    const bool on = ncclComm != nullptr && world > 1;
    N.shardComm = on ? ncclComm : nullptr;
    N.shardRank = on ? rank : 0;
    N.shardWorld = on ? world : 1;
    return GFX_OK;
}

int gfx_nrc_accumulate(gfx_ctx* ctx, void* stream, const GfxFrameParams* params) { return nrcPass(ctx, stream, params, 0); }
int gfx_nrc_propagate(gfx_ctx* ctx, void* stream, const GfxFrameParams* params) { return nrcPass(ctx, stream, params, 1); }
int gfx_nrc_shuffle(gfx_ctx* ctx, void* stream, const GfxFrameParams* params) { return nrcPass(ctx, stream, params, 2); }

} // extern "C"
