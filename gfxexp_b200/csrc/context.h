// context.h — host-side state behind the opaque gfx_ctx of include/gfxb200.h.
#pragma once
#include "scene.cuh"
#include <string>
#include <vector>
#include <cstdio>
#include <cstring>

namespace gfx {

struct SceneState {
    float4* vertices = nullptr;
    uint4* triangles = nullptr;
    DevMesh* meshes = nullptr;
    GfxMaterialDesc* materials = nullptr;
    DevInstance* instances = nullptr;
    uint32_t* instanceMeshSlots = nullptr;
    uint2* geomToInstMesh = nullptr;
    uint32_t* geomTriOffsets = nullptr; // numGeoms + 1
    float* primWeights = nullptr;
    float* primCdf = nullptr;
    float* geomWeights = nullptr;
    float* geomCdf = nullptr;
    float* instWeights = nullptr;
    float* instCdf = nullptr;
    float* instIntegral = nullptr;
    float* primProb = nullptr;
    float* geomProb = nullptr;
    float* instProb = nullptr;
    float4* lightTris = nullptr;
    uint32_t* instGuide = nullptr;
    uint32_t* primGuide = nullptr;
    uint32_t* lightTriBase = nullptr;      // per flattened geometry
    uint32_t* emissiveGeoms = nullptr;     // list of flattened geometry indices with an emissive material
    uint32_t numEmissiveGeoms = 0, numLightTris = 0;
    uint32_t numMeshes = 0, numMaterials = 0, numInstances = 0, numInstanceMeshSlots = 0;
    uint32_t numGeoms = 0, numFlatTris = 0, numMeshTris = 0, numVertices = 0;
    bool uploaded = false;
    bool staticLightDistsBuilt = false;
    bool lightTrisDirty = true;
    // flattened light pick (scene.cuh, lights.cu): tables + the scratch its stream-ordered rebuild needs
    float4* pickGuide = nullptr;           // 2 x kPickGuideSize
    float4* normalMats = nullptr;          // kNormalMatStride x numInstances
    // image textures of the materials (lights.cu uploadTextures)
    float4* texPool = nullptr;
    uint4* texTable = nullptr;
    uint4* materialTextures = nullptr;
    uint4* bumpTable = nullptr;            // per material, see DevScene::bumpTable
    float4* bumpTexels = nullptr;          // texPool, or bumpDefaultTexel for a scene without bump maps (not owned)
    float4* bumpDefaultTexel = nullptr;
    // environment light (lights.cu uploadEnvLight): texels + the importance map's distributions
    float4* envTexels = nullptr;
    float* envPdf = nullptr;
    float* envCdf = nullptr;
    float* envTopPdf = nullptr;
    float* envTopCdf = nullptr;
    uint32_t envW = 0, envH = 0;
    float envIntegral = 0.0f;              // integral of the importance map; 0 for a black map, which is no light to sample
    uint2* pickPieces = nullptr;           // pickCapacity + 2
    uint32_t* pickKeyAt = nullptr;         // kPickGuideSize + 1
    uint4* pickQueue[2] = { nullptr, nullptr };
    uint2* pickBoundaries = nullptr;
    uint32_t* pickCounters = nullptr;      // 4 words
    uint32_t* pickSortKeys[2] = { nullptr, nullptr };
    uint32_t* pickSortVals[2] = { nullptr, nullptr };
    void* pickSortTemp = nullptr;
    size_t pickSortTempBytes = 0;
    uint32_t pickCapacity = 0;
    uint32_t* pickFlagsHost = nullptr;     // pinned
    cudaEvent_t pickFlagsEvent = nullptr;
    bool pickFlagsPending = false, pickBuiltOnce = false, pickDirty = true;
    std::vector<DevMesh> hostMeshes;
    std::vector<DevInstance> hostInstances;
    // pinned staging for gfx_scene_update_instances (per-frame instance animation)
    DevInstance* pinnedInstances[2] = { nullptr, nullptr };
    cudaEvent_t pinnedInstancesFree[2] = { nullptr, nullptr };
    uint32_t pinnedInstancesNext = 0;
    void release();
};

struct BvhState {
    void* nodes = nullptr;       // GfxBvhNode8[numNodes]
    uint32_t* primRefs = nullptr;
    float4* tris = nullptr;      // GfxTriangleStorage[numTris]
    float4* leafTris = nullptr;  // traversal copy: TriangleStorage per primitive reference, in leaf order (see finishBvh)
    uint4* travNodes = nullptr;  // traversal copy of the nodes, child slots in octant order (see finishBvh)
    uint32_t* sceneBounds = nullptr;
    uint32_t* overflowFlag = nullptr;
    void* scratch = nullptr;     // build scratch arena, kept between builds (bvh_build.cu)
    size_t scratchBytes = 0;
    uint32_t builtForTris = 0;   // triangle count the output arrays are sized for
    uint32_t leafTrisCapacity = 0;
    uint32_t travNodesCapacity = 0;
    uint32_t numNodes = 0, numPrimRefs = 0, numTris = 0, levels = 0;
    float sceneMin[3] = { 0, 0, 0 }, sceneMax[3] = { 0, 0, 0 };
    bool ready = false;
    void release();
};

struct FrameState {
    uint32_t W = 0, H = 0;
    uint4* gb0[2] = { nullptr, nullptr };
    float2* gb1[2] = { nullptr, nullptr };
    float4* gb2[2] = { nullptr, nullptr };
    uint4* gb3[2] = { nullptr, nullptr };
    unsigned long long* rng = nullptr;
    float4* reservoir[2] = { nullptr, nullptr };
    float2* reservoirInfo[2] = { nullptr, nullptr };
    float4* beauty = nullptr;
    uint32_t* presentRgba8 = nullptr; // gfx_present_launch output, allocated on first use
    float4* albedo = nullptr;
    float4* normal = nullptr;
    float2* neighborDeltas = nullptr;
    unsigned long long* stats = nullptr; // 4 counters
    // wavefront visibility queue (SoA ray records compacted with warp ballots, traced by persistent threads)
    float4* rayQueue = nullptr;      // 2 x float4 per ray: (org, tmin) (dir, tmax)
    uint32_t* rayPixel = nullptr;    // pixel that asked for the ray
    uint32_t* rayCounters = nullptr; // [0] rays queued, [1] rays fetched
    uint8_t* visibility = nullptr;   // per pixel: 1 = unoccluded
    // wavefront path tracer (pathtrace.cu), allocated on first use
    float4* ptAlphaPdf = nullptr;
    float4* ptRadiance = nullptr;
    float4* ptExtRays[2] = { nullptr, nullptr };
    uint32_t* ptExtPixel[2] = { nullptr, nullptr };
    uint4* ptExtHits = nullptr;
    float4* ptShadowPending = nullptr;
    uint32_t* ptCounters = nullptr;
    // NRC frame buffers (nrc_pathtrace.cu), allocated on first use; layouts in include/gfxb200.h GFX_BUF_NRC_*
    struct Nrc {
        uint32_t numSuffixes = 0, queryCapacity = 0;
        float* inferenceQuery = nullptr;
        uint4* terminalInfo = nullptr;
        float* inferredRadiance = nullptr;
        float* frameContribution = nullptr;
        float* trainQuery[2] = { nullptr, nullptr };
        float* trainTarget[2] = { nullptr, nullptr };
        uint4* trainVertexInfo = nullptr;
        uint32_t* suffixTerminal = nullptr;
        uint32_t* shufflers = nullptr;
        uint32_t* state = nullptr;          // 32 words, see GFX_BUF_NRC_STATE
        // per-path state of the wavefront NRC path tracer (per pixel) ...
        float4* pathA = nullptr;            // primaryPathSpread, curSqrtPathSpread, flags|pathLength, linearTileIndex
        float4* pathB = nullptr;            // prevLocalThroughput
        float4* shadowPending2 = nullptr;   // per shadow slot: unoccluded directContNEE, tile (or ~0)
        // ... and per tile (one training path per tile)
        uint32_t* tilePrev = nullptr;       // prevTrainDataIndex
        uint32_t* tileSuffixEnded = nullptr;// trainingSuffixEndsWithCache
        uint32_t* stagedFlags = nullptr;    // want | fromRayGen<<1 | pathLength<<8
        uint32_t* stagedIndex = nullptr;    // index the vertex staged in this round received
        float* stagedQuery = nullptr;       // 14 floats
        float4* stagedThroughput = nullptr;
        float4* stagedNEE = nullptr;
        // strip sharding across ranks (gfx_nrc_shard): every rank traces its rows; the training vertices are numbered
        // globally through an all-gather of the per-round counts and the records are merged before the shuffle
        void* shardComm = nullptr;          // ncclComm_t of the ranks that share the frame
        int shardRank = 0, shardWorld = 1;
        uint32_t* shardCounts = nullptr;    // [0 .. world) gathered counts of this round, [64] this rank's count
        bool lastTraceIndirect = false;     // the last NRC path-trace launch was GFX_PT_NRC_INDIRECT: gfx_nrc_accumulate adds
        bool created = false;
    } nrc;
    // rearchitected ReSTIR (restir_rearch.cu), allocated on first use
    struct Rearch {
        float4* preSampledLights = nullptr;   // 128 x 1024 x 48 B
        unsigned long long* rngs = nullptr;
        uint32_t* sampleVis[2] = { nullptr, nullptr };
        float4* rays = nullptr;
        uint32_t* rayPixel = nullptr;
        uint32_t* rayMask = nullptr;
        uint32_t* counters = nullptr;
        uint32_t raysPerPixel = 0;
        bool created = false;
    } rearch;
    // ReGIR grid (regir.cu), (re)allocated by gfx_regir_build_cells when the grid dimensions change
    struct Regir {
        uint32_t dim[3] = { 0, 0, 0 };
        uint32_t numCells = 0, numSlots = 0;
        float gridOrigin[3] = { 0, 0, 0 }, gridCellSize[3] = { 0, 0, 0 };
        float4* slots[2] = { nullptr, nullptr };
        unsigned long long* slotRngs = nullptr;
        uint32_t* perCellNumAccesses = nullptr;
        uint32_t* lastAccessFrameIndices = nullptr;
        uint32_t* numActiveCells = nullptr;
        bool created = false;
    } regir;
    // SVGF state
    float4* svgfLighting[2] = { nullptr, nullptr };  // lighting rgb + variance, ping-pong
    float4* svgfMoments[2] = { nullptr, nullptr };   // first/second luminance moments + history length
    float4* svgfPrevLighting = nullptr;
    float4* svgfAlbedo = nullptr;
    float4* svgfNormal = nullptr;
    float2* svgfPrevScreenPos = nullptr;
    float4* svgfFinal[2] = { nullptr, nullptr };
    float* svgfDepth[2] = { nullptr, nullptr };
    float4* svgfDebugVisualize = nullptr; // gfx_svgf_debug_visualize output, allocated on first use
    bool created = false;
    void release();
};

} // namespace gfx

// Per-kernel CUDA-event timing (gfx_timing_enable / gfx_timing_read): every launch site is wrapped in a KernelTimerScope;
// when timing is off the scope is a branch on a bool.
struct KernelTimer {
    struct Rec {
        const char* label;
        cudaEvent_t start, stop;
    };
    bool enabled = false;
    std::vector<Rec> recs;
    std::vector<cudaEvent_t> pool;
    cudaEvent_t get() {
        if (!pool.empty()) {
            cudaEvent_t e = pool.back();
            pool.pop_back();
            return e;
        }
        cudaEvent_t e;
        cudaEventCreate(&e);
        return e;
    }
};

struct gfx_ctx {
    int device = 0;
    KernelTimer timer;
    std::string lastError;
    uint64_t launches = 0;
    uint32_t* traceFetchCounter = nullptr; // device counter of the wavefront trace kernel
    gfx::SceneState scene;
    gfx::BvhState bvh;
    gfx::FrameState frame;

    void setError(const std::string &msg) { lastError = msg; }
    gfx::DevScene devScene() const;
    gfx::DevScene devScene(const GfxFrameParams* p) const; // + the frame's environment-light switches
    gfx::DevFrame devFrame() const;
};

struct KernelTimerScope {
    gfx_ctx* ctx;
    cudaStream_t stream;
    size_t index;
    bool on;
    KernelTimerScope(gfx_ctx* c, cudaStream_t s, const char* label) : ctx(c), stream(s), index(0), on(c->timer.enabled) {
        if (!on)
            return;
        KernelTimer::Rec r{ label, c->timer.get(), c->timer.get() };
        cudaEventRecord(r.start, s);
        index = c->timer.recs.size();
        c->timer.recs.push_back(r);
    }
    ~KernelTimerScope() {
        if (on)
            cudaEventRecord(ctx->timer.recs[index].stop, stream);
    }
};
#define GFX_TIMED(ctx, stream, label) KernelTimerScope timedScope_##__LINE__(ctx, stream, label)

#define GFX_CUDA(ctx, call) \
    do { \
        const cudaError_t err_ = (call); \
        if (err_ != cudaSuccess) { \
            char buf_[512]; \
            snprintf(buf_, sizeof(buf_), "%s:%d: %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(err_)); \
            (ctx)->setError(buf_); \
            return err_ == cudaErrorMemoryAllocation ? GFX_ERR_OUT_OF_MEMORY : GFX_ERR_CUDA; \
        } \
    } while (0)

namespace gfx {
int buildBvh(gfx_ctx* ctx, cudaStream_t stream, uint32_t flags);
int finishBvh(gfx_ctx* ctx, cudaStream_t stream);
int launchPresent(gfx_ctx* ctx, cudaStream_t stream, const GfxPresentParams* params); // derived traversal tables of a built or imported BVH
int traceRays(gfx_ctx* ctx, cudaStream_t stream, const GfxRay* dRays, uint32_t numRays, GfxHitObject* dHits, int mode);
int traceRaysDebug(gfx_ctx* ctx, cudaStream_t stream, const GfxRay* dRays, uint32_t numRays, GfxHitObject* dHits, int mode,
                   int kernel);
int resetVisibilityQueue(gfx_ctx* ctx, cudaStream_t stream);
int traceVisibilityQueue(gfx_ctx* ctx, cudaStream_t stream);
int buildLightDistributions(gfx_ctx* ctx, cudaStream_t stream, uint32_t bufferIndex);
int uploadEnvLight(gfx_ctx* ctx, const float* rgba, uint32_t width, uint32_t height);
int uploadTextures(gfx_ctx* ctx, const GfxSceneDesc* sd);
int debugEnvLight(gfx_ctx* ctx, cudaStream_t stream, int op, const float* dIn, uint32_t n, float* dOut);
int debugShading(gfx_ctx* ctx, cudaStream_t stream, int op, const float* material, const float* dIn, uint32_t n, float* dOut);
int ensureBumpTable(gfx_ctx* ctx); // lights.cu, before a launch with enableBumpMapping
int debugBump(gfx_ctx* ctx, cudaStream_t stream, int op, uint32_t matSlot, const float* dIn, uint32_t n, float* dOut);
int debugLightPick(gfx_ctx* ctx, cudaStream_t stream, const float* dUl, uint32_t n, uint32_t* dFlat, uint32_t* dChain);
int debugLightSample(gfx_ctx* ctx, cudaStream_t stream, int op, const float* params, const float* dIn, uint32_t n, float* dOut);
size_t lightPickSortTempBytes(uint32_t capacity);
int launchGBuffer(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p);
int launchReSTIR(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int pass);
int launchReSTIRRearch(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int pass);
int ensureRearch(gfx_ctx* ctx, uint32_t raysPerPixel);
int launchSVGF(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int pass, uint32_t stage);
int launchSVGFDebugVisualize(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int view, float motionVectorOffset,
                             float motionVectorScale, uint32_t numFilteringStages);
int launchPathTrace(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int variant);
int launchPathTraceNrc(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, bool indirect); // GFX_PT_NRC[_INDIRECT]
int launchNrcVisualizePrediction(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p);
void regirGrid(const GfxFrameParams* p, uint32_t dim[3], float origin[3], float cellSize[3]); // regir.cu
int ensurePathTraceBuffers(gfx_ctx* ctx);
int ensureNrcFrame(gfx_ctx* ctx);
void* ncclSymbol(const char* name); // peer.cu: NCCL entry points resolved at run time from the NCCL the host process loaded
int launchRegirBuildCells(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, uint32_t frameIndex, int useTemporalReuse);
int launchRegirUpdateAccess(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, uint32_t frameIndex);
void releaseRegir(gfx_ctx* ctx);
int launchNrcPreprocess(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, uint32_t offsetToSelectUnbiasedTile,
                        uint32_t offsetToSelectTrainingPath, int isNewSequence);
int launchNrcPass(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* p, int pass); // 0 accumulate, 1 propagate, 2 shuffle
DevFrameParams makeDevParams(const gfx_ctx* ctx, const GfxFrameParams* p);
// GFX_SVGF_SUBPIXEL_JITTER: *jitter tells whether it applies to the frame (only with GFX_SVGF_ENABLE_TEMPORAL_AA), and then
// *sample = (ox, 1 - oy) is the sample's offset from the pixel's top-left corner in top-down pixel coordinates.  Refuses a
// frame that also sets enableJittering (GFX_ERR_INVALID_ARGUMENT).
int svgfSubPixelSample(gfx_ctx* ctx, const GfxFrameParams* p, bool* jitter, float2* sample);
} // namespace gfx
