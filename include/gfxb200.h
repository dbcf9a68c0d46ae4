/* gfxb200.h — C ABI of the H100-native per-frame hot path (BVH build/traverse, G-buffer,
 * ReSTIR DI, SVGF, NRC).  This is the drop-in boundary that stands where the reference's
 * OptiX wrapper and per-app launch sites stand today (SURVEY.md §8b):
 *
 *   optixu::Pipeline::launch(stream, plp, W, H, 1)        utils/optix_util.h:2149-2151
 *   optixu::Pipeline::setRayGenerationProgram(entry)      utils/optix_util.h:2116
 *   Scene::updateASs() -> GAS/IAS rebuild                 common/common_host.h:1027-1100
 *   Scene::setupLightGeomDistributions / setupLightInstDistribution
 *                                                          common/common_host.h:1102-1359
 *   cudau::Kernel::operator() / launchWithThreadDim        utils/cuda_util.h:421-436
 *   NeuralRadianceCache::{initialize,finalize,infer,train} neural_radiance_caching/network_interface.h:22-27
 *
 * Conventions: every entry point is extern "C", returns 0 on success or a negative GfxStatus,
 * never throws; gfx_last_error_string() gives the message (the reference throws
 * std::runtime_error from CUDADRV_CHECK/OPTIX_CHECK, utils/optix_util_private.h:66-100).
 * `stream` is a cudaStream_t passed as void* (NULL = default stream).  Pointers marked
 * "host" are read/written with cudaMemcpy inside the call; everything else lives in HBM
 * owned by the context.  There is no CPU fallback: every call fails with GFX_ERR_NO_DEVICE
 * when no sm_90 (H100) device is present.
 */
#ifndef GFXB200_H
#define GFXB200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gfx_ctx gfx_ctx;

typedef enum GfxStatus {
    GFX_OK = 0,
    GFX_ERR_INVALID_ARGUMENT = -1,
    GFX_ERR_NO_DEVICE = -2,
    GFX_ERR_CUDA = -3,
    GFX_ERR_NOT_READY = -4,     /* e.g. launch before scene upload / BVH build */
    GFX_ERR_OUT_OF_MEMORY = -5,
    GFX_ERR_UNSUPPORTED = -6
} GfxStatus;

/* ---- scene description (host side, SoA per mesh) ------------------------------------- */

/* One GeometryInstance: vertex/triangle buffers + material slot
 * (shared::GeometryInstanceData, common/common_shared.h:1172-1186; shared::Vertex :1109-1114). */
typedef struct GfxMeshDesc {
    const float* positions;   /* host, 3 * numVertices */
    const float* normals;     /* host, 3 * numVertices */
    const float* tangents;    /* host, 3 * numVertices (Vertex::texCoord0Dir) */
    const float* texcoords;   /* host, 2 * numVertices */
    const uint32_t* triangles;/* host, 3 * numTriangles */
    uint32_t numVertices;
    uint32_t numTriangles;
    uint32_t materialSlot;
    uint32_t reserved;
} GfxMeshDesc;

typedef enum GfxBsdfType {
    GFX_BSDF_LAMBERT = 0,              /* common_device.cuh:335-385   p0 = reflectance */
    GFX_BSDF_DIFFUSE_AND_SPECULAR = 1, /* common_device.cuh:443-765   p0 = diffuse, p1 = specular F0, p2 = smoothness */
    GFX_BSDF_SIMPLE_PBR = 2            /* common_device.cuh:767-826   p0 = baseColor, p1 = (occlusion, roughness, metallic) */
} GfxBsdfType;

/* shared::MaterialData (common/common_shared.h:1131-1170).  The fields are the values of 1x1 textures *after* the texture unit's
 * UNORM8/sRGB decode; a material whose parameters vary over the surface names image textures instead
 * (GfxSceneDesc::materialTextures). */
typedef struct GfxMaterialDesc {
    float p0[3];
    float p2;
    float p1[3];
    uint32_t bsdfType;     /* GfxBsdfType */
    float emittance[3];
    uint32_t hasEmittance; /* mat.emittance != 0 */
} GfxMaterialDesc;

/* shared::InstanceData (common/common_shared.h:1241-1249). Matrices are row-major. */
typedef struct GfxInstanceDesc {
    float transform[12];          /* object -> world, 3x4 */
    float curToPrevTransform[12]; /* world(cur) -> world(prev), 3x4 */
    float normalMatrix[9];        /* transpose(inverse(upper-left 3x3)), common_host.cpp:2635 */
    float uniformScale;
    uint32_t firstMeshSlot;       /* range into GfxSceneDesc::instanceMeshSlots (InstanceData::geomInstSlots) */
    uint32_t numMeshSlots;
} GfxInstanceDesc;

/* One image texture of a material (Material::texReflectance / texSpecular / ... , common_host.cpp:1462-1533): RGBA fp32 texels,
 * row-major, as the texture unit would hand them to the filter, i.e. after the UNORM8 -> float and sRGB -> linear decode of the
 * reference's samplers (NormalizedFloat_sRGB for colour maps).  Sampled like the reference's material samplers - linear filter,
 * repeat addressing, level 0 (tex2DLod(..., 0.0f)) - restated in software (csrc/lighting.cuh textureFetchRepeat). */
typedef struct GfxTextureDesc {
    const float* texels;
    uint32_t width;
    uint32_t height;
} GfxTextureDesc;

typedef struct GfxSceneDesc {
    const GfxMeshDesc* meshes;
    const GfxMaterialDesc* materials;
    const GfxInstanceDesc* instances;
    const uint32_t* instanceMeshSlots;
    uint32_t numMeshes;
    uint32_t numMaterials;
    uint32_t numInstances;
    uint32_t numInstanceMeshSlots;
    /* environment light: Scene::envLightTexture + envLightImportanceMap (restir_di_shared.h:221-222), what
     * loadEnvironmentalTexture (common/common_host.cpp:2658-2711) produces from the -env-texture file.  RGBA fp32 texels of an
     * equirectangular map, row 0 at theta = 0 (+y), column 0 at phi = 0; the library clamps them to [0, 65504] and builds the
     * luminance x sin(theta) importance map (RegularConstantContinuousDistribution2D, common_shared.h:283-386).  Sampled with
     * the reference's sampler (linear filter, clamp addressing) restated in software.  NULL = no environment light. */
    const float* envTexels;
    uint32_t envWidth;
    uint32_t envHeight;
    /* image textures: materialTextures[4 * m + k] = index into `textures` of the map that replaces, in material m,
     * k = 0: p0 (.xyz: reflectance / diffuse / baseColor), 1: p1 (.xyz: specular F0 / occlusion-roughness-metallic),
     * 2: p2 (.x: smoothness), 3: emittance (must be 0xFFFFFFFF: textured emitters are not supported, gfx_scene_upload refuses
     * them) - or 0xFFFFFFFF for "use the constant of GfxMaterialDesc".  NULL = no material is textured. */
    const GfxTextureDesc* textures;
    const uint32_t* materialTextures;
    uint32_t numTextures;
    /* bump maps (Material::texNormal + bumpMapType, common_host.cpp:1344-1412; MaterialData::normal + readModifiedNormal,
     * common_device.cuh:205-240): bumpMaps[2 * m] = index into `textures` of material m's map, or 0xFFFFFFFF for the
     * reference's default, the 1x1 texel (127, 127, 255) / 255 of createNormalTexture (createImmTexture quantises 0.5 to
     * uint(255 * 0.5) = 127); bumpMaps[2 * m + 1] = its GfxBumpMapType (ignored, but must be valid, for 0xFFFFFFFF).  The maps
     * are UNORM-decoded texels of the same pool as the other textures - no sRGB decode (sampler_normFloat) - sampled at level 0
     * with repeat addressing.  gfx_scene_upload refuses an index past numTextures or an unknown type.  NULL = every material
     * has the default texel.  Only read when GfxFrameParams::enableBumpMapping is set. */
    const uint32_t* bumpMaps;
} GfxSceneDesc;

/* BumpMapTextureType (common_host.h): how a material's bump map is read (loadNormalTexture, common_host.cpp:1344-1356: a PNG
 * with more than one channel is a normal map, a one-channel PNG - and spnza_bricks_a_bump.png - a height map) */
typedef enum GfxBumpMapType {
    GFX_BUMP_NORMAL_MAP = 0, /* readModifiedNormalFromNormalMap: n = 2 rgb - 1, n.y = -n.y (calcDimInfo's isLeftHanded = true) */
    GFX_BUMP_HEIGHT_MAP = 1  /* readModifiedNormalFromHeightMap: tex2Dgather of channel 0, n = normalize(-dh/du, dh/dv, 1) with
                              * dh/du = (5/1024 W) (g.y - g.x), dh/dv = (5/1024 H) (g.x - g.w) */
} GfxBumpMapType;

/* ---- BVH formats (bit-identical to the reference structs) ---------------------------- */

/* shared::CompressedInternalNode_T<8>, 80 B (common/common_shared.h:757-917) */
typedef struct GfxBvhNode8 {
    float quantBoxOrigin[3];
    uint8_t quantBoxExpScale[3];
    uint8_t internalMask;
    uint32_t intNodeChildBaseIndex;
    uint32_t leafBaseIndex;
    uint8_t childMetas[8];
    uint8_t childQMin[3][8]; /* Xs, Ys, Zs */
    uint8_t childQMax[3][8];
} GfxBvhNode8;

/* shared::TriangleStorage, 48 B (common/common_shared.h:1017-1025). geomIndex enumerates
 * (instance, mesh-slot-in-instance) pairs in instance order, as Scene flattening does. */
typedef struct GfxTriangleStorage {
    float pA[3], pB[3], pC[3];
    uint32_t geomIndex;
    uint32_t primIndex;
    uint32_t padding;
} GfxTriangleStorage;

/* shared::HitObject, 32 B (common/common_shared.h:1065-1078) */
typedef struct GfxHitObject {
    float dist;
    uint32_t instIndex;
    uint32_t instUserData;
    uint32_t geomIndex;
    uint32_t primIndex;
    float bcA, bcB, bcC;
} GfxHitObject;

/* ray record of the wavefront trace entry point: 32 B */
typedef struct GfxRay {
    float org[3];
    float tmin;
    float dir[3];
    float tmax;
} GfxRay;

typedef struct GfxBvhInfo {
    uint32_t numNodes;
    uint32_t numPrimRefs;
    uint32_t numTriangles;
    uint32_t numGeoms;
    float sceneMin[3];
    float sceneMax[3];
} GfxBvhInfo;

typedef enum GfxTraceMode {
    GFX_TRACE_CLOSEST = 0, /* bvh::traverse semantics, tie -> smaller storage index */
    GFX_TRACE_ANY = 1,     /* visibility ray: dist = 0 if anything is hit in (tmin,tmax), else tmax */
    GFX_TRACE_STATS = 2    /* flag: also return bvh::TraversalStatistics per ray in instUserData
                              (internal nodes visited | triangles tested << 16) */
} GfxTraceMode;

/* ---- per-frame parameters ------------------------------------------------------------ */

/* shared::PerspectiveCamera (restir_di/restir_di_shared.h:45-60) */
typedef struct GfxCamera {
    float aspect;
    float fovY;
    float position[3];
    float orientation[9]; /* row-major 3x3 */
} GfxCamera;

/* shared::PerFramePipelineLaunchParameters + the per-launch bitfields of
 * PipelineLaunchParameters (restir_di/restir_di_shared.h:243-288). */
typedef struct GfxFrameParams {
    GfxCamera camera;
    GfxCamera prevCamera;
    uint32_t numAccumFrames;
    uint32_t frameIndex;
    uint32_t bufferIndex;              /* G-buffer double-buffer slot (frameIndex % 2) */
    float spatialNeighborRadius;
    uint32_t log2NumCandidateSamples;
    uint32_t numSpatialNeighbors;
    uint32_t useLowDiscrepancyNeighbors;
    uint32_t reuseVisibility;
    uint32_t enableTemporalReuse;
    uint32_t enableSpatialReuse;
    uint32_t useUnbiasedEstimator;
    uint32_t resetFlowBuffer;
    uint32_t enableJittering;
    uint32_t currentReservoirIndex;    /* plp.currentReservoirIndex */
    uint32_t spatialNeighborBaseIndex; /* plp.spatialNeighborBaseIndex */
    uint32_t tileOriginY;              /* multi-GPU: first row owned by this rank (0 on 1 GPU) */
    uint32_t tileRows;                 /* multi-GPU: rows owned by this rank (0 = all) */
    /* SVGF (svgf_shared.h PerFramePipelineLaunchParameters: isFirstFrame, enableTemporalAccumulation,
     * feedback1stFilteredResult, enableTemporalAA, modulateAlbedo, taaHistoryLength; svgf_main.cpp:1730-1736) */
    uint32_t svgfFlags;                /* GfxSVGFFlags */
    uint32_t taaHistoryLength;         /* 16 by default */
    /* path tracers (path_tracing_shared.h PerFramePipelineLaunchParameters::maxPathLength; 5 by default,
     * path_tracing_main.cpp:1519).  0 selects that default for GFX_PT_BASELINE / GFX_PT_REGIR and means
     * "no limit" for GFX_PT_NRC, as in neural_radiance_caching_main.cpp:2246 (infBounces) */
    uint32_t maxPathLength;
    /* NRC / ReGIR: scene.initialSceneAabb (neural_radiance_caching_main.cpp:1096,1139; regir_main.cpp:1012), the
     * box positions are normalised to, and PerFramePipelineLaunchParameters::radianceScale (10^log10RadianceScale,
     * neural_radiance_caching_main.cpp:2241) */
    float sceneAabbMin[3];
    float sceneAabbMax[3];
    float radianceScale;
    /* ReGIR (regir_shared.h:247-249, regir_main.cpp:1109,1733-1736): grid over sceneAabb (0,0,0 = 32 x 8 x 32),
     * 2^3 candidates per light slot, 2^2 resampled slots per shading point, jittered cell lookup */
    uint32_t regirGridDim[3];
    uint32_t regirLog2NumCandidatesPerLightSlot;
    uint32_t regirLog2NumCandidatesPerCell;
    uint32_t regirEnableCellRandomization;
    /* rearchitected ReSTIR (restir_di_main.cpp:1945-1949, 2326-2335) */
    uint32_t reuseVisibilityForTemporal;        /* true by default */
    uint32_t reuseVisibilityForSpatiotemporal;  /* false by default */
    float radiusThresholdForSpatialVisReuse;    /* 10 px by default */
    /* environment light (PerFramePipelineLaunchParameters::envLightPowerCoeff, envLightRotation, enableEnvLight,
     * restir_di_shared.h:249-250,269): used when the scene has an environment map; probToSampleEnvLight = 0.25 (:6) */
    uint32_t enableEnvLight;
    float envLightPowerCoeff;
    float envLightRotation;
    /* perFramePlp.enableBumpMapping, the "Enable Bump Mapping" checkbox (false by default: restir_di_main.cpp:1986, 2005, 2345;
     * path_tracing_main.cpp:1516, 1537, 1765; regir_main.cpp:1728, 1755, 2011; neural_radiance_caching_main.cpp:1857, 1887,
     * 2251).  When set, every shading frame built from a surface - gfx_gbuffer_launch (so also the ReSTIR passes, which read
     * the frame back from the G-buffer) and the first hit and bounces of GFX_PT_BASELINE, GFX_PT_REGIR, GFX_PT_NRC and
     * GFX_PT_NRC_VISUALIZE_PREDICTION - is tilted by applyBumpMapping(readModifiedNormal(GfxSceneDesc::bumpMaps of the
     * material, texCoord)) before anything reads it.  As in the reference, a material without a map is tilted too, by about
     * 0.3 degrees (the default texel decodes to (-1/255, 1/255, 1)).  The SVGF app has no such switch: GFX_PT_SVGF ignores
     * the flag, and since gfx_gbuffer_launch (with or without GFX_SVGF_SUBPIXEL_JITTER) does not, an SVGF host leaves it 0. */
    uint32_t enableBumpMapping;
} GfxFrameParams;

typedef enum GfxSVGFFlags {
    GFX_SVGF_IS_FIRST_FRAME = 1,
    GFX_SVGF_ENABLE_TEMPORAL_ACCUMULATION = 2,
    GFX_SVGF_FEEDBACK_1ST_FILTERED_RESULT = 4,
    GFX_SVGF_ENABLE_TEMPORAL_AA = 8,
    GFX_SVGF_MODULATE_ALBEDO = 16,
    GFX_SVGF_MOLLIFY_SPECULAR = 32,   /* mollifySpecular (svgf_shared.h:225, svgf_main.cpp:1733, 1995; on in the SVGF app by default):
                                       * GFX_PT_SVGF sets up the BSDFs of the bounces (not of the first vertex) regularised */
    GFX_SVGF_SUBPIXEL_JITTER = 64     /* the SVGF app's TAA sub-pixel jitter (svgf_main.cpp:1410-1424, 2005-2008); only together
                                       * with GFX_SVGF_ENABLE_TEMPORAL_AA, as in the app.  The library computes the offset
                                       * (ox, oy) = (halton(2, i), halton(3, i)), i = frameIndex % taaHistoryLength (0 means 16);
                                       * the app's table has 256 entries, so a taaHistoryLength above 256 goes beyond what the app
                                       * can run.  gfx_gbuffer_launch casts the primary ray through (x + ox, y + 1 - oy) in
                                       * top-down pixel coordinates and measures the motion vector from that sample position, and
                                       * GFX_SVGF_FILL_BACKGROUND looks the environment up through it; no random number is drawn.
                                       * A frame that also sets enableJittering is refused with GFX_ERR_INVALID_ARGUMENT. */
} GfxSVGFFlags;

/* ReSTIR DI entry points (restir_di/restir_di_main.cpp:63-74 ReSTIREntryPoint) */
typedef enum GfxReSTIRPass {
    GFX_RESTIR_INITIAL_RIS = 0,                 /* performInitialRIS */
    GFX_RESTIR_INITIAL_AND_TEMPORAL_BIASED = 1, /* performInitialAndTemporalRISBiased */
    GFX_RESTIR_INITIAL_AND_TEMPORAL_UNBIASED = 2,
    GFX_RESTIR_SPATIAL_BIASED = 3,              /* performSpatialRISBiased */
    GFX_RESTIR_SPATIAL_UNBIASED = 4,
    GFX_RESTIR_SHADING = 5,                     /* shading */
    /* rearchitected renderer (restir_di_main.cpp:2423-2493; RearchitectedReSTIREntryPoint :76-87).  The
     * temporal / spatial / unbiased variants of the last two are selected by params->enableTemporalReuse,
     * enableSpatialReuse (pass 0 for both on the first frame of a sequence) and useUnbiasedEstimator. */
    GFX_RESTIR_PRESAMPLE_LIGHTS = 6,            /* performLightPreSampling: 128 subsets x 1024 lights */
    GFX_RESTIR_PER_PIXEL_RIS = 7,               /* performPerPixelRIS: candidates from the tile's subset */
    GFX_RESTIR_TRACE_SHADOW_RAYS = 8,           /* traceShadowRays[With{Temporal,Spatial,SpatioTemporal}Reuse{Biased,Unbiased}] */
    GFX_RESTIR_SHADE_AND_RESAMPLE = 9           /* shadeAndResample[With{Temporal,Spatial,Spatiotemporal}Reuse] */
} GfxReSTIRPass;

/* path tracer entry points (path_tracing/path_tracing_main.cpp:52-57 PathTracingEntryPoint) */
typedef enum GfxPathTraceVariant {
    GFX_PT_BASELINE = 0,                        /* pathTraceBaseline */
    GFX_PT_NRC = 1,                             /* pathTraceNRC (neural_radiance_caching_main.cpp:2281-2289):
                                                 * needs gfx_nrc_preprocess first; fills the NRC buffers below */
    GFX_PT_REGIR = 2,                           /* regir's pathTraceReGIR (regir_main.cpp:2051-2057): NEE resamples the
                                                 * cell reservoirs built by gfx_regir_build_cells */
    GFX_PT_NRC_VISUALIZE_PREDICTION = 3,        /* visualizePrediction (neural_radiance_caching/gpu_kernels/
                                                 * optix_pathtracing_kernels.cu:702-778): for every pixel of the G-buffer
                                                 * params->bufferIndex (the whole frame), a primary hit writes its radiance
                                                 * query to row y * W + x of GFX_BUF_NRC_INFERENCE_QUERY (a miss leaves its row
                                                 * as it was); every pixel's terminal info becomes alpha 1, pathLength 1,
                                                 * hasQuery = hit, not a training pixel or unbiased tile; the state block's
                                                 * numInferenceQueries becomes pad128(W*H), so that gfx_nrc_frame_infer infers
                                                 * exactly those rows (:2371-2387).  Show the result with
                                                 * GFX_PRESENT_NRC_PREDICTION.  GFX_ERR_NOT_READY before the frame has NRC
                                                 * buffers (gfx_nrc_preprocess creates them), GFX_ERR_UNSUPPORTED on a context
                                                 * sharded with gfx_nrc_shard(world > 1).  The next NRC frame overwrites
                                                 * everything it writes. */
    GFX_PT_SVGF = 4,                            /* the SVGF app's path tracer (svgf/gpu_kernels/optix_pathtracing_kernels.cu:
                                                 * 130-513, svgf_main.cpp:2118-2126) up to its temporal accumulation, which is
                                                 * GFX_SVGF_TEMPORAL_ACCUMULATE: from the G-buffer params->bufferIndex it writes
                                                 * one sample of max(contribution, 0) per pixel to GFX_BUF_BEAUTY_ACCUM and the
                                                 * first vertex's DH-reflectance estimate to GFX_BUF_ALBEDO_ACCUM (0 for a miss;
                                                 * params->numAccumFrames is not used).  The first vertex takes the G-buffer's
                                                 * shading normal as its geometric normal and frame; no Russian roulette at path
                                                 * length 2; GFX_SVGF_MOLLIFY_SPECULAR in params->svgfFlags regularises the
                                                 * bounces' BSDFs.  Rows params->tileOriginY / tileRows. */
    GFX_PT_NRC_INDIRECT = 5                     /* GFX_PT_NRC for a frame whose direct light at the primary vertex comes from
                                                 * ReSTIR DI: the same paths, RNG draws, Russian roulette, cache termination,
                                                 * training records and sharding rules, but the rendering radiance
                                                 * (GFX_BUF_NRC_FRAME_CONTRIBUTION) leaves out the primary hit's emission, the
                                                 * environment seen directly, the primary vertex's NEE (its shadow ray is traced
                                                 * for training paths only) and, at path length 2, the implicit emitter and
                                                 * environment terms; the training targets keep them.  The gfx_nrc_accumulate
                                                 * that follows adds instead of blending (see there). */
} GfxPathTraceVariant;

/* SVGF entry points (svgf/svgf_main.cpp:2127-2172) */
typedef enum GfxSVGFPass {
    GFX_SVGF_TEMPORAL_ACCUMULATE = 0, /* demodulate + reprojectPreviousAccumulation + EMA (svgf/gpu_kernels/optix_pathtracing_kernels.cu:55-128,325-378) */
    GFX_SVGF_ESTIMATE_VARIANCE = 1,   /* estimateVariance (svgf.cu:30-134) */
    GFX_SVGF_ATROUS = 2,              /* applyATrousFilter_box3x3(stage) (svgf.cu:221-354) */
    GFX_SVGF_FILL_BACKGROUND = 3,     /* fillBackground (svgf.cu:378-461) */
    GFX_SVGF_MODULATE_TAA = 4,        /* applyAlbedoModulationAndTemporalAntiAliasing (svgf.cu:533-611) */
    GFX_SVGF_FEEDBACK_NOISY_LIGHTING = 5 /* feedbackNoisyLighting (svgf.cu:356-374): lighting plane 0 -> GFX_BUF_SVGF_PREV_LIGHTING,
                                          * the SVGF app's frame with SVGF off and temporal accumulation on (svgf_main.cpp:2159-2164);
                                          * FILL_BACKGROUND / MODULATE_TAA then take stage 0 */
} GfxSVGFPass;

/* buffers that can be read back for parity checks (logical row-major (x,y) order) */
typedef enum GfxBufferId {
    GFX_BUF_GBUFFER0 = 0,   /* uint32 x4 : instSlot, geomInstSlot, primIndex, qbcB | qbcC<<16 */
    GFX_BUF_GBUFFER1 = 1,   /* float  x2 : motion vector */
    GFX_BUF_GBUFFER2 = 2,   /* float3 position + uint32 qGeometricNormal */
    GFX_BUF_GBUFFER3 = 3,   /* uint32 x4 : qShadingNormal, qShadingTangent, qTexCoord, matSlot */
    GFX_BUF_RNG = 4,        /* uint64    : PCG32 state */
    GFX_BUF_RESERVOIR = 5,  /* 12 floats : emittance3, position3, normal3, sumWeights, streamLength(u32) | atInfinity<<31, pad */
    GFX_BUF_RESERVOIR_INFO = 6, /* float x2 : recPDFEstimate, targetDensity */
    GFX_BUF_BEAUTY_ACCUM = 7,   /* float x4 */
    GFX_BUF_ALBEDO_ACCUM = 8,   /* float x4 */
    GFX_BUF_NORMAL_ACCUM = 9,   /* float x4 */
    GFX_BUF_SVGF_LIGHTING_VARIANCE = 10, /* float x4 : noisy/filtered lighting rgb + variance */
    GFX_BUF_SVGF_FINAL = 11,    /* float x4 */
    GFX_BUF_SVGF_MOMENTS = 12,  /* float x4 : firstMoment, secondMoment, sampleInfo(u32), 0 */
    GFX_BUF_SVGF_PREV_LIGHTING = 13, /* float x4 : prevNoisyLightingBuffer */
    GFX_BUF_SVGF_ALBEDO = 14,   /* float x4 : dhReflectance */
    GFX_BUF_SVGF_DEPTH = 15,    /* float : GL-style depth, background 1.0 */
    /* NRC frame buffers (neural_radiance_caching_shared.h:258-279); linear, not image shaped.
     * numSuffixes = ceil(W/4) * ceil(H/4) (= W*H/16 of neural_radiance_caching_main.cpp:1151 for multiples of 4) */
    GFX_BUF_NRC_INFERENCE_QUERY = 16,   /* float x14 RadianceQuery x pad128(W*H + numSuffixes) */
    GFX_BUF_NRC_TERMINAL_INFO = 17,     /* uint32 x4 x W*H : alpha rgb (float bits), hasQuery | pathLength<<1 | isTrainingPixel<<9 | isUnbiasedTile<<10 */
    GFX_BUF_NRC_INFERRED_RADIANCE = 18, /* float x3 x pad128(W*H + numSuffixes) */
    GFX_BUF_NRC_FRAME_CONTRIBUTION = 19,/* float x3 x W*H : perFrameContributionBuffer */
    GFX_BUF_NRC_TRAIN_QUERY = 20,       /* [2] float x14 x 131072 : [0] path tracer output, [1] shuffled */
    GFX_BUF_NRC_TRAIN_TARGET = 21,      /* [2] float x3 x 131072 */
    GFX_BUF_NRC_TRAIN_VERTEX_INFO = 22, /* uint32 x4 x 131072 : localThroughput rgb, prevVertexDataIndex | pathLength<<23 */
    GFX_BUF_NRC_TRAIN_SUFFIX_TERMINAL = 23, /* uint32 x numSuffixes : prevVertexDataIndex | hasQuery<<23 | pathLength<<24 */
    GFX_BUF_NRC_STATE = 24,             /* uint32 x32 : numTrainingData[2], tileSize[2][2], offsetToSelectUnbiasedTile,
                                         * offsetToSelectTrainingPath, targetMin/Max (ordered ints) [2][2][3] at 8,
                                         * targetAvg [2][3] at 20, numInferenceQueries at 26 */
    /* ReGIR grid (regir_shared.h:207-216); numSlots = numCells * 512 */
    GFX_BUF_REGIR_SLOTS = 25,           /* [2] 16 words x numSlots : Reservoir<LightSample> + ReservoirInfo as one 64-byte record:
                                         * emittance3 sumWeights | position3 streamLength|atInfinity<<31 | normal3 recPDFEstimate |
                                         * targetDensity 0 0 0 */
    GFX_BUF_REGIR_SLOT_RNG = 26,        /* uint64 x numSlots : lightSlotRngs */
    GFX_BUF_REGIR_CELL_ACCESSES = 27,   /* uint32 x numCells : perCellNumAccesses */
    GFX_BUF_REGIR_LAST_ACCESS = 28,     /* uint32 x numCells : lastAccessFrameIndices */
    GFX_BUF_REGIR_NUM_ACTIVE_CELLS = 29,/* uint32 x2 : numActiveCellsArray */
    /* rearchitected ReSTIR */
    GFX_BUF_SAMPLE_VISIBILITY = 30,     /* [2] uint32 per pixel : SampleVisibility bits (restir_di_shared.h:146-164) */
    GFX_BUF_PRESAMPLED_LIGHTS = 31,     /* 12 words x 131072 : emittance3 areaPDensity | position3 atInfinity | normal3 0 */
    GFX_BUF_PRESAMPLE_RNG = 32,         /* uint64 x 131072 : lightPreSamplingRngs */
    /* output side */
    GFX_BUF_PRESENT_RGBA8 = 33,         /* uint32 per pixel, R | G << 8 | B << 16 | A << 24 : gfx_present_launch */
    GFX_BUF_SVGF_DEBUG_VISUALIZE = 34   /* float x4 per pixel, w = 1 : gfx_svgf_debug_visualize (debugVisualizeBuffer) */
} GfxBufferId;

/* ---- context ------------------------------------------------------------------------- */
int gfx_ctx_create(int device, gfx_ctx** out);
void gfx_ctx_destroy(gfx_ctx* ctx);
const char* gfx_last_error_string(gfx_ctx* ctx);
int gfx_synchronize(gfx_ctx* ctx, void* stream);
/* number of kernels this library has launched since the context was created */
uint64_t gfx_kernel_launch_count(gfx_ctx* ctx);

/* per-kernel timing for bench.py's roofline: when enabled every kernel launch of this library is bracketed by CUDA
 * events on its stream; gfx_timing_read synchronises, sums the elapsed times per kernel label since the last read
 * and returns the number of labels written (at most `capacity`). */
typedef struct GfxKernelTiming {
    char label[48];
    float totalMs;
    uint32_t launches;
} GfxKernelTiming;
int gfx_timing_enable(gfx_ctx* ctx, int enable);
int gfx_timing_read(gfx_ctx* ctx, GfxKernelTiming* out, uint32_t capacity, uint32_t* numWritten);

/* ---- output side (SURVEY.md 8f-4) -------------------------------------------------------------------------------------
 * What the reference does between the accumulation buffers and a picture: copyToLinearBuffers + visualizeToOutputBuffer
 * (restir_di/gpu_kernels/copy_buffers.cu:6-28,32-80: normals are normalised and shown as 0.5 + 0.5 n), the display shader's
 * tone map (common/shaders/drawOptiXResult.frag; the screenshot path saveImage(float4*, SDRImageSaverConfig),
 * common/common_host.cpp:2859-2897, is the same arithmetic on the CPU): non-finite colours -> 0,
 * lum = sRGB luminance, colour *= (1 - exp(-brightnessScale * lum)) / lum, then sRGB_gamma_s (basic_types.h:5405-5410) and
 * 8-bit packing min(uint(v * 255), 255).  The packed image is what the reference's own
 * saveImage(path, width, height, const uint32_t*) (common_host.cpp:2715) writes with stb.
 *
 * The debug views of the reference's NRC and ReGIR apps (visualizeToOutputBuffer, neural_radiance_caching/gpu_kernels/
 * copy_buffers.cu:32-130 and regir/gpu_kernels/copy_buffers.cu:62-76,95-108) are further modes and flags.  They read the
 * frame's buffers at the pixel (after FLIP_Y), replace or tint the colour, and then go through the same alpha override, tone
 * map, gamma and packing (the reference tints first and its display shader tone-maps afterwards):
 *   GFX_PRESENT_NRC_PREDICTION   if the terminal info has a query: max(inferred radiance, 0), / radianceScale when that is
 *                                > 0, x (diffuse + specular reflectance) of the query row; then x alpha, w = 1; else 0
 *                                (copy_buffers.cu:52-67).  After GFX_PT_NRC_VISUALIZE_PREDICTION + gfx_nrc_frame_infer this
 *                                is the cache's prediction at the primary hits.
 *   GFX_PRESENT_NRC_PATH_LENGTH  blue -> green -> red ramp of the terminal info's pathLength, t = min((pathLength - 1) / 5, 1)
 *                                (:96-112); meaningful after an NRC frame
 *   GFX_PRESENT_FLOW             clamp(motionVectorScale * mv + motionVectorOffset, 0, 1) for x and y of GFX_BUF_GBUFFER1,
 *                                z = motionVectorOffset, w = 1 (:87-94)
 *   GFX_PRESENT_NRC_TRAINING_PATHS  flag: training pixels x (1, .25, 1, 1), other pixels of unbiased tiles x (.25, 1, .25, 1)
 *                                (:118-127), in every mode
 *   GFX_PRESENT_REGIR_CELLS      flag, COLOR mode only (ignored in the others): rgb x the colour of the ReGIR cell that holds
 *                                GFX_BUF_GBUFFER2's position (FNV-1 hash of the cell index -> PCG32 -> HSVtoRGB).  The grid is
 *                                gfx_regir_build_cells' over frame->sceneAabbMin/Max and frame->regirGridDim (0 = 32 x 8 x 32).
 * The NRC views read GFX_BUF_NRC_TERMINAL_INFO, _INFERRED_RADIANCE and _INFERENCE_QUERY (GFX_ERR_NOT_READY before the frame
 * has NRC buffers); the G-buffers are those of frame->bufferIndex.  The new modes do not read the source buffer.  A new mode
 * or flag needs `frame` (GFX_ERR_INVALID_ARGUMENT without); COLOR and NORMAL without the new flags never read the fields
 * after alphaForOverride, so callers built against the six-field struct keep working. */
typedef enum GfxPresentMode {
    GFX_PRESENT_COLOR = 0,
    GFX_PRESENT_NORMAL = 1,
    GFX_PRESENT_NRC_PREDICTION = 2,
    GFX_PRESENT_NRC_PATH_LENGTH = 3,
    GFX_PRESENT_FLOW = 4
} GfxPresentMode;
#define GFX_PRESENT_TONE_MAP 1u
#define GFX_PRESENT_SRGB_GAMMA 2u
#define GFX_PRESENT_FLIP_Y 4u
#define GFX_PRESENT_NRC_TRAINING_PATHS 8u
#define GFX_PRESENT_REGIR_CELLS 16u
typedef struct GfxPresentParams {
    int32_t sourceBuffer;      /* a float4-per-pixel frame buffer: GFX_BUF_BEAUTY_ACCUM, _ALBEDO_ACCUM, _NORMAL_ACCUM, GFX_BUF_SVGF_FINAL ... */
    uint32_t sourceIndex;
    int32_t mode;              /* GfxPresentMode */
    uint32_t flags;            /* GFX_PRESENT_* */
    float brightnessScale;     /* 10^brightness of the reference UI */
    float alphaForOverride;    /* >= 0: written instead of the source alpha (SDRImageSaverConfig::alphaForOverride) */
    /* the debug views only (see above): */
    const GfxFrameParams* frame;  /* host: bufferIndex, radianceScale, sceneAabbMin/Max, regirGridDim */
    float motionVectorScale;      /* 10^-1 by default (neural_radiance_caching_main.cpp:2462) */
    float motionVectorOffset;     /* 0.5 by default */
} GfxPresentParams;
/* writes GFX_BUF_PRESENT_RGBA8 (read it with gfx_buffer_download or gfx_buffer_device_ptr) */
int gfx_present_launch(gfx_ctx* ctx, void* stream, const GfxPresentParams* params);

/* ---- multi-GPU: one-sided seam-row exchange over NVLink peer memory (csrc/peer.cu) -------------------------------
 * The reference is a single-GPU program; a strip-sharded frame (SURVEY.md 8e) needs the reservoirs of `halo` rows across
 * each seam.  Each rank exports the IPC handles of its reservoir buffers and of its flag block
 * (bufferId = GFX_BUF_PEER_FLAGS), the neighbours open them (link 0 = the rank above, 1 = the rank below), and an
 * exchange is: push my seam rows into the neighbour's buffer, raise sequence `value` in its flag word, wait for my own
 * flag word to reach `value`.  All calls are asynchronous on `stream`.  gfx_peer_status reports whether a wait timed out
 * (neighbour died): the GPU is never left spinning. */
#define GFX_BUF_PEER_FLAGS (-1)
int gfx_peer_export(gfx_ctx* ctx, int bufferId, uint32_t index, void* handle64);
int gfx_peer_open(gfx_ctx* ctx, uint32_t link, int bufferId, uint32_t index, const void* handle64);
int gfx_peer_push_rows(gfx_ctx* ctx, void* stream, uint32_t link, int bufferId, uint32_t index, uint32_t rowLo, uint32_t rowHi);
int gfx_peer_signal(gfx_ctx* ctx, void* stream, uint32_t link, uint32_t flagIndex, uint32_t value);
int gfx_peer_wait(gfx_ctx* ctx, void* stream, uint32_t flagIndex, uint32_t value);
int gfx_peer_status(gfx_ctx* ctx, void* stream, uint32_t* timedOut);
int gfx_peer_close(gfx_ctx* ctx);

/* ---- scene, acceleration structure, light distributions ------------------------------ */
/* replaces Scene::initialize + createTriangleMeshes/createInstance uploads
 * (common/common_host.h:912-969, common/common_host.cpp:2178-2429,2582-2656) */
int gfx_scene_upload(gfx_ctx* ctx, const GfxSceneDesc* scene);
/* per-frame instance update (InstanceController::update, common/common_host.h:798-856) */
int gfx_scene_update_instances(gfx_ctx* ctx, void* stream, const GfxInstanceDesc* instances, uint32_t numInstances);

/* replaces Scene::updateASs (common/common_host.h:1027-1100): Morton-sorted LBVH over the
 * world-space triangles of all instances, collapsed to CompressedInternalNode_T<8>. */
/* flags: bits 0-7 = maximum triangles per leaf (0 = 2).  Hierarchy: default = top-down binned SAH (best trees, build
 * time in the tens of milliseconds: static scenes); GFX_BVH_BUILD_PLOC = PLOC clustering (within ~6 % of the SAH trees
 * in frame time, 8 ms for 2.9 M triangles); GFX_BVH_BUILD_FAST = Karras LBVH (fastest build, per-frame rebuilds of
 * animated scenes).  bits 16-23 = PLOC search radius (0 = 16, at most 64). */
#define GFX_BVH_BUILD_FAST 0x100u
#define GFX_BVH_BUILD_PLOC 0x200u
int gfx_bvh_build(gfx_ctx* ctx, void* stream, uint32_t flags);
int gfx_bvh_info(gfx_ctx* ctx, GfxBvhInfo* info);
/* read the built BVH back in the reference layout (host buffers sized from gfx_bvh_info) */
int gfx_bvh_export(gfx_ctx* ctx, GfxBvhNode8* nodes, uint32_t* primRefs, GfxTriangleStorage* tris);
/* adopt a BVH built elsewhere in the reference layout (e.g. by bvh::buildGeometryBVH<8>) */
int gfx_bvh_import(gfx_ctx* ctx, const GfxBvhNode8* nodes, uint32_t numNodes,
                   const uint32_t* primRefs, uint32_t numPrimRefs,
                   const GfxTriangleStorage* tris, uint32_t numTris);

/* wavefront trace: bvh::traverse<8> (common/bvh_builder.cpp:1653-1663) for a batch of rays.
 * rays/hits are DEVICE pointers in the _device variant and HOST pointers otherwise. */
int gfx_trace_device(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays,
                     GfxHitObject* hits, int mode);
int gfx_trace(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays,
              GfxHitObject* hits, int mode);
/* test hook of the traversal kernels: the records and modes of gfx_trace_device (DEVICE pointers) through kernel
 * 0 = the wavefront kernel of gfx_trace, 1 = the wavefront kernel with postponed leaf tests of the ReSTIR visibility queue
 * (mode GFX_TRACE_ANY only), 2 = the fused traversal of the G-buffer pass and the lighting any-hit test, one ray per thread.
 * Other kernels or modes: GFX_ERR_INVALID_ARGUMENT. */
int gfx_trace_debug(gfx_ctx* ctx, void* stream, const GfxRay* rays, uint32_t numRays,
                    GfxHitObject* hits, int mode, int kernel);

/* replaces Scene::setupLightGeomDistributions (static part, once) and
 * Scene::setupLightInstDistribution (per frame) + ext/cubd ExclusiveSum */
int gfx_light_dist_build(gfx_ctx* ctx, void* stream, uint32_t bufferIndex);
/* test hook for the flattened light pick that gfx_light_dist_build derives from those distributions: for n DEVICE floats ul in
 * [0, 1) writes the key (light-record index, or bit 30 set for sampleLight's probability-0 early outs,
 * restir_di_shared.h:356-409) found by the flattened table and by the three nested DiscreteDistribution1D::sample calls */
int gfx_light_pick_debug(gfx_ctx* ctx, void* stream, const float* ul, uint32_t n, uint32_t* keysFlat, uint32_t* keysChain);
/* test hook of the environment light (GfxSceneDesc::envTexels): n DEVICE pairs in, n DEVICE triples out.
 * op 0: RegularConstantContinuousDistribution2D::sample(u0, u1) -> (u, v, uvPDF); 1: evaluatePDF(u, v) -> (pdf, 0, 0);
 * 2: the software tex2DLod of the map at (u, v) -> rgb */
int gfx_env_light_debug(gfx_ctx* ctx, void* stream, int op, const float* in, uint32_t n, float* out);
/* test hook of light sampling as the renderers call it (lighting.cuh, pathtrace.cuh).  params: 3 HOST floats {envLightRotation,
 * envLightPowerCoeff, enableEnvLight != 0}, read as a frame's GfxFrameParams.  in / out: n DEVICE records of 16 floats each, unused
 * output slots 0, integers as their bits.
 * op 0: sampleLight(ul, u0, u1): in (ul, u0, u1); out (key of the flattened pick, position, normal, emittance, areaPDensity, the
 *       chain's lightProb (0 for a probability-0 early out), 0);
 * op 1: sampleLightUnlessDark(ul, u0, u1, shadingPoint, shadingNormal, vOutLocalZ): in (ul, u0, u1, point.xyz, normal.xyz,
 *       vOutLocalZ); out as op 0 with slot 12 = 1 for "dark";
 * op 2: classifyLight + finishLightSample (the two-phase candidate loop, guide entry from pickGuideFetch) on op 1's inputs and outputs;
 * op 3: sampleEnvLight(u0, u1): in (u0, u1); out (direction, areaPDensity, emittance);
 * op 4: the miss programs' density of the environment along a direction: in (direction, prevDirPDensity, probToSampleEnv); out
 *       (hypAreaPDensity, misWeight, u, v);
 * op 5: computeSurfacePointAtHit's hypAreaPDensity: in (instance slot, geometry index in the instance, primitive, bcB, bcC); out
 *       (hypAreaPDensity), 0 for indices out of range;
 * op 6: chooseEnvForCandidate(i, n, ul): in (i, n, ul); op 7: chooseEnvForNee(ul): in (ul); out (environment chosen, remapped ul,
 *       probToSampleCurLightType).
 * GFX_ERR_NOT_READY before gfx_scene_upload, before gfx_light_dist_build has built the light pick of the current transforms, and for
 * ops 3 and 4 without an environment map; GFX_ERR_INVALID_ARGUMENT for another op or a missing pointer. */
int gfx_light_sample_debug(gfx_ctx* ctx, void* stream, int op, const float* params, const float* in, uint32_t n, float* out);
/* test hook of the shading layer every renderer shares (BSDFs, sampling warps, encoders, frames); needs no scene.
 * material: 9 HOST floats {bsdfType, p0[3], p1[3], p2, regularize != 0}, read as setupBSDFBody reads a material with 1x1
 * textures (regularize = BSDFFlags::Regularize).  in / out: n DEVICE records of 8 floats each, unused output slots 0, integer
 * codes as their bits.  op 0: evaluate(vGiven, vSampled) -> rgb; 1: evaluatePDF(vGiven, vSampled); 2: sampleThroughput(vGiven,
 * u0, u1) -> (rgb, vSampled, dirPDensity); 3: evaluateDHReflectanceEstimate(vGiven) -> rgb; 4: concentricSampleDisk(u0, u1);
 * 5: cosineSampleHemisphere(u0, u1); 6: toPolarYUp(v) -> (phi, theta); 7: fromPolarYUp(phi, theta); 8: encodeVector(v);
 * 9: decodeVector(code); 10: encodeBarycentric(bc); 11: decodeBarycentric(code); 12: encodeTexCoords(u, v);
 * 13: decodeTexCoords(code); 14: makeCoordinateSystem(normal) -> (tangent, bitangent); 15: offsetRayOrigin(p, n).
 * GFX_ERR_INVALID_ARGUMENT for another op or a missing pointer. */
int gfx_shading_debug(gfx_ctx* ctx, void* stream, int op, const float* material, const float* in, uint32_t n, float* out);
/* test hook of the bump mapping (GfxSceneDesc::bumpMaps), n DEVICE records in and out:
 * op 0: readModifiedNormal of material matSlot's map at (u, v): 2 floats in, 3 out;
 * op 1: applyBumpMapping(modified normal, frame): 12 floats in (modified normal, tangent, bitangent, normal), 9 out (the frame);
 * op 2: the four channel-0 texels of the 2x2 footprint at (u, v) of material matSlot's map in tex2Dgather's order: 2 floats in,
 *       8 out = the software gather of the kernels, then the texture unit's tld4 on a CUDA texture object made from the same map
 *       (a uchar4 cudaArray holding round(255 texel), normalised-float read, repeat addressing, linear filter).
 * GFX_ERR_NOT_READY before gfx_scene_upload, GFX_ERR_INVALID_ARGUMENT for another op or a material slot out of range. */
int gfx_bump_debug(gfx_ctx* ctx, void* stream, int op, uint32_t matSlot, const float* in, uint32_t n, float* out);
/* host read-back of the instance-level distribution for parity: weights/cdf sized numInstances */
int gfx_light_dist_export(gfx_ctx* ctx, float* instWeights, float* instCdf, float* integral);

/* ---- frame state ---------------------------------------------------------------------- */
/* allocates G-buffers x2, reservoirs x2, rng, accumulation buffers (restir_di_main.cpp:1225-1330) */
int gfx_frame_create(gfx_ctx* ctx, uint32_t width, uint32_t height);
/* seeds one PCG32 per pixel, row-major, from std::mt19937_64(seed) (restir_di_main.cpp:1309-1321) */
int gfx_rng_seed(gfx_ctx* ctx, uint64_t seed);
/* Halton(2,3) concentric-disk neighbour table of 1024 entries (restir_di_main.cpp:1489-1542) */
int gfx_restir_setup_neighbor_table(gfx_ctx* ctx);
int gfx_buffer_download(gfx_ctx* ctx, void* stream, int bufferId, uint32_t index, void* host, size_t bytes);
int gfx_buffer_upload(gfx_ctx* ctx, void* stream, int bufferId, uint32_t index, const void* host, size_t bytes);
/* device pointer of a frame buffer (for NCCL collectives / torch views) */
void* gfx_buffer_device_ptr(gfx_ctx* ctx, int bufferId, uint32_t index, size_t* bytes);

/* counters accumulated by the frame kernels: out4[0] = rays traced (primary + visibility), others reserved */
int gfx_stats_read(gfx_ctx* ctx, void* stream, uint64_t* out4, int reset);

/* ---- launches -------------------------------------------------------------------------- */
/* replaces gBuffer.optixPipeline.launch (restir_di_main.cpp:2366; RG/CH/MS setupGBuffers) */
int gfx_gbuffer_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params);
/* replaces restir.setEntryPoint(pass) + restir.optixPipeline.launch (restir_di_main.cpp:2378-2421) */
int gfx_restir_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int pass);
/* replaces the svgf.cu kernels (svgf_main.cpp:2127-2172) */
int gfx_svgf_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int pass, uint32_t stage);
/* The SVGF app's "Buffer to Display" debug views: debugVisualize(bufferToDisplay, motionVectorOffset, motionVectorScale,
 * numFilteringStages) (svgf/gpu_kernels/visualize.cu:6-87).  Writes GFX_BUF_SVGF_DEBUG_VISUALIZE (allocated and zeroed on the
 * first call; downloading it before then is refused) on the rows params->tileOriginY / tileRows, pixel (x, y) of every plane to
 * pixel (x, y) of the view, w = 1.  The app launches Noisy Beauty and Variance after GFX_SVGF_ESTIMATE_VARIANCE and before the
 * first a-trous stage, only with SVGF on, and the other views after GFX_SVGF_MODULATE_TAA (svgf_main.cpp:2138-2145, 2175-2185).
 * Show the buffer with gfx_present_launch(GFX_PRESENT_COLOR): GFX_PRESENT_TONE_MAP | GFX_PRESENT_SRGB_GAMMA for Noisy Beauty,
 * Variance and Filtered Variance, no flags for the others (:1907-1911).  Final Rendering (the app's value 7) is not a view: it
 * is the present of GFX_BUF_SVGF_FINAL.
 *   NOISY_BEAUTY       lighting plane 0 rgb, x the SVGF albedo with GFX_SVGF_MODULATE_ALBEDO
 *   VARIANCE           sqrt(lighting plane 0 .w) in r, g and b
 *   FILTERED_VARIANCE  sqrt(lighting plane numFilteringStages % 2 .w); the app passes 5 with SVGF off too, so there it shows
 *                      plane 1 as the last frame with SVGF on left it
 *   ALBEDO             the SVGF albedo (the thresholded DH reflectance of the temporal pass; 1 at background pixels)
 *   NORMAL             0.5 n + 0.5 of the shading normal the temporal pass decoded.  The app reads its G-buffer, which it never
 *                      clears (svgf_main.cpp:2036-2042), so its background pixels show stale normals; here n = 0 there, and they
 *                      show (0.5, 0.5, 0.5).  The normal is not bump-mapped: the SVGF app has no bump mapping.
 *   MOTION_VECTOR      mv = (W, H) * ((x + 0.5, y + 0.5) / (W, H) - prevScreenPos), the prevScreenPos of the temporal pass (hits)
 *                      and of GFX_SVGF_FILL_BACKGROUND (background); clamp(scale * mv + offset, 0, 1) in r and g, b = offset
 *   SAMPLE_COUNT       min(count / 255, 1), count = the low 24 bits of GFX_BUF_SVGF_MOMENTS[params->bufferIndex].z
 * The app passes offset 0.5 and scale 10^-1 (its slider's default, :1724, 2143) and 5 stages.  A view outside 0..6:
 * GFX_ERR_INVALID_ARGUMENT; before gfx_frame_create: GFX_ERR_NOT_READY. */
typedef enum GfxSVGFView {            /* shared::BufferToDisplay (svgf_shared.h:247-256), same numbers */
    GFX_SVGF_VIEW_NOISY_BEAUTY = 0, GFX_SVGF_VIEW_VARIANCE = 1, GFX_SVGF_VIEW_FILTERED_VARIANCE = 2,
    GFX_SVGF_VIEW_ALBEDO = 3, GFX_SVGF_VIEW_NORMAL = 4, GFX_SVGF_VIEW_MOTION_VECTOR = 5, GFX_SVGF_VIEW_SAMPLE_COUNT = 6
} GfxSVGFView;
int gfx_svgf_debug_visualize(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int view,
                             float motionVectorOffset, float motionVectorScale, uint32_t numFilteringStages);
/* replaces pathTracing.setEntryPoint(variant) + pathTracing.optixPipeline.launch (path_tracing_main.cpp:1780-1789):
 * one sample per pixel of the unidirectional path tracer (NEE + MIS + Russian roulette, params->maxPathLength)
 * starting from the G-buffer of params->bufferIndex; running mean into GFX_BUFFER_BEAUTY_ACCUM. */
int gfx_pathtrace_launch(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, int variant);

/* ---- batched launches ------------------------------------------------------------------------
 * One call for a list of launches (a whole strip frame of the multi-GPU driver: ~35 kernels in ~1.3 ms at 8 GPUs, where one
 * host round trip per launch through a binding layer would make the host the bottleneck).  Each record is executed in order on
 * `stream` exactly like the entry point it names: GFX_OP_LIGHT_DIST = gfx_light_dist_build(a = bufferIndex), GFX_OP_GBUFFER =
 * gfx_gbuffer_launch(params), GFX_OP_RESTIR = gfx_restir_launch(params, a = pass), GFX_OP_PEER_PUSH_ROWS =
 * gfx_peer_push_rows(a = link, b = buffer id, c = index, d = rowLo, e = rowHi), GFX_OP_PEER_SIGNAL = gfx_peer_signal(a = link,
 * b = flag index, c = value), GFX_OP_PEER_WAIT = gfx_peer_wait(a = flag index, b = value).  Stops at the first failing record
 * and returns its status. */
#define GFX_OP_LIGHT_DIST 0
#define GFX_OP_GBUFFER 1
#define GFX_OP_RESTIR 2
#define GFX_OP_PEER_PUSH_ROWS 3
#define GFX_OP_PEER_SIGNAL 4
#define GFX_OP_PEER_WAIT 5
typedef struct GfxBatchOp {
    uint32_t op;
    uint32_t a, b, c, d, e;
    uint32_t pad[2];
    GfxFrameParams params;
} GfxBatchOp;
int gfx_launch_batch(gfx_ctx* ctx, void* stream, const GfxBatchOp* ops, uint32_t numOps);

/* One ReSTIR DI frame of a screen strip, every launch of it, in one call: what restir_di_main.cpp:2303-2421 does per frame
 * (light distribution, G-buffer, initial(+temporal) RIS, spatial passes, shading; `params` is mutated between launches exactly
 * like the host mutates plp, and left as after the last launch) restricted to the rows [y0, y1) of rank `rank` of `world`, with
 * the G-buffer recomputed on `halo` more rows on each side and the reservoir / reservoir-info seam rows exchanged with the
 * neighbour ranks by one-sided pushes over the peer links opened with gfx_peer_open (usePeer = 1; *peerSeq is the running
 * sequence number of the exchanges, in/out).  world = 1 renders the full frame (y0 = 0, y1 = H).  The caller all-gathers the
 * beauty strips afterwards (gfx_framebuffer_allgather or its own collective). */
typedef struct GfxStripFrame {
    uint32_t frameIndex, numSpatialPasses, unbiased, temporal;
    uint32_t y0, y1, halo;
    uint32_t rank, world, usePeer;
    uint32_t peerSeq;
} GfxStripFrame;
int gfx_restir_strip_frame(gfx_ctx* ctx, void* stream, GfxFrameParams* params, GfxStripFrame* strip);

/* The one mandatory collective of a strip-sharded frame (SURVEY.md 8e-1): all-gathers the composited beauty strips.  Rank r of
 * the communicator contributes the rows [r * rowsPerRank, (r + 1) * rowsPerRank) of its GFX_BUF_BEAUTY_ACCUM; `dstFramebuffer`
 * (DEVICE, W * H float4, may be the beauty buffer itself: in-place all-gather) receives the full frame on every rank.
 * `ncclComm` is the host's ncclComm_t; the library resolves the NCCL entry points at the call from the NCCL the process has
 * loaded (it never loads one itself), so libgfxb200.so has no link-time NCCL dependency.  Stream-ordered on `stream`. */
int gfx_framebuffer_allgather(gfx_ctx* ctx, void* ncclComm, void* stream, uint32_t rowsPerRank, void* dstFramebuffer);
/* the same for strips of unequal height (cost-balanced strips): rank r owns rows [rowStarts[r], rowStarts[r + 1]), rowStarts has
 * world + 1 entries; one ncclBroadcast per strip inside an NCCL group (= one launch) */
int gfx_framebuffer_allgatherv(gfx_ctx* ctx, void* ncclComm, void* stream, const uint32_t* rowStarts, uint32_t world, void* dstFramebuffer);

/* ---- ReGIR cell reservoirs (regir_main.cpp:2033-2068) --------------------------------- */
/* replaces kernelBuildCellReservoirs / kernelBuildCellReservoirsAndTemporalReuse (build_cell_reservoirs.cu:71-233):
 * streaming RIS of 2^log2NumCandidatesPerLightSlot light samples per slot against the intensity reaching the cell,
 * optionally merged with the slot's reservoir of the previous frame; cells unused for more than 8 frames are skipped */
int gfx_regir_build_cells(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t frameIndex, int useTemporalReuse);
/* replaces kernelUpdateLastAccessFrameIndices (build_cell_reservoirs.cu:235-248), after the path tracer */
int gfx_regir_update_access(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t frameIndex);

/* ---- NRC network (network_interface.h:14-28) ------------------------------------------ */
typedef struct gfx_nrc gfx_nrc;
/* numHiddenLayers: 1..8 (GFX_ERR_INVALID_ARGUMENT otherwise), and only depths whose training and inference kernels fit in
 * the device's shared memory per block (cudaDevAttrMaxSharedMemoryPerBlockOptin); a deeper network is rejected with
 * GFX_ERR_UNSUPPORTED and an error string that names the kernel, its need and the limit.  On an H100 (232 448 bytes)
 * that is 1..7: at 8 the CUDA-core training kernel (the only one for more than 3 hidden layers) needs 236 544 bytes of
 * dynamic shared memory alone.  gfx_nrc_create builds the hash-grid network: it is
 * gfx_nrc_create_with_encoding(ctx, GFX_NRC_POSITION_ENCODING_HASH_GRID, ...). */
int gfx_nrc_create(gfx_ctx* ctx, uint32_t numHiddenLayers, float learningRate, gfx_nrc** out);
/* NeuralRadianceCache::initialize(posEnc, numHiddenLayers, learningRate) (network_interface.cu:48-121); the values are those
 * of PositionEncoding (network_interface.h:5-8).  The position (query floats 0..2) is encoded by
 *   TRIANGLE_WAVE  TriangleWave(12 frequencies): network inputs 0..35, input 12 d + f of position dim d and frequency f
 *                  (triangle_wave.h:47-81); OneBlob 36..55, Identity 56..61, ones 62..63.  The encoding has no parameters:
 *                  numParams = the MLP's matrix weights.  Adam epsilon 1e-8.
 *   HASH_GRID      HashGrid(16 levels x 2 features): inputs 0..31; OneBlob 32..51, Identity 52..57, ones 58..63.
 *                  numParams = matrix weights + 991 232 grid entries.  Adam epsilon 1e-15.
 * Any other value is GFX_ERR_INVALID_ARGUMENT.  The depth limits are the same for both.  Switching the encoding at run
 * time is gfx_nrc_destroy + create, as in the reference. */
#define GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE 0
#define GFX_NRC_POSITION_ENCODING_HASH_GRID 1
int gfx_nrc_create_with_encoding(gfx_ctx* ctx, int positionEncoding, uint32_t numHiddenLayers, float learningRate,
                                 gfx_nrc** out);
void gfx_nrc_destroy(gfx_nrc* nrc);
/* inputData: device float[14, numData] (column per query), predictionData: device float[3, numData];
 * numData % 128 == 0 (network_interface.cu:141-147) */
int gfx_nrc_infer(gfx_nrc* nrc, void* stream, const float* inputData, float* predictionData, uint32_t numData);
int gfx_nrc_train(gfx_nrc* nrc, void* stream, const float* inputData, const float* targetData,
                  uint32_t numData, float* lossOnHost);
/* gfx_nrc_create leaves the cache as NeuralRadianceCache::initialize leaves tiny-cuda-nn's Trainer (seed 1337): Xavier-uniform MLP
 * matrices and U(-1e-4, 1e-4) hash-grid entries drawn from pcg32 in tiny-cuda-nn's order (trainer.h:54-109, gpu_matrix.h:292-307,
 * grid.h:1267-1272, random.h:65-100), fp32 master = those values, training weights = their halves, inference (EMA) weights and
 * optimizer state zero.  gfx_nrc_reset re-initialises with another Trainer seed.  A triangle-wave network draws the same
 * matrices (the same pcg32 prefix) and nothing after them. */
int gfx_nrc_reset(gfx_nrc* nrc, uint32_t seed);
/* state read-back for parity tests.  which: MASTER fp32[numParams]; TRAINING / INFERENCE half[numParams];
 * GRADIENTS fp32[numParams] = the loss-scaled (x128) gradients of the last gfx_nrc_train, rounded to half like
 * tiny-cuda-nn's gradient buffer (only after gfx_nrc_keep_gradients(nrc, 1)) */
#define GFX_NRC_READ_MASTER 0
#define GFX_NRC_READ_TRAINING 1
#define GFX_NRC_READ_INFERENCE 2
#define GFX_NRC_READ_GRADIENTS 3
int gfx_nrc_read(gfx_nrc* nrc, int which, void* hostOut, size_t bytes);
int gfx_nrc_keep_gradients(gfx_nrc* nrc, int on);
/* test hook: the encoded network input of numData DEVICE queries as gfx_nrc_infer's kernels produce it, 64 halves per query:
 * hash grid: HashGrid 32 | OneBlob 20 | Identity 6 | ones 6 (kernel_grid grid.h:132-255, kernel_one_blob_soa oneblob.h:110-139);
 * triangle wave: TriangleWave 36 | OneBlob 20 | Identity 6 | ones 2 (triangle_wave.h:47-81). */
int gfx_nrc_encode_debug(gfx_nrc* nrc, void* stream, const float* inputData, uint32_t numData, void* outHalf);
/* inference (EMA) weights as halves; gfx_nrc_set_params installs the same values as training, inference and master weights and
 * clears the optimizer state */
int gfx_nrc_get_params(gfx_nrc* nrc, void* hostHalfParams, size_t bytes);
int gfx_nrc_set_params(gfx_nrc* nrc, const void* hostHalfParams, size_t bytes);
uint32_t gfx_nrc_num_params(gfx_nrc* nrc);

/* ---- NRC frame: the launches around gfx_pathtrace_launch(GFX_PT_NRC) (neural_radiance_caching_main.cpp:2270-2368).
 * Buffers live in the frame (GFX_BUF_NRC_*); nothing in the sequence reads back to the host. ------------- */
/* replaces kernelPreprocessNRC (:2270-2276; nrc_setup_kernels.cu:6-49): tile-size controller, training-suffix reset */
int gfx_nrc_preprocess(gfx_ctx* ctx, void* stream, const GfxFrameParams* params, uint32_t offsetToSelectUnbiasedTile,
                       uint32_t offsetToSelectTrainingPath, int isNewSequence);
/* replaces neuralRadianceCache.infer on inferenceRadianceQueryBuffer (:2309-2316); the query count
 * pad128(W*H + #tiles) is read from device memory instead of synchronising with the host (:2291-2304) */
int gfx_nrc_frame_infer(gfx_ctx* ctx, gfx_nrc* nrc, void* stream);
/* replaces kernelAccumulateInferredRadianceValues / kernelPropagateRadianceValues / kernelShuffleTrainingData
 * (:2320-2348; nrc_setup_kernels.cu:51-92, 94-138, 140-216) */
/* gfx_nrc_accumulate after gfx_pathtrace_launch(GFX_PT_NRC_INDIRECT) (the context's last NRC path-trace launch) adds instead:
 * beauty += w * (frame contribution + alpha * cache), w = 1 / (1 + params->numAccumFrames).  Precondition: this frame's ReSTIR DI
 * shading pass has blended its direct light D into GFX_BUF_BEAUTY_ACCUM with the same numAccumFrames; the beauty is then the
 * running mean of D + the NRC path tracer's light beyond the primary vertex (ReSTIR DI + NRC as one estimator). */
int gfx_nrc_accumulate(gfx_ctx* ctx, void* stream, const GfxFrameParams* params);
int gfx_nrc_propagate(gfx_ctx* ctx, void* stream, const GfxFrameParams* params);
int gfx_nrc_shuffle(gfx_ctx* ctx, void* stream, const GfxFrameParams* params);
/* replaces the four neuralRadianceCache.train steps on quarters of the shuffled records (:2350-2365) */
int gfx_nrc_frame_train(gfx_ctx* ctx, gfx_nrc* nrc, void* stream, float* lossOnHost);

/* ---- NRC frame sharded by strips of rows over the ranks of one node (BASELINE config 5: ReSTIR DI + NRC, 3840x2160, 8 GPUs).
 * No counterpart in the reference (one GPU).  After gfx_nrc_shard every rank runs the sequence above on ITS rows
 * (params->tileOriginY / tileRows; gfx_nrc_frame_infer_rows instead of gfx_nrc_frame_infer) and all ranks must make the same
 * calls in the same order on `stream`:
 *   - gfx_pathtrace_launch(GFX_PT_NRC) numbers the training vertices over the whole frame: per path-tracing round one
 *     ncclAllGather of one word per rank (the vertex counts), so records, tile-size controller and buffer-overflow
 *     behaviour are those of the unsharded frame, bit for bit;
 *   - gfx_nrc_propagate ends with an ncclAllReduce (unsigned sum; every record is non-zero on one rank only) that leaves all
 *     records on all ranks; gfx_nrc_shuffle / gfx_nrc_frame_train then run replicated and keep the weights identical
 *     (the gradient accumulation is integer, hence order-independent).
 * ncclComm is the host's ncclComm_t over exactly `world` ranks; NULL or world <= 1 switches sharding off. */
int gfx_nrc_shard(gfx_ctx* ctx, void* ncclComm, int rank, int world);
/* inference of the rows [rowLo, rowHi) of the frame's terminal queries + the training-suffix queries of all tiles;
 * rowLo * width and width * height must be multiples of 128 */
int gfx_nrc_frame_infer_rows(gfx_ctx* ctx, gfx_nrc* nrc, void* stream, uint32_t rowLo, uint32_t rowHi);

#ifdef __cplusplus
}
#endif
#endif /* GFXB200_H */
