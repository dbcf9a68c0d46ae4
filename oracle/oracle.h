/* oracle/oracle.h — C API of the CPU oracle.  TEST INFRASTRUCTURE: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * liboracle.so.  The product library (libgfxb200.so) never links or calls it.
 *
 * The scene/parameter PODs are the ones of include/gfxb200.h (the interface spec), so one
 * set of host arrays feeds both sides of a parity test.
 *
 * Parity status (also in DESIGN.md): the reference has no golden vectors for this path and
 * cannot be built here, so this oracle is "parity unpinned" against the reference binary;
 * it is pinned against (a) the reference's struct-size static_asserts, (b) brute-force
 * closest-hit, (c) libm for detmath, (d) the analytic RIS expectation of
 * restir_di/RIS_Test/ris_test.ipynb (tests/test_oracle_*.py).
 */
#ifndef ORACLE_H
#define ORACLE_H
#include "../include/gfxb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_scene orc_scene;
typedef struct orc_frame orc_frame;

typedef struct OrcBuildConfig { /* bvh::GeometryBVHBuildConfig, common/bvh_builder.h:38-44 */
    float splittingBudget;
    float intNodeTravCost;
    float primIntersectCost;
    uint32_t minNumPrimsPerLeaf;
    uint32_t maxNumPrimsPerLeaf;
} OrcBuildConfig;

typedef struct OrcTraversalStats { /* bvh::TraversalStatistics (bvh_builder.h:79-86), summed over rays */
    uint64_t numAabbTests;
    uint64_t numTriTests;
    uint64_t numIntNodes;
    int32_t maxStackDepth;
    uint32_t numHits;
} OrcTraversalStats;

enum { ORC_TRACE_FIRST_FOUND = 0, ORC_TRACE_CANONICAL = 1, ORC_TRACE_BRUTE_FORCE = 2, ORC_TRACE_ANY = 3 };

/* scene = flattened geometries + SBVH (bvh::buildGeometryBVH<8>) + light distributions */
orc_scene* orc_scene_create(const GfxSceneDesc* scene, const OrcBuildConfig* cfg, int numThreads);
void orc_scene_destroy(orc_scene* s);
/* new instance transforms -> rebuild of the world-space BVH and of the light distributions; 0 on success */
int orc_scene_update_instances(orc_scene* s, const GfxInstanceDesc* instances, uint32_t numInstances);
double orc_scene_build_seconds(orc_scene* s);
void orc_bvh_info(orc_scene* s, GfxBvhInfo* info);
void orc_bvh_export(orc_scene* s, GfxBvhNode8* nodes, uint32_t* primRefs, GfxTriangleStorage* tris);
/* replace the BVH by one given in the reference layout (e.g. exported from the GPU builder) */
void orc_bvh_import(orc_scene* s, const GfxBvhNode8* nodes, uint32_t numNodes,
                    const uint32_t* primRefs, uint32_t numPrimRefs,
                    const GfxTriangleStorage* tris, uint32_t numTris);
/* structural validation of a BVH in the reference layout: every triangle referenced at least
 * once, every child box contains its subtree, leaf chains terminated. returns 0 if valid. */
int orc_bvh_validate(orc_scene* s, char* msg, size_t msgLen);
/* replace the BVH by the tree gfx_bvh_build(flags) builds on the GPU (gpu_bvh.cpp: binned SAH, or LBVH with
 * GFX_BVH_BUILD_FAST); -1 for GFX_BVH_BUILD_PLOC.  Works on a scene created without an SBVH build. */
int orc_bvh_build_gpu_style(orc_scene* s, uint32_t flags);
/* { small, big, huge } node counts of each level of the last SAH build above (at most maxLevels triples); returns the
 * number of levels */
uint32_t orc_bvh_sah_levels(orc_scene* s, uint32_t* counts, uint32_t maxLevels);
/* 0 if the two BVHs are the same tree: walked from the roots in parallel, every node field except the two base indices
 * and every leaf's reference words are equal; else 1 and the first difference, as a slot path from the root, in msg */
int orc_bvh_same_tree(orc_scene* a, orc_scene* b, char* msg, size_t msgLen);
void orc_trace(orc_scene* s, const GfxRay* rays, uint32_t numRays, GfxHitObject* hits, int mode,
               OrcTraversalStats* stats, int numThreads);
void orc_light_dist_export(orc_scene* s, float* instWeights, float* instCdf, float* integral);
/* environment light test hooks: op 0 sample (u0, u1) -> (u, v, uvPDF); 1 evaluatePDF(u, v); 2 texture fetch (u, v) -> rgb;
 * n pairs in, n triples out; -1 if the scene has no environment map */
int orc_env_query(orc_scene* s, int op, const float* in, uint32_t n, float* out);
int orc_light_sample_debug(orc_scene* s, int op, const float* params, const float* in, uint32_t n, float* out);

orc_frame* orc_frame_create(orc_scene* s, uint32_t width, uint32_t height);
void orc_frame_destroy(orc_frame* f);
void orc_rng_seed(orc_frame* f, uint64_t seed);
void orc_restir_setup_neighbor_table(orc_frame* f);
void* orc_buffer_ptr(orc_frame* f, int bufferId, uint32_t index, size_t* bytes);
/* measurement aid: enable / read-and-reset the candidate statistics of the initial RIS loop (5 counters, see render.cpp) */
void orc_ris_stats(int enable, unsigned long long* out5);
/* rays traced by the renderer entry points since the last reset (all threads) */
unsigned long long orc_rays_traced(int reset);
/* output side: float4 image -> tone-mapped / sRGB-encoded RGBA8 (present.cpp) */
void orc_present(const float* srcRGBA, uint32_t width, uint32_t height, const GfxPresentParams* config, uint32_t* image);
void orc_gbuffer(orc_frame* f, const GfxFrameParams* p, int numThreads);
void orc_restir(orc_frame* f, const GfxFrameParams* p, int pass, int numThreads);
/* unidirectional path tracer (GfxPathTraceVariant); returns the number of rays traced */
// GFX_PT_REGIR before a ReGIR build returns ORC_NOT_READY (the library returns GFX_ERR_NOT_READY) and writes nothing
#define ORC_NOT_READY UINT64_MAX
uint64_t orc_pathtrace(orc_frame* f, const GfxFrameParams* p, int variant, int numThreads);
/* rearchitected ReSTIR passes GFX_RESTIR_PRESAMPLE_LIGHTS .. GFX_RESTIR_SHADE_AND_RESAMPLE; returns shadow rays traced */
uint64_t orc_restir_rearch(orc_frame* f, const GfxFrameParams* p, int pass, int numThreads);
/* ReGIR (build_cell_reservoirs.cu): buildCellReservoirs[AndTemporalReuse], updateLastAccessFrameIndices;
 * buffers via orc_buffer_ptr(GFX_BUF_REGIR_*) once the grid exists */
void orc_regir_build_cells(orc_frame* f, const GfxFrameParams* p, uint32_t frameIndex, int useTemporalReuse, int numThreads);
void orc_regir_update_access(orc_frame* f, const GfxFrameParams* p, uint32_t frameIndex);
/* NRC bookkeeping kernels (nrc_setup_kernels.cu): preprocessNRC, accumulateInferredRadianceValues,
 * propagateRadianceValues, shuffleTrainingData; buffers via orc_buffer_ptr(GFX_BUF_NRC_*) */
void orc_nrc_preprocess(orc_frame* f, const GfxFrameParams* p, uint32_t offsetToSelectUnbiasedTile,
                        uint32_t offsetToSelectTrainingPath, int isNewSequence);
/* strip sharding of the NRC frame over ranks (the oracle's restatement of gfx_nrc_shard, for the gloo tests of the host logic):
 * `exchange` all-gathers numWords words per rank, `sum` all-reduces an unsigned 32-bit array in place; world <= 1 switches it off */
void orc_nrc_set_shard(orc_frame* f, int rank, int world, void (*exchange)(void* user, const uint32_t* mine, uint32_t numWords, uint32_t* all),
                       void (*sum)(void* user, uint32_t* words, uint64_t numWords), void* user);
void orc_nrc_accumulate(orc_frame* f, const GfxFrameParams* p);
void orc_nrc_propagate(orc_frame* f, const GfxFrameParams* p);
void orc_nrc_shuffle(orc_frame* f, const GfxFrameParams* p);
/* primary rays of the G-buffer pass (for the trace-only benchmarks) */
void orc_generate_primary_rays(const GfxFrameParams* p, uint32_t width, uint32_t height, GfxRay* rays);

#ifdef __cplusplus
}
#endif
#endif
