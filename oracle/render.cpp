// oracle/render.cpp — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// Per-pixel CPU restatement of the reference's G-buffer and ReSTIR DI programs:
//   setupGBuffers RG/CH/MS          restir_di/gpu_kernels/optix_gbuffer_kernels.cu:5-243
//   sampleLight<false>              restir_di/restir_di_shared.h:320-516
//   performDirectLighting           restir_di/restir_di_shared.h:518-557
//   evaluateVisibility              restir_di/restir_di_shared.h:559-582
//   testNeighbor                    restir_di/restir_di_shared.h:747-771
//   performInitialAndTemporalRIS    restir_di/gpu_kernels/optix_restir_di_kernels.cu:14-287
//   performSpatialRIS               restir_di/gpu_kernels/optix_restir_di_kernels.cu:303-547
//   shading                         restir_di/gpu_kernels/optix_restir_di_kernels.cu:559-637
//   light importance + CDFs         common/gpu_kernels/compute_light_probs.cu:22-46,68-82,115-174
// optixTrace is replaced by the restated bvh::traverse (canonical tie-break) — see bvh.h.
// Environment lights are not part of the synthetic configs (SURVEY.md §8a S3) and are omitted.
#include "oracle.h"
#include "bvh.h"
#include "shading.h"
#include "envlight.h"
#include <chrono>
#include <cstdio>
#include <random>
#include <vector>
#include <omp.h>

using namespace orc;

struct MeshData {
    std::vector<float> positions, normals, tangents, texcoords;
    std::vector<uint32_t> triangles;
    uint32_t numVertices, numTriangles, materialSlot;
    // emitterPrimDist (GeometryInstanceData::emitterPrimDist)
    std::vector<float> primWeights, primCdf;
    float primIntegral = 0.0f;
};
struct InstData {
    GfxInstanceDesc desc;
    std::vector<float> geomWeights, geomCdf; // lightGeomInstDist
    float geomIntegral = 0.0f;
};

struct orc_scene {
    std::vector<MeshData> meshes;
    std::vector<GfxMaterialDesc> materials;
    std::vector<InstData> instances;
    std::vector<uint32_t> instanceMeshSlots;
    // flattened geometry g -> (instance, mesh slot)
    std::vector<uint32_t> geomToInst, geomToMesh;
    GeometryBVH bvh;
    std::vector<uint32_t> sahLevels; // { small, big, huge } nodes per level of the last orc_bvh_build_gpu_style SAH build
    std::vector<float> instWeights, instCdf; // lightInstDist
    float instIntegral = 0.0f;
    double buildSeconds = 0.0;
    float sceneMin[3], sceneMax[3];
    OrcBuildConfig buildConfig;
    EnvLight env; // envLightTexture + envLightImportanceMap (restir_di_shared.h:221-222)
    std::vector<ImageTexture> textures;      // image textures of the materials ...
    std::vector<uint32_t> materialTextures;  // ... [4 * m + k]: texture of p0 / p1 / p2 / emittance or 0xFFFFFFFF (empty = none)
};

// plp.s->envLightTexture && plp.f->enableEnvLight; a map that is black everywhere (importance integral 0) is no light to sample
// and counts as none, as in the library (DESIGN.md, "Environment maps with black rows")
static inline bool useEnvLight(const orc_scene* s, const GfxFrameParams* p) {
    return s->env.present() && s->env.topIntegral > 0.0f && p->enableEnvLight;
}

// sequential fp32 exclusive scan (stands in for ext/cubd ExclusiveSum; SURVEY.md §8c item 4)
static float exclusiveScan(const std::vector<float> &w, std::vector<float> &cdf) {
    cdf.resize(w.size());
    float sum = 0.0f;
    for (size_t i = 0; i < w.size(); ++i) {
        cdf[i] = sum;
        sum = sum + w[i];
    }
    // DiscreteDistribution1D::finalize: integral = CDF[last] + weights[last] (common_shared.h:268-271)
    return w.empty() ? 0.0f : cdf.back() + w.back();
}

static inline float3 ld3(const std::vector<float> &a, uint32_t i) { return float3(a[3 * i], a[3 * i + 1], a[3 * i + 2]); }
static inline float2 ld2(const std::vector<float> &a, uint32_t i) { return float2(a[2 * i], a[2 * i + 1]); }
static inline Affine affine(const float* m) { Affine a; std::memcpy(a.m, m, 48); return a; }
static inline Mat3 mat3(const float* m) { Mat3 a; std::memcpy(a.m, m, 36); return a; }

static void buildLightDistributions(orc_scene* s) {
    // computeTriangleImportance (compute_light_probs.cu:22-46): lum(mean emittance at 3 verts) * area
    for (MeshData &mesh : s->meshes) {
        const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];
        mesh.primWeights.assign(mesh.numTriangles, 0.0f);
        for (uint32_t t = 0; t < mesh.numTriangles; ++t) {
            const float3 p0 = ld3(mesh.positions, mesh.triangles[3 * t + 0]);
            const float3 p1 = ld3(mesh.positions, mesh.triangles[3 * t + 1]);
            const float3 p2 = ld3(mesh.positions, mesh.triangles[3 * t + 2]);
            const float3 normal = cross(p1 - p0, p2 - p0);
            const float area = 0.5f * length(normal);
            float3 emittanceEstimate(0.0f);
            // tex2DLod(mat.emittance = 0, ...) reads zeros for a null texture object
            const float3 e = mat.hasEmittance ? float3(mat.emittance[0], mat.emittance[1], mat.emittance[2]) : float3(0.0f);
            emittanceEstimate += e;
            emittanceEstimate += e;
            emittanceEstimate += e;
            emittanceEstimate /= 3;
            mesh.primWeights[t] = sRGB_calcLuminance(emittanceEstimate) * area;
        }
        mesh.primIntegral = exclusiveScan(mesh.primWeights, mesh.primCdf);
    }
    // computeGeomInstImportance (:68-82) and computeInstImportance (:115-129)
    s->instWeights.assign(s->instances.size(), 0.0f);
    for (size_t i = 0; i < s->instances.size(); ++i) {
        InstData &inst = s->instances[i];
        inst.geomWeights.assign(inst.desc.numMeshSlots, 0.0f);
        for (uint32_t k = 0; k < inst.desc.numMeshSlots; ++k)
            inst.geomWeights[k] = s->meshes[s->instanceMeshSlots[inst.desc.firstMeshSlot + k]].primIntegral;
        inst.geomIntegral = exclusiveScan(inst.geomWeights, inst.geomCdf);
        s->instWeights[i] = pow2(inst.desc.uniformScale) * inst.geomIntegral;
    }
    s->instIntegral = exclusiveScan(s->instWeights, s->instCdf);
}

// (instance, mesh) pairs flattened into bvh::Geometry records in instance order
static std::vector<Geometry> collectGeometries(orc_scene* s) {
    s->geomToInst.clear();
    s->geomToMesh.clear();
    const uint32_t numInstances = (uint32_t)s->instances.size();
    // flatten (instance, mesh) pairs into bvh::Geometry records in instance order
    std::vector<Geometry> geoms;
    for (uint32_t i = 0; i < numInstances; ++i) {
        const GfxInstanceDesc &inst = s->instances[i].desc;
        for (uint32_t k = 0; k < inst.numMeshSlots; ++k) {
            const uint32_t meshSlot = s->instanceMeshSlots[inst.firstMeshSlot + k];
            const MeshData &m = s->meshes[meshSlot];
            Geometry g;
            g.vertices = reinterpret_cast<const uint8_t*>(m.positions.data());
            g.vertexStride = 12;
            g.numVertices = m.numVertices;
            g.triangles = m.triangles.data();
            g.numTriangles = m.numTriangles;
            g.preTransform = affine(inst.transform);
            geoms.push_back(g);
            s->geomToInst.push_back(i);
            s->geomToMesh.push_back(meshSlot);
        }
    }
    return geoms;
}

static void updateSceneBounds(orc_scene* s) {
    AABB box;
    for (const TriangleStorage &ts : s->bvh.triStorages) {
        box.unify(float3(ts.pA[0], ts.pA[1], ts.pA[2]));
        box.unify(float3(ts.pB[0], ts.pB[1], ts.pB[2]));
        box.unify(float3(ts.pC[0], ts.pC[1], ts.pC[2]));
    }
    for (int i = 0; i < 3; ++i) {
        s->sceneMin[i] = box.minP[i];
        s->sceneMax[i] = box.maxP[i];
    }
}

// world-space side of the scene: flattened geometry, BVH, bounds, light distributions
static void rebuildWorld(orc_scene* s, int numThreads) {
    const OrcBuildConfig* cfg = &s->buildConfig;
    s->bvh = GeometryBVH();
    s->sahLevels.clear();
    const std::vector<Geometry> geoms = collectGeometries(s);
    BuildConfig bc;
    bc.splittingBudget = cfg->splittingBudget;
    bc.intNodeTravCost = cfg->intNodeTravCost;
    bc.primIntersectCost = cfg->primIntersectCost;
    bc.minNumPrimsPerLeaf = cfg->minNumPrimsPerLeaf;
    bc.maxNumPrimsPerLeaf = cfg->maxNumPrimsPerLeaf;
    const auto t0 = std::chrono::steady_clock::now();
    // numThreads < 0: no SBVH build; the caller imports a BVH built elsewhere (orc_bvh_import) before tracing.
    // Used to validate / walk a GPU-built BVH of a scene whose single-threaded CPU build would take minutes.
    if (numThreads >= 0)
        buildGeometryBVH(geoms.data(), (uint32_t)geoms.size(), bc, &s->bvh);
    const auto t1 = std::chrono::steady_clock::now();
    s->buildSeconds = std::chrono::duration<double>(t1 - t0).count();
    updateSceneBounds(s);
    buildLightDistributions(s);
}

// the tree gfx_bvh_build(flags) emits (gpu_bvh.cpp) replaces the scene's BVH; works on a scene created without an SBVH
extern "C" int orc_bvh_build_gpu_style(orc_scene* s, uint32_t flags) {
    const std::vector<Geometry> geoms = collectGeometries(s);
    GeometryBVH bvh;
    std::vector<uint32_t> levels;
    const auto t0 = std::chrono::steady_clock::now();
    if (buildGpuStyleBVH(geoms.data(), (uint32_t)geoms.size(), flags, &bvh, &levels) != 0)
        return -1;
    s->buildSeconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    s->bvh = std::move(bvh);
    s->sahLevels = std::move(levels);
    updateSceneBounds(s);
    return 0;
}
extern "C" uint32_t orc_bvh_sah_levels(orc_scene* s, uint32_t* counts, uint32_t maxLevels) {
    const uint32_t numLevels = (uint32_t)(s->sahLevels.size() / 3);
    if (counts)
        std::memcpy(counts, s->sahLevels.data(), 3 * (size_t)std::min(numLevels, maxLevels) * 4);
    return numLevels;
}
extern "C" int orc_bvh_same_tree(orc_scene* a, orc_scene* b, char* msg, size_t msgLen) {
    const std::string d = sameTree(a->bvh, b->bvh);
    if (msgLen)
        snprintf(msg, msgLen, "%s", d.c_str());
    return d.empty() ? 0 : 1;
}

extern "C" orc_scene* orc_scene_create(const GfxSceneDesc* d, const OrcBuildConfig* cfg, int numThreads) {
    orc_scene* s = new orc_scene();
    s->meshes.resize(d->numMeshes);
    for (uint32_t i = 0; i < d->numMeshes; ++i) {
        const GfxMeshDesc &md = d->meshes[i];
        MeshData &m = s->meshes[i];
        m.numVertices = md.numVertices;
        m.numTriangles = md.numTriangles;
        m.materialSlot = md.materialSlot;
        m.positions.assign(md.positions, md.positions + 3 * (size_t)md.numVertices);
        m.normals.assign(md.normals, md.normals + 3 * (size_t)md.numVertices);
        m.tangents.assign(md.tangents, md.tangents + 3 * (size_t)md.numVertices);
        m.texcoords.assign(md.texcoords, md.texcoords + 2 * (size_t)md.numVertices);
        m.triangles.assign(md.triangles, md.triangles + 3 * (size_t)md.numTriangles);
    }
    s->materials.assign(d->materials, d->materials + d->numMaterials);
    s->instances.resize(d->numInstances);
    for (uint32_t i = 0; i < d->numInstances; ++i)
        s->instances[i].desc = d->instances[i];
    s->instanceMeshSlots.assign(d->instanceMeshSlots, d->instanceMeshSlots + d->numInstanceMeshSlots);

    if (!buildEnvLight(&s->env, d->envTexels, d->envWidth, d->envHeight)) { // a NaN texel: refused like gfx_scene_upload does
        delete s;
        return nullptr;
    }
    if (d->materialTextures && d->numTextures) {
        s->textures.resize(d->numTextures);
        for (uint32_t t = 0; t < d->numTextures; ++t) {
            s->textures[t].W = d->textures[t].width;
            s->textures[t].H = d->textures[t].height;
            s->textures[t].texels.assign(d->textures[t].texels, d->textures[t].texels + 4 * (size_t)d->textures[t].width * d->textures[t].height);
        }
        s->materialTextures.assign(d->materialTextures, d->materialTextures + 4 * (size_t)d->numMaterials);
    }
    s->buildConfig = *cfg;
    rebuildWorld(s, numThreads);
    return s;
}

// InstanceController::update (common/common_host.h:798-856) as seen from the hot path: new instance transforms (with their
// curToPrevTransform and normal matrices) arrive from the host, the acceleration structure over the moved geometry is
// rebuilt (Scene::updateASs) and the light distribution is recomputed (instance importances depend on the scale).
extern "C" int orc_scene_update_instances(orc_scene* s, const GfxInstanceDesc* instances, uint32_t numInstances) {
    if (!s || !instances || numInstances != s->instances.size())
        return -1;
    for (uint32_t i = 0; i < numInstances; ++i) {
        if (instances[i].firstMeshSlot != s->instances[i].desc.firstMeshSlot ||
            instances[i].numMeshSlots != s->instances[i].desc.numMeshSlots)
            return -2; // the topology of the scene is fixed; only transforms animate
        s->instances[i].desc = instances[i];
    }
    rebuildWorld(s, 0);
    return 0;
}
extern "C" void orc_scene_destroy(orc_scene* s) { delete s; }
extern "C" int orc_env_enabled(orc_scene* s, const GfxFrameParams* p) { return useEnvLight(s, p) ? 1 : 0; }
// test hooks of the environment light: op 0 = importance-map sample (u0, u1) -> (u, v, uvPDF), 1 = evaluatePDF(u, v) -> pdf,
// 2 = texture fetch (u, v) -> rgb; `in` holds n pairs, `out` n triples
extern "C" int orc_env_query(orc_scene* s, int op, const float* in, uint32_t n, float* out) {
    if (!s->env.present())
        return -1;
    for (uint32_t i = 0; i < n; ++i) {
        const float a = in[2 * i], b = in[2 * i + 1];
        float* o = out + 3 * i;
        if (op == 0) {
            s->env.sample(a, b, &o[0], &o[1], &o[2]);
        }
        else if (op == 1) {
            o[0] = s->env.evaluatePDF(a, b);
            o[1] = o[2] = 0.0f;
        }
        else {
            const float3 c = s->env.fetch(a, b);
            o[0] = c.x; o[1] = c.y; o[2] = c.z;
        }
    }
    return 0;
}
extern "C" double orc_scene_build_seconds(orc_scene* s) { return s->buildSeconds; }

extern "C" void orc_bvh_info(orc_scene* s, GfxBvhInfo* info) {
    info->numNodes = (uint32_t)s->bvh.intNodes.size();
    info->numPrimRefs = (uint32_t)s->bvh.primRefs.size();
    info->numTriangles = (uint32_t)s->bvh.triStorages.size();
    info->numGeoms = (uint32_t)s->geomToInst.size();
    for (int i = 0; i < 3; ++i) {
        info->sceneMin[i] = s->sceneMin[i];
        info->sceneMax[i] = s->sceneMax[i];
    }
}
extern "C" void orc_bvh_export(orc_scene* s, GfxBvhNode8* nodes, uint32_t* primRefs, GfxTriangleStorage* tris) {
    static_assert(sizeof(GfxBvhNode8) == sizeof(InternalNode8), "layout");
    static_assert(sizeof(GfxTriangleStorage) == sizeof(TriangleStorage), "layout");
    if (nodes) std::memcpy(nodes, s->bvh.intNodes.data(), s->bvh.intNodes.size() * sizeof(InternalNode8));
    if (primRefs) std::memcpy(primRefs, s->bvh.primRefs.data(), s->bvh.primRefs.size() * 4);
    if (tris) std::memcpy(tris, s->bvh.triStorages.data(), s->bvh.triStorages.size() * sizeof(TriangleStorage));
}
extern "C" void orc_bvh_import(orc_scene* s, const GfxBvhNode8* nodes, uint32_t numNodes,
                               const uint32_t* primRefs, uint32_t numPrimRefs,
                               const GfxTriangleStorage* tris, uint32_t numTris) {
    s->bvh.intNodes.resize(numNodes);
    std::memcpy(s->bvh.intNodes.data(), nodes, (size_t)numNodes * sizeof(InternalNode8));
    s->bvh.primRefs.assign(primRefs, primRefs + numPrimRefs);
    s->bvh.triStorages.resize(numTris);
    std::memcpy(s->bvh.triStorages.data(), tris, (size_t)numTris * sizeof(TriangleStorage));
    s->bvh.parentPointers.clear();
}

extern "C" int orc_bvh_validate(orc_scene* s, char* msg, size_t msgLen) {
    const GeometryBVH &bvh = s->bvh;
    const uint32_t numNodes = (uint32_t)bvh.intNodes.size();
    const uint32_t numTris = (uint32_t)bvh.triStorages.size();
    std::vector<uint32_t> refCount(numTris, 0);
    std::vector<uint8_t> visited(numNodes, 0);
    // iterative DFS; for every child compute the exact AABB of its subtree triangles and check
    // that the decoded quantised box contains it.
    struct Item { uint32_t node; };
    std::vector<AABB> subtreeBox(numNodes);
    std::vector<uint32_t> order;
    std::vector<uint32_t> st;
    if (numNodes == 0) return 0;
    st.push_back(0);
    while (!st.empty()) {
        const uint32_t n = st.back();
        st.pop_back();
        if (n >= numNodes) { snprintf(msg, msgLen, "node index %u out of range", n); return 1; }
        if (visited[n]) { snprintf(msg, msgLen, "node %u referenced twice", n); return 2; }
        visited[n] = 1;
        order.push_back(n);
        const InternalNode8 &node = bvh.intNodes[n];
        for (uint32_t slot = 0; slot < 8; ++slot) {
            if (!nodeChildIsValid(node, slot)) break;
            if ((node.internalMask >> slot) & 1)
                st.push_back(node.intNodeChildBaseIndex + popcnt(node.internalMask & ((1u << slot) - 1)));
        }
    }
    for (size_t oi = order.size(); oi-- > 0;) {
        const uint32_t n = order[oi];
        const InternalNode8 &node = bvh.intNodes[n];
        AABB nodeBox;
        for (uint32_t slot = 0; slot < 8; ++slot) {
            if (!nodeChildIsValid(node, slot)) break;
            AABB exact;
            if ((node.internalMask >> slot) & 1) {
                exact = subtreeBox[node.intNodeChildBaseIndex + popcnt(node.internalMask & ((1u << slot) - 1))];
            }
            else {
                uint32_t idx = node.leafBaseIndex + node.childMetas[slot];
                for (uint32_t guard = 0;; ++guard) {
                    if (idx >= bvh.primRefs.size() || guard > 100000) { snprintf(msg, msgLen, "leaf chain of node %u slot %u runs out of range", n, slot); return 3; }
                    const uint32_t pr = bvh.primRefs[idx];
                    const uint32_t si = pr & 0x7FFFFFFFu;
                    if (si >= numTris) { snprintf(msg, msgLen, "storage index %u out of range", si); return 4; }
                    ++refCount[si];
                    const TriangleStorage &ts = bvh.triStorages[si];
                    // SBVH references may be clipped; the un-clipped triangle box is an upper bound,
                    // so only un-split builds (every triangle referenced once) get the containment check.
                    exact.unify(float3(ts.pA[0], ts.pA[1], ts.pA[2]));
                    exact.unify(float3(ts.pB[0], ts.pB[1], ts.pB[2]));
                    exact.unify(float3(ts.pC[0], ts.pC[1], ts.pC[2]));
                    ++idx;
                    if (pr >> 31) break;
                }
            }
            const AABB q = nodeChildAabb(node, slot);
            if (bvh.primRefs.size() == numTris) {
                for (int d = 0; d < 3; ++d) {
                    if (q.minP[d] > exact.minP[d] || q.maxP[d] < exact.maxP[d]) {
                        snprintf(msg, msgLen, "node %u slot %u: quantised box does not contain its subtree on axis %d (%g..%g vs %g..%g)",
                                 n, slot, d, q.minP[d], q.maxP[d], exact.minP[d], exact.maxP[d]);
                        return 5;
                    }
                }
            }
            nodeBox.unify(exact);
        }
        subtreeBox[n] = nodeBox;
    }
    for (uint32_t i = 0; i < numTris; ++i)
        if (refCount[i] == 0) { snprintf(msg, msgLen, "triangle %u is never referenced", i); return 6; }
    for (uint32_t i = 0; i < numNodes; ++i)
        if (!visited[i]) { snprintf(msg, msgLen, "node %u unreachable", i); return 7; }
    if (msgLen) msg[0] = 0;
    return 0;
}

static inline float3 f3(const float* p) { return float3(p[0], p[1], p[2]); }

static inline void fixupHit(const orc_scene* s, HitObject* h) {
    // instIndex is not produced by the geometry-BVH traverser; fill it from the flattening table
    if (h->primIndex != UINT32_MAX)
        h->instIndex = s->geomToInst[h->geomIndex];
}

extern "C" void orc_trace(orc_scene* s, const GfxRay* rays, uint32_t numRays, GfxHitObject* hits, int mode,
                          OrcTraversalStats* stats, int numThreads) {
    static_assert(sizeof(GfxHitObject) == sizeof(HitObject), "layout");
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    uint64_t aabbTests = 0, triTests = 0, intNodes = 0, numHits = 0;
    int32_t maxDepth = -1;
#pragma omp parallel for schedule(dynamic, 256) num_threads(numThreads) reduction(+:aabbTests,triTests,intNodes,numHits) reduction(max:maxDepth)
    for (int64_t i = 0; i < (int64_t)numRays; ++i) {
        const GfxRay &r = rays[i];
        HitObject h;
        TraversalStatistics st = {};
        if (mode == ORC_TRACE_FIRST_FOUND)
            h = traverse(s->bvh, f3(r.org), f3(r.dir), r.tmin, r.tmax, stats ? &st : nullptr);
        else if (mode == ORC_TRACE_CANONICAL)
            h = traverseCanonical(s->bvh, f3(r.org), f3(r.dir), r.tmin, r.tmax);
        else if (mode == ORC_TRACE_BRUTE_FORCE)
            h = bruteForceClosest(s->bvh, f3(r.org), f3(r.dir), r.tmin, r.tmax);
        else {
            const bool any = traverseAny(s->bvh, f3(r.org), f3(r.dir), r.tmin, r.tmax);
            h = {};
            h.dist = any ? 0.0f : r.tmax;
            h.instIndex = h.geomIndex = UINT32_MAX;
            h.primIndex = any ? 0 : UINT32_MAX;
            h.bcA = h.bcB = h.bcC = NAN;
        }
        if (mode != ORC_TRACE_ANY)
            fixupHit(s, &h);
        std::memcpy(&hits[i], &h, sizeof(h));
        aabbTests += st.numAabbTests;
        triTests += st.numTriTests;
        intNodes += st.numIntNodes;
        maxDepth = std::max(maxDepth, st.maxStackDepth);
        numHits += h.primIndex != UINT32_MAX;
    }
    if (stats) {
        stats->numAabbTests = aabbTests;
        stats->numTriTests = triTests;
        stats->numIntNodes = intNodes;
        stats->maxStackDepth = maxDepth;
        stats->numHits = (uint32_t)numHits;
    }
}

extern "C" void orc_light_dist_export(orc_scene* s, float* w, float* cdf, float* integral) {
    if (w) std::memcpy(w, s->instWeights.data(), s->instWeights.size() * 4);
    if (cdf) std::memcpy(cdf, s->instCdf.data(), s->instCdf.size() * 4);
    if (integral) *integral = s->instIntegral;
}

// ---------------------------------------------------------------------------------------
// frame state
// ---------------------------------------------------------------------------------------
struct GB0 { uint32_t instSlot, geomInstSlot, primIndex, qbc; };   // GBuffer0Elements (restir_di_shared.h:182-188)
struct GB1 { float mvx, mvy; };                                    // GBuffer1Elements (:190-192)
struct GB2 { float px, py, pz; uint32_t qGeometricNormal; };       // GBuffer2Elements (:194-197)
struct GB3 { uint32_t qShadingNormal, qShadingTangent, qTexCoord, matSlot; }; // GBuffer3Elements (:199-204)
struct F4 { float x, y, z, w; };

struct LightSample { // restir_di_shared.h:89-96
    float3 emittance, position, normal;
    uint32_t atInfinity = 0;
};
struct Reservoir { // restir_di_shared.h:106-139
    LightSample sample;
    float sumWeights = 0.0f;
    uint32_t streamLength = 0;
    void initialize(const LightSample &s) { sample = s; sumWeights = 0; streamLength = 0; }
    bool update(const LightSample &newSample, float weight, float u) {
        sumWeights += weight;
        const bool accepted = u < weight / sumWeights;
        if (accepted)
            sample = newSample;
        ++streamLength;
        return accepted;
    }
};

struct orc_frame {
    orc_scene* scene;
    uint32_t W, H;
    std::vector<GB0> gb0[2];
    std::vector<GB1> gb1[2];
    std::vector<GB2> gb2[2];
    std::vector<GB3> gb3[2];
    std::vector<uint64_t> rng;
    // reservoir planes: [3][H*W] float4: (Le, sumW) (pos, M|atInf<<31) (n, 0)
    std::vector<F4> reservoir[2];
    std::vector<GB1> reservoirInfo[2]; // recPDFEstimate, targetDensity
    std::vector<F4> beauty, albedo, normal;
    std::vector<float2> neighborDeltas;
    struct orc_nrc_frame* nrc = nullptr; // NRC buffers, created on first use (nrc_pathtrace.inl)
    struct orc_regir* regir = nullptr;   // ReGIR grid, created on first use (regir.inl)
    struct orc_rearch* rearch = nullptr; // rearchitected ReSTIR state (restir_rearch.inl)
};

// the SVGF restatement (denoise.cpp, another translation unit) shows the environment behind miss pixels
extern "C" orc_scene* orc_frame_scene(orc_frame* f) { return f->scene; }
extern "C" orc_frame* orc_frame_create(orc_scene* s, uint32_t W, uint32_t H) {
    orc_frame* f = new orc_frame();
    f->scene = s;
    f->W = W;
    f->H = H;
    const size_t n = (size_t)W * H;
    for (int i = 0; i < 2; ++i) {
        f->gb0[i].assign(n, GB0{ 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu });
        f->gb1[i].assign(n, GB1{ 0, 0 });
        f->gb2[i].assign(n, GB2{ 0, 0, 0, 0 });
        f->gb3[i].assign(n, GB3{ 0, 0, 0, 0 });
        f->reservoir[i].assign(3 * n, F4{ 0, 0, 0, 0 });
        f->reservoirInfo[i].assign(n, GB1{ 0, 0 });
    }
    f->rng.assign(n, 0);
    f->beauty.assign(n, F4{ 0, 0, 0, 0 });
    f->albedo.assign(n, F4{ 0, 0, 0, 0 });
    f->normal.assign(n, F4{ 0, 0, 0, 0 });
    return f;
}
static void nrcFrameDestroy(struct orc_nrc_frame* n);
static void regirDestroy(struct orc_regir* r);
static void rearchDestroy(struct orc_rearch* r);
extern "C" void orc_frame_destroy(orc_frame* f) {
    if (f->nrc)
        nrcFrameDestroy(f->nrc);
    if (f->regir)
        regirDestroy(f->regir);
    if (f->rearch)
        rearchDestroy(f->rearch);
    delete f;
}

extern "C" void orc_rng_seed(orc_frame* f, uint64_t seed) { // restir_di_main.cpp:1309-1321
    std::mt19937_64 rngSeed(seed);
    for (uint32_t y = 0; y < f->H; ++y)
        for (uint32_t x = 0; x < f->W; ++x)
            f->rng[(size_t)y * f->W + x] = rngSeed();
}

extern "C" void orc_restir_setup_neighbor_table(orc_frame* f) { // restir_di_main.cpp:1489-1542
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
    f->neighborDeltas.resize(1024);
    for (uint32_t i = 0; i < 1024; ++i) {
        const float u0 = halton(2, i), u1 = halton(3, i);
        float r, theta;
        const float sx = 2 * u0 - 1;
        const float sy = 2 * u1 - 1;
        float2 d(0, 0);
        if (!(sx == 0 && sy == 0)) {
            if (sx >= -sy) {
                if (sx > sy) { r = sx; theta = sy / sx; }
                else { r = sy; theta = 2 - sx / sy; }
            }
            else {
                if (sx > sy) { r = -sy; theta = 6 + sx / sy; }
                else { r = -sx; theta = 4 + sy / sx; }
            }
            theta *= kPi / 4;
            // host-side table: libm in double, rounded once to float
            d.x = (float)(r * std::cos((double)theta));
            d.y = (float)(r * std::sin((double)theta));
        }
        f->neighborDeltas[i] = d;
    }
}

static void* nrcBufferPtr(orc_frame* f, int id, uint32_t index, size_t* bytes);
static void* regirBufferPtr(orc_frame* f, int id, uint32_t index, size_t* bytes);
static void* rearchBufferPtr(orc_frame* f, int id, uint32_t index, size_t* bytes);
extern "C" void* orc_buffer_ptr(orc_frame* f, int id, uint32_t index, size_t* bytes) {
    const size_t n = (size_t)f->W * f->H;
    void* p = nullptr;
    size_t b = 0;
    switch (id) {
    case GFX_BUF_GBUFFER0: p = f->gb0[index & 1].data(); b = n * 16; break;
    case GFX_BUF_GBUFFER1: p = f->gb1[index & 1].data(); b = n * 8; break;
    case GFX_BUF_GBUFFER2: p = f->gb2[index & 1].data(); b = n * 16; break;
    case GFX_BUF_GBUFFER3: p = f->gb3[index & 1].data(); b = n * 16; break;
    case GFX_BUF_RNG: p = f->rng.data(); b = n * 8; break;
    case GFX_BUF_RESERVOIR: p = f->reservoir[index & 1].data(); b = n * 48; break;
    case GFX_BUF_RESERVOIR_INFO: p = f->reservoirInfo[index & 1].data(); b = n * 8; break;
    case GFX_BUF_BEAUTY_ACCUM: p = f->beauty.data(); b = n * 16; break;
    case GFX_BUF_ALBEDO_ACCUM: p = f->albedo.data(); b = n * 16; break;
    case GFX_BUF_NORMAL_ACCUM: p = f->normal.data(); b = n * 16; break;
    default:
        if (id >= GFX_BUF_SAMPLE_VISIBILITY)
            return rearchBufferPtr(f, id, index, bytes);
        if (id >= GFX_BUF_REGIR_SLOTS)
            return regirBufferPtr(f, id, index, bytes);
        return nrcBufferPtr(f, id, index, bytes);
    }
    if (bytes) *bytes = b;
    return p;
}

// ---------------------------------------------------------------------------------------
// camera
// ---------------------------------------------------------------------------------------
struct Camera {
    float aspect, fovY;
    float3 position;
    Mat3 orientation;
    Mat3 invOrientation;
    float vh, vw; // 2*tan(fovY/2), aspect*vh  (host libm; identical numbers go to the GPU kernels)
};
static Mat3 invert3(const Mat3 &a) { // Matrix3x3::invert (basic_types.h:4150-4158): adjugate / det
    const float* m = a.m; // row-major: m[r*3+c]
    const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
    const float det = m00 * m11 * m22 + m01 * m12 * m20 + m02 * m10 * m21
        - m02 * m11 * m20 - m01 * m10 * m22 - m00 * m12 * m21;
    const float rdet = 1 / det;
    Mat3 r;
    r.m[0] = (m11 * m22 - m12 * m21) * rdet;
    r.m[1] = -(m01 * m22 - m02 * m21) * rdet;
    r.m[2] = (m01 * m12 - m02 * m11) * rdet;
    r.m[3] = -(m10 * m22 - m12 * m20) * rdet;
    r.m[4] = (m00 * m22 - m02 * m20) * rdet;
    r.m[5] = -(m00 * m12 - m02 * m10) * rdet;
    r.m[6] = (m10 * m21 - m11 * m20) * rdet;
    r.m[7] = -(m00 * m21 - m01 * m20) * rdet;
    r.m[8] = (m00 * m11 - m01 * m10) * rdet;
    return r;
}
static Camera makeCamera(const GfxCamera &c) {
    Camera cam;
    cam.aspect = c.aspect;
    cam.fovY = c.fovY;
    cam.position = f3(c.position);
    cam.orientation = mat3(c.orientation);
    cam.invOrientation = invert3(cam.orientation);
    cam.vh = 2 * std::tan(c.fovY * 0.5f);
    cam.vw = c.aspect * cam.vh;
    return cam;
}
static float2 calcScreenPosition(const Camera &cam, const float3 &posInWorld) { // restir_di_shared.h:51-59
    const float3 posInView = cam.invOrientation.mul(posInWorld - cam.position);
    const float2 posAtZ1(posInView.x / posInView.z, posInView.y / posInView.z);
    const float h = cam.vh;
    const float w = cam.aspect * h;
    return float2(1 - (posAtZ1.x + 0.5f * w) / w, 1 - (posAtZ1.y + 0.5f * h) / h);
}
static inline void primaryRay(const Camera &cam, uint32_t W, uint32_t H, uint32_t ix, uint32_t iy, float jx, float jy,
                              float3* origin, float3* direction) { // optix_gbuffer_kernels.cu:21-27
    const float x = (ix + jx) / W;
    const float y = (iy + jy) / H;
    *origin = cam.position;
    *direction = normalize(cam.orientation.mul(float3(cam.vw * (0.5f - x), cam.vh * (0.5f - y), 1)));
}

extern "C" void orc_generate_primary_rays(const GfxFrameParams* p, uint32_t W, uint32_t H, GfxRay* rays) {
    const Camera cam = makeCamera(p->camera);
    for (uint32_t y = 0; y < H; ++y)
        for (uint32_t x = 0; x < W; ++x) {
            float3 o, d;
            primaryRay(cam, W, H, x, y, 0.5f, 0.5f, &o, &d);
            GfxRay &r = rays[(size_t)y * W + x];
            r.org[0] = o.x; r.org[1] = o.y; r.org[2] = o.z;
            r.dir[0] = d.x; r.dir[1] = d.y; r.dir[2] = d.z;
            r.tmin = 0.0f;
            r.tmax = std::numeric_limits<float>::max();
        }
}

// BSDF::setup(mat, texCoord, 0.0f) (common_device.cuh:376-385, 778-826): constants, or the material's image textures at texCoord
static inline BSDF setupBsdf(const orc_scene* s, uint32_t matSlot, const float2 &texCoord) {
    const GfxMaterialDesc &m = s->materials[matSlot];
    BSDF b;
    if (s->materialTextures.empty()) {
        b.setup(m.bsdfType, m.p0, m.p1, m.p2);
        return b;
    }
    const uint32_t* tex = &s->materialTextures[4 * (size_t)matSlot];
    float p0[3] = { m.p0[0], m.p0[1], m.p0[2] }, p1[3] = { m.p1[0], m.p1[1], m.p1[2] }, p2 = m.p2;
    float t[4];
    if (tex[0] != 0xFFFFFFFFu) {
        s->textures[tex[0]].fetch(texCoord.x, texCoord.y, t);
        p0[0] = t[0]; p0[1] = t[1]; p0[2] = t[2];
    }
    if (tex[1] != 0xFFFFFFFFu) {
        s->textures[tex[1]].fetch(texCoord.x, texCoord.y, t);
        p1[0] = t[0]; p1[1] = t[1]; p1[2] = t[2];
    }
    if (tex[2] != 0xFFFFFFFFu) {
        s->textures[tex[2]].fetch(texCoord.x, texCoord.y, t);
        p2 = t[0];
    }
    b.setup(m.bsdfType, p0, p1, p2);
    return b;
}

// ---------------------------------------------------------------------------------------
// G-buffer — optix_gbuffer_kernels.cu:5-243
// ---------------------------------------------------------------------------------------
extern "C" void orc_gbuffer(orc_frame* f, const GfxFrameParams* p, int numThreads) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    const orc_scene* s = f->scene;
    const uint32_t W = f->W, H = f->H;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const Camera camera = makeCamera(p->camera);
    const Camera prevCamera = makeCamera(p->prevCamera);
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;

#pragma omp parallel for schedule(dynamic, 4) num_threads(numThreads)
    for (int64_t yy = y0; yy < (int64_t)y1; ++yy) {
        for (uint32_t x = 0; x < W; ++x) {
            const uint32_t y = (uint32_t)yy;
            const size_t pix = (size_t)y * W + x;
            float jx = 0.5f, jy = 0.5f;
            if (p->enableJittering) {
                PCG32RNG rng{ f->rng[pix] };
                jx = rng.getFloat0cTo1o();
                jy = rng.getFloat0cTo1o();
                f->rng[pix] = rng.state;
            }
            float3 origin, direction;
            primaryRay(camera, W, H, x, y, jx, jy, &origin, &direction);

            // HitPointParams defaults (:29-42)
            float3 albedo(0.0f);
            float3 positionInWorld(NAN), prevPositionInWorld(NAN), shadingNormalInWorld(NAN);
            uint32_t qGeometricNormalInWorld = 0, qTexCoord0DirInWorld = 0, qTexCoord = 0;
            uint32_t matSlot = 0xFFFFFFFFu, instSlot = 0xFFFFFFFFu, geomInstSlot = 0xFFFFFFFFu, primIndex = 0xFFFFFFFFu;
            uint16_t qbcB = 0, qbcC = 0;

            const HitObject hit = traverseCanonical(s->bvh, origin, direction, 0.0f, std::numeric_limits<float>::max());
            if (hit.primIndex != UINT32_MAX) {
                // closest-hit program (:112-199)
                instSlot = s->geomToInst[hit.geomIndex];
                geomInstSlot = s->geomToMesh[hit.geomIndex];
                primIndex = hit.primIndex;
                const InstData &inst = s->instances[instSlot];
                const MeshData &mesh = s->meshes[geomInstSlot];
                matSlot = mesh.materialSlot;
                const Affine xfm = affine(inst.desc.transform);
                const Affine curToPrev = affine(inst.desc.curToPrevTransform);
                const Mat3 normalMatrix = mat3(inst.desc.normalMatrix);

                const uint32_t i0 = mesh.triangles[3 * primIndex], i1 = mesh.triangles[3 * primIndex + 1], i2 = mesh.triangles[3 * primIndex + 2];
                const float bcB = hit.bcB;
                const float bcC = hit.bcC;
                const float bcA = 1 - (bcB + bcC);
                qbcB = encodeBarycentric(bcB);
                qbcC = encodeBarycentric(bcC);
                const float3 pA = ld3(mesh.positions, i0), pB = ld3(mesh.positions, i1), pC = ld3(mesh.positions, i2);
                const float3 positionInObj = bcA * pA + bcB * pB + bcC * pC;
                const float3 shadingNormalInObj = bcA * ld3(mesh.normals, i0) + bcB * ld3(mesh.normals, i1) + bcC * ld3(mesh.normals, i2);
                const float3 texCoord0DirInObj = bcA * ld3(mesh.tangents, i0) + bcB * ld3(mesh.tangents, i1) + bcC * ld3(mesh.tangents, i2);
                const float2 texCoord = bcA * ld2(mesh.texcoords, i0) + bcB * ld2(mesh.texcoords, i1) + bcC * ld2(mesh.texcoords, i2);
                const float3 geometricNormalInObj = cross(pB - pA, pC - pA);

                positionInWorld = xfm.point(positionInObj);
                prevPositionInWorld = curToPrev.point(positionInWorld);
                float3 geometricNormalInWorld = normalize(normalMatrix.mul(geometricNormalInObj));
                shadingNormalInWorld = normalize(normalMatrix.mul(shadingNormalInObj));
                float3 texCoord0DirInWorld = xfm.vector(texCoord0DirInObj);
                texCoord0DirInWorld = normalize(
                    texCoord0DirInWorld - dot(shadingNormalInWorld, texCoord0DirInWorld) * shadingNormalInWorld);
                if (!allFinite(shadingNormalInWorld)) {
                    geometricNormalInWorld = float3(0, 0, 1);
                    shadingNormalInWorld = float3(0, 0, 1);
                    texCoord0DirInWorld = float3(1, 0, 0);
                }
                qGeometricNormalInWorld = encodeVector(geometricNormalInWorld);
                qTexCoord = encodeTexCoords(texCoord);

                const BSDF bsdf = setupBsdf(s, matSlot, texCoord);
                const ReferenceFrame shadingFrame(shadingNormalInWorld, texCoord0DirInWorld);
                const float3 vOut = -direction;
                const float3 vOutLocal = shadingFrame.toLocal(normalize(vOut));
                shadingNormalInWorld = shadingFrame.normal;
                qTexCoord0DirInWorld = encodeVector(shadingFrame.tangent);
                albedo = bsdf.evaluateDHReflectanceEstimate(vOutLocal);
            }
            else {
                // miss program (:201-243), no environment texture
                const float3 vOut = -direction;
                const float3 pp = -vOut;
                float posPhi, posTheta;
                toPolarYUp(pp, &posPhi, &posTheta);
                const float phi = posPhi + p->envLightRotation;
                float u = phi / (2 * kPi);
                u -= std::floor(u);
                const float v = posTheta / kPi;
                positionInWorld = pp;
                prevPositionInWorld = pp;
                qGeometricNormalInWorld = encodeVector(vOut);
                shadingNormalInWorld = vOut;
                float sp, cp;
                dm_sincos(posPhi, &sp, &cp);
                qTexCoord0DirInWorld = encodeVector(float3(-cp, 0, -sp));
                qTexCoord = encodeTexCoords(float2(u, v));
                qbcB = encodeBarycentric(u);
                qbcC = encodeBarycentric(v);
            }

            // ray-gen epilogue (:56-109)
            const float2 curRasterPos(x + 0.5f, y + 0.5f);
            const float2 prevRasterPos = calcScreenPosition(prevCamera, prevPositionInWorld) * float2((float)W, (float)H);
            float2 motionVector = curRasterPos - prevRasterPos;
            if (p->resetFlowBuffer || std::isnan(prevPositionInWorld.x))
                motionVector = float2(0.0f, 0.0f);

            f->gb0[bufIdx][pix] = GB0{ instSlot, geomInstSlot, primIndex, (uint32_t)qbcB | ((uint32_t)qbcC << 16) };
            f->gb1[bufIdx][pix] = GB1{ motionVector.x, motionVector.y };
            f->gb2[bufIdx][pix] = GB2{ positionInWorld.x, positionInWorld.y, positionInWorld.z, qGeometricNormalInWorld };
            f->gb3[bufIdx][pix] = GB3{ encodeVector(shadingNormalInWorld), qTexCoord0DirInWorld, qTexCoord, matSlot };

            float3 prevAlbedoResult(0.0f), prevNormalResult(0.0f);
            if (p->numAccumFrames > 0) {
                prevAlbedoResult = float3(f->albedo[pix].x, f->albedo[pix].y, f->albedo[pix].z);
                prevNormalResult = float3(f->normal[pix].x, f->normal[pix].y, f->normal[pix].z);
            }
            const float curWeight = 1.0f / (1 + p->numAccumFrames);
            const float3 albedoResult = (1 - curWeight) * prevAlbedoResult + curWeight * albedo;
            const float3 normalResult = (1 - curWeight) * prevNormalResult + curWeight * shadingNormalInWorld;
            f->albedo[pix] = F4{ albedoResult.x, albedoResult.y, albedoResult.z, 1.0f };
            f->normal[pix] = F4{ normalResult.x, normalResult.y, normalResult.z, 1.0f };
        }
    }
}

// ---------------------------------------------------------------------------------------
// ReSTIR DI
// ---------------------------------------------------------------------------------------
static inline float convertToWeight(const float3 &c) { return (c.x + c.y + c.z) / 3; } // restir_di_shared.h:82-85

// which light sampleLight picked, for the test hook orc_light_sample_debug: stage 0 / 1 = the instance / geometry early out, 2 = a
// primitive; lightProb = the product of the three probabilities (set at stage 2 only)
struct LightPickInfo {
    uint32_t stage = 0, instSlot = 0, geomInstIndexInInst = 0, primIndex = 0;
    float lightProb = 0.0f;
};
static void sampleLight(const orc_scene* s, const GfxFrameParams* p, float ul, bool sampleEnvLight, float u0, float u1,
                        LightSample* lightSample, float* areaPDensity, LightPickInfo* pickInfo = nullptr) {
    // restir_di_shared.h:320-516, useSolidAngleSampling = false
    float3 emittance(0.0f);
    if (sampleEnvLight) { // :330-364
        float u, v, uvPDF;
        s->env.sample(u0, u1, &u, &v, &uvPDF);
        const float phi = 2 * kPi * u;
        const float theta = kPi * v;
        float posPhi = phi - p->envLightRotation;
        posPhi = posPhi - std::floor(posPhi / (2 * kPi)) * 2 * kPi;
        const float3 direction = fromPolarYUp(posPhi, theta);
        lightSample->position = direction;
        lightSample->atInfinity = 1;
        lightSample->normal = -direction;
        lightSample->emittance = float3(0.0f); // (left unset by the reference when sin(theta) == 0)
        // the PDF in texture space -> with respect to area: lim_{l -> inf} uvPDF / (2 pi^2 sin(theta)) / l^2
        const float sinTheta = dm_sin(theta);
        if (sinTheta == 0.0f) {
            *areaPDensity = 0.0f;
            return;
        }
        *areaPDensity = uvPDF / (2 * kPi * kPi * sinTheta);
        emittance = float3(kPi * p->envLightPowerCoeff);
        emittance *= s->env.fetch(u, v);
        lightSample->emittance = emittance;
        return;
    }
    float lightProb = 1.0f;

    DiscreteDistribution1D lightInstDist{ s->instWeights.data(), s->instCdf.data(), s->instIntegral, (uint32_t)s->instWeights.size() };
    float instProb, uGeomInst;
    const uint32_t instSlot = lightInstDist.sample(ul, &instProb, &uGeomInst);
    lightProb *= instProb;
    if (pickInfo)
        pickInfo->instSlot = instSlot;
    const InstData &inst = s->instances[instSlot];
    if (instProb == 0.0f) {
        *areaPDensity = 0.0f;
        return;
    }

    DiscreteDistribution1D lightGeomInstDist{ inst.geomWeights.data(), inst.geomCdf.data(), inst.geomIntegral, (uint32_t)inst.geomWeights.size() };
    float geomInstProb, uPrim;
    const uint32_t geomInstIndexInInst = lightGeomInstDist.sample(uGeomInst, &geomInstProb, &uPrim);
    const uint32_t geomInstSlot = s->instanceMeshSlots[inst.desc.firstMeshSlot + geomInstIndexInInst];
    lightProb *= geomInstProb;
    const MeshData &mesh = s->meshes[geomInstSlot];
    if (pickInfo) {
        pickInfo->stage = 1;
        pickInfo->geomInstIndexInInst = geomInstIndexInInst;
    }
    if (geomInstProb == 0.0f) {
        *areaPDensity = 0.0f;
        return;
    }

    DiscreteDistribution1D emitterPrimDist{ mesh.primWeights.data(), mesh.primCdf.data(), mesh.primIntegral, mesh.numTriangles };
    float primProb;
    const uint32_t primIndex = emitterPrimDist.sample(uPrim, &primProb);
    lightProb *= primProb;
    if (pickInfo) {
        pickInfo->stage = 2;
        pickInfo->primIndex = primIndex;
        pickInfo->lightProb = lightProb;
    }

    const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];
    const uint32_t i0 = mesh.triangles[3 * primIndex], i1 = mesh.triangles[3 * primIndex + 1], i2 = mesh.triangles[3 * primIndex + 2];
    const Affine xfm = affine(inst.desc.transform);
    const float3 pA = xfm.point(ld3(mesh.positions, i0));
    const float3 pB = xfm.point(ld3(mesh.positions, i1));
    const float3 pC = xfm.point(ld3(mesh.positions, i2));
    const float3 geomNormal = cross(pB - pA, pC - pA);

    float bcA = 0.5f * u0;
    float bcB = 0.5f * u1;
    const float offset = bcB - bcA;
    if (offset > 0)
        bcB += offset;
    else
        bcA -= offset;
    const float bcC = 1 - (bcA + bcB);

    const float recArea = 2.0f / length(geomNormal);
    *areaPDensity = lightProb * recArea;

    lightSample->position = bcA * pA + bcB * pB + bcC * pC;
    lightSample->atInfinity = 0;
    lightSample->normal = bcA * ld3(mesh.normals, i0) + bcB * ld3(mesh.normals, i1) + bcC * ld3(mesh.normals, i2);
    lightSample->normal = normalize(mat3(inst.desc.normalMatrix).mul(lightSample->normal));

    if (mat.hasEmittance) {
        emittance = float3(1.0f, 1.0f, 1.0f);
        // tex2DLod on a 1x1 texture: the texel, whatever the coordinate
        emittance *= float3(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
    }
    lightSample->emittance = emittance;
}

// the choice between the environment and the emitters that the streaming-RIS loops make for candidate i of n
// (optix_restir_di_kernels.cu:74-90, build_cell_reservoirs.cu:120-139): the first probToSampleEnvLight * n candidates go to the
// environment; returns sampleEnvLight and remaps ul
static bool chooseEnvForCandidate(const orc_scene* s, const GfxFrameParams* p, uint32_t i, uint32_t numCandidates, float* ul,
                                  float* probToSampleCurLightType) {
    *probToSampleCurLightType = 1.0f;
    if (!useEnvLight(s, p))
        return false;
    if (!(s->instIntegral > 0.0f))
        return true;
    const float prob = std::fmin(std::fmax(kProbToSampleEnvLight * numCandidates - i, 0.0f), 1.0f);
    if (*ul < prob) {
        *probToSampleCurLightType = kProbToSampleEnvLight;
        *ul = *ul / prob;
        return true;
    }
    *probToSampleCurLightType = 1.0f - kProbToSampleEnvLight;
    *ul = (*ul - prob) / (1 - prob);
    return false;
}

static bool evaluateVisibility(const orc_scene* s, const float3 &shadingPoint, const LightSample &ls) { // restir_di_shared.h:559-582
    float3 shadowRayDir = ls.atInfinity ? ls.position : (ls.position - shadingPoint);
    const float dist2 = sqLength(shadowRayDir);
    float dist = std::sqrt(dist2);
    shadowRayDir /= dist;
    if (ls.atInfinity)
        dist = 1e+10f;
    return !traverseAny(s->bvh, shadingPoint, shadowRayDir, 0.0f, dist * 0.9999f);
}

template <bool withVisibility>
static float3 performDirectLighting(const orc_scene* s, const float3 &shadingPoint, const float3 &vOutLocal,
                                    const ReferenceFrame &shadingFrame, const BSDF &bsdf, const LightSample &ls) { // :518-557
    float3 shadowRayDir = ls.atInfinity ? ls.position : (ls.position - shadingPoint);
    const float dist2 = sqLength(shadowRayDir);
    float dist = std::sqrt(dist2);
    shadowRayDir /= dist;
    const float3 shadowRayDirLocal = shadingFrame.toLocal(shadowRayDir);

    const float lpCos = dot(-shadowRayDir, ls.normal);
    const float spCos = shadowRayDirLocal.z;

    float visibility = 1.0f;
    if (withVisibility) {
        if (ls.atInfinity)
            dist = 1e+10f;
        if (traverseAny(s->bvh, shadingPoint, shadowRayDir, 0.0f, dist * 0.9999f))
            visibility = 0.0f;
    }

    if (visibility > 0 && lpCos > 0) {
        const float3 Le = ls.emittance / kPi;
        const float3 fsValue = bsdf.evaluate(vOutLocal, shadowRayDirLocal);
        const float G = lpCos * std::fabs(spCos) / dist2;
        return fsValue * Le * G;
    }
    return float3(0.0f);
}

static inline Reservoir loadReservoir(const orc_frame* f, uint32_t idx, size_t pix) {
    const size_t n = (size_t)f->W * f->H;
    const F4 a = f->reservoir[idx][pix], b = f->reservoir[idx][n + pix], c = f->reservoir[idx][2 * n + pix];
    Reservoir r;
    r.sample.emittance = float3(a.x, a.y, a.z);
    r.sumWeights = a.w;
    r.sample.position = float3(b.x, b.y, b.z);
    const uint32_t m = f2u(b.w);
    r.streamLength = m & 0x7FFFFFFFu;
    r.sample.atInfinity = m >> 31;
    r.sample.normal = float3(c.x, c.y, c.z);
    return r;
}
static inline void storeReservoir(orc_frame* f, uint32_t idx, size_t pix, const Reservoir &r) {
    const size_t n = (size_t)f->W * f->H;
    f->reservoir[idx][pix] = F4{ r.sample.emittance.x, r.sample.emittance.y, r.sample.emittance.z, r.sumWeights };
    f->reservoir[idx][n + pix] = F4{ r.sample.position.x, r.sample.position.y, r.sample.position.z,
                                     u2f((r.streamLength & 0x7FFFFFFFu) | (r.sample.atInfinity << 31)) };
    f->reservoir[idx][2 * n + pix] = F4{ r.sample.normal.x, r.sample.normal.y, r.sample.normal.z, 0.0f };
}

// The reservoir planes keep M in 31 bits next to atInfinity.  Spatial passes add up to 16 stream lengths per pass and any
// number of passes may run, so the sum saturates at 2^31 - 1 instead of wrapping into atInfinity.  Both inputs are at most
// 2^31 - 1, so the 32-bit sum cannot wrap.
static inline uint32_t saturatedStreamLength(uint32_t a, uint32_t b) { return std::min(a + b, 0x7FFFFFFFu); }

template <bool testGeometry>
static bool testNeighbor(const orc_frame* f, const Camera &camera, uint32_t nbBufIdx, int nbx, int nby, float dist, const float3 &normalInWorld) {
    // restir_di_shared.h:747-771
    if (nbx < 0 || nbx >= (int)f->W || nby < 0 || nby >= (int)f->H)
        return false;
    const size_t nbPix = (size_t)nby * f->W + nbx;
    if (f->gb0[nbBufIdx][nbPix].instSlot == 0xFFFFFFFFu)
        return false;
    if (testGeometry) {
        const GB2 &g2 = f->gb2[nbBufIdx][nbPix];
        const GB3 &g3 = f->gb3[nbBufIdx][nbPix];
        const float3 nbPositionInWorld(g2.px, g2.py, g2.pz);
        const float3 nbNormalInWorld = decodeVector(g3.qShadingNormal);
        const float nbDist = length(camera.position - nbPositionInWorld);
        if (std::fabs(nbDist - dist) / dist > 0.1f || dot(normalInWorld, nbNormalInWorld) < 0.9f)
            return false;
    }
    return true;
}

struct ShadingPoint { // the common prologue of the three ReSTIR programs
    float3 positionInWorld; // offset ray origin
    float3 vOutLocal;
    float dist;
    ReferenceFrame shadingFrame;
    BSDF bsdf;
};

// candidate statistics of the initial RIS loop: [0] zero density, [1] below the shading horizon, [2] light faces away,
// [3] otherwise exactly zero, [4] contributing
static bool g_risStatsEnabled = false;
static unsigned long long g_risStats[5] = { 0, 0, 0, 0, 0 };
extern "C" void orc_ris_stats(int enable, unsigned long long* out5) {
    if (out5)
        for (int i = 0; i < 5; ++i) out5[i] = g_risStats[i];
    for (int i = 0; i < 5; ++i) g_risStats[i] = 0;
    g_risStatsEnabled = enable != 0;
}

template <bool withTemporalRIS, bool useUnbiasedEstimator>
static void performInitialAndTemporalRIS(orc_frame* f, const GfxFrameParams* p, const Camera &camera, const Camera &prevCamera,
                                         uint32_t x, uint32_t y) { // optix_restir_di_kernels.cu:14-287
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t curBufIdx = p->bufferIndex & 1;

    const GB0 gb0 = f->gb0[curBufIdx][pix];
    const uint32_t instSlot = gb0.instSlot;
    if (instSlot == 0xFFFFFFFFu)
        return;
    const GB2 gb2 = f->gb2[curBufIdx][pix];
    const GB3 gb3 = f->gb3[curBufIdx][pix];

    float3 positionInWorld(gb2.px, gb2.py, gb2.pz);
    const float3 geometricNormalInWorld = decodeVector(gb2.qGeometricNormal);

    PCG32RNG rng{ f->rng[pix] };

    float3 vOut = camera.position - positionInWorld;
    const float frontHit = dot(vOut, geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
    positionInWorld = offsetRayOrigin(positionInWorld, frontHit * geometricNormalInWorld);
    const float dist = length(vOut);
    vOut /= dist;

    const float3 shadingNormalInWorld = decodeVector(gb3.qShadingNormal);
    const float3 shadingTangentInWorld = decodeVector(gb3.qShadingTangent);
    const ReferenceFrame shadingFrame(shadingNormalInWorld, shadingTangentInWorld);
    const float3 vOutLocal = shadingFrame.toLocal(vOut);
    const BSDF bsdf = setupBsdf(s, gb3.matSlot, decodeTexCoords(gb3.qTexCoord));

    const uint32_t curResIndex = p->currentReservoirIndex & 1;
    Reservoir reservoir;
    reservoir.initialize(LightSample());

    float selectedTargetDensity = 0.0f;
    const uint32_t numCandidates = 1u << p->log2NumCandidateSamples;
    for (uint32_t i = 0; i < numCandidates; ++i) {
        float ul = rng.getFloat0cTo1o();
        float probToSampleCurLightType;
        const bool sampleEnvLight = chooseEnvForCandidate(s, p, i, numCandidates, &ul, &probToSampleCurLightType);
        LightSample lightSample;
        float probDensity;
        const float u0 = rng.getFloat0cTo1o();
        const float u1 = rng.getFloat0cTo1o();
        sampleLight(s, p, ul, sampleEnvLight, u0, u1, &lightSample, &probDensity);
        const float3 cont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, lightSample);
        probDensity *= probToSampleCurLightType;
        const float targetDensity = convertToWeight(cont);
        const float weight = targetDensity / probDensity;
        if (g_risStatsEnabled) { // measurement aid for the CUDA side's staged light fetch; does not touch the results
            const float3 d = lightSample.position - positionInWorld;
            const bool belowHorizon = dot(d, shadingNormalInWorld) * vOutLocal.z <= 0.0f;
            const bool facesAway = dot(d, lightSample.normal) >= 0.0f;
            const bool dark = cont.x == 0.0f && cont.y == 0.0f && cont.z == 0.0f;
            const int bucket = !(probDensity > 0.0f) ? 0 : belowHorizon ? 1 : facesAway ? 2 : dark ? 3 : 4;
#pragma omp atomic
            g_risStats[bucket] += 1;
        }
        if (reservoir.update(lightSample, weight, rng.getFloat0cTo1o()))
            selectedTargetDensity = targetDensity;
    }

    float recPDFEstimate = reservoir.sumWeights / (selectedTargetDensity * reservoir.streamLength);
    if (!std::isfinite(recPDFEstimate)) {
        recPDFEstimate = 0.0f;
        selectedTargetDensity = 0.0f;
    }

    if (p->reuseVisibility && selectedTargetDensity > 0.0f) {
        if (!evaluateVisibility(s, positionInWorld, reservoir.sample)) {
            recPDFEstimate = 0.0f;
            selectedTargetDensity = 0.0f;
        }
    }

    if (withTemporalRIS) {
        const uint32_t prevBufIdx = (curBufIdx + 1) % 2;
        const uint32_t prevResIndex = (curResIndex + 1) % 2;

        bool neighborIsSelected = false;
        const uint32_t selfStreamLength = reservoir.streamLength;
        if (recPDFEstimate == 0.0f)
            reservoir.initialize(LightSample());
        uint32_t combinedStreamLength = selfStreamLength;
        const uint32_t maxPrevStreamLength = 20 * selfStreamLength;

        const GB1 gb1 = f->gb1[curBufIdx][pix];
        const int nbx = dm_f2int(x + 0.5f - gb1.mvx);
        const int nby = dm_f2int(y + 0.5f - gb1.mvy);

        const bool acceptedNeighbor = testNeighbor<!useUnbiasedEstimator>(f, camera, prevBufIdx, nbx, nby, dist, shadingNormalInWorld);
        if (acceptedNeighbor) {
            const size_t nbPix = (size_t)nby * f->W + nbx;
            const Reservoir neighbor = loadReservoir(f, prevResIndex, nbPix);
            const GB1 neighborInfo = f->reservoirInfo[prevResIndex][nbPix];
            const LightSample nbLightSample = neighbor.sample;
            const float3 cont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, nbLightSample);
            const float targetDensity = convertToWeight(cont);
            const uint32_t nbStreamLength = std::min(neighbor.streamLength, maxPrevStreamLength);
            const float weight = targetDensity * neighborInfo.mvx * nbStreamLength;
            if (reservoir.update(nbLightSample, weight, rng.getFloat0cTo1o())) {
                selectedTargetDensity = targetDensity;
                if (useUnbiasedEstimator)
                    neighborIsSelected = true;
            }
            combinedStreamLength += nbStreamLength;
        }
        reservoir.streamLength = combinedStreamLength;

        float weightForEstimate;
        if (useUnbiasedEstimator) { // :192-266, useMIS_RIS = true
            const LightSample selectedLightSample = reservoir.sample;
            float numWeight, denomWeight;
            {
                const float3 cont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, selectedLightSample);
                const float targetDensityForSelf = convertToWeight(cont);
                numWeight = targetDensityForSelf;
                denomWeight = targetDensityForSelf * selfStreamLength;
            }
            if (acceptedNeighbor) {
                const size_t nbPix = (size_t)nby * f->W + nbx;
                const GB2 nbGb2 = f->gb2[prevBufIdx][nbPix];
                const GB3 nbGb3 = f->gb3[prevBufIdx][nbPix];
                float3 nbPositionInWorld(nbGb2.px, nbGb2.py, nbGb2.pz);
                const float3 nbGeometricNormalInWorld = decodeVector(nbGb2.qGeometricNormal);
                const float3 nbVOut = normalize(prevCamera.position - nbPositionInWorld);
                const float nbFrontHit = dot(nbVOut, nbGeometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
                nbPositionInWorld = offsetRayOrigin(nbPositionInWorld, nbFrontHit * nbGeometricNormalInWorld);
                const BSDF nbBsdf = setupBsdf(s, nbGb3.matSlot, decodeTexCoords(nbGb3.qTexCoord));
                const ReferenceFrame nbShadingFrame(decodeVector(nbGb3.qShadingNormal), decodeVector(nbGb3.qShadingTangent));
                const float3 nbVOutLocal = nbShadingFrame.toLocal(nbVOut);
                const Reservoir neighbor = loadReservoir(f, prevResIndex, nbPix);
                const float3 cont = performDirectLighting<false>(s, nbPositionInWorld, nbVOutLocal, nbShadingFrame, nbBsdf, selectedLightSample);
                const float nbTargetDensity = convertToWeight(cont);
                const uint32_t nbStreamLength = std::min(neighbor.streamLength, maxPrevStreamLength);
                denomWeight += nbTargetDensity * nbStreamLength;
                if (neighborIsSelected)
                    numWeight = nbTargetDensity;
            }
            weightForEstimate = numWeight / denomWeight;
        }
        else {
            weightForEstimate = 1.0f / reservoir.streamLength;
        }

        recPDFEstimate = weightForEstimate * reservoir.sumWeights / selectedTargetDensity;
        if (!std::isfinite(recPDFEstimate)) {
            recPDFEstimate = 0.0f;
            selectedTargetDensity = 0.0f;
        }
    }

    f->rng[pix] = rng.state;
    storeReservoir(f, curResIndex, pix, reservoir);
    f->reservoirInfo[curResIndex][pix] = GB1{ recPDFEstimate, selectedTargetDensity };
}

template <bool useUnbiasedEstimator>
static void performSpatialRIS(orc_frame* f, const GfxFrameParams* p, const Camera &camera, const Camera &prevCamera,
                              uint32_t x, uint32_t y) { // optix_restir_di_kernels.cu:303-547
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;

    const GB0 gb0 = f->gb0[bufIdx][pix];
    if (gb0.instSlot == 0xFFFFFFFFu)
        return;
    const GB2 gb2 = f->gb2[bufIdx][pix];
    const GB3 gb3 = f->gb3[bufIdx][pix];

    float3 positionInWorld(gb2.px, gb2.py, gb2.pz);
    const float3 geometricNormalInWorld = decodeVector(gb2.qGeometricNormal);
    PCG32RNG rng{ f->rng[pix] };

    float3 vOut = camera.position - positionInWorld;
    const float frontHit = dot(vOut, geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
    positionInWorld = offsetRayOrigin(positionInWorld, frontHit * geometricNormalInWorld);
    const float dist = length(vOut);
    vOut /= dist;

    const ReferenceFrame shadingFrame(decodeVector(gb3.qShadingNormal), decodeVector(gb3.qShadingTangent));
    const float3 vOutLocal = shadingFrame.toLocal(vOut);
    const BSDF bsdf = setupBsdf(s, gb3.matSlot, decodeTexCoords(gb3.qTexCoord));

    const uint32_t srcResIndex = p->currentReservoirIndex & 1;
    const uint32_t dstResIndex = (srcResIndex + 1) % 2;

    Reservoir combinedReservoir;
    combinedReservoir.initialize(LightSample());
    float selectedTargetDensity = 0.0f;
    int32_t selectedNeighborIndex = -1;

    const Reservoir self = loadReservoir(f, srcResIndex, pix);
    const GB1 selfResInfo = f->reservoirInfo[srcResIndex][pix];
    if (selfResInfo.mvx > 0.0f) {
        combinedReservoir = self;
        selectedTargetDensity = selfResInfo.mvy;
    }
    uint32_t combinedStreamLength = self.streamLength;

    auto neighborCoord = [&](int nIdx, PCG32RNG &r, int* nbx, int* nby) {
        float radius = p->spatialNeighborRadius;
        float deltaX, deltaY;
        if (p->useLowDiscrepancyNeighbors) {
            const float2 delta = f->neighborDeltas[(p->spatialNeighborBaseIndex + nIdx) % 1024];
            deltaX = radius * delta.x;
            deltaY = radius * delta.y;
        }
        else {
            radius *= std::sqrt(r.getFloat0cTo1o());
            const float angle = 2 * kPi * r.getFloat0cTo1o();
            float sa, ca;
            dm_sincos(angle, &sa, &ca);
            deltaX = radius * ca;
            deltaY = radius * sa;
        }
        *nbx = dm_f2int(x + 0.5f + deltaX);
        *nby = dm_f2int(y + 0.5f + deltaY);
    };

    for (int nIdx = 0; nIdx < (int)p->numSpatialNeighbors; ++nIdx) {
        int nbx, nby;
        neighborCoord(nIdx, rng, &nbx, &nby);
        const bool acceptedNeighbor =
            testNeighbor<!useUnbiasedEstimator>(f, camera, bufIdx, nbx, nby, dist, shadingFrame.normal)
            && (nbx != (int)x || nby != (int)y);
        if (acceptedNeighbor) {
            const size_t nbPix = (size_t)nby * f->W + nbx;
            const Reservoir neighbor = loadReservoir(f, srcResIndex, nbPix);
            const GB1 neighborInfo = f->reservoirInfo[srcResIndex][nbPix];
            const LightSample nbLightSample = neighbor.sample;
            const float3 cont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, nbLightSample);
            const float targetDensity = convertToWeight(cont);
            const uint32_t nbStreamLength = neighbor.streamLength;
            const float weight = targetDensity * neighborInfo.mvx * nbStreamLength;
            if (combinedReservoir.update(nbLightSample, weight, rng.getFloat0cTo1o())) {
                selectedTargetDensity = targetDensity;
                if (useUnbiasedEstimator)
                    selectedNeighborIndex = nIdx;
            }
            combinedStreamLength = saturatedStreamLength(combinedStreamLength, nbStreamLength);
        }
    }
    combinedReservoir.streamLength = combinedStreamLength;

    float weightForEstimate = 0.0f;
    if (useUnbiasedEstimator) { // :414-529
        if (selectedTargetDensity > 0.0f) {
            const LightSample selectedLightSample = combinedReservoir.sample;
            float numWeight, denomWeight;
            bool visibility = true;
            {
                float3 cont;
                if (p->reuseVisibility)
                    cont = performDirectLighting<true>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, selectedLightSample);
                else
                    cont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, selectedLightSample);
                const float targetDensityForSelf = convertToWeight(cont);
                if (p->reuseVisibility)
                    visibility = targetDensityForSelf > 0.0f;
                numWeight = targetDensityForSelf;
                denomWeight = targetDensityForSelf * self.streamLength;
            }
            for (int nIdx = 0; nIdx < (int)p->numSpatialNeighbors; ++nIdx) {
                int nbx, nby;
                neighborCoord(nIdx, rng, &nbx, &nby);
                const bool acceptedNeighbor =
                    (nbx >= 0 && nbx < (int)f->W && nby >= 0 && nby < (int)f->H) && (nbx != (int)x || nby != (int)y);
                if (acceptedNeighbor) {
                    const size_t nbPix = (size_t)nby * f->W + nbx;
                    if (f->gb0[bufIdx][nbPix].instSlot == 0xFFFFFFFFu)
                        continue;
                    const GB2 nbGb2 = f->gb2[bufIdx][nbPix];
                    const GB3 nbGb3 = f->gb3[bufIdx][nbPix];
                    float3 nbPositionInWorld(nbGb2.px, nbGb2.py, nbGb2.pz);
                    const float3 nbGeometricNormalInWorld = decodeVector(nbGb2.qGeometricNormal);
                    const float3 nbVOut = normalize(prevCamera.position - nbPositionInWorld);
                    const float nbFrontHit = dot(nbVOut, nbGeometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
                    nbPositionInWorld = offsetRayOrigin(nbPositionInWorld, nbFrontHit * nbGeometricNormalInWorld);
                    const BSDF nbBsdf = setupBsdf(s, nbGb3.matSlot, decodeTexCoords(nbGb3.qTexCoord));
                    const ReferenceFrame nbShadingFrame(decodeVector(nbGb3.qShadingNormal), decodeVector(nbGb3.qShadingTangent));
                    const float3 nbVOutLocal = nbShadingFrame.toLocal(nbVOut);
                    const Reservoir neighbor = loadReservoir(f, srcResIndex, nbPix);
                    float3 cont;
                    if (p->reuseVisibility)
                        cont = performDirectLighting<true>(s, nbPositionInWorld, nbVOutLocal, nbShadingFrame, nbBsdf, selectedLightSample);
                    else
                        cont = performDirectLighting<false>(s, nbPositionInWorld, nbVOutLocal, nbShadingFrame, nbBsdf, selectedLightSample);
                    const float nbTargetDensity = convertToWeight(cont);
                    const uint32_t nbStreamLength = neighbor.streamLength;
                    denomWeight += nbTargetDensity * nbStreamLength;
                    if (nIdx == selectedNeighborIndex)
                        numWeight = nbTargetDensity;
                }
            }
            weightForEstimate = numWeight / denomWeight;
            if (p->reuseVisibility && !visibility)
                weightForEstimate = 0.0f;
        }
    }
    else {
        weightForEstimate = 1.0f / combinedReservoir.streamLength;
    }

    float recPDFEstimate = weightForEstimate * combinedReservoir.sumWeights / selectedTargetDensity;
    float targetDensityOut = selectedTargetDensity;
    if (!std::isfinite(recPDFEstimate)) {
        recPDFEstimate = 0.0f;
        targetDensityOut = 0.0f;
    }

    f->rng[pix] = rng.state;
    storeReservoir(f, dstResIndex, pix, combinedReservoir);
    f->reservoirInfo[dstResIndex][pix] = GB1{ recPDFEstimate, targetDensityOut };
}

static void shading(orc_frame* f, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y) { // :559-637
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const GB3 gb3 = f->gb3[bufIdx][pix];

    float3 contribution(0.01f, 0.01f, 0.01f);
    if (gb0.instSlot != 0xFFFFFFFFu) {
        const GB2 gb2 = f->gb2[bufIdx][pix];
        float3 positionInWorld(gb2.px, gb2.py, gb2.pz);
        const float3 geometricNormalInWorld = decodeVector(gb2.qGeometricNormal);
        const float3 vOut = normalize(camera.position - positionInWorld);
        const float frontHit = dot(vOut, geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
        positionInWorld = offsetRayOrigin(positionInWorld, frontHit * geometricNormalInWorld);

        const ReferenceFrame shadingFrame(decodeVector(gb3.qShadingNormal), decodeVector(gb3.qShadingTangent));
        const float3 vOutLocal = shadingFrame.toLocal(vOut);
        const GfxMaterialDesc &mat = s->materials[gb3.matSlot];
        const BSDF bsdf = setupBsdf(s, gb3.matSlot, decodeTexCoords(gb3.qTexCoord));

        const uint32_t curResIndex = p->currentReservoirIndex & 1;
        const Reservoir reservoir = loadReservoir(f, curResIndex, pix);
        const GB1 reservoirInfo = f->reservoirInfo[curResIndex][pix];

        contribution = float3(0.0f);
        if (vOutLocal.z > 0) {
            float3 emittance(0.0f);
            if (mat.hasEmittance)
                emittance = float3(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
            contribution += emittance / kPi;
        }

        const LightSample lightSample = reservoir.sample;
        float3 directCont(0.0f);
        const float recPDFEstimate = reservoirInfo.mvx;
        if (recPDFEstimate > 0 && std::isfinite(recPDFEstimate)) {
            const bool visDone = p->reuseVisibility &&
                (!p->enableTemporalReuse || (p->enableSpatialReuse && p->useUnbiasedEstimator));
            if (visDone)
                directCont = performDirectLighting<false>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, lightSample);
            else
                directCont = performDirectLighting<true>(s, positionInWorld, vOutLocal, shadingFrame, bsdf, lightSample);
        }
        contribution += recPDFEstimate * directCont;
    }
    else if (useEnvLight(s, p)) { // :620-629: the environment seen directly
        const float2 texCoord = decodeTexCoords(gb3.qTexCoord);
        contribution = p->envLightPowerCoeff * s->env.fetch(texCoord.x, texCoord.y);
    }

    float3 prevColorResult(0.0f);
    if (p->numAccumFrames > 0)
        prevColorResult = float3(f->beauty[pix].x, f->beauty[pix].y, f->beauty[pix].z);
    const float curWeight = 1.0f / (1 + p->numAccumFrames);
    const float3 colorResult = (1 - curWeight) * prevColorResult + curWeight * contribution;
    f->beauty[pix] = F4{ colorResult.x, colorResult.y, colorResult.z, 1.0f };
}

extern "C" void orc_restir(orc_frame* f, const GfxFrameParams* p, int pass, int numThreads) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    const Camera camera = makeCamera(p->camera);
    const Camera prevCamera = makeCamera(p->prevCamera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads)
    for (int64_t yy = y0; yy < (int64_t)y1; ++yy) {
        const uint32_t y = (uint32_t)yy;
        for (uint32_t x = 0; x < W; ++x) {
            switch (pass) {
            case GFX_RESTIR_INITIAL_RIS: performInitialAndTemporalRIS<false, false>(f, p, camera, prevCamera, x, y); break;
            case GFX_RESTIR_INITIAL_AND_TEMPORAL_BIASED: performInitialAndTemporalRIS<true, false>(f, p, camera, prevCamera, x, y); break;
            case GFX_RESTIR_INITIAL_AND_TEMPORAL_UNBIASED: performInitialAndTemporalRIS<true, true>(f, p, camera, prevCamera, x, y); break;
            case GFX_RESTIR_SPATIAL_BIASED: performSpatialRIS<false>(f, p, camera, prevCamera, x, y); break;
            case GFX_RESTIR_SPATIAL_UNBIASED: performSpatialRIS<true>(f, p, camera, prevCamera, x, y); break;
            case GFX_RESTIR_SHADING: shading(f, p, camera, x, y); break;
            default: break;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// path tracing (path_tracing/gpu_kernels/optix_pathtracing_kernels.cu)
// ---------------------------------------------------------------------------------------
#include "pathtrace.inl"
#include "nrc_pathtrace.inl"
#include "regir.inl"
#include "restir_rearch.inl"

extern "C" uint64_t orc_restir_rearch(orc_frame* f, const GfxFrameParams* p, int pass, int numThreads) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    return restirRearch(f, p, pass, numThreads);
}

// test hook of light sampling, the oracle's side of gfx_light_sample_debug (include/gfxb200.h) for ops 0 and 3-7: the same
// records of 16 floats, params = {envLightRotation, envLightPowerCoeff, enableEnvLight != 0}.  Op 0's key is the library's light
// record index (every triangle of every emissive geometry, in instance order) or its kPickNone code for an early out.
extern "C" int orc_light_sample_debug(orc_scene* s, int op, const float* params, const float* in, uint32_t n, float* out) {
    if (op < 0 || op > 7 || op == 1 || op == 2)
        return -2;
    if ((op == 3 || op == 4) && !s->env.present())
        return -1;
    GfxFrameParams p;
    std::memset(&p, 0, sizeof(p));
    p.envLightRotation = params[0];
    p.envLightPowerCoeff = params[1];
    p.enableEnvLight = params[2] != 0.0f ? 1u : 0u;
    const uint32_t kPickNone = 0x40000000u;
    std::vector<uint32_t> lightTriBase; // per flattened geometry, 0xFFFFFFFF for one without an emitter
    uint32_t numLightTris = 0;
    for (const InstData &inst : s->instances)
        for (uint32_t k = 0; k < inst.desc.numMeshSlots; ++k) {
            const MeshData &mesh = s->meshes[s->instanceMeshSlots[inst.desc.firstMeshSlot + k]];
            lightTriBase.push_back(s->materials[mesh.materialSlot].hasEmittance ? numLightTris : 0xFFFFFFFFu);
            if (s->materials[mesh.materialSlot].hasEmittance)
                numLightTris += mesh.numTriangles;
        }
    std::vector<uint32_t> geomBase(s->instances.size());
    for (size_t i = 0, g = 0; i < s->instances.size(); g += s->instances[i].desc.numMeshSlots, ++i)
        geomBase[i] = (uint32_t)g;
    auto bits = [](uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; };
    auto asUint = [](float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; };
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < (int64_t)n; ++r) {
        const float* a = in + 16 * r;
        float* o = out + 16 * r;
        for (int k = 0; k < 16; ++k)
            o[k] = 0.0f;
        if (op == 0) {
            LightSample ls;
            ls.emittance = ls.position = ls.normal = float3(0.0f);
            float density = 0.0f;
            LightPickInfo pick;
            sampleLight(s, &p, a[0], false, a[1], a[2], &ls, &density, &pick);
            const InstData &inst = s->instances[pick.instSlot];
            const uint32_t geomSlot = inst.desc.firstMeshSlot + pick.geomInstIndexInInst;
            uint32_t key;
            if (pick.stage == 0)
                key = kPickNone | 0x20000000u | pick.instSlot;
            else if (pick.stage == 1)
                key = kPickNone | geomSlot;
            else if (lightTriBase[geomBase[pick.instSlot] + pick.geomInstIndexInInst] == 0xFFFFFFFFu)
                key = kPickNone | 0x10000000u | geomSlot;
            else
                key = lightTriBase[geomBase[pick.instSlot] + pick.geomInstIndexInInst] + pick.primIndex;
            o[0] = bits(key);
            o[1] = ls.position.x; o[2] = ls.position.y; o[3] = ls.position.z;
            o[4] = ls.normal.x; o[5] = ls.normal.y; o[6] = ls.normal.z;
            o[7] = ls.emittance.x; o[8] = ls.emittance.y; o[9] = ls.emittance.z;
            o[10] = density;
            o[11] = pick.lightProb;
        }
        else if (op == 3) {
            LightSample ls;
            ls.emittance = ls.position = ls.normal = float3(0.0f);
            float density = 0.0f;
            sampleLight(s, &p, 0.0f, true, a[0], a[1], &ls, &density);
            o[0] = ls.position.x; o[1] = ls.position.y; o[2] = ls.position.z;
            o[3] = density;
            o[4] = ls.emittance.x; o[5] = ls.emittance.y; o[6] = ls.emittance.z;
        }
        else if (op == 4) {
            const EnvMissTerms m = envMissTerms(s, &p, float3(a[0], a[1], a[2]), a[3], a[4]);
            o[0] = m.hypAreaPDensity; o[1] = m.misWeight; o[2] = m.texCoord.x; o[3] = m.texCoord.y;
        }
        else if (op == 5) {
            const uint32_t instSlot = asUint(a[0]), geomInInst = asUint(a[1]), primIndex = asUint(a[2]);
            if (instSlot < s->instances.size() && geomInInst < s->instances[instSlot].desc.numMeshSlots) {
                const InstData &inst = s->instances[instSlot];
                const MeshData &mesh = s->meshes[s->instanceMeshSlots[inst.desc.firstMeshSlot + geomInInst]];
                if (primIndex < mesh.numTriangles) {
                    SurfacePoint sp;
                    computeSurfacePointAtHit(s, &p, inst, mesh, primIndex, a[3], a[4], &sp);
                    o[0] = sp.hypAreaPDensity;
                }
            }
        }
        else {
            float ul = op == 6 ? a[2] : a[0], prob = 0.0f;
            const bool env = op == 6 ? chooseEnvForCandidate(s, &p, asUint(a[0]), asUint(a[1]), &ul, &prob) : chooseEnvForNee(s, &p, &ul, &prob);
            o[0] = env ? 1.0f : 0.0f; o[1] = ul; o[2] = prob;
        }
    }
    return 0;
}
