// oracle/svgf_app.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of the SVGF app's own path tracer and of the
// pass it runs when SVGF is switched off:
//   pathTrace_rayGen_generic        svgf/gpu_kernels/optix_pathtracing_kernels.cu:193-337 (up to the temporal accumulation,
//                                   which denoise.cpp restates as GFX_SVGF_TEMPORAL_ACCUMULATE)
//   pathTrace_closestHit_generic    :381-468 (Russian roulette from pathLength 3, specular mollification)
//   miss program                    :482-513 (the path tracing app's body)
//   ReferenceFrame(normal)          common/common_device.cuh:158-160, makeCoordinateSystem (basic_types.h:2602-2609)
//   offsetRayOriginNaive            common/common_device.cuh:104-108, RayEpsilon = 1e-4 (:6)
//   BSDFFlags::Regularize           common/common_device.cuh:795-797 (DiffuseAndSpecular), :821-823 (SimplePBR)
//   feedbackNoisyLighting           svgf/gpu_kernels/svgf.cu:356-374
// The first vertex comes from this oracle's ray-cast G-buffer (GBuffer0's instance, mesh, primitive and barycentrics), as
// the GL G-buffer's position, normalised shading normal and texture coordinate would.  This file compiles render.cpp into
// its own library, liborc_svgf_app.so (Makefile.svgf_app, bound by tests/oracle_svgf_app.py), and links denoise.o, so the
// SVGF passes run on the frames of that library.
#include "render.cpp"

extern "C" {
struct orc_svgf;
void* orc_svgf_buffer_ptr(orc_svgf* s, int id, uint32_t index, size_t* bytes); // denoise.cpp
}

namespace {

// bsdf.setup(mat, texCoord, 0.0f, BSDFFlags::Regularize): the material's constants or texels as setupBsdf fetches them, then
// the smoothness halved (before the 0.999 clamp for DiffuseAndSpecular, after it for SimplePBR); Lambert ignores the flag
BSDF setupBsdfRegularized(const orc_scene* s, uint32_t matSlot, const float2 &texCoord) {
    const GfxMaterialDesc &m = s->materials[matSlot];
    float p0[3] = { m.p0[0], m.p0[1], m.p0[2] }, p1[3] = { m.p1[0], m.p1[1], m.p1[2] }, p2 = m.p2;
    if (!s->materialTextures.empty()) {
        const uint32_t* tex = &s->materialTextures[4 * (size_t)matSlot];
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
    }
    BSDF b;
    b.setup<true>(m.bsdfType, p0, p1, p2);
    return b;
}

ReferenceFrame frameFromNormal(const float3 &normal) { // ReferenceFrame(const Normal3D &)
    ReferenceFrame fr;
    fr.normal = normal;
    makeCoordinateSystem(normal, &fr.tangent, &fr.bitangent);
    return fr;
}

float3 offsetRayOriginNaive(const float3 &p, const float3 &geometricNormal) {
    return p + 1e-4f * geometricNormal;
}

// RGB max(contribution, RGB(0)) = std::fmax per component: a NaN becomes 0
float maxZero(float v) { return v > 0.0f ? v : 0.0f; }

void svgfAppPixel(orc_frame* f, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y, PathTraceCounters* counters) {
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const uint32_t maxPathLength = p->maxPathLength ? p->maxPathLength : 5u; // svgf_main.cpp:1729
    const bool mollifySpecular = (p->svgfFlags & GFX_SVGF_MOLLIFY_SPECULAR) != 0;
    if (gb0.instSlot == 0xFFFFFFFFu) { // :213-219
        f->beauty[pix] = F4{ 0.0f, 0.0f, 0.0f, 1.0f };
        f->albedo[pix] = F4{ 0.0f, 0.0f, 0.0f, 0.0f };
        return;
    }
    const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
    const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
    const InstData* inst = &s->instances[gb0.instSlot];
    const MeshData* mesh = &s->meshes[gb0.geomInstSlot];
    SurfacePoint sp;
    computeSurfacePointFromGBuffer(s, *inst, *mesh, gb0.primIndex, bcB, bcC, &sp);

    float3 contribution(0.0f);
    float3 alpha(1.0f);
    const float initImportance = sRGB_calcLuminance(alpha);
    PCG32RNG rng{ f->rng[pix] };

    // shading on the first hit (:233-268)
    float3 positionInWorld = sp.positionInWorld;
    const float3 shadingNormalInWorld = sp.shadingNormalInWorld;
    float3 dhReflectance;
    float3 vIn;
    float dirPDensity;
    {
        const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];
        const float3 geometricNormalInWorld = shadingNormalInWorld;
        const float3 vOut = normalize(camera.position - positionInWorld);
        const float frontHit = dot(vOut, geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
        const ReferenceFrame shadingFrame = frameFromNormal(shadingNormalInWorld);
        positionInWorld = offsetRayOriginNaive(positionInWorld, frontHit * geometricNormalInWorld);
        const float3 vOutLocal = shadingFrame.toLocal(vOut);

        if (vOutLocal.z > 0 && mat.hasEmittance) {
            const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
            contribution += alpha * emittance / kPi;
        }
        const BSDF bsdf = setupBsdf(s, mesh->materialSlot, sp.texCoord);
        dhReflectance = bsdf.evaluateDHReflectanceEstimate(vOutLocal);
        contribution += alpha * performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);

        float3 vInLocal;
        const float uDir0 = rng.getFloat0cTo1o();
        const float uDir1 = rng.getFloat0cTo1o();
        alpha *= bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
        vIn = shadingFrame.fromLocal(vInLocal);
    }

    // path extension loop (:270-317) with the closest-hit program (:381-468) inlined
    float prevDirPDensity = dirPDensity;
    uint32_t pathLength = 1;
    float3 rayOrg = positionInWorld;
    float3 rayDir = vIn;
    while (true) {
        const bool isValidSampling = prevDirPDensity > 0.0f && std::isfinite(prevDirPDensity);
        if (!isValidSampling)
            break;
        ++pathLength;
        const bool maxLengthTerminate = pathLength >= maxPathLength;

        ++counters->closestRays;
        const HitObject hit = traverseCanonical(s->bvh, rayOrg, rayDir, 0.0f, std::numeric_limits<float>::max());
        if (hit.primIndex == UINT32_MAX) { // miss program (:482-513)
            contribution += alpha * evaluateEnvLightOnMiss(s, p, rayDir, prevDirPDensity);
            break;
        }

        inst = &s->instances[s->geomToInst[hit.geomIndex]];
        mesh = &s->meshes[s->geomToMesh[hit.geomIndex]];
        computeSurfacePointAtHit(s, p, *inst, *mesh, hit.primIndex, hit.bcB, hit.bcC, &sp);
        const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];

        const float3 vOut = normalize(-rayDir);
        const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
        const ReferenceFrame shadingFrame(sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
        positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
        const float3 vOutLocal = shadingFrame.toLocal(vOut);

        // implicit light sampling with MIS (:422-435)
        if (vOutLocal.z > 0 && mat.hasEmittance) {
            const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
            const float dist2 = sqLength(positionInWorld - rayOrg);
            const float lightPDensity = sp.hypAreaPDensity * dist2 / vOutLocal.z;
            const float bsdfPDensity = prevDirPDensity;
            const float misWeight = pow2(bsdfPDensity) / (pow2(bsdfPDensity) + pow2(lightPDensity));
            contribution += alpha * emittance * (misWeight / kPi);
        }

        // Russian roulette (:437-444): none at pathLength 2, the random number is drawn all the same
        float continueProb = 1.0f;
        if (pathLength > 2)
            continueProb = std::fmin(sRGB_calcLuminance(alpha) / initImportance, 1.0f);
        if (rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate)
            break;
        alpha /= continueProb;

        // specular mollification after the first vertex (:446-450)
        const BSDF bsdf = mollifySpecular ? setupBsdfRegularized(s, mesh->materialSlot, sp.texCoord)
                                          : setupBsdf(s, mesh->materialSlot, sp.texCoord);
        contribution += alpha * performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);

        float3 vInLocal;
        const float uDir0 = rng.getFloat0cTo1o();
        const float uDir1 = rng.getFloat0cTo1o();
        alpha *= bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
        rayOrg = positionInWorld;
        rayDir = shadingFrame.fromLocal(vInLocal);
        prevDirPDensity = dirPDensity;
    }
    f->rng[pix] = rng.state;
    // :318-319; the 0.001 threshold of :331-333 is the temporal pass's
    f->beauty[pix] = F4{ maxZero(contribution.x), maxZero(contribution.y), maxZero(contribution.z), 1.0f };
    f->albedo[pix] = F4{ dhReflectance.x, dhReflectance.y, dhReflectance.z, 1.0f };
}

} // namespace

// gfx_pathtrace_launch(GFX_PT_SVGF) on the rows params->tileOriginY / tileRows; returns the number of rays traced
extern "C" uint64_t orc_svgf_app_pathtrace(orc_frame* f, const GfxFrameParams* p, int numThreads) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    const Camera camera = makeCamera(p->camera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    uint64_t rays = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays)
    for (int64_t yy = y0; yy < (int64_t)y1; ++yy) {
        PathTraceCounters counters;
        for (uint32_t x = 0; x < W; ++x)
            svgfAppPixel(f, p, camera, x, (uint32_t)yy, &counters);
        rays += counters.closestRays + counters.visibilityRays;
    }
    return rays;
}

// gfx_svgf_launch(GFX_SVGF_FEEDBACK_NOISY_LIGHTING): lighting plane 0 -> prevNoisyLighting on the rows of the frame params
extern "C" void orc_svgf_app_feedback_noisy_lighting(orc_svgf* sv, const GfxFrameParams* p, uint32_t W, uint32_t H) {
    const F4* src = (const F4*)orc_svgf_buffer_ptr(sv, GFX_BUF_SVGF_LIGHTING_VARIANCE, 0, nullptr);
    F4* dst = (F4*)orc_svgf_buffer_ptr(sv, GFX_BUF_SVGF_PREV_LIGHTING, 0, nullptr);
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    for (size_t i = (size_t)y0 * W; i < (size_t)y1 * W; ++i)
        dst[i] = src[i];
}
