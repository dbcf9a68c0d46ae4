// oracle/bump.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of the reference's bump mapping, the apps' "Enable Bump
// Mapping" switch (perFramePlp.enableBumpMapping, GfxFrameParams::enableBumpMapping; GfxSceneDesc::bumpMaps):
//   applyBumpMapping                             common/common_device.cuh:176-203
//   readModifiedNormalFromNormalMap / HeightMap  common/common_device.cuh:205-240 (sample<float4> = tex2DLod, :143-147)
//   createNormalTexture's default 1x1 texel      common/common_host.cpp:1396-1412
// at the sites where the apps tilt their shading frames: the G-buffer pass (optix_gbuffer_kernels.cu:151-154, 175-178), the
// first hit and the closest hit of the path tracers (path_tracing optix_pathtracing_kernels.cu:117-121, 252-255; regir :200-203,
// 336-339; neural_radiance_caching :182-185, 398-401) and visualizePrediction (:740-743).
// Like views.cpp, this file compiles render.cpp into its own library, liborc_bump.so (Makefile.bump, bound by
// tests/oracle_bump.py): the functions below are the oracle's G-buffer pass, path tracers and visualizePrediction pass restated
// with the bump at those sites (orc_bump_*), on the helpers of render.cpp; every other pass is render.cpp's own.  The bump maps
// of a scene are attached to it after orc_scene_create (orc_bump_attach).
#include "render.cpp"
#include <map>
#include <mutex>

// applyBumpMapping: atan of the quotient (z may be <= 0), the normal not renormalised; Matrix3x3(tangent, bitangent, normal) * v
// is fromLocal(v)
static ReferenceFrame applyBumpMapping(const float3 &modNormalInTF, const ReferenceFrame &frameToModify) {
    const float projLength = std::sqrt(modNormalInTF.x * modNormalInTF.x + modNormalInTF.y * modNormalInTF.y);
    if (projLength < 1e-3f)
        return frameToModify;
    const float tiltAngle = dm_atan(projLength / modNormalInTF.z);
    float qSin, qCos;
    dm_sincos(tiltAngle / 2, &qSin, &qCos);
    const float qX = (-modNormalInTF.y / projLength) * qSin;
    const float qY = (modNormalInTF.x / projLength) * qSin;
    const float qW = qCos;
    const float3 modTangentInTF(1 - 2 * qY * qY, 2 * qX * qY, -2 * qY * qW);
    const float3 modBitangentInTF(2 * qX * qY, 1 - 2 * qX * qX, 2 * qX * qW);
    ReferenceFrame bumpShadingFrame;
    bumpShadingFrame.tangent = frameToModify.fromLocal(modTangentInTF);
    bumpShadingFrame.bitangent = frameToModify.fromLocal(modBitangentInTF);
    bumpShadingFrame.normal = frameToModify.fromLocal(modNormalInTF);
    return bumpShadingFrame;
}

// tex2Dgather<float4>(tex, u, v, 0), channel 0, repeat addressing: the linear filter's 2x2 footprint (i0 = floor(frac(u) W - 0.5),
// i1 = i0 + 1, wrapped; one texel on when the fraction is above 255.5 / 256) in tld4's order x = (i0, j1), y = (i1, j1),
// z = (i1, j0), w = (i0, j0)
static uint32_t gatherIndex(float xB, uint32_t W) {
    const float fx = std::floor(xB);
    const int ix = dm_f2int(fx) + ((xB - fx) * 256.0f > 255.5f ? 1 : 0);
    return ix < 0 ? W - 1 : ((uint32_t)ix >= W ? (uint32_t)ix - W : (uint32_t)ix);
}
static void gatherRepeat(const ImageTexture &t, float u, float v, float out[4]) {
    const uint32_t x0 = gatherIndex((u - std::floor(u)) * t.W - 0.5f, t.W), y0 = gatherIndex((v - std::floor(v)) * t.H - 0.5f, t.H);
    const uint32_t x1 = x0 + 1 >= t.W ? 0u : x0 + 1, y1 = y0 + 1 >= t.H ? 0u : y0 + 1;
    out[0] = t.texels[4 * ((size_t)y1 * t.W + x0)];
    out[1] = t.texels[4 * ((size_t)y1 * t.W + x1)];
    out[2] = t.texels[4 * ((size_t)y0 * t.W + x1)];
    out[3] = t.texels[4 * ((size_t)y0 * t.W + x0)];
}
// readModifiedNormalFromNormalMap (:205-213, y flipped: calcDimInfo's isLeftHanded) / readModifiedNormalFromHeightMap (:227-238)
static float3 readModifiedNormal(const ImageTexture &t, uint32_t type, float u, float v) {
    if (type == GFX_BUMP_HEIGHT_MAP) {
        float h[4];
        gatherRepeat(t, u, v, h);
        const float coeff = 5.0f / 1024;
        const float dhdu = (coeff * t.W) * (h[1] - h[0]);
        const float dhdv = (coeff * t.H) * (h[0] - h[3]);
        return normalize(float3(-dhdu, dhdv, 1));
    }
    float texValue[4];
    t.fetch(u, v, texValue);
    float3 modLocalNormal(texValue[0], texValue[1], texValue[2]);
    modLocalNormal = 2.0f * modLocalNormal - float3(1.0f);
    modLocalNormal.y *= -1;
    return modLocalNormal;
}

// the bump maps of a scene: its textures (UNORM texels) and GfxSceneDesc::bumpMaps (empty = every material has the default)
struct BumpMaps {
    std::vector<ImageTexture> textures;
    std::vector<uint32_t> table;
};
static std::map<const orc_scene*, BumpMaps> g_bumpMaps;
static std::mutex g_bumpMapsMutex;

static const BumpMaps* bumpMapsOf(const orc_scene* s) {
    std::lock_guard<std::mutex> lock(g_bumpMapsMutex);
    const auto it = g_bumpMaps.find(s);
    return it == g_bumpMaps.end() ? nullptr : &it->second;
}
extern "C" void orc_bump_attach(orc_scene* s, const GfxSceneDesc* d) {
    BumpMaps b;
    if (d->bumpMaps) {
        b.textures.resize(d->numTextures);
        for (uint32_t t = 0; t < d->numTextures; ++t) {
            b.textures[t].W = d->textures[t].width;
            b.textures[t].H = d->textures[t].height;
            b.textures[t].texels.assign(d->textures[t].texels, d->textures[t].texels + 4 * (size_t)d->textures[t].width * d->textures[t].height);
        }
        b.table.assign(d->bumpMaps, d->bumpMaps + 2 * (size_t)d->numMaterials);
    }
    std::lock_guard<std::mutex> lock(g_bumpMapsMutex);
    g_bumpMaps[s] = std::move(b);
}
extern "C" void orc_bump_detach(orc_scene* s) {
    std::lock_guard<std::mutex> lock(g_bumpMapsMutex);
    g_bumpMaps.erase(s);
}

// createNormalTexture's default: the 1x1 UNORM8 texel (127, 127, 255), a normal map
static const ImageTexture &defaultBumpTexel() {
    static const ImageTexture t = [] {
        ImageTexture d;
        d.W = d.H = 1;
        d.texels = { 127.0f / 255.0f, 127.0f / 255.0f, 1.0f, 1.0f };
        return d;
    }();
    return t;
}
static const ImageTexture &bumpTextureOf(const BumpMaps* b, uint32_t matSlot, uint32_t* type) {
    const uint32_t tex = (b && !b->table.empty()) ? b->table[2 * (size_t)matSlot] : 0xFFFFFFFFu;
    *type = tex == 0xFFFFFFFFu ? (uint32_t)GFX_BUMP_NORMAL_MAP : b->table[2 * (size_t)matSlot + 1];
    return tex == 0xFFFFFFFFu ? defaultBumpTexel() : b->textures[tex];
}
// the frame of a shading point as every bump-mapping app builds it
static ReferenceFrame shadingFrameAt(const orc_scene* s, const GfxFrameParams* p, uint32_t matSlot, const float2 &texCoord,
                                     const float3 &shadingNormal, const float3 &tangent) {
    const ReferenceFrame frame(shadingNormal, tangent);
    if (!p->enableBumpMapping)
        return frame;
    uint32_t type;
    const ImageTexture &t = bumpTextureOf(bumpMapsOf(s), matSlot, &type);
    return applyBumpMapping(readModifiedNormal(t, type, texCoord.x, texCoord.y), frame);
}

// test hooks, the oracle's side of gfx_bump_debug: op 0 readModifiedNormal (2 floats in, 3 out), 1 applyBumpMapping (12 in, 9 out),
// 2 the gather (2 in, 4 out); -1 for a material slot out of range.  And dm_atan over an array, for its bound against libm.
extern "C" int orc_bump_query(orc_scene* s, int op, uint32_t matSlot, const float* in, uint32_t n, float* out) {
    if (op != 1 && matSlot >= s->materials.size())
        return -1;
    const BumpMaps* b = bumpMapsOf(s);
    for (uint32_t i = 0; i < n; ++i) {
        if (op == 1) {
            const float* a = in + 12 * (size_t)i;
            ReferenceFrame frame;
            frame.tangent = float3(a[3], a[4], a[5]);
            frame.bitangent = float3(a[6], a[7], a[8]);
            frame.normal = float3(a[9], a[10], a[11]);
            const ReferenceFrame r = applyBumpMapping(float3(a[0], a[1], a[2]), frame);
            const float o[9] = { r.tangent.x, r.tangent.y, r.tangent.z, r.bitangent.x, r.bitangent.y, r.bitangent.z, r.normal.x, r.normal.y, r.normal.z };
            std::memcpy(out + 9 * (size_t)i, o, sizeof(o));
            continue;
        }
        const float u = in[2 * (size_t)i], v = in[2 * (size_t)i + 1];
        uint32_t type;
        const ImageTexture &t = bumpTextureOf(b, matSlot, &type);
        if (op == 0) {
            const float3 m = readModifiedNormal(t, type, u, v);
            out[3 * (size_t)i] = m.x; out[3 * (size_t)i + 1] = m.y; out[3 * (size_t)i + 2] = m.z;
        }
        else {
            gatherRepeat(t, u, v, out + 4 * (size_t)i);
        }
    }
    return 0;
}
extern "C" void orc_bump_dm_atan(const float* x, float* y, size_t n) { for (size_t i = 0; i < n; ++i) y[i] = dm_atan(x[i]); }

// ---------------------------------------------------------------------------------------
// render.cpp's G-buffer pass, pathtrace.inl / regir.inl / nrc_pathtrace.inl's path tracers and views.cpp's visualizePrediction
// pass with the bump at the frame sites (shadingFrameAt)
// ---------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------
// G-buffer — optix_gbuffer_kernels.cu:5-243
// ---------------------------------------------------------------------------------------
extern "C" void orc_bump_gbuffer(orc_frame* f, const GfxFrameParams* p, int numThreads) {
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
                const ReferenceFrame shadingFrame = shadingFrameAt(s, p, matSlot, texCoord, shadingNormalInWorld, texCoord0DirInWorld);
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

static void pathTracePixelBump(orc_frame* f, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y,
                           PathTraceCounters* counters) {
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
    const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
    const uint32_t maxPathLength = p->maxPathLength ? p->maxPathLength : 5u; // 0 = the hosts' default (path_tracing_main.cpp:1519)

    float3 contribution(0.001f, 0.001f, 0.001f);
    if (gb0.instSlot != 0xFFFFFFFFu) {
        const InstData* inst = &s->instances[gb0.instSlot];
        const MeshData* mesh = &s->meshes[gb0.geomInstSlot];
        SurfacePoint sp;
        computeSurfacePointFromGBuffer(s, *inst, *mesh, gb0.primIndex, bcB, bcC, &sp);

        float3 alpha(1.0f);
        const float initImportance = sRGB_calcLuminance(alpha);
        PCG32RNG rng{ f->rng[pix] };

        // shading on the first hit (:106-146)
        float3 positionInWorld = sp.positionInWorld;
        float3 vIn;
        float dirPDensity;
        {
            const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];
            const float3 vOut = normalize(camera.position - positionInWorld);
            const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            positionInWorld = offsetRayOrigin(positionInWorld, frontHit * sp.geometricNormalInWorld);
            const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh->materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
            const float3 vOutLocal = shadingFrame.toLocal(vOut);

            contribution = float3(0.0f);
            if (vOutLocal.z > 0 && mat.hasEmittance) {
                const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
                contribution += alpha * emittance / kPi;
            }
            const BSDF bsdf = setupBsdf(s, mesh->materialSlot, sp.texCoord);
            contribution += alpha * performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);

            float3 vInLocal;
            const float uDir0 = rng.getFloat0cTo1o();
            const float uDir1 = rng.getFloat0cTo1o();
            alpha *= bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
            vIn = shadingFrame.fromLocal(vInLocal);
        }

        // path extension loop (:148-194) with the closest-hit program (:218-300) inlined
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
            if (hit.primIndex == UINT32_MAX) { // miss program (:310-341): implicit environment light sampling with MIS
                contribution += alpha * evaluateEnvLightOnMiss(s, p, rayDir, prevDirPDensity);
                break;
            }

            inst = &s->instances[s->geomToInst[hit.geomIndex]];
            mesh = &s->meshes[s->geomToMesh[hit.geomIndex]];
            computeSurfacePointAtHit(s, p, *inst, *mesh, hit.primIndex, hit.bcB, hit.bcC, &sp);
            const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];

            const float3 vOut = normalize(-rayDir);
            const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh->materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
            positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
            const float3 vOutLocal = shadingFrame.toLocal(vOut);

            // implicit light sampling with MIS (:262-275)
            if (vOutLocal.z > 0 && mat.hasEmittance) {
                const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
                const float dist2 = sqLength(positionInWorld - rayOrg); // sqDistance(rayOrigin, positionInWorld)
                const float lightPDensity = sp.hypAreaPDensity * dist2 / vOutLocal.z;
                const float bsdfPDensity = prevDirPDensity;
                const float misWeight = pow2(bsdfPDensity) / (pow2(bsdfPDensity) + pow2(lightPDensity));
                contribution += alpha * emittance * (misWeight / kPi);
            }

            // Russian roulette (:277-281)
            const float continueProb = std::fmin(sRGB_calcLuminance(alpha) / initImportance, 1.0f);
            if (rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate)
                break;
            alpha /= continueProb;

            const BSDF bsdf = setupBsdf(s, mesh->materialSlot, sp.texCoord);
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
    }
    else if (useEnvLight(s, p)) { // :200-207: the environment seen directly; the miss program left (u, v) in the barycentrics
        contribution = p->envLightPowerCoeff * s->env.fetch(bcB, bcC);
    }

    float3 prevColorResult(0.0f);
    if (p->numAccumFrames > 0)
        prevColorResult = float3(f->beauty[pix].x, f->beauty[pix].y, f->beauty[pix].z);
    const float curWeight = 1.0f / (1 + p->numAccumFrames);
    const float3 colorResult = (1 - curWeight) * prevColorResult + curWeight * contribution;
    f->beauty[pix] = F4{ colorResult.x, colorResult.y, colorResult.z, 1.0f };
}

static void regirPathTracePixelBump(orc_frame* f, orc_regir* r, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y,
                                PathTraceCounters* counters) {
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
    const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));

    float3 contribution(0.001f, 0.001f, 0.001f);
    if (gb0.instSlot != 0xFFFFFFFFu) {
        const InstData* inst = &s->instances[gb0.instSlot];
        const MeshData* mesh = &s->meshes[gb0.geomInstSlot];
        SurfacePoint sp;
        computeSurfacePointFromGBuffer(s, *inst, *mesh, gb0.primIndex, bcB, bcC, &sp);

        float3 alpha(1.0f);
        const float initImportance = sRGB_calcLuminance(alpha);
        PCG32RNG rng{ f->rng[pix] };
        float3 positionInWorld = sp.positionInWorld;
        float3 vIn;
        float dirPDensity;
        {
            const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];
            const float3 vOut = normalize(camera.position - positionInWorld);
            const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            positionInWorld = offsetRayOrigin(positionInWorld, frontHit * sp.geometricNormalInWorld);
            const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh->materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
            const float3 vOutLocal = shadingFrame.toLocal(vOut);
            contribution = float3(0.0f);
            if (vOutLocal.z > 0 && mat.hasEmittance) {
                const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
                contribution += alpha * emittance / kPi;
            }
            const BSDF bsdf = setupBsdf(s, mesh->materialSlot, sp.texCoord);
            contribution += alpha * regirNextEventEstimation(s, r, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);
            float3 vInLocal;
            const float uDir0 = rng.getFloat0cTo1o();
            const float uDir1 = rng.getFloat0cTo1o();
            alpha *= bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
            vIn = shadingFrame.fromLocal(vInLocal);
        }

        float prevDirPDensity = dirPDensity;
        uint32_t pathLength = 1;
        float3 rayOrg = positionInWorld;
        float3 rayDir = vIn;
        while (true) {
            const bool isValidSampling = prevDirPDensity > 0.0f && std::isfinite(prevDirPDensity);
            if (!isValidSampling)
                break;
            ++pathLength;
            const bool maxLengthTerminate = pathLength >= (p->maxPathLength ? p->maxPathLength : 5u);
            // useReGIR: length limit and Russian roulette before the trace (:254-263) ...
            if (maxLengthTerminate)
                break;
            {
                const float continueProb = std::fmin(sRGB_calcLuminance(alpha) / initImportance, 1.0f);
                if (rng.getFloat0cTo1o() >= continueProb)
                    break;
                alpha /= continueProb;
            }

            ++counters->closestRays;
            const HitObject hit = traverseCanonical(s->bvh, rayOrg, rayDir, 0.0f, std::numeric_limits<float>::max());
            if (hit.primIndex == UINT32_MAX)
                break;

            inst = &s->instances[s->geomToInst[hit.geomIndex]];
            mesh = &s->meshes[s->geomToMesh[hit.geomIndex]];
            computeSurfacePointAtHit(s, p, *inst, *mesh, hit.primIndex, hit.bcB, hit.bcC, &sp);
            sp.hypAreaPDensity = 0.0f; // never written by computeSurfacePoint<false, ...>: see the header of this file
            const GfxMaterialDesc &mat = s->materials[mesh->materialSlot];

            const float3 vOut = normalize(-rayDir);
            const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh->materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
            positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
            const float3 vOutLocal = shadingFrame.toLocal(vOut);

            // ... and, because useImplicitLightSampling is on, once more in the closest-hit program (:343-364)
            if (vOutLocal.z > 0 && mat.hasEmittance) {
                const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
                const float dist2 = sqLength(positionInWorld - rayOrg);
                const float lightPDensity = sp.hypAreaPDensity * dist2 / vOutLocal.z;
                const float bsdfPDensity = prevDirPDensity;
                const float misWeight = pow2(bsdfPDensity) / (pow2(bsdfPDensity) + pow2(lightPDensity));
                contribution += alpha * emittance * (misWeight / kPi);
            }
            const float continueProb = std::fmin(sRGB_calcLuminance(alpha) / initImportance, 1.0f);
            if (rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate)
                break;
            alpha /= continueProb;

            const BSDF bsdf = setupBsdf(s, mesh->materialSlot, sp.texCoord);
            contribution += alpha * regirNextEventEstimation(s, r, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);

            float3 vInLocal;
            const float uDir0 = rng.getFloat0cTo1o();
            const float uDir1 = rng.getFloat0cTo1o();
            alpha *= bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
            rayOrg = positionInWorld;
            rayDir = shadingFrame.fromLocal(vInLocal);
            prevDirPDensity = dirPDensity;
        }
        f->rng[pix] = rng.state;
    }
    else if (useEnvLight(s, p)) { // regir/gpu_kernels/optix_pathtracing_kernels.cu:283-290; the ReGIR ray type's miss program is empty
        contribution = p->envLightPowerCoeff * s->env.fetch(bcB, bcC);
    }

    float3 prevColorResult(0.0f);
    if (p->numAccumFrames > 0)
        prevColorResult = float3(f->beauty[pix].x, f->beauty[pix].y, f->beauty[pix].z);
    const float curWeight = 1.0f / (1 + p->numAccumFrames);
    const float3 colorResult = (1 - curWeight) * prevColorResult + curWeight * contribution;
    f->beauty[pix] = F4{ colorResult.x, colorResult.y, colorResult.z, 1.0f };
}

static uint64_t regirPathTraceBump(orc_frame* f, const GfxFrameParams* p, int numThreads) {
    orc_regir* r = f->regir;
    if (!r)
        return ORC_NOT_READY;
    const Camera camera = makeCamera(p->camera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    uint64_t rays = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays)
    for (int64_t yy = y0; yy < (int64_t)y1; ++yy) {
        PathTraceCounters counters;
        for (uint32_t x = 0; x < W; ++x)
            regirPathTracePixelBump(f, r, p, camera, x, (uint32_t)yy, &counters);
        rays += counters.closestRays + counters.visibilityRays;
    }
    return rays;
}

// ray generation up to the path extension loop (:95-283)
static void nrcRayGenBump(orc_frame* f, orc_nrc_frame* n, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y,
                      PathTraceCounters* counters) {
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
    const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
    NrcPathState &st = n->paths[pix];
    st = NrcPathState();

    const uint32_t tileSizeX = n->state[NRC_TILE_SIZE + 2 * bufIdx], tileSizeY = n->state[NRC_TILE_SIZE + 2 * bufIdx + 1];
    const uint32_t numPixelsInTile = tileSizeX * tileSizeY;
    const uint32_t localLinearIndex = (y % tileSizeY) * tileSizeX + (x % tileSizeX);
    st.isTrainingPath = (localLinearIndex + n->state[NRC_OFFSET_TRAINING_PATH]) % numPixelsInTile == 0;
    const uint32_t numTilesX = (f->W + tileSizeX - 1) / tileSizeX;
    const uint32_t tileX = x / tileSizeX, tileY = y / tileSizeY;
    st.linearTileIndex = tileY * numTilesX + tileX;
    const uint32_t localLinearTileIndex = (tileY % 4) * 4 + (tileX % 4);
    st.isUnbiasedTrainingTile = (localLinearTileIndex + n->state[NRC_OFFSET_UNBIASED_TILE]) % 16 == 0;

    st.contribution = float3(0.001f, 0.001f, 0.001f);
    st.renderingPathEndsWithCache = false;
    st.trainingSuffixEndsWithCache = false;
    st.pathLength = 1;
    if (gb0.instSlot == 0xFFFFFFFFu) {
        if (useEnvLight(s, p)) // :323-331: the environment seen directly, (u, v) left in the barycentrics by the miss program
            st.contribution = p->envLightPowerCoeff * s->env.fetch(bcB, bcC);
        return;
    }

    const InstData &inst = s->instances[gb0.instSlot];
    const MeshData &mesh = s->meshes[gb0.geomInstSlot];
    SurfacePoint sp;
    computeSurfacePointFromGBuffer(s, inst, mesh, gb0.primIndex, bcB, bcC, &sp);

    float3 alpha(1.0f);
    PCG32RNG rng{ f->rng[pix] };
    const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];

    float3 vOut = camera.position - sp.positionInWorld;
    const float primaryDist2 = sqLength(vOut);
    vOut /= std::sqrt(primaryDist2);
    const float primaryDotVN = dot(vOut, sp.geometricNormalInWorld);
    const float frontHit = primaryDotVN >= 0.0f ? 1.0f : -1.0f;
    const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
    st.primaryPathSpread = primaryDist2 / (4 * kPi * std::fabs(primaryDotVN));

    const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh.materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
    const float3 vOutLocal = shadingFrame.toLocal(vOut);

    float3 contribution(0.0f);
    if (vOutLocal.z > 0 && mat.hasEmittance) {
        const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
        contribution += alpha * emittance / kPi;
    }
    const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);
    const float3 directContNEE = performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);
    contribution += alpha * directContNEE;

    float3 vInLocal;
    float dirPDensity;
    const float uDir0 = rng.getFloat0cTo1o();
    const float uDir1 = rng.getFloat0cTo1o();
    const float3 localThroughput = bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
    alpha *= localThroughput;

    st.prevTrainDataIndex = kInvalidVertexDataIndex;
    if (st.isTrainingPath) {
        NrcStagedVertex &sv = n->staged[st.linearTileIndex];
        sv.want = true;
        sv.fromRayGen = true;
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, sv.query);
        sv.localThroughput = localThroughput;
        sv.directContNEE = directContNEE;
        sv.pathLength = st.pathLength;
    }

    st.active = true;
    st.rng = rng;
    st.alpha = alpha;
    st.contribution = contribution;
    st.prevDirPDensity = dirPDensity;
    st.curSqrtPathSpread = 0.0f;
    st.prevLocalThroughput = localThroughput;
    st.rayOrg = positionInWorld;
    st.rayDir = shadingFrame.fromLocal(vInLocal);
}

// one iteration of the path extension loop (:285-311) with the closest-hit program (:363-623) inlined
static void nrcExtendBump(orc_frame* f, orc_nrc_frame* n, const GfxFrameParams* p, size_t pix, PathTraceCounters* counters) {
    const orc_scene* s = f->scene;
    NrcPathState &st = n->paths[pix];
    const bool isValidSampling = st.prevDirPDensity > 0.0f && std::isfinite(st.prevDirPDensity);
    if (!isValidSampling) {
        st.active = false;
        return;
    }
    ++st.pathLength;
    const bool maxLengthTerminate = (st.pathLength >= p->maxPathLength && p->maxPathLength > 0) || st.pathLength >= kMaxNrcRounds;
    st.active = false; // rwPayload.terminate = true

    ++counters->closestRays;
    const HitObject hit = traverseCanonical(s->bvh, st.rayOrg, st.rayDir, 0.0f, std::numeric_limits<float>::max());
    if (hit.primIndex == UINT32_MAX) { // pathTrace_miss_generic (:625-672)
        if (useEnvLight(s, p)) {
            const float3 directContImplicit = evaluateEnvLightOnMiss(s, p, st.rayDir, st.prevDirPDensity, true);
            if (!st.renderingPathEndsWithCache)
                st.contribution += st.alpha * directContImplicit;
            if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
                float* tgt = &n->trainTarget[0][3 * (size_t)st.prevTrainDataIndex];
                const float3 add = st.prevLocalThroughput * directContImplicit;
                tgt[0] += add.x; tgt[1] += add.y; tgt[2] += add.z;
            }
        }
        return;
    }

    const InstData &inst = s->instances[s->geomToInst[hit.geomIndex]];
    const MeshData &mesh = s->meshes[s->geomToMesh[hit.geomIndex]];
    SurfacePoint sp;
    computeSurfacePointAtHit(s, p, inst, mesh, hit.primIndex, hit.bcB, hit.bcC, &sp);
    const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];

    const float3 vOut = normalize(-st.rayDir);
    const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
    const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh.materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
    const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
    const float3 vOutLocal = shadingFrame.toLocal(vOut);

    const float dist2 = sqLength(positionInWorld - st.rayOrg);
    st.curSqrtPathSpread += std::sqrt(dist2 / (st.prevDirPDensity * std::fabs(vOutLocal.z)));

    // implicit light sampling (:417-445)
    if (vOutLocal.z > 0 && mat.hasEmittance) {
        const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
        const float lightPDensity = sp.hypAreaPDensity * dist2 / vOutLocal.z;
        const float bsdfPDensity = st.prevDirPDensity;
        const float misWeight = pow2(bsdfPDensity) / (pow2(bsdfPDensity) + pow2(lightPDensity));
        const float3 directContImplicit = emittance * (misWeight / kPi);
        if (!st.renderingPathEndsWithCache)
            st.contribution += st.alpha * directContImplicit;
        if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
            float* tgt = &n->trainTarget[0][3 * (size_t)st.prevTrainDataIndex];
            const float3 add = st.prevLocalThroughput * directContImplicit;
            tgt[0] += add.x; tgt[1] += add.y; tgt[2] += add.z;
        }
    }

    // Russian roulette (:447-469)
    bool performRR = true;
    bool terminatedByRR = false;
    float recContinueProb = 1.0f;
    if (st.isTrainingPath)
        performRR = st.pathLength > 2;
    if (performRR) {
        const float continueProb = std::fmin(sRGB_calcLuminance(st.alpha) / sRGB_calcLuminance(float3(1.0f)), 1.0f);
        if (st.rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate) {
            if (st.renderingPathEndsWithCache && st.isTrainingPath && st.isUnbiasedTrainingTile)
                return;
            terminatedByRR = true;
        }
        recContinueProb = 1.0f / continueProb;
    }

    const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);

    // path termination by the spread heuristic (:474-531)
    bool endsWithCache = pow2(st.curSqrtPathSpread) > kPathTerminationFactor * st.primaryPathSpread;
    if (st.renderingPathEndsWithCache && st.isTrainingPath && st.isUnbiasedTrainingTile)
        endsWithCache = false;
    if (endsWithCache) {
        float query[14];
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, query);
        if (!st.renderingPathEndsWithCache) {
            std::memcpy(&n->inferenceQuery[14 * pix], query, sizeof(query));
            writeTerminalInfo(n, pix, st.alpha, st.pathLength, true, st.isTrainingPath, st.isUnbiasedTrainingTile);
            st.renderingPathEndsWithCache = true;
            if (st.isTrainingPath)
                st.curSqrtPathSpread = 0;
            else
                return;
        }
        else {
            if (!st.trainingSuffixEndsWithCache) {
                const size_t offset = (size_t)f->W * f->H;
                std::memcpy(&n->inferenceQuery[14 * (offset + st.linearTileIndex)], query, sizeof(query));
                n->suffixTerminal[st.linearTileIndex] = packSuffixTerminal(st.prevTrainDataIndex, true, st.pathLength);
                st.trainingSuffixEndsWithCache = true;
            }
            return;
        }
    }

    if (terminatedByRR)
        return;
    st.alpha *= recContinueProb;
    if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
        uint32_t* vi = &n->trainVertexInfo[4 * (size_t)st.prevTrainDataIndex];
        for (int c = 0; c < 3; ++c)
            vi[c] = f2u(u2f(vi[c]) * recContinueProb);
    }

    const float3 directContNEE = performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, st.rng, counters);
    if (!st.renderingPathEndsWithCache)
        st.contribution += st.alpha * directContNEE;

    float3 vInLocal;
    float dirPDensity;
    const float uDir0 = st.rng.getFloat0cTo1o();
    const float uDir1 = st.rng.getFloat0cTo1o();
    const float3 localThroughput = bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
    st.alpha *= localThroughput;
    st.rayOrg = positionInWorld;
    st.rayDir = shadingFrame.fromLocal(vInLocal);
    st.prevDirPDensity = dirPDensity;
    st.prevLocalThroughput = localThroughput;
    st.active = true; // rwPayload.terminate = false

    if (st.isTrainingPath && !st.trainingSuffixEndsWithCache) {
        NrcStagedVertex &sv = n->staged[st.linearTileIndex];
        sv.want = true;
        sv.fromRayGen = false;
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, sv.query);
        sv.localThroughput = localThroughput;
        sv.directContNEE = directContNEE;
        sv.pathLength = st.pathLength;
    }
}

static uint64_t nrcPathTraceBump(orc_frame* f, const GfxFrameParams* p, int numThreads) {
    orc_nrc_frame* n = nrcFrame(f);
    const Camera camera = makeCamera(p->camera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const uint32_t tileSizeX = n->state[NRC_TILE_SIZE + 2 * bufIdx], tileSizeY = n->state[NRC_TILE_SIZE + 2 * bufIdx + 1];
    const uint32_t numTilesX = (W + tileSizeX - 1) / tileSizeX, numTilesY = (H + tileSizeY - 1) / tileSizeY;
    std::vector<uint32_t> tileToPixel((size_t)numTilesX * numTilesY, 0u);
    for (auto &sv : n->staged)
        sv.want = false;

    // a strip of rows (tileOriginY / tileRows) is one rank's share of a sharded frame
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    for (size_t pix = 0; pix < (size_t)W * H; ++pix)
        if (pix < (size_t)y0 * W || pix >= (size_t)y1 * W)
            n->paths[pix].active = false;
    uint64_t rays = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays)
    for (int64_t y = y0; y < (int64_t)y1; ++y) {
        PathTraceCounters counters;
        for (uint32_t x = 0; x < W; ++x) {
            nrcRayGenBump(f, n, p, camera, x, (uint32_t)y, &counters);
            const NrcPathState &st = n->paths[(size_t)y * W + x];
            if (st.isTrainingPath)
                tileToPixel[st.linearTileIndex] = (uint32_t)(y * W + x);
        }
        rays += counters.closestRays + counters.visibilityRays;
    }
    nrcCommitStagedVertices(f, n, p, tileToPixel);

    for (uint32_t round = 0; round < kMaxNrcRounds; ++round) {
        uint64_t numActive = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays, numActive)
        for (int64_t y = y0; y < (int64_t)y1; ++y) {
            PathTraceCounters counters;
            for (uint32_t x = 0; x < W; ++x) {
                const size_t pix = (size_t)y * W + x;
                if (!n->paths[pix].active)
                    continue;
                nrcExtendBump(f, n, p, pix, &counters);
                numActive += n->paths[pix].active ? 1 : 0;
            }
            rays += counters.closestRays + counters.visibilityRays;
        }
        if (!nrcCommitStagedVertices(f, n, p, tileToPixel, numActive != 0))
            break;
    }

    // ray-gen epilogue (:312-360)
    for (size_t pix = (size_t)y0 * W; pix < (size_t)y1 * W; ++pix) {
        const NrcPathState &st = n->paths[pix];
        if (f->gb0[bufIdx][pix].instSlot != 0xFFFFFFFFu) {
            f->rng[pix] = st.rng.state;
            if (st.isTrainingPath && !st.trainingSuffixEndsWithCache)
                n->suffixTerminal[st.linearTileIndex] = packSuffixTerminal(st.prevTrainDataIndex, false, st.pathLength);
        }
        if (!st.renderingPathEndsWithCache)
            writeTerminalInfo(n, pix, float3(0.0f), st.pathLength, false, st.isTrainingPath, st.isUnbiasedTrainingTile);
        n->frameContribution[3 * pix + 0] = st.contribution.x;
        n->frameContribution[3 * pix + 1] = st.contribution.y;
        n->frameContribution[3 * pix + 2] = st.contribution.z;
    }
    return rays;
}

extern "C" uint64_t orc_bump_pathtrace(orc_frame* f, const GfxFrameParams* p, int variant, int numThreads) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    if (variant == GFX_PT_NRC)
        return nrcPathTraceBump(f, p, numThreads);
    if (variant == GFX_PT_REGIR)
        return regirPathTraceBump(f, p, numThreads);
    const Camera camera = makeCamera(p->camera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    uint64_t rays = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays)
    for (int64_t yy = y0; yy < (int64_t)y1; ++yy) {
        PathTraceCounters counters;
        for (uint32_t x = 0; x < W; ++x)
            pathTracePixelBump(f, p, camera, x, (uint32_t)yy, &counters);
        rays += counters.closestRays + counters.visibilityRays;
    }
    return rays;
}

// visualizePrediction: the radiance query of every primary hit, built like nrcRayGen builds it, at row y * W + x (a miss
// leaves its row as it was); terminal info alpha 1, pathLength 1, hasQuery = hit; the host then infers W*H queries
// (neural_radiance_caching_main.cpp:2376-2384), pad128 like every inference launch here
extern "C" void orc_bump_nrc_visualize_prediction(orc_frame* f, const GfxFrameParams* p) {
    orc_nrc_frame* n = nrcFrame(f);
    const orc_scene* s = f->scene;
    const Camera camera = makeCamera(p->camera);
    const uint32_t bufIdx = p->bufferIndex & 1;
    for (size_t pix = 0; pix < (size_t)f->W * f->H; ++pix) {
        const GB0 gb0 = f->gb0[bufIdx][pix];
        const bool hit = gb0.instSlot != 0xFFFFFFFFu;
        if (hit) {
            const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
            const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
            const InstData &inst = s->instances[gb0.instSlot];
            const MeshData &mesh = s->meshes[gb0.geomInstSlot];
            SurfacePoint sp;
            computeSurfacePointFromGBuffer(s, inst, mesh, gb0.primIndex, bcB, bcC, &sp);
            float3 vOut = camera.position - sp.positionInWorld;
            const float primaryDist2 = sqLength(vOut);
            vOut /= std::sqrt(primaryDist2);
            const float primaryDotVN = dot(vOut, sp.geometricNormalInWorld);
            const float frontHit = primaryDotVN >= 0.0f ? 1.0f : -1.0f;
            const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
            const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh.materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
            const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);
            createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, &n->inferenceQuery[14 * pix]);
        }
        writeTerminalInfo(n, pix, float3(1.0f), 1, hit, false, false);
    }
    n->state[NRC_NUM_INFERENCE_QUERIES] = (f->W * f->H + 127) / 128 * 128;
}
