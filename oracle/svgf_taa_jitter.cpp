// oracle/svgf_taa_jitter.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of the SVGF app's TAA sub-pixel jitter,
// GFX_SVGF_SUBPIXEL_JITTER:
//   subPixelOffsets          svgf/svgf_main.cpp:1410-1424 (halton(2, i), halton(3, i)), chosen at :2005-2008 as
//                            subPixelOffsets[frameIndex % taaHistoryLength] when enableTemporalAA is on
//   the jittered G-buffer    :2015-2028 addOffset(matV2C, ox, oy) + shaders/draw_g_buffers.{vert,frag}
//   fillBackground           svgf/gpu_kernels/svgf.cu:404-441, computeEnvDirection(..., true)
// The app rasterises with the offset added to the projection: after the perspective divide the fragment at GL pixel centre
// (X + 0.5, Y + 0.5) shows the point whose unjittered projection is (X + ox, Y + oy).  qRotateY(pi) in matW2V makes GL's x run
// as this renderer's does, and GL counts rows from the bottom, so in top-down pixel coordinates the sample lies at
// (x + ox, y + 1 - oy), the position fillBackground writes directly (svgf.cu:406-408).
//
// This file compiles the SVGF app's oracle (svgf_app.cpp, which compiles render.cpp) into its own library,
// liborc_svgf_taa_jitter.so (Makefile.svgf_taa_jitter, bound by tests/oracle_svgf_taa_jitter.py), and links denoise.o.  Frames
// the jitter does not apply to go through the existing orc_gbuffer / orc_svgf_pass unchanged.
#include "svgf_app.cpp"

extern "C" {
int orc_svgf_pass(orc_svgf* s, const GfxFrameParams* p, int pass, uint32_t stage, int numThreads); // denoise.cpp
}

extern "C" void orc_svgf_subpixel_offset(uint32_t i, float* offset) {
    offset[0] = dm_halton(2, i);
    offset[1] = dm_halton(3, i);
}

// whether the jitter applies to the frame (the flag together with GFX_SVGF_ENABLE_TEMPORAL_AA); sample = (ox, 1 - oy), the
// sample's offset from the pixel's top-left corner, top-down
extern "C" int orc_svgf_subpixel_sample(const GfxFrameParams* p, float* sample) {
    sample[0] = sample[1] = 0.5f;
    if (!(p->svgfFlags & GFX_SVGF_SUBPIXEL_JITTER) || !(p->svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_AA))
        return 0;
    const uint32_t taaHistoryLength = p->taaHistoryLength ? p->taaHistoryLength : 16;
    float offset[2];
    orc_svgf_subpixel_offset(p->frameIndex % taaHistoryLength, offset);
    sample[0] = offset[0];
    sample[1] = 1.0f - offset[1];
    return 1;
}

namespace {

// orc_gbuffer (render.cpp) with the primary ray through (x, y) + sample and the motion vector measured from the sample
void gbufferSubPixelJitter(orc_frame* f, const GfxFrameParams* p, const float sample[2], int numThreads) {
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
            const float jx = sample[0], jy = sample[1]; // no random number drawn
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

            // ray-gen epilogue (:56-109): the current raster position is the sample, the point's unjittered projection, from
            // which GL's motion vector is taken (draw_g_buffers.vert/.frag)
            const float2 curRasterPos(x + jx, y + jy);
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

} // namespace

// gfx_gbuffer_launch: -1 for a frame that sets both GFX_SVGF_SUBPIXEL_JITTER and enableJittering, as the library refuses it
extern "C" int orc_gbuffer_taa_jitter(orc_frame* f, const GfxFrameParams* p, int numThreads) {
    if ((p->svgfFlags & GFX_SVGF_SUBPIXEL_JITTER) && p->enableJittering)
        return -1;
    float sample[2];
    if (!orc_svgf_subpixel_sample(p, sample)) {
        orc_gbuffer(f, p, numThreads);
        return 0;
    }
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    gbufferSubPixelJitter(f, p, sample, numThreads);
    return 0;
}

// gfx_svgf_launch(GFX_SVGF_FILL_BACKGROUND, numFilteringStages) on the oracle's SVGF state `s` of frame `f`: orc_svgf_pass, then
// with the jitter and the environment light the miss pixels' lighting again, looked up through the sample
// (svgf.cu:434-441); the albedo and prevScreenPos (from the pixel centre, :443-449) are the pass's own
extern "C" int orc_svgf_fill_background_taa_jitter(orc_svgf* s, orc_frame* f, const GfxFrameParams* p, uint32_t numFilteringStages,
                                                   int numThreads) {
    if ((p->svgfFlags & GFX_SVGF_SUBPIXEL_JITTER) && p->enableJittering)
        return -1;
    orc_svgf_pass(s, p, GFX_SVGF_FILL_BACKGROUND, numFilteringStages, numThreads);
    float sample[2];
    orc_scene* scene = f->scene;
    if (!orc_svgf_subpixel_sample(p, sample) || !orc_env_enabled(scene, p))
        return 0;
    const uint32_t W = f->W, H = f->H;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    F4* lighting = (F4*)orc_svgf_buffer_ptr(s, GFX_BUF_SVGF_LIGHTING_VARIANCE, numFilteringStages % 2, nullptr);
    const Camera camera = makeCamera(p->camera);
    for (uint32_t y = y0; y < y1; ++y) {
        for (uint32_t x = 0; x < W; ++x) {
            const size_t pix = (size_t)y * W + x;
            if (f->gb0[bufIdx][pix].instSlot != 0xFFFFFFFFu)
                continue;
            float3 origin, direction;
            primaryRay(camera, W, H, x, y, sample[0], sample[1], &origin, &direction);
            float posPhi, posTheta;
            toPolarYUp(direction, &posPhi, &posTheta);
            float phi = posPhi + p->envLightRotation;
            phi += p->envLightRotation; // as written in the reference (:418-420): added twice when the environment light is on
            float u = phi / (2 * kPi);
            u -= std::floor(u);
            const float uv[2] = { u, posTheta / kPi };
            float rgb[3];
            orc_env_query(scene, 2, uv, 1, rgb);
            const float3 finalLighting = p->envLightPowerCoeff * float3(rgb[0], rgb[1], rgb[2]);
            lighting[pix] = F4{ finalLighting.x, finalLighting.y, finalLighting.z, 0.0f };
        }
    }
    return 0;
}
