// gbuffer.cu — primary visibility + G-buffer as one fused kernel.
//
// Replaces gBuffer.optixPipeline.launch(W, H, 1) (restir_di/restir_di_main.cpp:2366) and its three
// OptiX programs RG/CH/MS setupGBuffers (restir_di/gpu_kernels/optix_gbuffer_kernels.cu:5-110,
// 112-199, 201-243): pinhole ray generation, closest hit through the software BVH, attribute
// interpolation, object->world, motion vector, DH-reflectance albedo, polar/UNORM16 encoding,
// running-mean albedo/normal accumulation.
//
// Thread mapping: 8x4-pixel tiles per warp (block 8x8 like the reference's PURE_CUDA kernels) so a
// warp's primary rays stay coherent in the BVH while every G-buffer plane is still written in
// 128-byte row segments.
#include "traverse.cuh"
#include "shading.cuh"
#include "lighting.cuh"
#include "context.h"

namespace gfx {

GFX_D f2 calcScreenPosition(const DevCamera &cam, const f3 &posInWorld) { // restir_di_shared.h:51-59
    const f3 posInView = mul3x3(cam.invOrientation, posInWorld - cam.position);
    const f2 posAtZ1(posInView.x / posInView.z, posInView.y / posInView.z);
    const float h = cam.vh;
    const float w = cam.aspect * h;
    return f2(1 - (posAtZ1.x + 0.5f * w) / w, 1 - (posAtZ1.y + 0.5f * h) / h);
}

GFX_D void countRays(const DevFrame &frame, uint32_t n) {
    // one atomic per warp; every lane of the warp reaches this point (no early kernel exits)
    const uint32_t total = __reduce_add_sync(0xFFFFFFFFu, n);
    if ((threadIdx.x + threadIdx.y * blockDim.x) % 32 == 0 && total)
        atomicAdd(frame.stats, (unsigned long long)total);
}

// JITTER: GFX_SVGF_SUBPIXEL_JITTER, the primary ray through (x, y) + sample (svgfSubPixelSample) and no random number drawn.
// BUMP: GfxFrameParams::enableBumpMapping, a kernel of its own so that the frames without it run the code they ran before it existed
template <bool JITTER, bool BUMP>
GFX_D uint32_t gbufferPixel(const DevScene &scene, const DevFrame &frame, const DevFrameParams &p, float2 sample) {
    const uint32_t x = blockIdx.x * 8 + threadIdx.x;
    const uint32_t y = p.y0 + blockIdx.y * 8 + threadIdx.y;
    if (x >= frame.W || y >= p.y1)
        return 0;
    const size_t pix = (size_t)y * frame.W + x;
    const uint32_t bufIdx = p.bufferIndex;

    float jx = 0.5f, jy = 0.5f;
    if (JITTER) {
        jx = sample.x;
        jy = sample.y;
    }
    else if (p.enableJittering) {
        PCG32RNG rng{ frame.rng[pix] };
        jx = rng.getFloat0cTo1o();
        jy = rng.getFloat0cTo1o();
        frame.rng[pix] = rng.state;
    }
    // ray generation (:21-27)
    const float fx = (x + jx) / frame.W;
    const float fy = (y + jy) / frame.H;
    const f3 origin = p.camera.position;
    const f3 direction = normalize(mul3x3(p.camera.orientation, f3(p.camera.vw * (0.5f - fx), p.camera.vh * (0.5f - fy), 1)));

    f3 albedo(0.0f);
    f3 positionInWorld(NAN), prevPositionInWorld(NAN), shadingNormalInWorld(NAN);
    uint32_t qGeometricNormalInWorld = 0, qTexCoord0DirInWorld = 0, qTexCoord = 0;
    uint32_t matSlot = 0xFFFFFFFFu, instSlot = 0xFFFFFFFFu, geomInstSlot = 0xFFFFFFFFu, primIndex = 0xFFFFFFFFu;
    uint32_t qbcB = 0, qbcC = 0;

    // (a shared-memory stack as in the wavefront kernels gains nothing here: primary rays are coherent)
    const Hit hit = traverseBvh<false>(scene.bvh, origin, direction, 0.0f, 3.402823466e+38f);
    if (hit.storageIndex != 0xFFFFFFFFu) {
        // closest-hit program (:112-199)
        const uint2 im = __ldg(scene.geomToInstMesh + hit.geomIndex);
        instSlot = im.x;
        geomInstSlot = im.y;
        primIndex = hit.primIndex;
        const DevInstance* inst = scene.instances + instSlot;
        const DevMesh mesh = scene.meshes[geomInstSlot];
        matSlot = mesh.materialSlot;

        const uint4 tri = __ldg(scene.triangles + mesh.triBase + primIndex);
        const float4* vA = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.x);
        const float4* vB = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.y);
        const float4* vC = scene.vertices + 3 * (size_t)(mesh.vertexBase + tri.z);
        const float4 a0 = __ldg(vA), a1 = __ldg(vA + 1), a2 = __ldg(vA + 2);
        const float4 b0 = __ldg(vB), b1 = __ldg(vB + 1), b2 = __ldg(vB + 2);
        const float4 c0 = __ldg(vC), c1 = __ldg(vC + 1), c2 = __ldg(vC + 2);

        const float bcB = hit.bcB;
        const float bcC = hit.bcC;
        const float bcA = 1 - (bcB + bcC);
        qbcB = encodeBarycentric(bcB);
        qbcC = encodeBarycentric(bcC);
        const f3 pA(a0.x, a0.y, a0.z), pB(b0.x, b0.y, b0.z), pC(c0.x, c0.y, c0.z);
        const f3 positionInObj = bcA * pA + bcB * pB + bcC * pC;
        const f3 shadingNormalInObj = bcA * f3(a1.x, a1.y, a1.z) + bcB * f3(b1.x, b1.y, b1.z) + bcC * f3(c1.x, c1.y, c1.z);
        const f3 texCoord0DirInObj = bcA * f3(a2.x, a2.y, a2.z) + bcB * f3(b2.x, b2.y, b2.z) + bcC * f3(c2.x, c2.y, c2.z);
        const f2 texCoord = bcA * f2(a0.w, a1.w) + bcB * f2(b0.w, b1.w) + bcC * f2(c0.w, c1.w);
        const f3 geometricNormalInObj = cross(pB - pA, pC - pA);

        positionInWorld = xfmPoint(inst->transform, positionInObj);
        prevPositionInWorld = xfmPoint(inst->curToPrevTransform, positionInWorld);
        f3 geometricNormalInWorld = normalize(mul3x3(inst->normalMatrix, geometricNormalInObj));
        shadingNormalInWorld = normalize(mul3x3(inst->normalMatrix, shadingNormalInObj));
        f3 texCoord0DirInWorld = xfmVector(inst->transform, texCoord0DirInObj);
        texCoord0DirInWorld = normalize(
            texCoord0DirInWorld - dot(shadingNormalInWorld, texCoord0DirInWorld) * shadingNormalInWorld);
        if (!allFinite(shadingNormalInWorld)) {
            geometricNormalInWorld = f3(0, 0, 1);
            shadingNormalInWorld = f3(0, 0, 1);
            texCoord0DirInWorld = f3(1, 0, 0);
        }
        qGeometricNormalInWorld = encodeVector(geometricNormalInWorld);
        qTexCoord = encodeTexCoords(texCoord);

        const BSDF bsdf = setupBsdf(scene, matSlot, texCoord);
        ReferenceFrame shadingFrame(shadingNormalInWorld, texCoord0DirInWorld);
        if (BUMP) // optix_gbuffer_kernels.cu:175-178 (restir_di, regir), :151-154 (path_tracing, NRC)
            shadingFrame = bumpShadingFrame(scene, matSlot, texCoord, shadingFrame);
        const f3 vOut = -direction;
        const f3 vOutLocal = shadingFrame.toLocal(normalize(vOut));
        shadingNormalInWorld = shadingFrame.normal;
        qTexCoord0DirInWorld = encodeVector(shadingFrame.tangent);
        albedo = bsdf.evaluateDHReflectanceEstimate(vOutLocal);
    }
    else {
        // miss program (:201-243); the synthetic configs carry no environment texture
        const f3 vOut = -direction;
        const f3 pp = -vOut;
        float posPhi, posTheta;
        toPolarYUp(pp, &posPhi, &posTheta);
        const float phi = posPhi + p.envLightRotation;
        float u = phi / (2 * kPi);
        u -= floorf(u);
        const float v = posTheta / kPi;
        positionInWorld = pp;
        prevPositionInWorld = pp;
        qGeometricNormalInWorld = encodeVector(vOut);
        shadingNormalInWorld = vOut;
        float sp, cp;
        dm_sincos(posPhi, &sp, &cp);
        qTexCoord0DirInWorld = encodeVector(f3(-cp, 0, -sp));
        qTexCoord = encodeTexCoords(f2(u, v));
        qbcB = encodeBarycentric(u);
        qbcC = encodeBarycentric(v);
    }

    // ray-gen epilogue (:56-109).  With the jitter the current raster position is the sample's: it is where the point
    // projects without the offset, and GL's prevScreenPos = pixel centre - (that - previous projection) is what
    // k_svgfTemporal computes from this motion vector.
    const f2 curRasterPos = JITTER ? f2(x + jx, y + jy) : f2(x + 0.5f, y + 0.5f);
    const f2 prevRasterPos = calcScreenPosition(p.prevCamera, prevPositionInWorld) * f2((float)frame.W, (float)frame.H);
    f2 motionVector = curRasterPos - prevRasterPos;
    if (p.resetFlowBuffer || isnan(prevPositionInWorld.x))
        motionVector = f2(0.0f, 0.0f);

    frame.gb0[bufIdx][pix] = make_uint4(instSlot, geomInstSlot, primIndex, qbcB | (qbcC << 16));
    frame.gb1[bufIdx][pix] = make_float2(motionVector.x, motionVector.y);
    frame.gb2[bufIdx][pix] = make_float4(positionInWorld.x, positionInWorld.y, positionInWorld.z, __uint_as_float(qGeometricNormalInWorld));
    frame.gb3[bufIdx][pix] = make_uint4(encodeVector(shadingNormalInWorld), qTexCoord0DirInWorld, qTexCoord, matSlot);

    f3 prevAlbedoResult(0.0f), prevNormalResult(0.0f);
    if (p.numAccumFrames > 0) {
        const float4 pa = frame.albedo[pix], pn = frame.normal[pix];
        prevAlbedoResult = f3(pa.x, pa.y, pa.z);
        prevNormalResult = f3(pn.x, pn.y, pn.z);
    }
    const float curWeight = 1.0f / (1 + p.numAccumFrames);
    const f3 albedoResult = (1 - curWeight) * prevAlbedoResult + curWeight * albedo;
    const f3 normalResult = (1 - curWeight) * prevNormalResult + curWeight * shadingNormalInWorld;
    frame.albedo[pix] = make_float4(albedoResult.x, albedoResult.y, albedoResult.z, 1.0f);
    frame.normal[pix] = make_float4(normalResult.x, normalResult.y, normalResult.z, 1.0f);
    return 1;
}

template <bool BUMP>
__global__ void __launch_bounds__(64) k_gbuffer(DevScene scene, DevFrame frame, DevFrameParams p) {
    countRays(frame, gbufferPixel<false, BUMP>(scene, frame, p, make_float2(0.5f, 0.5f)));
}

template <bool BUMP>
__global__ void __launch_bounds__(64) k_gbufferSubPixelJitter(DevScene scene, DevFrame frame, DevFrameParams p, float2 sample) {
    countRays(frame, gbufferPixel<true, BUMP>(scene, frame, p, sample));
}

int launchGBuffer(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params) {
    bool jitter;
    float2 sample;
    int rc = svgfSubPixelSample(ctx, params, &jitter, &sample);
    if (rc == GFX_OK && params->enableBumpMapping)
        rc = ensureBumpTable(ctx);
    if (rc != GFX_OK)
        return rc;
    const DevFrameParams p = makeDevParams(ctx, params);
    if (p.y1 <= p.y0)
        return GFX_OK;
    const dim3 block(8, 8);
    const dim3 grid((ctx->frame.W + 7) / 8, (p.y1 - p.y0 + 7) / 8);
    GFX_TIMED(ctx, stream, "gbuffer");
    const bool bump = params->enableBumpMapping != 0;
    if (jitter && bump)
        k_gbufferSubPixelJitter<true><<<grid, block, 0, stream>>>(ctx->devScene(), ctx->devFrame(), p, sample);
    else if (jitter)
        k_gbufferSubPixelJitter<false><<<grid, block, 0, stream>>>(ctx->devScene(), ctx->devFrame(), p, sample);
    else if (bump)
        k_gbuffer<true><<<grid, block, 0, stream>>>(ctx->devScene(), ctx->devFrame(), p);
    else
        k_gbuffer<false><<<grid, block, 0, stream>>>(ctx->devScene(), ctx->devFrame(), p);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

} // namespace gfx
