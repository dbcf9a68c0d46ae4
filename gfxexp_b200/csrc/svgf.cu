// svgf.cu — SVGF passes as sm_90a kernels.
//
// Replaces the PURE_CUDA kernels of svgf/gpu_kernels/svgf.cu (estimateVariance :30-134,
// applyATrousFilter_box3x3 :221-354, fillBackground :378-461,
// applyAlbedoModulationAndTemporalAntiAliasing :533-611, feedbackNoisyLighting :356-374; launch sites
// svgf/svgf_main.cpp:2127-2172)
// and the temporal-accumulation epilogue of the SVGF path tracer
// (svgf/gpu_kernels/optix_pathtracing_kernels.cu:12-128 reprojectPreviousAccumulation, :325-378
// demodulation + EMA + moments).  Config 4 runs them on restir_di's output: the inputs are this
// library's G-buffers, the beauty buffer and the DH-reflectance albedo buffer.
//
// The reference reads everything through 2-D surfaces with no on-chip reuse; here every plane is a
// linear float4/float array, a block is a 32x8 pixel tile (one warp = one 512-byte row segment per
// plane) and the dilated taps of the à-trous stages come through the read-only path (L1/L2): the
// footprint of one stage is ~68 B/px compulsory (SURVEY.md §8d) against 126 MB of L2.
// exp() is detmath's and pow(x,128) is seven squarings, exactly as in the oracle; compiled with
// -fmad=false, so outputs are bit-identical to oracle/denoise.cpp.
#include "shading.cuh"
#include "lighting.cuh"
#include "context.h"

namespace gfx {

struct DevSvgf {
    uint32_t W, H;
    const uint4* gb0[2];
    const float2* gb1[2];
    const float4* gb2[2];
    const uint4* gb3[2];
    const float4* beauty;
    const float4* albedoAccum;
    float4* lighting[2];
    float4* moments[2];
    float4* prevLighting;
    float4* albedo;
    float* depth[2];
    float4* normal;           // decoded shading normal of the current frame (written by the temporal pass): the filters
                              // read it instead of running decodeVector (two sincos) per tap and stage
    float4* finalLighting[2];
    float2* prevScreenPos;
    float m22, m23;
    uint32_t svgfFlags, taaHistoryLength;
};

GFX_D float pow128(float x) {
    x = x * x; x = x * x; x = x * x; x = x * x; x = x * x; x = x * x; x = x * x;
    return x;
}
GFX_D float calcDepthWeight(float nbDepth, float depth, float dzdx, float dzdy, int32_t dx, int32_t dy) { // svgf.cu:6-12
    const float sigma_z = 1.0f;
    const float eps = 1e-6f;
    return dm_exp(-fabsf(nbDepth - depth) / (sigma_z * fabsf(dzdx * dx + dzdy * dy) + eps));
}
GFX_D float calcNormalWeight(const f3 &nbNormal, const f3 &normal) { // svgf.cu:14-18
    return pow128(fmaxf(0.0f, dot(nbNormal, normal)));
}
GFX_D float calcLuminanceWeight(float nbLuminance, float luminance, float localMeanStdDev) { // svgf.cu:20-26
    const float sigma_l = 4.0f;
    const float eps = 1e-6f;
    return dm_exp(-fabsf(nbLuminance - luminance) / (sigma_l * localMeanStdDev + eps));
}
GFX_D int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
GFX_D f3 xyz(const float4 &v) { return f3(v.x, v.y, v.z); }
GFX_D f3 rgbSafeDivide(const f3 &a, const f3 &b) {
    return f3(b.x != 0 ? a.x / b.x : 0.0f, b.y != 0 ? a.y / b.y : 0.0f, b.z != 0 ? a.z / b.z : 0.0f);
}

#define SVGF_PIXEL() \
    const int x = blockIdx.x * 32 + threadIdx.x; \
    const int y = (int)p.y0 + blockIdx.y * 8 + threadIdx.y; \
    const int W = (int)s.W, H = (int)s.H; \
    if (x >= W || y >= (int)p.y1) \
        return; \
    const size_t pix = (size_t)y * W + x;

// ---- temporal accumulation ---------------------------------------------------------------
__global__ void __launch_bounds__(256) k_svgfTemporal(DevSvgf s, DevFrameParams p) {
    SVGF_PIXEL();
    const uint32_t curBufIdx = p.bufferIndex;
    const uint32_t prevBufIdx = (curBufIdx + 1) % 2;
    const uint4 gb0 = s.gb0[curBufIdx][pix];
    const uint4 gb3 = s.gb3[curBufIdx][pix];
    const uint32_t instSlot = gb0.x;
    const uint32_t materialSlot = gb3.w;
    if (instSlot == 0xFFFFFFFFu) {
        s.depth[curBufIdx][pix] = 1.0f;
        s.normal[pix] = make_float4(0, 0, 0, 0);
        s.lighting[0][pix] = make_float4(0, 0, 0, 0);
        s.moments[curBufIdx][pix] = make_float4(0, 0, 0, 0);
        return;
    }
    const float4 gb2 = s.gb2[curBufIdx][pix];
    const f3 positionInWorld(gb2.x, gb2.y, gb2.z);
    const f3 shadingNormalInWorld = decodeVector(gb3.x);
    s.normal[pix] = make_float4(shadingNormalInWorld.x, shadingNormalInWorld.y, shadingNormalInWorld.z, 0.0f);

    const f3 posInView = mul3x3(p.camera.invOrientation, positionInWorld - p.camera.position);
    const float zv = -posInView.z;
    const float ndcZ = (s.m22 * zv + s.m23) / (-zv);
    s.depth[curBufIdx][pix] = 0.5f * ndcZ + 0.5f;

    const f3 contribution = xyz(s.beauty[pix]);
    f3 dhReflectance = xyz(s.albedoAccum[pix]);
    dhReflectance.x = dhReflectance.x < 0.001f ? 0.0f : dhReflectance.x;
    dhReflectance.y = dhReflectance.y < 0.001f ? 0.0f : dhReflectance.y;
    dhReflectance.z = dhReflectance.z < 0.001f ? 0.0f : dhReflectance.z;
    s.albedo[pix] = make_float4(dhReflectance.x, dhReflectance.y, dhReflectance.z, 0.0f);

    const float2 mv = s.gb1[curBufIdx][pix];
    const f2 prevScreenPos((x + 0.5f - mv.x) / W, (y + 0.5f - mv.y) / H);
    s.prevScreenPos[pix] = make_float2(prevScreenPos.x, prevScreenPos.y);

    f3 prevNoisyLighting(0.0f);
    float prevFirstMoment = 0.0f, prevSecondMoment = 0.0f;
    uint32_t prevCount = 0, prevAcceptFlags = 0;
    const bool enableTemporalAccumulation = (s.svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_ACCUMULATION) != 0;
    const bool outOfScreen = (prevScreenPos.x < 0.0f || prevScreenPos.y < 0.0f || prevScreenPos.x >= 1.0f || prevScreenPos.y >= 1.0f);
    if (enableTemporalAccumulation && !outOfScreen) {
        const f2 prevViewportPos(W * prevScreenPos.x, H * prevScreenPos.y);
        const int ppx = dm_f2int(prevViewportPos.x), ppy = dm_f2int(prevViewportPos.y);
        const f2 fDelta = prevViewportPos - (f2((float)ppx, (float)ppy) + f2(0.5f, 0.5f));
        const int dlx = fDelta.x < 0 ? -1 : 1, dly = fDelta.y < 0 ? -1 : 1;
        const int nbx[4] = { ppx, clampi(ppx + dlx, 0, W - 1), ppx, clampi(ppx + dlx, 0, W - 1) };
        const int nby[4] = { ppy, ppy, clampi(ppy + dly, 0, H - 1), clampi(ppy + dly, 0, H - 1) };
        float sumWeights = 0.0f;
        float prevFloatSampleCount = 0;
        uint32_t acceptableFlags = 0;
        const float sx = fabsf(fDelta.x);
        const float t = fabsf(fDelta.y);
        const float weights[4] = { (1 - sx) * (1 - t), sx * (1 - t), (1 - sx) * t, sx * t };
#pragma unroll
        for (uint32_t i = 0; i < 4; ++i) {
            const size_t nb = (size_t)nby[i] * W + nbx[i];
            const uint32_t nbInst = s.gb0[prevBufIdx][nb].x;
            const uint4 nbGb3 = s.gb3[prevBufIdx][nb];
            if (nbInst != instSlot || nbGb3.w != materialSlot)
                continue;
            if (dot(decodeVector(nbGb3.x), shadingNormalInWorld) <= 0.85f)
                continue;
            const float4 nbGb2 = s.gb2[prevBufIdx][nb];
            if (sqLength(f3(nbGb2.x, nbGb2.y, nbGb2.z) - positionInWorld) > 0.1f)
                continue;
            const float weight = weights[i];
            const float4 nbLighting = s.prevLighting[nb];
            const float4 nbMoments = s.moments[prevBufIdx][nb];
            prevNoisyLighting += weight * xyz(nbLighting);
            prevFirstMoment += weight * nbMoments.x;
            prevSecondMoment += weight * nbMoments.y;
            prevFloatSampleCount += weight * (__float_as_uint(nbMoments.z) & 0xFFFFFFu);
            sumWeights += weight;
            acceptableFlags |= (1u << i);
        }
        if (sumWeights > 0) {
            prevNoisyLighting /= sumWeights;
            prevFirstMoment /= sumWeights;
            prevSecondMoment /= sumWeights;
            prevCount = dm_f2uint(floorf(prevFloatSampleCount / sumWeights + 0.5f));
            prevAcceptFlags = acceptableFlags;
        }
    }

    f3 demCont = rgbSafeDivide(contribution, dhReflectance);
    float luminance = sRGB_calcLuminance(demCont);
    float sqLuminance = pow2f(luminance);

    if ((s.svgfFlags & GFX_SVGF_IS_FIRST_FRAME) || !enableTemporalAccumulation) {
        prevCount = 0;
        prevAcceptFlags = 0;
    }
    const uint32_t sampleCount = min(prevCount + 1, 65535u);
    if (enableTemporalAccumulation) {
        if (sampleCount > 1) {
            float curWeight = 1.0f / 5;
            if (sampleCount < 5)
                curWeight = 1.0f / sampleCount;
            const float prevWeight = 1.0f - curWeight;
            demCont = prevWeight * prevNoisyLighting + curWeight * demCont;
            luminance = prevWeight * prevFirstMoment + curWeight * luminance;
            sqLuminance = prevWeight * prevSecondMoment + curWeight * sqLuminance;
        }
    }
    s.lighting[0][pix] = make_float4(demCont.x, demCont.y, demCont.z, 0.0f);
    s.moments[curBufIdx][pix] = make_float4(luminance, sqLuminance,
                                            __uint_as_float((sampleCount & 0xFFFFFFu) | (prevAcceptFlags << 24)), 0.0f);
}

// ---- estimateVariance (svgf.cu:30-134) ---------------------------------------------------
__global__ void __launch_bounds__(256) k_svgfVariance(DevSvgf s, DevFrameParams p) {
    SVGF_PIXEL();
    const uint32_t curBufIdx = p.bufferIndex;
    if (s.gb0[curBufIdx][pix].x == 0xFFFFFFFFu)
        return;
    const float4 m = s.moments[curBufIdx][pix];
    float firstMoment = m.x;
    float secondMoment = m.y;
    const uint32_t count = __float_as_uint(m.z) & 0xFFFFFFu;
    if (count < 4) {
        const float filterKernel[] = { 0.00598f, 0.060626f, 0.241843f, 0.383103f, 0.241843f, 0.060626f, 0.00598f };
        const float centerWeight = pow2f(filterKernel[3]);
        float sumFirstMoments = centerWeight * firstMoment;
        float sumSecondMoments = centerWeight * secondMoment;
        const float* depthBuf = s.depth[curBufIdx];
        const float depth = depthBuf[pix];
        const int32_t dx = x < W / 2 ? 1 : -1;
        const int32_t dy = y < H / 2 ? 1 : -1;
        const float hnbDepth = depthBuf[(size_t)y * W + (x + dx)];
        const float vnbDepth = depthBuf[(size_t)(y + dy) * W + x];
        const float dzdx = (hnbDepth - depth) * dx;
        const float dzdy = (vnbDepth - depth) * dy;
        const f3 normal = xyz(s.normal[pix]);
        float sumWeights = centerWeight;
        for (int i = -3; i <= 3; ++i) {
            const int nbPixY = y + i;
            if (nbPixY < 0 || nbPixY >= H)
                continue;
            const float hy = filterKernel[i + 3];
            for (int j = -3; j <= 3; ++j) {
                const int nbPixX = x + j;
                if (nbPixX < 0 || nbPixX >= W)
                    continue;
                if (i == 0 && j == 0)
                    continue;
                const float hx = filterKernel[j + 3];
                const size_t nb = (size_t)nbPixY * W + nbPixX;
                const float nbDepth = depthBuf[nb];
                if (nbDepth == 1.0f)
                    continue;
                const f3 nbNormal = xyz(s.normal[nb]);
                const float wz = calcDepthWeight(nbDepth, depth, dzdx, dzdy, j, i);
                const float wn = calcNormalWeight(nbNormal, normal);
                const float weight = hx * hy * wz * wn;
                const float4 nbm = s.moments[curBufIdx][nb];
                sumFirstMoments += weight * nbm.x;
                sumSecondMoments += weight * nbm.y;
                sumWeights += weight;
            }
        }
        firstMoment = sumFirstMoments / sumWeights;
        secondMoment = sumSecondMoments / sumWeights;
    }
    const float variance = fmaxf(secondMoment - pow2f(firstMoment), 0.0f);
    s.lighting[0][pix].w = variance;
}

// ---- à-trous box 3x3 (svgf.cu:221-354) ---------------------------------------------------
__global__ void __launch_bounds__(256) k_svgfATrous(DevSvgf s, DevFrameParams p, uint32_t filterStageIndex) {
    SVGF_PIXEL();
    const int32_t stepWidth = 1 << filterStageIndex; // 1, 2, 4, 8, 16
    const uint32_t curBufIdx = p.bufferIndex;
    const float4* __restrict__ src = s.lighting[filterStageIndex % 2];
    float4* __restrict__ dst = s.lighting[(filterStageIndex + 1) % 2];
    if (s.gb0[curBufIdx][pix].x == 0xFFFFFFFFu)
        return;
    const bool feedback = (s.svgfFlags & GFX_SVGF_FEEDBACK_1ST_FILTERED_RESULT) != 0;

    const float4 srcLv = __ldg(src + pix);
    if (filterStageIndex == 0 && !feedback)
        s.prevLighting[pix] = srcLv;
    const float luminance = sRGB_calcLuminance(xyz(srcLv));

    const float* __restrict__ depthBuf = s.depth[curBufIdx];
    const float4* __restrict__ normals = s.normal;
    const float depth = __ldg(depthBuf + pix);
    const int32_t dx = x < W / 2 ? 1 : -1;
    const int32_t dy = y < H / 2 ? 1 : -1;
    const float hnbDepth = __ldg(depthBuf + (size_t)y * W + (x + dx));
    const float vnbDepth = __ldg(depthBuf + (size_t)(y + dy) * W + x);
    const float dzdx = (hnbDepth - depth) * dx;
    const float dzdy = (vnbDepth - depth) * dy;
    const f3 normal = xyz(__ldg(normals + pix));

    const float gaussKernel[] = { 1 / 4.0f, 1 / 2.0f, 1 / 4.0f };
    float sumLocalVars = 0.0f;
    float sumVarWeights = 0.0f;
#pragma unroll
    for (int i = -1; i <= 1; ++i) {
        const int nbPixY = clampi(y + i, 0, H - 1);
        const float hy = gaussKernel[i + 1];
#pragma unroll
        for (int j = -1; j <= 1; ++j) {
            const int nbPixX = clampi(x + j, 0, W - 1);
            const float hx = gaussKernel[j + 1];
            const float weight = hx * hy;
            sumLocalVars += weight * __ldg(&src[(size_t)nbPixY * W + nbPixX].w);
            sumVarWeights += weight;
        }
    }
    const float localMeanStdDev = sqrtf(sumLocalVars / sumVarWeights);

    const float centerWeight = 1.0f;
    float sumWeights = centerWeight;
    f3 dstLighting = centerWeight * xyz(srcLv);
    float dstVariance = pow2f(centerWeight) * srcLv.w;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        if (k == 4)
            continue;
        const int ox = (k % 3 - 1) * stepWidth, oy = (k / 3 - 1) * stepWidth;
        const int nbx = x + ox, nby = y + oy;
        if (nbx < 0 || nbx >= W || nby < 0 || nby >= H)
            continue;
        const float h = 1.0f;
        const size_t nb = (size_t)nby * W + nbx;
        const float nbDepth = __ldg(depthBuf + nb);
        if (nbDepth == 1.0f)
            continue;
        const f3 nbNormal = xyz(__ldg(normals + nb));
        const float wz = calcDepthWeight(nbDepth, depth, dzdx, dzdy, ox, oy);
        const float wn = calcNormalWeight(nbNormal, normal);
        const float4 nbLv = __ldg(src + nb);
        const float nbLuminance = sRGB_calcLuminance(xyz(nbLv));
        const float wl = calcLuminanceWeight(nbLuminance, luminance, localMeanStdDev);
        const float weight = h * wz * wn * wl;
        dstLighting += weight * xyz(nbLv);
        dstVariance += pow2f(weight) * nbLv.w;
        sumWeights += weight;
    }
    dstLighting /= sumWeights;
    dstVariance /= pow2f(sumWeights);
    const float4 out = make_float4(dstLighting.x, dstLighting.y, dstLighting.z, dstVariance);
    dst[pix] = out;
    if (filterStageIndex == 0 && feedback)
        s.prevLighting[pix] = out;
}

// ---- fillBackground (svgf.cu:378-461) -----------------------------------------------------
// JITTER: GFX_SVGF_SUBPIXEL_JITTER, the environment seen through (x, y) + sample (computeEnvDirection(..., true), :404-408,
// :436); prevScreenPos stays the pixel centre's (:443)
template <bool JITTER>
GFX_D void svgfBackgroundPixel(const DevSvgf &s, const DevFrameParams &p, uint32_t numFilteringStages, const DevEnvLight &env,
                               float2 sample) {
    SVGF_PIXEL();
    const uint32_t curBufIdx = p.bufferIndex;
    if (s.gb0[curBufIdx][pix].x != 0xFFFFFFFFu)
        return;
    f3 finalLighting(0.001f, 0.001f, 0.001f);
    const float fx = (x + 0.5f) / W;
    const float fy = (y + 0.5f) / H;
    f3 direction = normalize(mul3x3(p.camera.orientation, f3(p.camera.vw * (0.5f - fx), p.camera.vh * (0.5f - fy), 1)));
    if (env.enabled) { // :431-437; without the jitter the camera's sub-pixel offset is the pixel centre
        f3 envDirection = direction;
        if (JITTER) {
            const float jfx = (x + sample.x) / W;
            const float jfy = (y + sample.y) / H;
            envDirection = normalize(mul3x3(p.camera.orientation, f3(p.camera.vw * (0.5f - jfx), p.camera.vh * (0.5f - jfy), 1)));
        }
        float posPhi, posTheta;
        toPolarYUp(envDirection, &posPhi, &posTheta);
        float phi = posPhi + env.rotation;
        phi += env.rotation; // as written in the reference (:418-420): the rotation is added twice when the environment light is on
        float u = phi / (2 * kPi);
        u -= floorf(u);
        const float v = posTheta / kPi;
        finalLighting = env.powerCoeff * envFetch(env, u, v);
    }
    const float* o = p.prevCamera.orientation;
    direction = f3(o[0] * direction.x + o[3] * direction.y + o[6] * direction.z,
                   o[1] * direction.x + o[4] * direction.y + o[7] * direction.z,
                   o[2] * direction.x + o[5] * direction.y + o[8] * direction.z);
    direction /= direction.z;
    const f2 prevScreenPos(0.5f - direction.x / p.prevCamera.vw, 0.5f - direction.y / p.prevCamera.vh);
    s.lighting[numFilteringStages % 2][pix] = make_float4(finalLighting.x, finalLighting.y, finalLighting.z, 0.0f);
    s.albedo[pix] = make_float4(1.0f, 1.0f, 1.0f, 0.0f);
    s.prevScreenPos[pix] = make_float2(prevScreenPos.x, prevScreenPos.y);
}

__global__ void __launch_bounds__(256) k_svgfBackground(DevSvgf s, DevFrameParams p, uint32_t numFilteringStages, DevEnvLight env) {
    svgfBackgroundPixel<false>(s, p, numFilteringStages, env, make_float2(0.5f, 0.5f));
}

__global__ void __launch_bounds__(256) k_svgfBackgroundSubPixelJitter(DevSvgf s, DevFrameParams p, uint32_t numFilteringStages,
                                                                      DevEnvLight env, float2 sample) {
    svgfBackgroundPixel<true>(s, p, numFilteringStages, env, sample);
}

// ---- albedo modulation + TAA (svgf.cu:465-611) -------------------------------------------
__global__ void __launch_bounds__(256) k_svgfModulateTAA(DevSvgf s, DevFrameParams p, uint32_t numFilteringStages) {
    SVGF_PIXEL();
    const uint32_t curBufIdx = p.bufferIndex;
    const uint32_t prevBufIdx = (curBufIdx + 1) % 2;
    const float4* __restrict__ src = s.lighting[numFilteringStages % 2];
    const bool modulateAlbedo = (s.svgfFlags & GFX_SVGF_MODULATE_ALBEDO) != 0;

    f3 finalLighting = xyz(src[pix]);
    if (modulateAlbedo)
        finalLighting *= xyz(s.albedo[pix]);

    if ((s.svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_AA) && !(s.svgfFlags & GFX_SVGF_IS_FIRST_FRAME)) {
        const float4* __restrict__ prevFinal = s.finalLighting[prevBufIdx];
        const float2 psp = s.prevScreenPos[pix];
        f3 prevFinalLighting(0.0f);
        const bool outOfScreen = (psp.x < 0.0f || psp.y < 0.0f || psp.x >= 1.0f || psp.y >= 1.0f);
        if (!outOfScreen) {
            const f2 prevViewportPos(W * psp.x, H * psp.y);
            const int ppx = dm_f2int(prevViewportPos.x), ppy = dm_f2int(prevViewportPos.y);
            const f2 fDelta = prevViewportPos - (f2((float)ppx, (float)ppy) + f2(0.5f, 0.5f));
            const int dlx = fDelta.x < 0 ? -1 : 1, dly = fDelta.y < 0 ? -1 : 1;
            const int bx = ppx, by = ppy;
            const int cx = clampi(ppx + dlx, 0, W - 1), cy = clampi(ppy + dly, 0, H - 1);
            float sumWeights = 0.0f;
            const float sx = fabsf(fDelta.x);
            const float t = fabsf(fDelta.y);
            {
                const float weight = (1 - sx) * (1 - t);
                prevFinalLighting += weight * xyz(prevFinal[(size_t)by * W + bx]);
                sumWeights += weight;
            }
            {
                const float weight = sx * (1 - t);
                prevFinalLighting += weight * xyz(prevFinal[(size_t)by * W + cx]);
                sumWeights += weight;
            }
            {
                const float weight = (1 - sx) * t;
                prevFinalLighting += weight * xyz(prevFinal[(size_t)cy * W + bx]);
                sumWeights += weight;
            }
            {
                const float weight = sx * t;
                prevFinalLighting += weight * xyz(prevFinal[(size_t)cy * W + cx]);
                sumWeights += weight;
            }
            if (sumWeights != 0) {
                const float r = 1 / sumWeights;
                prevFinalLighting = f3(prevFinalLighting.x * r, prevFinalLighting.y * r, prevFinalLighting.z * r);
            }
            else {
                prevFinalLighting = f3(0.0f);
            }
        }

        f3 nbBoxMin = finalLighting, nbBoxMax = finalLighting, nbCrossMin = finalLighting, nbCrossMax = finalLighting;
#pragma unroll
        for (int i = -1; i <= 1; ++i) {
#pragma unroll
            for (int j = -1; j <= 1; ++j) {
                if (i == 0 && j == 0)
                    continue;
                const size_t nb = (size_t)clampi(y + i, 0, H - 1) * W + clampi(x + j, 0, W - 1);
                f3 nbValue = xyz(src[nb]);
                if (modulateAlbedo)
                    nbValue *= xyz(s.albedo[nb]);
                nbBoxMin = min3(nbBoxMin, nbValue);
                nbBoxMax = max3(nbBoxMax, nbValue);
                if (i == 0 || j == 0) {
                    nbCrossMin = min3(nbCrossMin, nbValue);
                    nbCrossMax = max3(nbCrossMax, nbValue);
                }
            }
        }
        const f3 nbMin = 0.5f * (nbBoxMin + nbCrossMin);
        const f3 nbMax = 0.5f * (nbBoxMax + nbCrossMax);
        prevFinalLighting = min3(max3(prevFinalLighting, nbMin), nbMax);

        const float curWeight = 1.0f / s.taaHistoryLength;
        const float prevWeight = 1.0f - curWeight;
        finalLighting = prevWeight * prevFinalLighting + curWeight * finalLighting;
    }
    s.finalLighting[curBufIdx][pix] = make_float4(finalLighting.x, finalLighting.y, finalLighting.z, 1.0f);
}

// ---- feedbackNoisyLighting (svgf.cu:356-374) ----------------------------------------------
// With SVGF off and temporal accumulation on, the next frame's reprojection reads the unfiltered lighting of this one.
__global__ void __launch_bounds__(256) k_svgfFeedbackNoisyLighting(DevSvgf s, DevFrameParams p) {
    SVGF_PIXEL();
    s.prevLighting[pix] = s.lighting[0][pix];
}

// ---- debugVisualize (visualize.cu:6-87) ----------------------------------------------------
// The app reads its lighting, albedo and moment planes at the launch index and its G-buffers (normal, prevScreenPos) at
// glPix(launch index), and writes the view at glPix(launch index).  That is the indexing of every SVGF kernel of the app:
// applyAlbedoModulationAndTemporalAntiAliasing too reads the lighting at the launch index and writes finalLightingBuffer at
// glPix (svgf.cu:555, 610), and the display shows both buffers through the same shader.  The planes here are top-down, like
// GFX_BUF_SVGF_FINAL, so pixel (x, y) of every plane is pixel (x, y) of the view: no flip.
__global__ void __launch_bounds__(256) k_svgfDebugVisualize(DevSvgf s, DevFrameParams p, float4* out, int view,
                                                            float motionVectorOffset, float motionVectorScale,
                                                            uint32_t numFilteringStages) {
    SVGF_PIXEL();
    float4 color = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    switch (view) {
    case GFX_SVGF_VIEW_NOISY_BEAUTY: {
        f3 lighting = xyz(s.lighting[0][pix]);
        if (s.svgfFlags & GFX_SVGF_MODULATE_ALBEDO)
            lighting *= xyz(s.albedo[pix]);
        color = make_float4(lighting.x, lighting.y, lighting.z, 1.0f);
    } break;
    case GFX_SVGF_VIEW_VARIANCE: {
        const float stdDev = sqrtf(s.lighting[0][pix].w);
        color = make_float4(stdDev, stdDev, stdDev, 1.0f);
    } break;
    case GFX_SVGF_VIEW_FILTERED_VARIANCE: {
        const float stdDev = sqrtf(s.lighting[numFilteringStages % 2][pix].w);
        color = make_float4(stdDev, stdDev, stdDev, 1.0f);
    } break;
    case GFX_SVGF_VIEW_ALBEDO: {
        const float4 albedo = s.albedo[pix];
        color = make_float4(albedo.x, albedo.y, albedo.z, 1.0f);
    } break;
    case GFX_SVGF_VIEW_NORMAL: {
        const f3 n = 0.5f * xyz(s.normal[pix]) + f3(0.5f);
        color = make_float4(n.x, n.y, n.z, 1.0f);
    } break;
    case GFX_SVGF_VIEW_MOTION_VECTOR: {
        const float2 prevScreenPos = s.prevScreenPos[pix];
        const f2 curScreenPos((x + 0.5f) / W, (y + 0.5f) / H);
        const f2 motionVector((float)W * (curScreenPos.x - prevScreenPos.x), (float)H * (curScreenPos.y - prevScreenPos.y));
        color = make_float4(fminf(fmaxf(motionVectorScale * motionVector.x + motionVectorOffset, 0.0f), 1.0f),
                            fminf(fmaxf(motionVectorScale * motionVector.y + motionVectorOffset, 0.0f), 1.0f),
                            motionVectorOffset, 1.0f);
    } break;
    default: { // GFX_SVGF_VIEW_SAMPLE_COUNT: the field k_svgfVariance reads
        const uint32_t count = __float_as_uint(s.moments[p.bufferIndex][pix].z) & 0xFFFFFFu;
        const float value = fminf(count / 255.0f, 1.0f);
        color = make_float4(value, value, value, 1.0f);
    } break;
    }
    out[pix] = color;
}

namespace {

DevSvgf makeDevSvgf(const gfx_ctx* ctx, const GfxFrameParams* params) {
    const FrameState &F = ctx->frame;
    DevSvgf s;
    s.W = F.W;
    s.H = F.H;
    for (int i = 0; i < 2; ++i) {
        s.gb0[i] = F.gb0[i];
        s.gb1[i] = F.gb1[i];
        s.gb2[i] = F.gb2[i];
        s.gb3[i] = F.gb3[i];
        s.lighting[i] = F.svgfLighting[i];
        s.moments[i] = F.svgfMoments[i];
        s.depth[i] = F.svgfDepth[i];
        s.finalLighting[i] = F.svgfFinal[i];
    }
    s.beauty = F.beauty;
    s.albedoAccum = F.albedo;
    s.prevLighting = F.svgfPrevLighting;
    s.albedo = F.svgfAlbedo;
    s.prevScreenPos = F.svgfPrevScreenPos;
    s.normal = F.svgfNormal;
    // camera(aspect, fovY, 0.1, 1000) depth row (svgf_main.cpp:1473-1478, basic_types.h:4899-4917)
    const float nearZ = 0.1f, farZ = 1000.0f;
    const float dz = farZ - nearZ;
    s.m22 = -(nearZ + farZ) / dz;
    s.m23 = -2 * farZ * nearZ / dz;
    s.svgfFlags = params->svgfFlags;
    s.taaHistoryLength = params->taaHistoryLength ? params->taaHistoryLength : 16;
    return s;
}

} // namespace

int launchSVGF(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params, int pass, uint32_t stage) {
    // The depth gradient of both filters reads the neighbour x + (x < W/2 ? 1 : -1) and row y + (y < H/2 ? 1 : -1): pixel -1 and
    // row -1 on frames one pixel wide or high, as in the reference (svgf.cu:75-78, 268-271).  Such frames are refused.
    if ((pass == GFX_SVGF_ESTIMATE_VARIANCE || pass == GFX_SVGF_ATROUS) && (ctx->frame.W < 2 || ctx->frame.H < 2)) {
        ctx->setError("gfx_svgf_launch: the variance and à-trous passes need a frame of at least 2x2 pixels");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    bool jitter;
    float2 sample;
    const int rc = svgfSubPixelSample(ctx, params, &jitter, &sample);
    if (rc != GFX_OK)
        return rc;
    const DevFrameParams p = makeDevParams(ctx, params);
    if (p.y1 <= p.y0)
        return GFX_OK;
    const FrameState &F = ctx->frame;
    const DevSvgf s = makeDevSvgf(ctx, params);

    const dim3 block(32, 8);
    const dim3 grid((F.W + 31) / 32, (p.y1 - p.y0 + 7) / 8);
    switch (pass) {
    case GFX_SVGF_TEMPORAL_ACCUMULATE: { GFX_TIMED(ctx, stream, "svgf_temporal"); k_svgfTemporal<<<grid, block, 0, stream>>>(s, p); } break;
    case GFX_SVGF_ESTIMATE_VARIANCE: { GFX_TIMED(ctx, stream, "svgf_variance"); k_svgfVariance<<<grid, block, 0, stream>>>(s, p); } break;
    case GFX_SVGF_ATROUS:
        if (stage > 4) {
            ctx->setError("gfx_svgf_launch: à-trous stage must be 0..4 (svgf.cu:232-239)");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        { GFX_TIMED(ctx, stream, "svgf_atrous"); k_svgfATrous<<<grid, block, 0, stream>>>(s, p, stage); }
        break;
    case GFX_SVGF_FILL_BACKGROUND: {
        GFX_TIMED(ctx, stream, "svgf_background");
        if (jitter)
            k_svgfBackgroundSubPixelJitter<<<grid, block, 0, stream>>>(s, p, stage, ctx->devScene(params).env, sample);
        else
            k_svgfBackground<<<grid, block, 0, stream>>>(s, p, stage, ctx->devScene(params).env);
    } break;
    case GFX_SVGF_MODULATE_TAA: { GFX_TIMED(ctx, stream, "svgf_modulate_taa"); k_svgfModulateTAA<<<grid, block, 0, stream>>>(s, p, stage); } break;
    case GFX_SVGF_FEEDBACK_NOISY_LIGHTING: { GFX_TIMED(ctx, stream, "svgf_feedback_noisy_lighting"); k_svgfFeedbackNoisyLighting<<<grid, block, 0, stream>>>(s, p); } break;
    default:
        ctx->setError("gfx_svgf_launch: unknown pass");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

int launchSVGFDebugVisualize(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params, int view, float motionVectorOffset,
                             float motionVectorScale, uint32_t numFilteringStages) {
    if (view < GFX_SVGF_VIEW_NOISY_BEAUTY || view > GFX_SVGF_VIEW_SAMPLE_COUNT) {
        ctx->setError("gfx_svgf_debug_visualize: the view must be 0..6 (GfxSVGFView); Final Rendering is the present of "
                      "GFX_BUF_SVGF_FINAL");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    FrameState &F = ctx->frame;
    if (!F.svgfDebugVisualize) {
        const size_t n = (size_t)F.W * F.H;
        GFX_CUDA(ctx, cudaMalloc(&F.svgfDebugVisualize, n * 16));
        GFX_CUDA(ctx, cudaMemsetAsync(F.svgfDebugVisualize, 0, n * 16, stream));
    }
    const DevFrameParams p = makeDevParams(ctx, params);
    if (p.y1 <= p.y0)
        return GFX_OK;
    const DevSvgf s = makeDevSvgf(ctx, params);
    const dim3 block(32, 8);
    const dim3 grid((F.W + 31) / 32, (p.y1 - p.y0 + 7) / 8);
    {
        GFX_TIMED(ctx, stream, "svgf_debug_visualize");
        k_svgfDebugVisualize<<<grid, block, 0, stream>>>(s, p, F.svgfDebugVisualize, view, motionVectorOffset, motionVectorScale,
                                                         numFilteringStages);
    }
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

} // namespace gfx
