// oracle/denoise.cpp — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// CPU restatement of the reference's SVGF:
//   temporal accumulation  svgf/gpu_kernels/optix_pathtracing_kernels.cu:12-128 (reprojectPreviousAccumulation),
//                          :325-378 (demodulation, EMA 1/5, moments)
//   estimateVariance       svgf/gpu_kernels/svgf.cu:30-134
//   à-trous (box 3x3)      svgf/gpu_kernels/svgf.cu:6-26 (weights), :221-354
//   fillBackground         svgf/gpu_kernels/svgf.cu:378-461
//   albedo modulation+TAA  svgf/gpu_kernels/svgf.cu:465-531, :533-611
// Inputs are the G-buffers / beauty / albedo of an orc_frame (config 4 runs SVGF on restir_di's
// output).  Where the reference reads GL-rasterised G-buffers this restatement reads the ray-cast
// ones: world position (GBuffer2), decoded shading normal (GBuffer3), instSlot (GBuffer0), matSlot
// (GBuffer3), prevScreenPos = (raster - motionVector) / imageSize (GBuffer1), and a GL-style depth
// derived from the view-space z with camera(aspect, fovY, 0.1, 1000) (svgf_main.cpp:1473-1478,
// basic_types.h:4899-4917), background = 1.0.  exp() is detmath's, pow(x,128) is seven squarings
// (both sides), so the CUDA path can match bit for bit.
#include "oracle.h"
#include "shading.h"
#include <vector>
#include <omp.h>

using namespace orc;

struct F4 { float x, y, z, w; };
struct U4 { uint32_t x, y, z, w; };
struct F2 { float x, y; };

struct orc_svgf {
    orc_frame* frame;
    uint32_t W, H;
    std::vector<F4> lighting[2];   // lighting_variance_buffers
    std::vector<F4> moments[2];    // momentPair_sampleInfo_buffer per temporal set
    std::vector<F4> prevLighting;  // prevNoisyLightingBuffer
    std::vector<F4> albedo;        // albedoBuffer
    std::vector<float> depth[2];   // depthBuffer per temporal set
    std::vector<F4> finalLighting[2];
    std::vector<F2> prevScreenPos; // GBuffer2Elements::prevScreenPos (current frame)
};

extern "C" orc_svgf* orc_svgf_create(orc_frame* f, uint32_t W, uint32_t H) {
    orc_svgf* s = new orc_svgf();
    s->frame = f;
    s->W = W;
    s->H = H;
    const size_t n = (size_t)W * H;
    for (int i = 0; i < 2; ++i) {
        s->lighting[i].assign(n, F4{ 0, 0, 0, 0 });
        s->moments[i].assign(n, F4{ 0, 0, 0, 0 });
        s->depth[i].assign(n, 0.0f);
        s->finalLighting[i].assign(n, F4{ 0, 0, 0, 0 });
    }
    s->prevLighting.assign(n, F4{ 0, 0, 0, 0 });
    s->albedo.assign(n, F4{ 0, 0, 0, 0 });
    s->prevScreenPos.assign(n, F2{ 0, 0 });
    return s;
}
extern "C" void orc_svgf_destroy(orc_svgf* s) { delete s; }

extern "C" void* orc_svgf_buffer_ptr(orc_svgf* s, int id, uint32_t index, size_t* bytes) {
    const size_t n = (size_t)s->W * s->H;
    void* p = nullptr;
    size_t b = 0;
    switch (id) {
    case GFX_BUF_SVGF_LIGHTING_VARIANCE: p = s->lighting[index & 1].data(); b = n * 16; break;
    case GFX_BUF_SVGF_FINAL: p = s->finalLighting[index & 1].data(); b = n * 16; break;
    case GFX_BUF_SVGF_MOMENTS: p = s->moments[index & 1].data(); b = n * 16; break;
    case GFX_BUF_SVGF_PREV_LIGHTING: p = s->prevLighting.data(); b = n * 16; break;
    case GFX_BUF_SVGF_ALBEDO: p = s->albedo.data(); b = n * 16; break;
    case GFX_BUF_SVGF_DEPTH: p = s->depth[index & 1].data(); b = n * 4; break;
    default: break;
    }
    if (bytes) *bytes = b;
    return p;
}

namespace {

struct Cam {
    float3 position;
    Mat3 orientation, invOrientation;
    float vh, vw, aspect;
    float m22, m23; // camera(aspect, fovY, 0.1, 1000) depth row
};
Mat3 invert3(const Mat3 &a) { // basic_types.h:4150-4158
    const float* m = a.m;
    const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
    const float det = m00 * m11 * m22 + m01 * m12 * m20 + m02 * m10 * m21
        - m02 * m11 * m20 - m01 * m10 * m22 - m00 * m12 * m21;
    const float rdet = 1 / det;
    Mat3 r;
    r.m[0] = (m11 * m22 - m12 * m21) * rdet; r.m[1] = -(m01 * m22 - m02 * m21) * rdet; r.m[2] = (m01 * m12 - m02 * m11) * rdet;
    r.m[3] = -(m10 * m22 - m12 * m20) * rdet; r.m[4] = (m00 * m22 - m02 * m20) * rdet; r.m[5] = -(m00 * m12 - m02 * m10) * rdet;
    r.m[6] = (m10 * m21 - m11 * m20) * rdet; r.m[7] = -(m00 * m21 - m01 * m20) * rdet; r.m[8] = (m00 * m11 - m01 * m10) * rdet;
    return r;
}
Cam makeCam(const GfxCamera &c) {
    Cam cam;
    cam.position = float3(c.position[0], c.position[1], c.position[2]);
    std::memcpy(cam.orientation.m, c.orientation, 36);
    cam.invOrientation = invert3(cam.orientation);
    cam.aspect = c.aspect;
    cam.vh = 2 * std::tan(c.fovY * 0.5f);
    cam.vw = c.aspect * cam.vh;
    const float near = 0.1f, far = 1000.0f; // svgf_main.cpp:1473-1478
    const float dz = far - near;
    cam.m22 = -(near + far) / dz;
    cam.m23 = -2 * far * near / dz;
    return cam;
}

inline float pow128(float x) { // std::pow(x, sigma_n = 128) as seven squarings
    x = x * x; x = x * x; x = x * x; x = x * x; x = x * x; x = x * x; x = x * x;
    return x;
}
inline float calcDepthWeight(float nbDepth, float depth, float dzdx, float dzdy, int32_t dx, int32_t dy) { // svgf.cu:6-12
    const float sigma_z = 1.0f;
    const float eps = 1e-6f;
    return dm_exp(-std::fabs(nbDepth - depth) / (sigma_z * std::fabs(dzdx * dx + dzdy * dy) + eps));
}
inline float calcNormalWeight(const float3 &nbNormal, const float3 &normal) { // svgf.cu:14-18
    return pow128(std::fmax(0.0f, dot(nbNormal, normal)));
}
inline float calcLuminanceWeight(float nbLuminance, float luminance, float localMeanStdDev) { // svgf.cu:20-26
    const float sigma_l = 4.0f;
    const float eps = 1e-6f;
    return dm_exp(-std::fabs(nbLuminance - luminance) / (sigma_l * localMeanStdDev + eps));
}
inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
inline float3 xyz(const F4 &v) { return float3(v.x, v.y, v.z); }
inline float3 rgbSafeDivide(const float3 &a, const float3 &b) { // RGB::safeDivide (basic_types.h:5224-5229)
    return float3(b.x != 0 ? a.x / b.x : 0.0f, b.y != 0 ? a.y / b.y : 0.0f, b.z != 0 ? a.z / b.z : 0.0f);
}

struct View {
    const U4* gb0[2];
    const F2* gb1[2];
    const F4* gb2[2];
    const U4* gb3[2];
    const F4* beauty;
    const F4* albedoAccum;
};
View makeView(orc_frame* f) {
    View v;
    for (uint32_t i = 0; i < 2; ++i) {
        v.gb0[i] = (const U4*)orc_buffer_ptr(f, GFX_BUF_GBUFFER0, i, nullptr);
        v.gb1[i] = (const F2*)orc_buffer_ptr(f, GFX_BUF_GBUFFER1, i, nullptr);
        v.gb2[i] = (const F4*)orc_buffer_ptr(f, GFX_BUF_GBUFFER2, i, nullptr);
        v.gb3[i] = (const U4*)orc_buffer_ptr(f, GFX_BUF_GBUFFER3, i, nullptr);
    }
    v.beauty = (const F4*)orc_buffer_ptr(f, GFX_BUF_BEAUTY_ACCUM, 0, nullptr);
    v.albedoAccum = (const F4*)orc_buffer_ptr(f, GFX_BUF_ALBEDO_ACCUM, 0, nullptr);
    return v;
}

// ---- temporal accumulation ---------------------------------------------------------------
void temporalAccumulate(orc_svgf* s, const View &v, const GfxFrameParams* p, const Cam &cam, int x, int y) {
    const int W = (int)s->W, H = (int)s->H;
    const size_t pix = (size_t)y * W + x;
    const uint32_t curBufIdx = p->bufferIndex & 1;
    const uint32_t prevBufIdx = (curBufIdx + 1) % 2;
    const U4 gb0 = v.gb0[curBufIdx][pix];
    const U4 gb3 = v.gb3[curBufIdx][pix];
    const uint32_t instSlot = gb0.x;
    const uint32_t materialSlot = gb3.w;
    if (instSlot == 0xFFFFFFFFu) {
        s->depth[curBufIdx][pix] = 1.0f;
        s->lighting[0][pix] = F4{ 0, 0, 0, 0 };
        s->moments[curBufIdx][pix] = F4{ 0, 0, 0, 0 };
        return;
    }
    const F4 gb2 = v.gb2[curBufIdx][pix];
    const float3 positionInWorld(gb2.x, gb2.y, gb2.z);
    const float3 shadingNormalInWorld = decodeVector(gb3.x);

    // GL-style depth of the hit point
    const float3 posInView = cam.invOrientation.mul(positionInWorld - cam.position);
    const float zv = -posInView.z;
    const float ndcZ = (cam.m22 * zv + cam.m23) / (-zv);
    s->depth[curBufIdx][pix] = 0.5f * ndcZ + 0.5f;

    const float3 contribution = xyz(v.beauty[pix]);
    float3 dhReflectance = xyz(v.albedoAccum[pix]);
    // optix_pathtracing_kernels.cu:325-336: tiny DH reflectance is treated as zero
    dhReflectance.x = dhReflectance.x < 0.001f ? 0.0f : dhReflectance.x;
    dhReflectance.y = dhReflectance.y < 0.001f ? 0.0f : dhReflectance.y;
    dhReflectance.z = dhReflectance.z < 0.001f ? 0.0f : dhReflectance.z;
    s->albedo[pix] = F4{ dhReflectance.x, dhReflectance.y, dhReflectance.z, 0.0f };

    const F2 mv = v.gb1[curBufIdx][pix];
    const float2 prevScreenPos((x + 0.5f - mv.x) / W, (y + 0.5f - mv.y) / H);
    s->prevScreenPos[pix] = F2{ prevScreenPos.x, prevScreenPos.y };

    // reprojectPreviousAccumulation (:55-128)
    float3 prevNoisyLighting(0.0f);
    float prevFirstMoment = 0.0f, prevSecondMoment = 0.0f;
    uint32_t prevCount = 0, prevAcceptFlags = 0;
    const bool enableTemporalAccumulation = (p->svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_ACCUMULATION) != 0;
    const bool outOfScreen = (prevScreenPos.x < 0.0f || prevScreenPos.y < 0.0f || prevScreenPos.x >= 1.0f || prevScreenPos.y >= 1.0f);
    if (enableTemporalAccumulation && !outOfScreen) {
        const float2 prevViewportPos(W * prevScreenPos.x, H * prevScreenPos.y);
        const int ppx = dm_f2int(prevViewportPos.x), ppy = dm_f2int(prevViewportPos.y);
        const float2 fDelta = prevViewportPos - (float2((float)ppx, (float)ppy) + float2(0.5f, 0.5f));
        const int dlx = fDelta.x < 0 ? -1 : 1, dly = fDelta.y < 0 ? -1 : 1;
        const int nbx[4] = { ppx, clampi(ppx + dlx, 0, W - 1), ppx, clampi(ppx + dlx, 0, W - 1) };
        const int nby[4] = { ppy, ppy, clampi(ppy + dly, 0, H - 1), clampi(ppy + dly, 0, H - 1) };
        float sumWeights = 0.0f;
        float prevFloatSampleCount = 0;
        uint32_t acceptableFlags = 0;
        const float sx = std::fabs(fDelta.x);
        const float t = std::fabs(fDelta.y);
        const float weights[4] = { (1 - sx) * (1 - t), sx * (1 - t), (1 - sx) * t, sx * t };
        for (uint32_t i = 0; i < 4; ++i) {
            const size_t nb = (size_t)nby[i] * W + nbx[i];
            const uint32_t nbInst = v.gb0[prevBufIdx][nb].x;
            const U4 nbGb3 = v.gb3[prevBufIdx][nb];
            if (nbInst != instSlot || nbGb3.w != materialSlot)
                continue;
            if (dot(decodeVector(nbGb3.x), shadingNormalInWorld) <= 0.85f)
                continue;
            const F4 nbGb2 = v.gb2[prevBufIdx][nb];
            if (sqLength(float3(nbGb2.x, nbGb2.y, nbGb2.z) - positionInWorld) > 0.1f)
                continue;
            const float weight = weights[i];
            const F4 nbLighting = s->prevLighting[nb];
            const F4 nbMoments = s->moments[prevBufIdx][nb];
            prevNoisyLighting += weight * xyz(nbLighting);
            prevFirstMoment += weight * nbMoments.x;
            prevSecondMoment += weight * nbMoments.y;
            prevFloatSampleCount += weight * (f2u(nbMoments.z) & 0xFFFFFFu);
            sumWeights += weight;
            acceptableFlags |= (1u << i);
        }
        if (sumWeights > 0) {
            prevNoisyLighting /= sumWeights;
            prevFirstMoment /= sumWeights;
            prevSecondMoment /= sumWeights;
            prevCount = dm_f2uint(std::floor(prevFloatSampleCount / sumWeights + 0.5f)); // roundf for x >= 0
            prevAcceptFlags = acceptableFlags;
        }
    }

    float3 demCont = rgbSafeDivide(contribution, dhReflectance);
    float luminance = sRGB_calcLuminance(demCont);
    float sqLuminance = pow2(luminance);

    if ((p->svgfFlags & GFX_SVGF_IS_FIRST_FRAME) || !enableTemporalAccumulation) {
        prevCount = 0;
        prevAcceptFlags = 0;
    }
    const uint32_t sampleCount = std::min(prevCount + 1, 65535u);
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
    s->lighting[0][pix] = F4{ demCont.x, demCont.y, demCont.z, 0.0f };
    s->moments[curBufIdx][pix] = F4{ luminance, sqLuminance, u2f((sampleCount & 0xFFFFFFu) | (prevAcceptFlags << 24)), 0.0f };
}

// ---- estimateVariance (svgf.cu:30-134) ---------------------------------------------------
void estimateVariance(orc_svgf* s, const View &v, const GfxFrameParams* p, int x, int y) {
    const int W = (int)s->W, H = (int)s->H;
    const size_t pix = (size_t)y * W + x;
    const uint32_t curBufIdx = p->bufferIndex & 1;
    if (v.gb0[curBufIdx][pix].x == 0xFFFFFFFFu)
        return;
    const F4 m = s->moments[curBufIdx][pix];
    float firstMoment = m.x;
    float secondMoment = m.y;
    const uint32_t count = f2u(m.z) & 0xFFFFFFu;
    if (count < 4) {
        const float filterKernel[] = { 0.00598f, 0.060626f, 0.241843f, 0.383103f, 0.241843f, 0.060626f, 0.00598f };
        const float centerWeight = pow2(filterKernel[3]);
        float sumFirstMoments = centerWeight * firstMoment;
        float sumSecondMoments = centerWeight * secondMoment;
        const float depth = s->depth[curBufIdx][pix];
        const int32_t dx = x < W / 2 ? 1 : -1;
        const int32_t dy = y < H / 2 ? 1 : -1;
        const float hnbDepth = s->depth[curBufIdx][(size_t)y * W + (x + dx)];
        const float vnbDepth = s->depth[curBufIdx][(size_t)(y + dy) * W + x];
        const float dzdx = (hnbDepth - depth) * dx;
        const float dzdy = (vnbDepth - depth) * dy;
        const float3 normal = decodeVector(v.gb3[curBufIdx][pix].x);
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
                const float nbDepth = s->depth[curBufIdx][nb];
                if (nbDepth == 1.0f)
                    continue;
                const float3 nbNormal = decodeVector(v.gb3[curBufIdx][nb].x);
                const float wz = calcDepthWeight(nbDepth, depth, dzdx, dzdy, j, i);
                const float wn = calcNormalWeight(nbNormal, normal);
                const float weight = hx * hy * wz * wn;
                const F4 nbm = s->moments[curBufIdx][nb];
                sumFirstMoments += weight * nbm.x;
                sumSecondMoments += weight * nbm.y;
                sumWeights += weight;
            }
        }
        firstMoment = sumFirstMoments / sumWeights;
        secondMoment = sumSecondMoments / sumWeights;
    }
    const float variance = std::fmax(secondMoment - pow2(firstMoment), 0.0f);
    s->lighting[0][pix].w = variance;
}

// ---- à-trous box 3x3 (svgf.cu:221-354) ---------------------------------------------------
void applyATrous(orc_svgf* s, const View &v, const GfxFrameParams* p, uint32_t filterStageIndex, int x, int y) {
    const int W = (int)s->W, H = (int)s->H;
    const size_t pix = (size_t)y * W + x;
    const int32_t stepWidths[] = { 1, 2, 4, 8, 16 };
    const int32_t stepWidth = stepWidths[filterStageIndex];
    const uint32_t curBufIdx = p->bufferIndex & 1;
    const std::vector<F4> &src = s->lighting[filterStageIndex % 2];
    std::vector<F4> &dst = s->lighting[(filterStageIndex + 1) % 2];
    if (v.gb0[curBufIdx][pix].x == 0xFFFFFFFFu)
        return;
    const bool feedback = (p->svgfFlags & GFX_SVGF_FEEDBACK_1ST_FILTERED_RESULT) != 0;

    const F4 srcLv = src[pix];
    if (filterStageIndex == 0 && !feedback)
        s->prevLighting[pix] = srcLv;
    const float luminance = sRGB_calcLuminance(xyz(srcLv));

    const float depth = s->depth[curBufIdx][pix];
    const int32_t dx = x < W / 2 ? 1 : -1;
    const int32_t dy = y < H / 2 ? 1 : -1;
    const float hnbDepth = s->depth[curBufIdx][(size_t)y * W + (x + dx)];
    const float vnbDepth = s->depth[curBufIdx][(size_t)(y + dy) * W + x];
    const float dzdx = (hnbDepth - depth) * dx;
    const float dzdy = (vnbDepth - depth) * dy;
    const float3 normal = decodeVector(v.gb3[curBufIdx][pix].x);

    const float gaussKernel[] = { 1 / 4.0f, 1 / 2.0f, 1 / 4.0f };
    float sumLocalVars = 0.0f;
    float sumVarWeights = 0.0f;
    for (int i = -1; i <= 1; ++i) {
        const int nbPixY = clampi(y + i, 0, H - 1);
        const float hy = gaussKernel[i + 1];
        for (int j = -1; j <= 1; ++j) {
            const int nbPixX = clampi(x + j, 0, W - 1);
            const float hx = gaussKernel[j + 1];
            const float weight = hx * hy;
            sumLocalVars += weight * src[(size_t)nbPixY * W + nbPixX].w;
            sumVarWeights += weight;
        }
    }
    const float localMeanStdDev = std::sqrt(sumLocalVars / sumVarWeights);

    const float centerWeight = 1.0f;
    float sumWeights = centerWeight;
    float3 dstLighting = centerWeight * xyz(srcLv);
    float dstVariance = pow2(centerWeight) * srcLv.w;
    for (int k = 0; k < 9; ++k) {
        if (k == 4)
            continue;
        const int ox = (k % 3 - 1) * stepWidth, oy = (k / 3 - 1) * stepWidth;
        const int nbx = x + ox, nby = y + oy;
        if (nbx < 0 || nbx >= W || nby < 0 || nby >= H)
            continue;
        const float h = 1.0f;
        const size_t nb = (size_t)nby * W + nbx;
        const float nbDepth = s->depth[curBufIdx][nb];
        if (nbDepth == 1.0f)
            continue;
        const float3 nbNormal = decodeVector(v.gb3[curBufIdx][nb].x);
        const float wz = calcDepthWeight(nbDepth, depth, dzdx, dzdy, ox, oy);
        const float wn = calcNormalWeight(nbNormal, normal);
        const F4 nbLv = src[nb];
        const float nbLuminance = sRGB_calcLuminance(xyz(nbLv));
        const float wl = calcLuminanceWeight(nbLuminance, luminance, localMeanStdDev);
        const float weight = h * wz * wn * wl;
        dstLighting += weight * xyz(nbLv);
        dstVariance += pow2(weight) * nbLv.w;
        sumWeights += weight;
    }
    dstLighting /= sumWeights;
    dstVariance /= pow2(sumWeights);
    const F4 out{ dstLighting.x, dstLighting.y, dstLighting.z, dstVariance };
    dst[pix] = out;
    if (filterStageIndex == 0 && feedback)
        s->prevLighting[pix] = out;
}

extern "C" orc_scene* orc_frame_scene(orc_frame* f);
extern "C" int orc_env_enabled(orc_scene* s, const GfxFrameParams* p);
extern "C" int orc_env_query(orc_scene* s, int op, const float* in, uint32_t n, float* out);

// ---- fillBackground (svgf.cu:378-461) -----------------------------------------------------
void fillBackground(orc_svgf* s, const View &v, const GfxFrameParams* p, const Cam &cam, const Cam &prevCam,
                    uint32_t numFilteringStages, int x, int y) {
    const int W = (int)s->W, H = (int)s->H;
    const size_t pix = (size_t)y * W + x;
    const uint32_t curBufIdx = p->bufferIndex & 1;
    if (v.gb0[curBufIdx][pix].x != 0xFFFFFFFFu)
        return;
    float3 finalLighting(0.001f, 0.001f, 0.001f);
    const float fx = (x + 0.5f) / W;
    const float fy = (y + 0.5f) / H;
    float3 direction = normalize(cam.orientation.mul(float3(cam.vw * (0.5f - fx), cam.vh * (0.5f - fy), 1)));
    orc_scene* scene = orc_frame_scene(s->frame);
    if (orc_env_enabled(scene, p)) { // :431-437; the sub-pixel offset is the pixel centre (no TAA jitter in this host)
        float posPhi, posTheta;
        toPolarYUp(direction, &posPhi, &posTheta);
        float phi = posPhi + p->envLightRotation;
        phi += p->envLightRotation; // as written in the reference (:418-420): added twice when the environment light is on
        float u = phi / (2 * kPi);
        u -= std::floor(u);
        const float uv[2] = { u, posTheta / kPi };
        float rgb[3];
        orc_env_query(scene, 2, uv, 1, rgb);
        finalLighting = p->envLightPowerCoeff * float3(rgb[0], rgb[1], rgb[2]);
    }
    // transpose(prevCamera.orientation) * direction
    const float* o = prevCam.orientation.m;
    direction = float3(o[0] * direction.x + o[3] * direction.y + o[6] * direction.z,
                       o[1] * direction.x + o[4] * direction.y + o[7] * direction.z,
                       o[2] * direction.x + o[5] * direction.y + o[8] * direction.z);
    direction /= direction.z;
    const float2 prevScreenPos(0.5f - direction.x / prevCam.vw, 0.5f - direction.y / prevCam.vh);
    s->lighting[numFilteringStages % 2][pix] = F4{ finalLighting.x, finalLighting.y, finalLighting.z, 0.0f };
    s->albedo[pix] = F4{ 1.0f, 1.0f, 1.0f, 0.0f };
    s->prevScreenPos[pix] = F2{ prevScreenPos.x, prevScreenPos.y };
}

// ---- albedo modulation + TAA (svgf.cu:465-611) -------------------------------------------
void modulateAndTAA(orc_svgf* s, const GfxFrameParams* p, uint32_t numFilteringStages, int x, int y) {
    const int W = (int)s->W, H = (int)s->H;
    const size_t pix = (size_t)y * W + x;
    const uint32_t curBufIdx = p->bufferIndex & 1;
    const uint32_t prevBufIdx = (curBufIdx + 1) % 2;
    const std::vector<F4> &src = s->lighting[numFilteringStages % 2];
    const bool modulateAlbedo = (p->svgfFlags & GFX_SVGF_MODULATE_ALBEDO) != 0;

    float3 finalLighting = xyz(src[pix]);
    if (modulateAlbedo)
        finalLighting *= xyz(s->albedo[pix]);

    if ((p->svgfFlags & GFX_SVGF_ENABLE_TEMPORAL_AA) && !(p->svgfFlags & GFX_SVGF_IS_FIRST_FRAME)) {
        const std::vector<F4> &prevFinal = s->finalLighting[prevBufIdx];
        const F2 psp = s->prevScreenPos[pix];
        // reprojectPreviousAccumulation (:465-531)
        float3 prevFinalLighting(0.0f);
        const bool outOfScreen = (psp.x < 0.0f || psp.y < 0.0f || psp.x >= 1.0f || psp.y >= 1.0f);
        if (!outOfScreen) {
            const float2 prevViewportPos(W * psp.x, H * psp.y);
            const int ppx = dm_f2int(prevViewportPos.x), ppy = dm_f2int(prevViewportPos.y);
            const float2 fDelta = prevViewportPos - (float2((float)ppx, (float)ppy) + float2(0.5f, 0.5f));
            const int dlx = fDelta.x < 0 ? -1 : 1, dly = fDelta.y < 0 ? -1 : 1;
            const int bx = ppx, by = ppy;
            const int cx = clampi(ppx + dlx, 0, W - 1), cy = clampi(ppy + dly, 0, H - 1);
            float sumWeights = 0.0f;
            const float sx = std::fabs(fDelta.x);
            const float t = std::fabs(fDelta.y);
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
            // RGB::safeDivide(float) (basic_types.h:5216-5223): multiply by the reciprocal when non-zero
            if (sumWeights != 0) {
                const float r = 1 / sumWeights;
                prevFinalLighting = float3(prevFinalLighting.x * r, prevFinalLighting.y * r, prevFinalLighting.z * r);
            }
            else {
                prevFinalLighting = float3(0.0f);
            }
        }

        float3 nbBoxMin = finalLighting, nbBoxMax = finalLighting, nbCrossMin = finalLighting, nbCrossMax = finalLighting;
        for (int i = -1; i <= 1; ++i) {
            for (int j = -1; j <= 1; ++j) {
                if (i == 0 && j == 0)
                    continue;
                const size_t nb = (size_t)clampi(y + i, 0, H - 1) * W + clampi(x + j, 0, W - 1);
                float3 nbValue = xyz(src[nb]);
                if (modulateAlbedo)
                    nbValue *= xyz(s->albedo[nb]);
                nbBoxMin = min3(nbBoxMin, nbValue);
                nbBoxMax = max3(nbBoxMax, nbValue);
                if (i == 0 || j == 0) {
                    nbCrossMin = min3(nbCrossMin, nbValue);
                    nbCrossMax = max3(nbCrossMax, nbValue);
                }
            }
        }
        const float3 nbMin = 0.5f * (nbBoxMin + nbCrossMin);
        const float3 nbMax = 0.5f * (nbBoxMax + nbCrossMax);
        prevFinalLighting = min3(max3(prevFinalLighting, nbMin), nbMax);

        const float curWeight = 1.0f / p->taaHistoryLength;
        const float prevWeight = 1.0f - curWeight;
        finalLighting = prevWeight * prevFinalLighting + curWeight * finalLighting;
    }
    s->finalLighting[curBufIdx][pix] = F4{ finalLighting.x, finalLighting.y, finalLighting.z, 1.0f };
}

} // namespace

// Returns GFX_ERR_INVALID_ARGUMENT, and runs nothing, for the variance and à-trous passes on a frame narrower or shorter than
// 2 pixels, whose depth-gradient neighbour lies outside the frame (gfx_svgf_launch refuses them alike); GFX_OK otherwise.
extern "C" int orc_svgf_pass(orc_svgf* s, const GfxFrameParams* p, int pass, uint32_t stage, int numThreads) {
    const int W = (int)s->W, H = (int)s->H;
    if ((pass == GFX_SVGF_ESTIMATE_VARIANCE || pass == GFX_SVGF_ATROUS) && (W < 2 || H < 2))
        return GFX_ERR_INVALID_ARGUMENT;
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    const View v = makeView(s->frame);
    const Cam cam = makeCam(p->camera);
    const Cam prevCam = makeCam(p->prevCamera);
    const int y0 = (int)p->tileOriginY, y1 = p->tileRows ? std::min(H, (int)(p->tileOriginY + p->tileRows)) : H;
#pragma omp parallel for schedule(dynamic, 4) num_threads(numThreads)
    for (int y = y0; y < y1; ++y) {
        for (int x = 0; x < W; ++x) {
            switch (pass) {
            case GFX_SVGF_TEMPORAL_ACCUMULATE: temporalAccumulate(s, v, p, cam, x, y); break;
            case GFX_SVGF_ESTIMATE_VARIANCE: estimateVariance(s, v, p, x, y); break;
            case GFX_SVGF_ATROUS: applyATrous(s, v, p, stage, x, y); break;
            case GFX_SVGF_FILL_BACKGROUND: fillBackground(s, v, p, cam, prevCam, stage, x, y); break;
            case GFX_SVGF_MODULATE_TAA: modulateAndTAA(s, p, stage, x, y); break;
            default: break;
            }
        }
    }
    return GFX_OK;
}
