// present.cu — the output side of a frame (SURVEY.md §8f-4): accumulation buffer -> tone-mapped, sRGB-encoded RGBA8.
//
// Replaces, in one kernel, copyToLinearBuffers + visualizeToOutputBuffer (restir_di/gpu_kernels/copy_buffers.cu:6-28,32-80),
// the display shader common/shaders/drawOptiXResult.frag with GL_FRAMEBUFFER_SRGB, and the arithmetic of the screenshot
// writer saveImage(float4*, SDRImageSaverConfig) (common/common_host.cpp:2859-2897), whose order of operations is followed:
// tone map, gamma, pack.  exp / pow come from detmath.h so that the oracle produces the same codes bit for bit.
// HBM-bound: 16 B read + 4 B written per pixel.
//
// The debug views of the NRC and ReGIR apps (neural_radiance_caching/gpu_kernels/copy_buffers.cu:32-130,
// regir/gpu_kernels/copy_buffers.cu:62-76,95-108) are the k_present<true> instantiation; k_present<false> is the plain
// COLOR / NORMAL path.
#include "pathtrace.cuh"

namespace gfx {

GFX_D float srgbGamma(float value) { // sRGB_gamma_s, basic_types.h:5405-5410
    if (value <= 0.0031308f)
        return 12.92f * value;
    return 1.055f * dm_pow(value, 1.0f / 2.4f) - 0.055f;
}

// what the views read besides the source buffer
struct PresentViews {
    const uint4* terminalInfo;
    const float* inferredRadiance;
    const float* inferenceQuery;
    const float2* motionVector; // GBuffer1 of frame->bufferIndex
    const float4* gbuffer2;
    float radianceScale, motionVectorScale, motionVectorOffset;
    DevRegir grid; // dimX..Z, gridOrigin, gridCellSize only
};

GFX_D uint32_t getFNV1Hash32(uint32_t x) { // regir/gpu_kernels/copy_buffers.cu:46-60, over the 4 bytes of x
    uint32_t hash = 2166136261u;
    for (int i = 0; i < 4; ++i)
        hash = (16777619u * hash) ^ ((x >> (8 * i)) & 0xFFu);
    return hash;
}

GFX_D f3 HSVtoRGB(float h, float s, float v) { // basic_types.h:5365-5388
    if (s == 0)
        return f3(v, v, v);
    const float hm = h - floorf(h);
    const int32_t hi = static_cast<int32_t>(hm * 6);
    const float f = hm * 6 - hi;
    const float m = v * (1 - s);
    const float n = v * (1 - s * f);
    const float k = v * (1 - s * (1 - f));
    if (hi == 0) return f3(v, k, m);
    if (hi == 1) return f3(n, v, m);
    if (hi == 2) return f3(m, v, k);
    if (hi == 3) return f3(m, n, v);
    if (hi == 4) return f3(k, m, v);
    if (hi == 5) return f3(v, m, n);
    return f3(0.0f);
}

GFX_D f3 calcCellColor(const DevRegir &grid, const f3 &positionInWorld) { // regir/gpu_kernels/copy_buffers.cu:62-76
    PCG32RNG rng{ (static_cast<uint64_t>(getFNV1Hash32(calcCellLinearIndex(grid, positionInWorld))) << 32) | 3018421212u };
    const float h = rng.getFloat0cTo1o();
    const float s = 0.5f + 0.5f * rng.getFloat0cTo1o();
    const float v = 0.5f + 0.5f * rng.getFloat0cTo1o();
    return HSVtoRGB(h, s, v);
}

// the view's value before alpha override / tone map / gamma (neural_radiance_caching/gpu_kernels/copy_buffers.cu:49-127)
GFX_D float4 viewValue(const PresentViews &w, int mode, uint32_t flags, size_t i, float4 v) {
    if (mode == GFX_PRESENT_NRC_PREDICTION) { // :52-67
        const uint4 t = w.terminalInfo[i];
        f3 radiance(0.0f);
        if (t.w & 1u) {
            const float* r = w.inferredRadiance + 3 * i;
            radiance = max3(f3(r[0], r[1], r[2]), f3(0.0f));
            if (w.radianceScale > 0)
                radiance /= w.radianceScale;
            const float* q = w.inferenceQuery + 14 * i;
            radiance *= (f3(q[8], q[9], q[10]) + f3(q[11], q[12], q[13]));
        }
        const f3 c = f3(__uint_as_float(t.x), __uint_as_float(t.y), __uint_as_float(t.z)) * radiance;
        v = make_float4(c.x, c.y, c.z, 1.0f);
    }
    else if (mode == GFX_PRESENT_FLOW) { // :87-94
        const float2 mv = w.motionVector[i];
        v = make_float4(fminf(fmaxf(w.motionVectorScale * mv.x + w.motionVectorOffset, 0.0f), 1.0f),
                        fminf(fmaxf(w.motionVectorScale * mv.y + w.motionVectorOffset, 0.0f), 1.0f), w.motionVectorOffset, 1.0f);
    }
    else if (mode == GFX_PRESENT_NRC_PATH_LENGTH) { // :96-112; the 8-bit field promotes to int
        const int32_t pathLength = (int32_t)((w.terminalInfo[i].w >> 1) & 0xFFu);
        const float t = fminf((pathLength - 1) / 5.0f, 1.0f);
        const f3 R(1.0f, 0.0f, 0.0f), G(0.0f, 1.0f, 0.0f), B(0.0f, 0.0f, 1.0f);
        f3 c;
        if (t < 0.5f) {
            const float tt = 2 * t;
            c = B * (1.0f - tt) + G * tt;
        }
        else {
            const float tt = 2 * (t - 0.5f);
            c = G * (1.0f - tt) + R * tt;
        }
        v = make_float4(c.x, c.y, c.z, 1.0f);
    }
    else if (mode == GFX_PRESENT_COLOR && (flags & GFX_PRESENT_REGIR_CELLS)) { // regir copy_buffers.cu:99-107
        const float4 g = w.gbuffer2[i];
        const f3 cellColor = calcCellColor(w.grid, f3(g.x, g.y, g.z));
        v.x *= cellColor.x;
        v.y *= cellColor.y;
        v.z *= cellColor.z;
    }
    if (flags & GFX_PRESENT_NRC_TRAINING_PATHS) { // :118-127
        const uint32_t t = w.terminalInfo[i].w;
        if ((t >> 9) & 1u) {
            v.x *= 1.0f; v.y *= 0.25f; v.z *= 1.0f; v.w *= 1.0f;
        }
        else if ((t >> 10) & 1u) {
            v.x *= 0.25f; v.y *= 1.0f; v.z *= 0.25f; v.w *= 1.0f;
        }
    }
    return v;
}

template <bool kViews>
__global__ void k_present(const float4* __restrict__ src, uint32_t* __restrict__ dst, uint32_t W, uint32_t H, int mode,
                          uint32_t flags, float brightnessScale, float alphaForOverride, PresentViews views) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H)
        return;
    const uint32_t sy = (flags & GFX_PRESENT_FLIP_Y) ? H - 1 - y : y;
    float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (!kViews || mode == GFX_PRESENT_COLOR || mode == GFX_PRESENT_NORMAL)
        v = src[(size_t)sy * W + x];
    if (mode == GFX_PRESENT_NORMAL) { // copy_buffers.cu:22-25 then :59-66
        f3 n(v.x, v.y, v.z);
        if (n.x != 0 || n.y != 0 || n.z != 0)
            n = normalize(n);
        v = make_float4(0.5f + 0.5f * n.x, 0.5f + 0.5f * n.y, 0.5f + 0.5f * n.z, 1.0f);
    }
    if constexpr (kViews)
        v = viewValue(views, mode, flags, (size_t)sy * W + x, v);
    if (alphaForOverride >= 0.0f)
        v.w = alphaForOverride;
    if (flags & GFX_PRESENT_TONE_MAP) {
        float r = v.x, g = v.y, b = v.z;
        if (!(isfinite(r) && isfinite(g) && isfinite(b)))
            r = g = b = 0.0f;
        const float lum = 0.2126729f * r + 0.7151522f * g + 0.0721750f * b;
        const float lumT = 1 - dm_exp(-(brightnessScale * lum)); // simpleToneMap_s
        const float s = lum > 0.0f ? lumT / lum : 0.0f;
        v.x = r * s;
        v.y = g * s;
        v.z = b * s;
    }
    if (flags & GFX_PRESENT_SRGB_GAMMA) {
        v.x = srgbGamma(v.x);
        v.y = srgbGamma(v.y);
        v.z = srgbGamma(v.z);
    }
    dst[(size_t)y * W + x] = (min(dm_f2uint(v.x * 255), 255u) << 0) | (min(dm_f2uint(v.y * 255), 255u) << 8) |
                             (min(dm_f2uint(v.z * 255), 255u) << 16) | (min(dm_f2uint(v.w * 255), 255u) << 24);
}

} // namespace gfx

using namespace gfx;

extern "C" void* gfx_buffer_device_ptr(gfx_ctx* ctx, int bufferId, uint32_t index, size_t* bytes);

namespace gfx {

int launchPresent(gfx_ctx* ctx, cudaStream_t stream, const GfxPresentParams* p) {
    FrameState &F = ctx->frame;
    const size_t n = (size_t)F.W * F.H;
    if (p->sourceBuffer == GFX_BUF_PRESENT_RGBA8 || p->mode < GFX_PRESENT_COLOR || p->mode > GFX_PRESENT_FLOW) {
        ctx->setError("gfx_present_launch: bad source buffer or mode");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    // the fields after alphaForOverride are read only for the views (older callers pass the six-field struct)
    const bool views = p->mode > GFX_PRESENT_NORMAL || (p->flags & (GFX_PRESENT_NRC_TRAINING_PATHS | GFX_PRESENT_REGIR_CELLS));
    const void* src = nullptr;
    if (p->mode == GFX_PRESENT_COLOR || p->mode == GFX_PRESENT_NORMAL) {
        size_t bytes = 0;
        src = gfx_buffer_device_ptr(ctx, p->sourceBuffer, p->sourceIndex, &bytes);
        if (!src || bytes != n * 16) {
            ctx->setError("gfx_present_launch: the source must be a float4-per-pixel frame buffer");
            return GFX_ERR_INVALID_ARGUMENT;
        }
    }
    PresentViews w = {};
    if (views) {
        const GfxFrameParams* fp = p->frame;
        if (!fp) {
            ctx->setError("gfx_present_launch: the NRC / ReGIR / flow views need GfxPresentParams::frame");
            return GFX_ERR_INVALID_ARGUMENT;
        }
        const bool nrcView = p->mode == GFX_PRESENT_NRC_PREDICTION || p->mode == GFX_PRESENT_NRC_PATH_LENGTH ||
                             (p->flags & GFX_PRESENT_NRC_TRAINING_PATHS);
        if (nrcView && !F.nrc.created) {
            ctx->setError("gfx_present_launch: no NRC frame yet");
            return GFX_ERR_NOT_READY;
        }
        const FrameState::Nrc &N = F.nrc;
        w.terminalInfo = N.terminalInfo;
        w.inferredRadiance = N.inferredRadiance;
        w.inferenceQuery = N.inferenceQuery;
        w.motionVector = F.gb1[fp->bufferIndex & 1];
        w.gbuffer2 = F.gb2[fp->bufferIndex & 1];
        w.radianceScale = fp->radianceScale;
        w.motionVectorScale = p->motionVectorScale;
        w.motionVectorOffset = p->motionVectorOffset;
        uint32_t dim[3];
        float origin[3], cellSize[3];
        regirGrid(fp, dim, origin, cellSize);
        w.grid.dimX = dim[0];
        w.grid.dimY = dim[1];
        w.grid.dimZ = dim[2];
        w.grid.gridOrigin = f3(origin[0], origin[1], origin[2]);
        w.grid.gridCellSize = f3(cellSize[0], cellSize[1], cellSize[2]);
    }
    if (!F.presentRgba8)
        GFX_CUDA(ctx, cudaMalloc(&F.presentRgba8, n * 4));
    const dim3 block(32, 8), grid((F.W + 31) / 32, (F.H + 7) / 8);
    { GFX_TIMED(ctx, stream, "present");
    if (views)
        k_present<true><<<grid, block, 0, stream>>>(static_cast<const float4*>(src), F.presentRgba8, F.W, F.H, p->mode, p->flags,
                                                    p->brightnessScale, p->alphaForOverride, w);
    else
        k_present<false><<<grid, block, 0, stream>>>(static_cast<const float4*>(src), F.presentRgba8, F.W, F.H, p->mode, p->flags,
                                                     p->brightnessScale, p->alphaForOverride, w); }
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

} // namespace gfx
