// nrc.cu — the Neural Radiance Cache network on sm_90a.
//
// Replaces NeuralRadianceCache::{initialize,infer,train} (neural_radiance_caching/network_interface.cu:
// 48-157) and the tiny-cuda-nn kernels behind it (ext/tiny-cuda-nn: kernel_grid<half,3,2>
// encodings/grid.h:132-304, kernel_one_blob encodings/oneblob.h:83-108, kernel_mlp_fused<64,...>
// src/fully_fused_mlp.cu:47-129 — nvcuda::wmma 16x16x16 half —, relative_l2_luminance_loss,
// adam_step, ema_step_half_precision).
//
// Inference (2.2 M queries per 1080p frame): each 128-thread CTA (one warpgroup) takes 128 queries
// (hash grid + one-blob + identity -> 64 fp16 features) into shared memory in the K-major core-matrix
// layout, then runs the 64->64->...->16 MLP on Hopper's warpgroup tensor-core instruction:
// wgmma.mma_async m64nNk16 (N = 64|16, fp16 in, fp32 accumulate), two per K step for the two 64-row
// halves of the tile, accumulators in registers; ReLU + fp16 rounding in registers, activations written
// back to the same shared-memory tile for the next layer.  Weights (18 KB) stay resident in shared
// memory, pre-arranged in the core-matrix layout by k_nrcPrepWeights.  No activation ever touches HBM:
// the compulsory traffic is 56 B in + 12 B out per query (SURVEY.md §8d).
//
// Training (4 x 16 384 samples per frame) is latency-bound: one block = 128 samples, weights and activations in shared
// memory, every matrix product on wgmma (k_nrcTrainTc) for 1..3 hidden layers; deeper networks, whose activation tiles do
// not fit, train on CUDA cores (k_nrcTrain).  Weight gradients are accumulated with 64-bit fixed-point atomics.
//
// Both of NeuralRadianceCache::initialize's position encodings are built (gfx_nrc_create_with_encoding): the hash grid above,
// and the triangle wave (triangle_wave.h:47-81), which has no parameters and no grid stage - k_nrcInferMlp<kEncTriangleWave> is
// its whole inference, and the training kernels skip layer 0's data gradient and the encoding backward for it.  The kernels
// are templated on the encoding; the hash-grid instantiations are the code that was here before.
#include "context.h"
#include <cuda_fp16.h>
#include <random>
#include <vector>
#include <cmath>

namespace gfx {

constexpr uint32_t kInputDims = 14, kOutputDims = 3, kWidth = 64, kPaddedOutput = 16;
constexpr uint32_t kLevels = 16, kLog2HashmapSize = 15, kBaseResolution = 16;
constexpr float kLossScale = 128.0f;

struct NrcLevel {
    uint32_t offset;      // grid entries
    uint32_t hashmapSize;
    float scale;
    uint32_t resolution;
};
struct NrcLevels { NrcLevel l[kLevels]; };

} // namespace gfx

struct gfx_nrc {
    gfx_ctx* ctx = nullptr;
    int positionEncoding = GFX_NRC_POSITION_ENCODING_HASH_GRID;
    uint32_t numHiddenLayers = 2;
    float learningRate = 1e-2f;
    float adamEpsilon = 1e-15f;   // network_interface.cu:94 (triangle wave 1e-8), :119 (hash grid 1e-15)
    uint32_t numMatrixWeights = 0, numParams = 0;
    gfx::NrcLevels levels;
    __half* params = nullptr;     // current fp16 weights
    __half* paramsEma = nullptr;  // inference weights
    float* master = nullptr;
    float* m1 = nullptr;
    float* m2 = nullptr;
    uint32_t* steps = nullptr;
    unsigned long long* grads = nullptr; // loss-scaled gradients as 64-bit fixed point (2^-30 units): integer atomics
                                         // commute, so a training step is bit-reproducible whatever the block schedule
    float* loss = nullptr;        // device scalar
    uint4* ummaWeights = nullptr; // EMA MLP weights in the K-major core-matrix shared-memory layout
    uint4* trainBlobFwd = nullptr; // training weights, core-matrix layouts: W_l [N x 64] and W_l^T [64 x K] K-major blobs
    uint4* trainBlobT = nullptr;
    float4* positions = nullptr;   // split inference scratch: packed query positions, grid features [tile][level][row] half2
    __half2* features = nullptr;
    uint32_t scratchQueries = 0;
    float* gradsFloat = nullptr;   // gfx_nrc_keep_gradients: the loss-scaled gradients of the last training step
    bool keepGradients = false;
    uint32_t globalStep = 0;
    bool ummaDirty = true;
};

namespace gfx {

GFX_D float quarticCdf(float x, float invRadius) { // tiny-cuda-nn common_device.h:478-483
    const float u = x * invRadius;
    const float u2 = u * u;
    const float u4 = u2 * u2;
    return fmaxf(0.0f, fminf(1.0f, (15.0f / 16.0f) * u * (1 - (2.0f / 3.0f) * u2 + (1.0f / 5.0f) * u4) + 0.5f));
}

// index % size without an integer division: hashed levels have power-of-two tables, dense levels only wrap for
// out-of-range positions
GFX_D uint32_t nrcWrap(uint32_t index, uint32_t size) {
    if ((size & (size - 1u)) == 0u)
        return index & (size - 1u);
    return index < size ? index : index % size;
}

// grid_index's per-axis multipliers of one level (grid.h:76-111): the dense strides (0 for an axis the table does not reach),
// or the coherent hash's primes when the dense grid outgrows the table.  Returns whether the level is hashed.
GFX_D bool nrcLevelMultipliers(const NrcLevel &lv, uint32_t (&mul)[3]) {
    uint32_t stride = 1;
    uint32_t strides[3];
    bool used[3];
#pragma unroll
    for (uint32_t dim = 0; dim < 3; ++dim) {
        used[dim] = stride <= lv.hashmapSize;
        strides[dim] = stride;
        if (used[dim])
            stride *= lv.resolution;
    }
    const bool hashed = lv.hashmapSize < stride;
    const uint32_t primes[3] = { 1u, 2654435761u, 805459861u };
#pragma unroll
    for (uint32_t dim = 0; dim < 3; ++dim)
        mul[dim] = hashed ? primes[dim] : (used[dim] ? strides[dim] : 0u);
    return hashed;
}

// The cell of one level that a position falls in: pos_fract (common_device.h:425-431), then grid_index for its 8 corners.
// The per-axis terms of the dense stride sum or of the coherent prime hash are computed once, a corner is one 3-input add/xor
// plus the wrap.  Everything that depends only on the level is warp-uniform.  Corner bit d of idx selects the upper neighbour
// along axis d.
struct NrcCell {
    float frac[3];
    uint32_t term[3][2];
    uint32_t size;
    bool hashed;
    GFX_D NrcCell(const NrcLevel &lv, const float p[3]) {
        uint32_t mul[3];
        hashed = nrcLevelMultipliers(lv, mul);
        size = lv.hashmapSize;
#pragma unroll
        for (uint32_t d = 0; d < 3; ++d) {
            frac[d] = p[d] * lv.scale + 0.5f;
            const int tmp = (int)floorf(frac[d]);
            frac[d] -= (float)tmp;
            term[d][0] = (uint32_t)tmp * mul[d];
            term[d][1] = term[d][0] + mul[d];
        }
    }
    // the corner's entry of the level's table (two features)
    GFX_D uint32_t entry(uint32_t idx) const {
        const uint32_t a = term[0][idx & 1u], b = term[1][(idx >> 1) & 1u], c = term[2][(idx >> 2) & 1u];
        return nrcWrap(hashed ? (a ^ b ^ c) : (a + b + c), size);
    }
    // the corner's trilinear weight
    GFX_D float weight(uint32_t idx) const {
        float w = 1;
#pragma unroll
        for (uint32_t d = 0; d < 3; ++d)
            w *= (idx & (1u << d)) == 0 ? 1 - frac[d] : frac[d];
        return w;
    }
};

// OneBlob: 5 dims x 4 bins -> features 32..51, identity 52..57, ones 58..63 (q = the 14 query floats; q[0..2] unused)
GFX_D void nrcEncodeTail(const float* q, __half* tail) {
#pragma unroll
    for (uint32_t d = 0; d < 5; ++d) {
        const float x = q[3 + d];
        // kernel_one_blob_soa (tiny-cuda-nn oneblob.h:110-139; the composite encoding runs its nested encodings on SoA
        // slices): CDF at the five bin boundaries k / 4, each summed over the three periodic images
        float leftCdf = quarticCdf(-x, 4.0f) + quarticCdf(-x - 1.0f, 4.0f) + quarticCdf(-x + 1.0f, 4.0f);
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
            const float rightBoundary = 0.25f * (float)(k + 1); // scalbnf(k + 1, -2)
            const float rightCdf = quarticCdf(rightBoundary - x, 4.0f) + quarticCdf(rightBoundary - x - 1.0f, 4.0f) +
                                   quarticCdf(rightBoundary - x + 1.0f, 4.0f);
            tail[d * 4 + k] = __float2half(rightCdf - leftCdf);
            leftCdf = rightCdf;
        }
    }
#pragma unroll
    for (uint32_t d = 0; d < 6; ++d)
        tail[20 + d] = __float2half(q[8 + d]);
#pragma unroll
    for (uint32_t k = 26; k < 32; ++k)
        tail[k] = __float2half(1.0f);
}

// Encodes one query into 64 halves, delivered 8 at a time (chunk c = features 8c..8c+7) through `emit`.
// Arithmetic mirrors oracle/nrc.cpp::encode (half accumulation of the trilinear blend like kernel_grid).
template <typename Emit>
GFX_D void nrcEncode(const NrcLevels &levels, const __half* __restrict__ table, const float* __restrict__ in, Emit emit) {
    float q[kInputDims];
#pragma unroll
    for (uint32_t d = 0; d < kInputDims; ++d)
        q[d] = in[d];
    __half feat[8];
    // One level at a time: the encoder is bound by the L1's divergent-gather rate, not by issue.  The 8 gathers are all
    // issued before the blend uses them: a corner's wrap may branch, and a load cannot move above a branch, so a blend step
    // between them would wait for each gather in turn.
#pragma unroll 1
    for (uint32_t l = 0; l < kLevels; ++l) {
        const NrcLevel lv = levels.l[l];
        const __half2* grid = reinterpret_cast<const __half2*>(table + (size_t)lv.offset * 2);
        const NrcCell cell(lv, q);
        __half2 v[8];
#pragma unroll
        for (uint32_t idx = 0; idx < 8; ++idx)
            v[idx] = __ldg(grid + cell.entry(idx));
        __half r0 = __float2half(0.0f), r1 = __float2half(0.0f);
#pragma unroll
        for (uint32_t idx = 0; idx < 8; ++idx) {
            const float weight = cell.weight(idx);
            r0 = __float2half(__half2float(r0) + __half2float(__float2half(weight * __low2float(v[idx]))));
            r1 = __float2half(__half2float(r1) + __half2float(__float2half(weight * __high2float(v[idx]))));
        }
        feat[(l & 3) * 2 + 0] = r0;
        feat[(l & 3) * 2 + 1] = r1;
        if ((l & 3) == 3)
            emit(l >> 2, feat);
    }
    __half tail[32];
    nrcEncodeTail(q, tail);
#pragma unroll
    for (uint32_t c = 0; c < 4; ++c)
        emit(4 + c, tail + 8 * c);
}

// triangle_wave_encoding (tiny-cuda-nn encodings/triangle_wave.h:47-81), frequency f of one position coordinate.  The only
// products, f * 0.25f and |.| * 4, are exact, so FMA contraction cannot change the result.
GFX_D float nrcTriangleWave(float p, uint32_t f) {
    const float x = scalbnf(p, (int)f - 1);
    const float val = x + (float)f * 0.25f;
    return fabsf(val - floorf(val) - 0.5f) * 4 - 1;
}

// quartic_cdf (common_device.h:478-483) as the reference's own tiny-cuda-nn build evaluates it: nvcc contracts its polynomial
// into three FMAs (the triangle-wave network is pinned bit for bit against that build, tests/golden/tcnn_nrc_triwave.npz)
GFX_D float quarticCdfContracted(float x, float invRadius) {
    const float u = x * invRadius;
    const float u2 = u * u;
    const float u4 = u2 * u2;
    const float inner = __fmaf_rn(1.0f / 5.0f, u4, __fmaf_rn(-(2.0f / 3.0f), u2, 1.0f));
    return fmaxf(0.0f, fminf(1.0f, __fmaf_rn((15.0f / 16.0f) * u, inner, 0.5f)));
}

// The triangle-wave network's one-blob + identity (q = the 14 query floats).  TriangleWave prefers the AoS layout, so the
// Composite encoding runs every nested encoding in AoS (composite.h:253-262) and OneBlob takes kernel_one_blob (oneblob.h:83-108)
// with one_blob_subwarp_aligned (:47-69): the CDF at the four left bin boundaries k / 4, each summed over the three periodic
// images; bin k < 3 ends at bin k + 1's left CDF, the last bin at "bin 0's left CDF + 1".  Identity is x * 1 + 0 (identity.h:67).
GFX_D void nrcEncodeTailAos(const float* q, __half* tail) {
#pragma unroll
    for (uint32_t d = 0; d < 5; ++d) {
        const float x = q[3 + d];
        float cdf[4];
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
            const float left = 0.25f * (float)k; // scalbnf(k, -2)
            cdf[k] = quarticCdfContracted(left - x, 4.0f) + quarticCdfContracted(left - x - 1.0f, 4.0f) +
                     quarticCdfContracted(left - x + 1.0f, 4.0f);
        }
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k)
            tail[d * 4 + k] = __float2half((k < 3 ? cdf[k + 1] : cdf[0] + 1.0f) - cdf[k]);
    }
#pragma unroll
    for (uint32_t d = 0; d < 6; ++d)
        tail[20 + d] = __float2half(q[8 + d] + 0.0f);
}

// The triangle-wave network's 64 inputs from the 14 query floats, in registers, delivered 8 at a time like nrcEncode:
// TriangleWave(3 dims x 12 frequencies) feature-major in 0..35 (input 12 d + f), then one-blob 36..55 and identity 56..61,
// and the ones Composite pads the last nested encoding with (composite.h:100-111, 231-237) in 62..63.  OneBlob's min_alignment
// of 4 divides 36, so nothing is padded between the triangle wave and the one-blob.
template <typename Emit>
GFX_D void nrcEncodeTriWave(const float (&q)[kInputDims], Emit emit) {
    __half feat[64];
#pragma unroll
    for (uint32_t d = 0; d < 3; ++d)
#pragma unroll
        for (uint32_t f = 0; f < 12; ++f)
            feat[12 * d + f] = __float2half(nrcTriangleWave(q[d], f));
    __half tail[26];
    nrcEncodeTailAos(q, tail);
#pragma unroll
    for (uint32_t k = 0; k < 26; ++k)
        feat[36 + k] = tail[k];
    feat[62] = feat[63] = __float2half(1.0f);
#pragma unroll
    for (uint32_t c = 0; c < 8; ++c)
        emit(c, feat + 8 * c);
}

// the network's input encoding of one query read from global memory (the kernels are templated on the encoding)
constexpr uint32_t kEncTriangleWave = GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE, kEncHashGrid = GFX_NRC_POSITION_ENCODING_HASH_GRID;
template <uint32_t kEnc, typename Emit>
GFX_D void nrcEncodeQuery(const NrcLevels &levels, const __half* __restrict__ table, const float* __restrict__ in, Emit emit) {
    if constexpr (kEnc == kEncHashGrid) {
        nrcEncode(levels, table, in, emit);
    }
    else {
        float q[kInputDims];
#pragma unroll
        for (uint32_t d = 0; d < kInputDims; ++d)
            q[d] = in[d];
        nrcEncodeTriWave(q, emit);
    }
}

// 8 halves -> one 16-byte core-matrix row
GFX_D uint4 packHalf8(const __half* f) {
    uint4 v;
    v.x = (uint32_t)__half_as_ushort(f[0]) | ((uint32_t)__half_as_ushort(f[1]) << 16);
    v.y = (uint32_t)__half_as_ushort(f[2]) | ((uint32_t)__half_as_ushort(f[3]) << 16);
    v.z = (uint32_t)__half_as_ushort(f[4]) | ((uint32_t)__half_as_ushort(f[5]) << 16);
    v.w = (uint32_t)__half_as_ushort(f[6]) | ((uint32_t)__half_as_ushort(f[7]) << 16);
    return v;
}

// ---------------------------------------------------------------------------------------------
// wgmma helpers (PTX for sm_90a)
// ---------------------------------------------------------------------------------------------
GFX_D uint32_t smemU32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// shared-memory matrix descriptor, K-major, no swizzle (cute::GmmaDescriptor, layout INTERLEAVE): core matrices are
// 8 rows x 16 B stored contiguously; LBO = byte distance between the two K-halves of one MMA (K = 16),
// SBO = byte distance between consecutive 8-row groups.
GFX_D uint64_t makeSmemDesc(uint32_t addr, uint32_t lboBytes, uint32_t sboBytes) {
    uint64_t d = 0;
    d |= (uint64_t)((addr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lboBytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sboBytes >> 4) & 0x3FFFu) << 32;
    return d; // base_offset 0, layout_type 0 (no swizzle)
}

// The accumulator fragment of wgmma m64nNk16 (f32): in warp w, lane l holds rows 16 w + l / 4 + 8 i (i = 0, 1) and, per
// 8-column group j, columns 8 j + 2 (l % 4) + e (e = 0, 1) in d[4 j + 2 i + e].
GFX_D uint32_t fragRow(uint32_t tid, uint32_t i) { return ((tid >> 5) << 4) + ((tid & 31u) >> 2) + 8u * i; }
GFX_D uint32_t fragCol(uint32_t tid, uint32_t j) { return 8u * j + 2u * (tid & 3u); }

// D[64 x 64] (+)= A[64 x 16] B[64 x 16]^T, both operands K-major in shared memory
GFX_D void wgmma64(float (&d)[32], uint64_t aDesc, uint64_t bDesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(aDesc), "l"(bDesc), "r"(accumulate) : "memory");
}
// D[64 x 16] (+)= A[64 x 16] B[16 x 16]^T
GFX_D void wgmma16(float (&d)[8], uint64_t aDesc, uint64_t bDesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(aDesc), "l"(bDesc), "r"(accumulate) : "memory");
}
GFX_D void wgmmaFence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
GFX_D void wgmmaCommit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
GFX_D void wgmmaWait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from touching accumulator registers across the asynchronous MMA (cutlass warpgroup_fence_operand)
template <int N>
GFX_D void fenceAccumulators(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i)
        asm volatile("" : "+f"(d[i]) :: "memory");
}

// One layer of the 128-row tile: acc[h] = A rows 64 h .. 64 h + 63 x W^T, K = 16 kSteps.  A: chunk stride aChunk bytes
// (8 K values per chunk, 16 B per row), W: the [N x K] K-major blob, chunk stride N * 16.  Returns when the MMAs are done.
GFX_D void mlpLayer64(float (&acc)[2][32], uint32_t aAddr, uint32_t aChunk, uint32_t wAddr, uint32_t kSteps) {
    wgmmaFence();
    for (uint32_t k = 0; k < kSteps; ++k) {
        const uint64_t bDesc = makeSmemDesc(wAddr + 2 * k * (kWidth * 16), kWidth * 16, 128);
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h)
            wgmma64(acc[h], makeSmemDesc(aAddr + h * 1024 + 2 * k * aChunk, aChunk, 128), bDesc, k > 0 ? 1u : 0u);
    }
    wgmmaCommit();
    wgmmaWait();
    fenceAccumulators(acc[0]);
    fenceAccumulators(acc[1]);
}
GFX_D void mlpLayer16(float (&acc)[2][8], uint32_t aAddr, uint32_t aChunk, uint32_t wAddr) {
    wgmmaFence();
#pragma unroll
    for (uint32_t k = 0; k < kWidth / 16; ++k) {
        const uint64_t bDesc = makeSmemDesc(wAddr + 2 * k * (kPaddedOutput * 16), kPaddedOutput * 16, 128);
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h)
            wgmma16(acc[h], makeSmemDesc(aAddr + h * 1024 + 2 * k * aChunk, aChunk, 128), bDesc, k > 0 ? 1u : 0u);
    }
    wgmmaCommit();
    wgmmaWait();
    fenceAccumulators(acc[0]);
    fenceAccumulators(acc[1]);
}

// hidden-layer epilogue: ReLU, fp16, back into a [128 x 64] K-major tile (element (r, k) at (k / 8) * 2048 + r * 16 + (k % 8) * 2)
GFX_D void storeReluTile(const float (&acc)[2][32], uint8_t* tile, uint32_t tid) {
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
        for (uint32_t j = 0; j < 8; ++j)
#pragma unroll
            for (uint32_t i = 0; i < 2; ++i) {
                const uint32_t r = h * 64 + fragRow(tid, i);
                const __half2 v = __floats2half2_rn(fmaxf(acc[h][4 * j + 2 * i], 0.0f), fmaxf(acc[h][4 * j + 2 * i + 1], 0.0f));
                *reinterpret_cast<__half2*>(tile + j * (128 * 16) + r * 16 + (tid & 3u) * 4) = v;
            }
}

GFX_D void mbarInit(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smemU32(bar)), "r"(count) : "memory");
}
GFX_D void mbarWait(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n"
        :: "r"(smemU32(bar)), "r"(phase) : "memory");
}
GFX_D void fenceProxyAsync() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
GFX_D void bulkLoad(void* smemDst, const void* globalSrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smemU32(smemDst)), "l"(globalSrc), "r"(bytes), "r"(smemU32(bar)) : "memory");
}
GFX_D void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smemU32(bar)), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------------------------------------
// k_nrcPrepWeights: MLP weights W_l [out][in] -> per-layer K-major core-matrix blobs of W_l ([N x 64]):
//   byte offset(layer, n, k) = layerBase + (k / 8) * (N * 16) + n * 16 + (k % 8) * 2
// and, for training (blobT not null), of W_l^T ([64 x K], 64 rows per K-chunk)
// ---------------------------------------------------------------------------------------------
__global__ void k_nrcPrepWeights(const __half* __restrict__ w, uint32_t numHiddenLayers, __half* __restrict__ blob,
                                 __half* __restrict__ blobT) {
    const uint32_t total = numHiddenLayers * kWidth * kWidth + kPaddedOutput * kWidth;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        uint32_t layer = i / (kWidth * kWidth), rem = i % (kWidth * kWidth), N = kWidth;
        if (layer >= numHiddenLayers) {
            layer = numHiddenLayers;
            rem = i - numHiddenLayers * kWidth * kWidth;
            N = kPaddedOutput;
        }
        const uint32_t n = rem / kWidth, k = rem % kWidth;
        blob[layer * kWidth * kWidth + (k / 8) * (N * 8) + n * 8 + (k % 8)] = w[i];
        if (blobT)
            blobT[layer * kWidth * kWidth + (n / 8) * (kWidth * 8) + k * 8 + (n % 8)] = w[i];
    }
}

// ---------------------------------------------------------------------------------------------
// k_nrcInfer: fused encode + MLP on wgmma. 128 threads (one warpgroup), persistent over 128-query tiles.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kTileRows = 128;
constexpr uint32_t kATileBytes = kTileRows * kWidth * 2; // 16 KB: 8 K-chunks x 128 rows x 16 B

// query q encoded into row `row` of a [128 x 64] K-major tile (chunk c of 8 features at c * 2048 + row * 16), zeros past numData
template <uint32_t kEnc>
GFX_D void encodeTileRow(const NrcLevels &levels, const __half* __restrict__ table, const float* __restrict__ input, uint32_t q,
                         uint32_t numData, uint8_t* tile, uint32_t row) {
    if (q < numData) {
        nrcEncodeQuery<kEnc>(levels, table, input + (size_t)q * kInputDims, [&](uint32_t c, const __half* f) {
            *reinterpret_cast<uint4*>(tile + c * (kTileRows * 16) + row * 16) = packHalf8(f);
        });
    }
    else {
#pragma unroll
        for (uint32_t c = 0; c < 8; ++c)
            *reinterpret_cast<uint4*>(tile + c * (kTileRows * 16) + row * 16) = make_uint4(0, 0, 0, 0);
    }
}

// The MLP over one 128-row tile whose inputs are in sA (overwritten by the hidden activations): per hidden layer mlpLayer64
// and the ReLU epilogue, then the 16-wide output layer, whose accumulators go to out(acc)
template <typename Out>
GFX_D void mlpTile(uint8_t* sA, uint32_t wAddr, uint32_t numHiddenLayers, uint32_t tid, Out out) {
    const uint32_t aAddr = smemU32(sA);
    for (uint32_t layer = 0; layer <= numHiddenLayers; ++layer) {
        // make the generic-proxy writes of sA (and of the weights) visible to the tensor core
        fenceProxyAsync();
        __syncthreads();
        const uint32_t wLayer = wAddr + layer * kWidth * kWidth * 2;
        if (layer < numHiddenLayers) {
            float acc[2][32];
            mlpLayer64(acc, aAddr, kTileRows * 16, wLayer, kWidth / 16);
            __syncthreads(); // every warp's MMAs have read the A tile before it is overwritten
            storeReluTile(acc, sA, tid);
        }
        else {
            float acc[2][8];
            mlpLayer16(acc, aAddr, kTileRows * 16, wLayer);
            out(acc);
        }
    }
}

// the network outputs (columns 0..2) of the output layer's accumulators: write(tile row, column, value); they are held by
// lanes with l % 4 < 2
template <typename Write>
GFX_D void forEachOutput(const float (&acc)[2][8], uint32_t tid, Write write) {
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
        for (uint32_t i = 0; i < 2; ++i)
#pragma unroll
            for (uint32_t e = 0; e < 2; ++e) {
                const uint32_t r = h * 64 + fragRow(tid, i), c = fragCol(tid, 0) + e;
                if (c < kOutputDims)
                    write(r, c, acc[h][2 * i + e]);
            }
}

template <uint32_t kEnc>
__global__ void __launch_bounds__(128) k_nrcInfer(NrcLevels levels, const __half* __restrict__ table,
                                                  const uint4* __restrict__ ummaWeights, uint32_t numHiddenLayers,
                                                  const float* __restrict__ input, float* __restrict__ output,
                                                  uint32_t numDataImm, const uint32_t* __restrict__ numDataPtr) {
    // the batch size either comes with the launch or lives in device memory (NRC frame: W*H + #tiles, known
    // only on the device; the reference synchronises with the host for it)
    const uint32_t numData = numDataPtr ? *numDataPtr : numDataImm;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* sA = smem;                                    // activation tile (A operand)
    uint8_t* sW = smem + kATileBytes;                      // all weight blobs (B operands)

    const uint32_t tid = threadIdx.x;
    const uint32_t weightBytes = (numHiddenLayers * kWidth * kWidth + kPaddedOutput * kWidth) * 2;

    // resident weights (18 KB, once per persistent CTA): cooperative 16-byte copies
    for (uint32_t i = tid; i < weightBytes / 16; i += 128)
        reinterpret_cast<uint4*>(sW)[i] = __ldg(ummaWeights + i);

    const uint32_t wAddr = smemU32(sW);

    const uint32_t numTiles = (numData + kTileRows - 1) / kTileRows;
    for (uint32_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
        encodeTileRow<kEnc>(levels, table, input, tile * kTileRows + tid, numData, sA, tid);
        mlpTile(sA, wAddr, numHiddenLayers, tid, [&](const float (&acc)[2][8]) {
            // trim_and_cast_from: half output -> float
            forEachOutput(acc, tid, [&](uint32_t r, uint32_t c, float v) {
                const uint32_t row = tile * kTileRows + r;
                if (row < numData)
                    output[(size_t)row * kOutputDims + c] = __half2float(__float2half(v));
            });
        });
        // all warps are done with the A tile before the next tile overwrites it
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// Inference, split form (default): the hash grid is the part of the network that is bound by divergent gathers - 128 dependent
// 4-byte reads per query out of a 2 MB table, i.e. 128 L1 wavefronts, while the tensor cores sit almost idle.  One LEVEL of the
// table is only 128 KB, though (level 0: 16 KB), which fits in an H100 SM's shared memory (227 KB per block), where a 32-lane
// gather is a few clocks instead of tens.  So:
//   k_nrcPackPositions   positions of the [N][14] queries -> float4 stream (read once per level below);
//   k_nrcGridEncode      grid = 16 levels x R replicas, one CTA per SM: the CTA pulls ITS level's table into shared memory with
//                        cp.async.bulk (TMA) + mbarrier once, then streams its share of the queries through it: coalesced
//                        position read, 8 shared-memory gathers, trilinear blend in half exactly like kernel_grid
//                        (grid.h:132-255), coalesced half2 store into features[tile][level][row] (8 KB per 128-query tile);
//   k_nrcInferMlp        per 128-query tile: two TMA bulk copies bring the tile's queries (7 KB) and grid features (8 KB) into
//                        shared memory (double-buffered: the next tile is in flight), the threads add one-blob + identity and
//                        lay the A tile out in core matrices, wgmma runs the 64->64->...->16 MLP as above, and the
//                        radiance leaves through a TMA bulk store.
// The features are the same halves, bit for bit, as nrcEncode's (tests/test_gpu_nrc.py::test_split_encoding_is_bit_exact).
// ---------------------------------------------------------------------------------------------
__global__ void k_nrcPackPositions(const float* __restrict__ input, float4* __restrict__ positions, uint32_t numDataImm,
                                   const uint32_t* __restrict__ numDataPtr) {
    const uint32_t numData = numDataPtr ? *numDataPtr : numDataImm;
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < numData; q += gridDim.x * blockDim.x) {
        const float* in = input + (size_t)q * kInputDims;
        positions[q] = make_float4(in[0], in[1], in[2], 0.0f);
    }
}

constexpr uint32_t kEncodeThreads = 1024;
constexpr uint32_t kTileFeatureBytes = kLevels * 128 * 4; // 8 KB per 128-query tile: [level][row] half2

__global__ void __launch_bounds__(kEncodeThreads, 1) k_nrcGridEncode(NrcLevels levels, const __half* __restrict__ table,
                                                                      const float4* __restrict__ positions,
                                                                      __half2* __restrict__ features, uint32_t replicas,
                                                                      uint32_t numDataImm, const uint32_t* __restrict__ numDataPtr) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t numData = numDataPtr ? *numDataPtr : numDataImm;
    const uint32_t level = blockIdx.x / replicas, replica = blockIdx.x % replicas;
    const NrcLevel lv = levels.l[level];
    const uint32_t tableBytes = lv.hashmapSize * 4u;
    if (threadIdx.x == 0) {
        mbarInit(&bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbarExpectTx(&bar, tableBytes);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(table + (size_t)lv.offset * 2);
        for (uint32_t off = 0; off < tableBytes; off += 32768u)
            bulkLoad(smem + off, src + off, min(32768u, tableBytes - off), &bar);
    }
    __syncthreads();
    mbarWait(&bar, 0);
    __half2* grid = reinterpret_cast<__half2*>(smem);

    // Dense levels index x + y * res + z * res^2 with res a multiple of 16: the queries of a warp are consecutive pixels, whose
    // positions typically run along ONE grid axis, so along y or z all 32 lanes would hit the same shared-memory bank (the dense
    // levels' CTAs would take twice as long as the hashed ones' and set the kernel's duration).  Entries are therefore
    // permuted inside each aligned row of 32: entry i lives at i ^ swz(i >> 5), swz(r) = (r ^ (r >> 5)) & 31 - y and z
    // neighbours land in different banks.  Hashed levels are spread by the hash already.
    uint32_t mul[3];
    const bool swizzle = !nrcLevelMultipliers(lv, mul) && (lv.hashmapSize & 31u) == 0u;
    const uint32_t swzMask = swizzle ? 31u : 0u;
    if (swizzle) {
        const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, numRows = lv.hashmapSize >> 5;
        for (uint32_t row = warp; row < numRows; row += kEncodeThreads / 32) {
            const __half2 v = grid[row * 32 + lane];
            __syncwarp();
            grid[row * 32 + (lane ^ ((row ^ (row >> 5)) & 31u))] = v;
        }
        __syncthreads();
    }

    // this replica's share of the 128-query tiles
    const uint32_t numTiles = (numData + 127u) / 128u;
    const uint32_t tilesPer = (numTiles + replicas - 1) / replicas;
    const uint32_t qBegin = min(replica * tilesPer, numTiles) * 128u;
    const uint32_t qEnd = min(min((replica + 1) * tilesPer, numTiles) * 128u, numData);

    for (uint32_t q = qBegin + threadIdx.x; q < qEnd; q += kEncodeThreads) {
        const float4 p = __ldg(positions + q);
        const float in[3] = { p.x, p.y, p.z };
        const NrcCell cell(lv, in);
        __half2 r = __floats2half2_rn(0.0f, 0.0f);
#pragma unroll
        for (uint32_t idx = 0; idx < 8; ++idx) {
            const float weight = cell.weight(idx);
            uint32_t index = cell.entry(idx);
            index ^= ((index >> 5) ^ (index >> 10)) & swzMask;
            const float2 v = __half22float2(grid[index]);
            // result += (half)(weight * (float)value) in half precision (grid.h:233-238); __hadd2 rounds the exact sum once,
            // which equals the float-add-then-round-to-half the oracle spells out (the fp32 sum of two halves only rounds when
            // the smaller one is below a quarter ulp of the larger)
            r = __hadd2(r, __floats2half2_rn(weight * v.x, weight * v.y));
        }
        features[((size_t)(q >> 7) * kLevels + level) * 128u + (q & 127u)] = r;
    }
}

// queries of one tile and, for the hash grid, its grid features, landed by TMA
template <uint32_t kEnc> struct NrcTileStage {
    float query[128 * kInputDims];    // 7168 B
    __half2 feat[kLevels * 128];      // 8192 B
};
template <> struct NrcTileStage<kEncTriangleWave> { // the triangle wave is computed from the queries alone
    float query[128 * kInputDims];
};

// k_nrcInferMlp<kEncTriangleWave> is the whole triangle-wave inference: no grid stage in front of it, the thread that owns a row
// computes its 64 inputs from the staged query in registers.
template <uint32_t kEnc>
__global__ void __launch_bounds__(128) k_nrcInferMlp(const uint4* __restrict__ ummaWeights, uint32_t numHiddenLayers,
                                                     const float* __restrict__ input, const __half2* __restrict__ features,
                                                     float* __restrict__ output, uint32_t numDataImm,
                                                     const uint32_t* __restrict__ numDataPtr) {
    using Stage = NrcTileStage<kEnc>;
    const uint32_t numData = numDataPtr ? *numDataPtr : numDataImm;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* sA = smem;                                                        // activation tile (A operand), 16 KB
    Stage* stage = reinterpret_cast<Stage*>(smem + kATileBytes);               // 2 x 15 KB (triangle wave: 2 x 7 KB)
    float* sOut = reinterpret_cast<float*>(smem + kATileBytes + 2 * sizeof(Stage)); // 128 x 3 floats
    uint8_t* sW = smem + kATileBytes + 2 * sizeof(Stage) + 128 * kOutputDims * 4;   // weight blobs (B operands)
    __shared__ __align__(8) uint64_t stageBar[2];

    const uint32_t tid = threadIdx.x;
    const uint32_t weightBytes = (numHiddenLayers * kWidth * kWidth + kPaddedOutput * kWidth) * 2;
    const uint32_t numTiles = numData / kTileRows;

    auto requestTile = [&](uint32_t tile, uint32_t b) { // thread 0 only
        fenceProxyAsync();
        mbarExpectTx(&stageBar[b], (uint32_t)sizeof(Stage));
        bulkLoad(stage[b].query, input + (size_t)tile * 128 * kInputDims, 128 * kInputDims * 4, &stageBar[b]);
        if constexpr (kEnc == kEncHashGrid)
            bulkLoad(stage[b].feat, features + (size_t)tile * kLevels * 128, kTileFeatureBytes, &stageBar[b]);
    };

    if (tid == 0) {
        mbarInit(&stageBar[0], 1);
        mbarInit(&stageBar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (blockIdx.x < numTiles)
            requestTile(blockIdx.x, 0);
    }
    for (uint32_t i = tid; i < weightBytes / 16; i += 128)
        reinterpret_cast<uint4*>(sW)[i] = __ldg(ummaWeights + i);
    __syncthreads();

    const uint32_t wAddr = smemU32(sW);
    uint32_t stagePhase0 = 0, stagePhase1 = 0, buf = 0;

    for (uint32_t tile = blockIdx.x; tile < numTiles; tile += gridDim.x, buf ^= 1u) {
        // prefetch the next tile into the other buffer (every thread finished reading it one tile ago: the end-of-tile barrier)
        if (tid == 0 && tile + gridDim.x < numTiles)
            requestTile(tile + gridDim.x, buf ^ 1u);
        if (buf == 0) {
            mbarWait(&stageBar[0], stagePhase0);
            stagePhase0 ^= 1u;
        }
        else {
            mbarWait(&stageBar[1], stagePhase1);
            stagePhase1 ^= 1u;
        }
        const Stage &st = stage[buf];

        // ---- this thread's row of the A tile: chunk c (8 features = 16 B) at c * 2048 + row * 16
        if constexpr (kEnc == kEncTriangleWave) {
            float q[kInputDims];
#pragma unroll
            for (uint32_t d = 0; d < kInputDims; ++d)
                q[d] = st.query[tid * kInputDims + d];
            nrcEncodeTriWave(q, [&](uint32_t c, const __half* f) {
                *reinterpret_cast<uint4*>(sA + c * (kTileRows * 16) + tid * 16) = packHalf8(f);
            });
        }
        else {
#pragma unroll
            for (uint32_t c = 0; c < 4; ++c) { // hash grid: levels 4c .. 4c + 3
                uint4 v;
                v.x = *reinterpret_cast<const uint32_t*>(&st.feat[(4 * c + 0) * 128 + tid]);
                v.y = *reinterpret_cast<const uint32_t*>(&st.feat[(4 * c + 1) * 128 + tid]);
                v.z = *reinterpret_cast<const uint32_t*>(&st.feat[(4 * c + 2) * 128 + tid]);
                v.w = *reinterpret_cast<const uint32_t*>(&st.feat[(4 * c + 3) * 128 + tid]);
                *reinterpret_cast<uint4*>(sA + c * (kTileRows * 16) + tid * 16) = v;
            }
            float q[kInputDims];
            q[0] = q[1] = q[2] = 0.0f;
#pragma unroll
            for (uint32_t d = 3; d < kInputDims; ++d)
                q[d] = st.query[tid * kInputDims + d];
            __half tail[32];
            nrcEncodeTail(q, tail);
#pragma unroll
            for (uint32_t c = 0; c < 4; ++c)
                *reinterpret_cast<uint4*>(sA + (4 + c) * (kTileRows * 16) + tid * 16) = packHalf8(tail + 8 * c);
        }

        mlpTile(sA, wAddr, numHiddenLayers, tid, [&](const float (&acc)[2][8]) {
            // the previous tile's bulk store must have read sOut before it is overwritten
            if (tid == 0)
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            __syncthreads();
            // trim_and_cast_from: half output -> float
            forEachOutput(acc, tid, [&](uint32_t r, uint32_t c, float v) { sOut[r * kOutputDims + c] = __half2float(__float2half(v)); });
        });
        // all warps are done reading the A tile / the stage and writing sOut before the next tile overwrites them
        fenceProxyAsync();
        __syncthreads();
        if (tid == 0) { // radiance of the tile: one TMA bulk store of 1536 contiguous bytes
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         :: "l"(output + (size_t)tile * 128 * kOutputDims), "r"(smemU32(sOut)), "r"(128u * kOutputDims * 4u) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (tid == 0)
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// test hook: the 64 encoded halves per query as k_nrcInferMlp assembles them - hash grid: the features of pack -> grid encode,
// then the tail; triangle wave: nrcEncodeTriWave
template <uint32_t kEnc>
__global__ void k_nrcAssembleEncoding(const float* __restrict__ input, const __half2* __restrict__ features, uint32_t numData,
                                      __half* __restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= numData)
        return;
    __half* o = out + (size_t)q * 64;
    float qv[kInputDims];
    for (uint32_t d = 0; d < kInputDims; ++d)
        qv[d] = input[(size_t)q * kInputDims + d];
    if constexpr (kEnc == kEncHashGrid) {
        for (uint32_t l = 0; l < kLevels; ++l) {
            const __half2 v = features[((size_t)(q >> 7) * kLevels + l) * 128u + (q & 127u)];
            o[2 * l] = __low2half(v);
            o[2 * l + 1] = __high2half(v);
        }
        __half tail[32];
        nrcEncodeTail(qv, tail);
        for (uint32_t k = 0; k < 32; ++k)
            o[32 + k] = tail[k];
    }
    else {
        nrcEncodeTriWave(qv, [&](uint32_t c, const __half* f) {
            for (uint32_t e = 0; e < 8; ++e)
                o[c * 8 + e] = f[e];
        });
    }
}

// ---------------------------------------------------------------------------------------------
// training step on CUDA cores: block = 128 samples
// ---------------------------------------------------------------------------------------------
// deterministic gradient accumulation: 2^-30 fixed point in 64 bits (range +-8.6e9, resolution 9.3e-10 on loss-scaled values)
constexpr float kGradFixedScale = 1073741824.0f;
GFX_D void atomicAddFixed(unsigned long long* p, float v) {
    atomicAdd(p, (unsigned long long)__float2ll_rn(v * kGradFixedScale));
}
GFX_D float fixedToFloat(unsigned long long v) {
    return (float)((double)(long long)v * (1.0 / 1073741824.0));
}

// RelativeL2Luminance (relative_l2_luminance.h:41-88) of one sample with network output o[0..2]: returns its loss term and
// writes dL/dy, loss-scaled and fp16 like tiny-cuda-nn's backward buffers, to d[0..15] (zero for the padding and for invalid
// samples)
GFX_D float nrcRelativeL2Luminance(const __half* o, const float* __restrict__ target, bool valid, uint32_t numData, __half* d) {
    float loss = 0.0f;
    const uint32_t nTotal = numData * kOutputDims;
    const float r = __half2float(o[0]), g = __half2float(o[1]), b = __half2float(o[2]);
    const float luminance = 0.299f * r + 0.587f * g + 0.114f * b;
    const float denom = luminance * luminance + 0.01f;
#pragma unroll
    for (uint32_t k = 0; k < kPaddedOutput; ++k) {
        float gr = 0.0f;
        if (k < kOutputDims && valid) {
            const float difference = __half2float(o[k]) - target[k];
            loss += difference * difference / denom / nTotal;
            gr = kLossScale * (2 * difference / denom) / nTotal;
        }
        d[k] = __float2half(gr);
    }
    return loss;
}

// hash-grid backward (kernel_grid_backward, grid.h:306-429) of one sample at position in[0..2]: the gradients of the first 32
// network inputs, grad(2 l + e) for feature e of level l, scattered to the corners of each level's cell
template <typename Grad>
GFX_D void nrcGridBackward(const NrcLevels &levels, const float* __restrict__ in, Grad grad, unsigned long long* gGrid) {
    const float p[3] = { in[0], in[1], in[2] };
    for (uint32_t l = 0; l < kLevels; ++l) {
        const NrcLevel lv = levels.l[l];
        const float g0 = grad(l * 2 + 0), g1 = grad(l * 2 + 1);
        if (g0 == 0.0f && g1 == 0.0f)
            continue;
        const NrcCell cell(lv, p);
#pragma unroll
        for (uint32_t idx = 0; idx < 8; ++idx) {
            const float weight = cell.weight(idx);
            const uint32_t gi = lv.offset * 2 + cell.entry(idx) * 2;
            atomicAddFixed(gGrid + gi, weight * g0);
            atomicAddFixed(gGrid + gi + 1, weight * g1);
        }
    }
}

// the 128-thread block's loss terms, summed per warp and then over the 4 warps, added to *lossOut
GFX_D void nrcBlockLoss(float localLoss, float* lossOut) {
    __shared__ float sLoss[4];
    for (int off = 16; off > 0; off >>= 1)
        localLoss += __shfl_xor_sync(0xFFFFFFFFu, localLoss, off);
    if ((threadIdx.x & 31) == 0)
        sLoss[threadIdx.x >> 5] = localLoss;
    __syncthreads();
    if (threadIdx.x == 0)
        atomicAdd(lossOut, sLoss[0] + sLoss[1] + sLoss[2] + sLoss[3]);
}

constexpr uint32_t kRowStride = 66; // halves per activation row in shared memory (conflict-free rows)

// kEnc = kEncTriangleWave: the encoding has no parameters, so NetworkWithInputEncoding::backward asks for no input gradient
// (network_with_input_encoding.h:92-99): no data gradient through layer 0 and no encoding backward
template <uint32_t kEnc>
__global__ void __launch_bounds__(128) k_nrcTrain(NrcLevels levels, const __half* __restrict__ params, uint32_t numMatrixWeights,
                                                  uint32_t numHiddenLayers, const float* __restrict__ input,
                                                  const float* __restrict__ target, uint32_t numData,
                                                  unsigned long long* __restrict__ grads, float* __restrict__ lossOut) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t H = numHiddenLayers;
    __half* sW = reinterpret_cast<__half*>(smem);                              // numMatrixWeights
    __half* sAct = sW + numMatrixWeights;                                      // (H + 1) x 128 x kRowStride
    __half* sD = sAct + (size_t)(H + 1) * 128 * kRowStride;                    // 128 x kRowStride

    const uint32_t tid = threadIdx.x;
    const uint32_t q = blockIdx.x * 128 + tid;
    const bool valid = q < numData;
    for (uint32_t i = tid; i < numMatrixWeights; i += 128)
        sW[i] = params[i];
    const __half* table = params + numMatrixWeights;

    __half* x = sAct + (size_t)tid * kRowStride;
    if (valid) {
        nrcEncodeQuery<kEnc>(levels, table, input + (size_t)q * kInputDims, [&](uint32_t c, const __half* f) {
#pragma unroll
            for (uint32_t e = 0; e < 8; ++e)
                x[c * 8 + e] = f[e];
        });
    }
    else {
        for (uint32_t e = 0; e < 64; ++e)
            x[e] = __float2half(0.0f);
    }
    __syncthreads();

    // forward
    for (uint32_t layer = 0; layer < H; ++layer) {
        const __half* W = sW + (size_t)layer * kWidth * kWidth;
        const __half* in = sAct + ((size_t)layer * 128 + tid) * kRowStride;
        __half* out = sAct + ((size_t)(layer + 1) * 128 + tid) * kRowStride;
        for (uint32_t j = 0; j < kWidth; ++j) {
            float acc = 0.0f;
#pragma unroll 8
            for (uint32_t i = 0; i < kWidth; ++i)
                acc += __half2float(W[j * kWidth + i]) * __half2float(in[i]);
            out[j] = __float2half(fmaxf(acc, 0.0f));
        }
    }
    __half o[kPaddedOutput];
    {
        const __half* W = sW + (size_t)H * kWidth * kWidth;
        const __half* in = sAct + ((size_t)H * 128 + tid) * kRowStride;
        for (uint32_t j = 0; j < kPaddedOutput; ++j) {
            float acc = 0.0f;
#pragma unroll 8
            for (uint32_t i = 0; i < kWidth; ++i)
                acc += __half2float(W[j * kWidth + i]) * __half2float(in[i]);
            o[j] = __float2half(acc);
        }
    }
    __half* d = sD + (size_t)tid * kRowStride;
    const float localLoss = nrcRelativeL2Luminance(o, target + (size_t)q * kOutputDims, valid, numData, d);
    __syncthreads();

    // output layer: dW, then dL/d(hidden)
    {
        const uint32_t base = H * kWidth * kWidth;
        const __half* hin = sAct + (size_t)H * 128 * kRowStride;
        for (uint32_t p = tid; p < kPaddedOutput * kWidth; p += 128) {
            const uint32_t j = p / kWidth, i = p % kWidth;
            float acc = 0.0f;
            for (uint32_t s = 0; s < 128; ++s)
                acc += __half2float(sD[s * kRowStride + j]) * __half2float(hin[s * kRowStride + i]);
            if (acc != 0.0f)
                atomicAddFixed(grads + base + p, acc);
        }
        const __half* W = sW + (size_t)H * kWidth * kWidth;
        const __half* myIn = hin + (size_t)tid * kRowStride;
        __half dNext[64];
        for (uint32_t i = 0; i < kWidth; ++i) {
            float acc = 0.0f;
#pragma unroll
            for (uint32_t j = 0; j < kPaddedOutput; ++j)
                acc += __half2float(W[j * kWidth + i]) * __half2float(d[j]);
            dNext[i] = (H > 0 && !(__half2float(myIn[i]) > 0.0f)) ? __float2half(0.0f) : __float2half(acc);
        }
        __syncthreads();
        for (uint32_t i = 0; i < kWidth; ++i)
            d[i] = dNext[i];
        __syncthreads();
    }
    for (int layer = (int)H - 1; layer >= 0; --layer) {
        const uint32_t base = (uint32_t)layer * kWidth * kWidth;
        const __half* hin = sAct + (size_t)layer * 128 * kRowStride;
        for (uint32_t p = tid; p < kWidth * kWidth; p += 128) {
            const uint32_t j = p / kWidth, i = p % kWidth;
            float acc = 0.0f;
            for (uint32_t s = 0; s < 128; ++s)
                acc += __half2float(sD[s * kRowStride + j]) * __half2float(hin[s * kRowStride + i]);
            if (acc != 0.0f)
                atomicAddFixed(grads + base + p, acc);
        }
        if (kEnc == kEncTriangleWave && layer == 0)
            break;
        const __half* W = sW + (size_t)layer * kWidth * kWidth;
        const __half* myIn = hin + (size_t)tid * kRowStride;
        __half dNext[64];
        for (uint32_t i = 0; i < kWidth; ++i) {
            float acc = 0.0f;
            for (uint32_t j = 0; j < kWidth; ++j)
                acc += __half2float(W[j * kWidth + i]) * __half2float(d[j]);
            dNext[i] = (layer > 0 && !(__half2float(myIn[i]) > 0.0f)) ? __float2half(0.0f) : __float2half(acc);
        }
        __syncthreads();
        for (uint32_t i = 0; i < kWidth; ++i)
            d[i] = dNext[i];
        __syncthreads();
    }

    // the first 32 input gradients, to the hash grid
    if (kEnc == kEncHashGrid && valid)
        nrcGridBackward(levels, input + (size_t)q * kInputDims, [&](uint32_t k) { return __half2float(d[k]); },
                        grads + numMatrixWeights);
    nrcBlockLoss(localLoss, lossOut);
}

// ---------------------------------------------------------------------------------------------
// k_nrcTrainTc: the same training step with every matrix product on wgmma (forward, data gradients, weight gradients).
//
// Per CTA = 128 samples (kernel_mlp_fused + kernel_mlp_fused_backward of tiny-cuda-nn work on the same 128-row chunks,
// ext/tiny-cuda-nn/src/fully_fused_mlp.cu:47-129, 150-259; the weight gradients are its three split-K CUTLASS GEMMs,
// :822-873).  All operands are K-major core-matrix tiles in shared memory:
//   forward        Z_l     [128 x N]  = A_l [128 x 64]            x W_l^T   (B = W_l blob  [N x 64],  as in k_nrcInfer)
//   data gradient  dA_l    [128 x 64] = dZ_l [128 x K]            x W_l     (B = W_l^T blob [64 x K], K = 64 or 16)
//   weight grad    dW_l    [K x 64]   = dZ_l^T [K(<=64) x 128]    x A_l     (A = transposed dZ tile, B = transposed A_l tile,
//                                                                            K = 128 samples; one M = 64 MMA per K step,
//                                                                            rows >= K of the accumulator are ignored)
// dZ_l lives in the sDz tile; each thread copies its own sample's rows of dZ_l and A_l into the transposed tiles.  The
// accumulators are wgmma register fragments, so the network output and the data gradient go back through shared memory to the
// rows they belong to.  Rounding points match k_nrcTrain (activations and gradients are fp16 between layers, fp32
// accumulation inside).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kTTileBytes = 64 * 128 * 2; // transposed tile: 16 K-chunks x 64 rows x 16 B

// element (row, k) of a [128 x 64] K-major tile
GFX_D __half tileHalf(const uint8_t* tile, uint32_t row, uint32_t k) {
    return *reinterpret_cast<const __half*>(tile + (k / 8) * (kTileRows * 16) + row * 16 + (k % 8) * 2);
}

template <uint32_t kEnc> // as k_nrcTrain: the triangle wave skips layer 0's data gradient and the encoding backward
__global__ void __launch_bounds__(128) k_nrcTrainTc(NrcLevels levels, const __half* __restrict__ params, uint32_t numMatrixWeights,
                                                    uint32_t numHiddenLayers, const uint4* __restrict__ blobFwd,
                                                    const uint4* __restrict__ blobT, const float* __restrict__ input,
                                                    const float* __restrict__ target, uint32_t numData,
                                                    unsigned long long* __restrict__ grads, float* __restrict__ lossOut) {
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t H = numHiddenLayers;
    const uint32_t weightBytes = numMatrixWeights * 2;
    uint8_t* sWf = smem;                                   // forward blobs
    uint8_t* sWt = sWf + weightBytes;                      // transposed blobs
    uint8_t* sAct = sWt + weightBytes;                     // (H + 1) activation tiles A_0..A_H, 16 KB each
    uint8_t* sDz = sAct + (H + 1) * kATileBytes;           // dZ tile [128 x 64] (K-major, rows = samples)
    uint8_t* sDzT = sDz + kATileBytes;                     // dZ^T tile [64 x 128] (rows = neurons, K = samples)
    uint8_t* sActT = sDzT + kTTileBytes;                   // A_l^T tile [64 x 128]
    __shared__ __align__(8) uint64_t weightBar;

    const uint32_t tid = threadIdx.x;
    const uint32_t q = blockIdx.x * 128 + tid;
    const bool valid = q < numData;

    if (tid == 0) {
        mbarInit(&weightBar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbarExpectTx(&weightBar, 2 * weightBytes);
        bulkLoad(sWf, blobFwd, weightBytes, &weightBar);
        bulkLoad(sWt, blobT, weightBytes, &weightBar);
    }

    encodeTileRow<kEnc>(levels, params + numMatrixWeights, input, q, numData, sAct, tid); // this thread's sample into A_0
    fenceProxyAsync();
    __syncthreads();
    mbarWait(&weightBar, 0);

    // ---- forward
    for (uint32_t layer = 0; layer < H; ++layer) {
        float acc[2][32];
        mlpLayer64(acc, smemU32(sAct + layer * kATileBytes), kTileRows * 16, smemU32(sWf) + layer * kWidth * kWidth * 2, kWidth / 16);
        storeReluTile(acc, sAct + (layer + 1) * kATileBytes, tid);
        fenceProxyAsync();
        __syncthreads();
    }
    float* sOutF = reinterpret_cast<float*>(sDzT); // [128][4]: the network output, back to the thread that owns the sample
    {
        float acc[2][8];
        mlpLayer16(acc, smemU32(sAct + H * kATileBytes), kTileRows * 16, smemU32(sWf) + H * kWidth * kWidth * 2);
        forEachOutput(acc, tid, [&](uint32_t r, uint32_t c, float v) { sOutF[r * 4 + c] = v; });
        __syncthreads();
    }

    // ---- loss + dL/dy -> this sample's row of dZ_H
    float localLoss;
    {
        const __half o[3] = { __float2half(sOutF[tid * 4 + 0]), __float2half(sOutF[tid * 4 + 1]), __float2half(sOutF[tid * 4 + 2]) };
        __half d[kPaddedOutput];
        localLoss = nrcRelativeL2Luminance(o, target + (size_t)q * kOutputDims, valid, numData, d);
#pragma unroll
        for (uint32_t c = 0; c < kPaddedOutput / 8; ++c)
            *reinterpret_cast<uint4*>(sDz + c * (kTileRows * 16) + tid * 16) = packHalf8(d + 8 * c);
    }
    __syncthreads(); // every thread has read its output row before sDzT is overwritten

    // ---- backward, layer H (output, K = 16) down to 0
    for (int layer = (int)H; layer >= 0; --layer) {
        const uint32_t K = layer == (int)H ? kPaddedOutput : kWidth; // width of dZ_l
        const uint8_t* aTile = sAct + layer * kATileBytes;
        // this sample's rows of dZ_l and A_l -> column tid of the transposed tiles ([64 x 128] K-major: element (row j, k = tid))
        {
            __half* dzT = reinterpret_cast<__half*>(sDzT + (tid / 8) * (64 * 16) + (tid % 8) * 2);
            __half* aT = reinterpret_cast<__half*>(sActT + (tid / 8) * (64 * 16) + (tid % 8) * 2);
#pragma unroll
            for (uint32_t c = 0; c < 8; ++c) {
                const uint4 v = *reinterpret_cast<const uint4*>(aTile + c * (kTileRows * 16) + tid * 16);
                const uint32_t w4[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (uint32_t e = 0; e < 4; ++e) {
                    aT[(c * 8 + 2 * e) * 8] = __ushort_as_half((unsigned short)(w4[e] & 0xFFFFu));
                    aT[(c * 8 + 2 * e + 1) * 8] = __ushort_as_half((unsigned short)(w4[e] >> 16));
                }
                if (c < K / 8) {
                    const uint4 g = *reinterpret_cast<const uint4*>(sDz + c * (kTileRows * 16) + tid * 16);
                    const uint32_t g4[4] = { g.x, g.y, g.z, g.w };
#pragma unroll
                    for (uint32_t e = 0; e < 4; ++e) {
                        dzT[(c * 8 + 2 * e) * 8] = __ushort_as_half((unsigned short)(g4[e] & 0xFFFFu));
                        dzT[(c * 8 + 2 * e + 1) * 8] = __ushort_as_half((unsigned short)(g4[e] >> 16));
                    }
                }
            }
        }
        fenceProxyAsync();
        __syncthreads();

        // weight gradient dW_l = dZ_l^T x A_l (K = 128 samples) -> fixed-point global accumulation of rows 0..K-1
        {
            float accW[32];
            wgmmaFence();
#pragma unroll
            for (uint32_t k = 0; k < kTileRows / 16; ++k)
                wgmma64(accW, makeSmemDesc(smemU32(sDzT) + 2 * k * (64 * 16), 64 * 16, 128),
                        makeSmemDesc(smemU32(sActT) + 2 * k * (64 * 16), 64 * 16, 128), k > 0 ? 1u : 0u);
            wgmmaCommit();
            wgmmaWait();
            fenceAccumulators(accW);
            const uint32_t base = (uint32_t)layer * kWidth * kWidth;
#pragma unroll
            for (uint32_t j = 0; j < 8; ++j)
#pragma unroll
                for (uint32_t i = 0; i < 2; ++i)
#pragma unroll
                    for (uint32_t e = 0; e < 2; ++e) {
                        const uint32_t r = fragRow(tid, i), c = fragCol(tid, j) + e;
                        const float g = accW[4 * j + 2 * i + e];
                        if (r < K && g != 0.0f)
                            atomicAddFixed(grads + base + r * kWidth + c, g);
                    }
        }
        if (kEnc == kEncTriangleWave && layer == 0)
            break;
        // data gradient dA_l = dZ_l x W_l (K steps of 16 over dZ's width) -> dZ_{l-1} (ReLU mask of A_l = relu(Z_{l-1})), or
        // the encoder gradient for layer 0, written over dZ_l
        {
            float accA[2][32];
            mlpLayer64(accA, smemU32(sDz), kTileRows * 16, smemU32(sWt) + layer * kWidth * kWidth * 2, K / 16);
            __syncthreads(); // every warp's MMAs have read dZ_l before it is overwritten
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h)
#pragma unroll
                for (uint32_t j = 0; j < 8; ++j)
#pragma unroll
                    for (uint32_t i = 0; i < 2; ++i) {
                        const uint32_t off = j * (kTileRows * 16) + (h * 64 + fragRow(tid, i)) * 16 + (tid & 3u) * 4;
                        const float2 act = __half22float2(*reinterpret_cast<const __half2*>(aTile + off));
                        const float g0 = (layer > 0 && !(act.x > 0.0f)) ? 0.0f : accA[h][4 * j + 2 * i];
                        const float g1 = (layer > 0 && !(act.y > 0.0f)) ? 0.0f : accA[h][4 * j + 2 * i + 1];
                        *reinterpret_cast<__half2*>(sDz + off) = __floats2half2_rn(g0, g1);
                    }
        }
        __syncthreads(); // dZ_{l-1} is complete
    }

    // ---- the first 32 input gradients (this sample's row of the dZ tile), to the hash grid
    if (kEnc == kEncHashGrid && valid)
        nrcGridBackward(levels, input + (size_t)q * kInputDims, [&](uint32_t k) { return __half2float(tileHalf(sDz, tid, k)); },
                        grads + numMatrixWeights);
    nrcBlockLoss(localLoss, lossOut);
}

// adam_step (adam.h:49-115) + ema_step_half_precision (ema.h:61-77); clears the gradient for the next step
__global__ void k_nrcAdamEma(uint32_t numParams, uint32_t numMatrixWeights, float learningRate, float epsilon, float emaDebiasOld,
                             float emaDebiasNew, unsigned long long* __restrict__ grads, float* __restrict__ master,
                             __half* __restrict__ params, __half* __restrict__ paramsEma, float* __restrict__ m1,
                             float* __restrict__ m2, uint32_t* __restrict__ steps) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= numParams)
        return;
    const float beta1 = 0.9f, beta2 = 0.99f, l2Reg = 1e-6f, emaDecay = 0.99f;
    float gradient = __half2float(__float2half(fixedToFloat(grads[i]))) / kLossScale;
    grads[i] = 0ull;
    const bool matrix = i < numMatrixWeights;
    if (matrix || gradient != 0) {
        const float weightFp = master[i];
        if (matrix)
            gradient += l2Reg * weightFp;
        const float gradientSq = gradient * gradient;
        const float firstMoment = m1[i] = beta1 * m1[i] + (1 - beta1) * gradient;
        const float secondMoment = m2[i] = beta2 * m2[i] + (1 - beta2) * gradientSq;
        float lr = learningRate;
        const uint32_t currentStep = ++steps[i];
        lr *= sqrtf(1 - powf(beta2, (float)currentStep)) / (1 - powf(beta1, (float)currentStep));
        const float effectiveLr = fminf(fmaxf(lr / (sqrtf(secondMoment) + epsilon), 0.0f), 3.402823466e+38f);
        const float newWeight = weightFp - effectiveLr * firstMoment;
        master[i] = newWeight;
        params[i] = __float2half(newWeight);
    }
    const float filtered = (__half2float(paramsEma[i]) * emaDecay * emaDebiasOld + __half2float(params[i]) * (1 - emaDecay)) * emaDebiasNew;
    paramsEma[i] = __float2half(filtered);
}

// gfx_nrc_keep_gradients: the gradients k_nrcAdamEma is about to consume, as the half values tiny-cuda-nn would hold
// (loss-scaled by 128), widened to float
__global__ void k_nrcKeepGradients(uint32_t n, const unsigned long long* __restrict__ grads, float* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        dst[i] = __half2float(__float2half(fixedToFloat(grads[i])));
}

__global__ void k_nrcFloatToHalf(uint32_t n, const float* __restrict__ src, __half* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        dst[i] = __float2half(src[i]);
}

__global__ void k_nrcHalfToFloat(uint32_t n, const __half* __restrict__ src, float* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        dst[i] = __half2float(src[i]);
}

static void setupLevels(gfx_nrc* n) { // grid.h:885-922
    uint32_t offset = 0;
    for (uint32_t l = 0; l < kLevels; ++l) {
        const float scale = exp2f(l * log2f(2.0f)) * kBaseResolution - 1.0f;
        const uint32_t resolution = (uint32_t)ceilf(scale) + 1;
        const double dense = pow((double)resolution, 3.0);
        uint32_t paramsInLevel = dense > (double)(0xFFFFFFFFu / 2) ? 0xFFFFFFFFu / 2 : resolution * resolution * resolution;
        paramsInLevel = (paramsInLevel + 7u) / 8u * 8u;
        paramsInLevel = paramsInLevel < (1u << kLog2HashmapSize) ? paramsInLevel : (1u << kLog2HashmapSize);
        n->levels.l[l] = NrcLevel{ offset, paramsInLevel, scale, resolution };
        offset += paramsInLevel;
    }
    n->numMatrixWeights = kWidth * kWidth * n->numHiddenLayers + kPaddedOutput * kWidth;
    // the triangle-wave encoding has no parameters (triangle_wave.h: n_params() == 0)
    n->numParams = n->numMatrixWeights + (n->positionEncoding == GFX_NRC_POSITION_ENCODING_HASH_GRID ? offset * 2 : 0u);
}

// tiny-cuda-nn's pcg32 (dependencies/pcg32/pcg32.h:46-116): 64-bit LCG, XSH-RR output
struct Pcg32 {
    uint64_t state, inc;
    explicit Pcg32(uint64_t initstate, uint64_t initseq = 1u) {
        state = 0u;
        inc = (initseq << 1u) | 1u;
        nextUint();
        state += initstate;
        nextUint();
    }
    uint32_t nextUint() {
        const uint64_t oldstate = state;
        state = oldstate * 0x5851f42d4c957f2dULL + inc;
        const uint32_t xorshifted = (uint32_t)(((oldstate >> 18u) ^ oldstate) >> 27u);
        const uint32_t rot = (uint32_t)(oldstate >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31));
    }
    float nextFloat() {
        union { uint32_t u; float f; } x;
        x.u = (nextUint() >> 9) | 0x3f800000u;
        return x.f - 1.0f;
    }
};

// The parameters a freshly constructed tcnn::Trainer holds (trainer.h:54-60, 72-109): rng = pcg32{seed_seq{seed}[0]};
// NetworkWithInputEncoding::initialize_params (network_with_input_encoding.h:133-156) initialises the network first -
// FullyFusedMLP: every weight matrix Xavier-uniform on the host, next_float() * 2 * scale - scale with
// scale = sqrt(6 / (fan_in + fan_out)) (fully_fused_mlp.cu:922-949, gpu_matrix.h:292-307) - then the encoding: the hash grid
// U(-1e-4, 1e-4) by generate_random_uniform (grid.h:1267-1272, random.h:65-100), a kernel in which thread i jumps the stream
// ahead by 4 i and writes elements i, i + T, i + 2T, i + 3T (T = total threads) with val * (upper - lower) + lower, one FMA
// under nvcc's default contraction.  One-blob, identity and the triangle wave have no parameters: for a triangle-wave network
// numParams == numMatrixWeights and nothing is drawn after the matrices.
static void tcnnInitialParams(uint32_t seed, uint32_t numHiddenLayers, uint32_t numMatrixWeights, uint32_t numParams,
                              std::vector<float>* master) {
    std::seed_seq seq{ seed };
    std::vector<uint32_t> seeds(2);
    seq.generate(seeds.begin(), seeds.end());
    Pcg32 rng(seeds.front());
    master->assign(numParams, 0.0f);
    size_t pos = 0;
    for (uint32_t m = 0; m <= numHiddenLayers; ++m) {
        const uint32_t rows = m == numHiddenLayers ? kPaddedOutput : kWidth, cols = kWidth; // fan_out = rows, fan_in = cols
        const float scale = 1.0f * std::sqrt(6.0f / (float)(cols + rows));
        for (uint32_t i = 0; i < rows * cols; ++i)
            (*master)[pos++] = rng.nextFloat() * 2.0f * scale - scale;
    }
    const size_t n = numParams - numMatrixWeights;
    if (n == 0) // no encoding parameters: no generate_random_uniform
        return;
    const size_t threadsNeeded = (n + 3) / 4;
    const size_t totalThreads = (threadsNeeded + 127) / 128 * 128; // n_blocks_linear(n_threads) * n_threads_linear
    std::vector<float> stream(totalThreads * 4);
    for (float &f : stream)
        f = rng.nextFloat();
    const float upper = 1e-4f, lower = -1e-4f;
    for (size_t i = 0; i < totalThreads; ++i)
        for (size_t j = 0; j < 4; ++j) {
            const size_t idx = i + totalThreads * j;
            if (idx >= n)
                break;
            (*master)[numMatrixWeights + idx] = fmaf(stream[i * 4 + j], upper - lower, lower);
        }
}

// Dynamic shared memory of the kernels whose footprint grows with the depth: the launches request these sizes, and
// gfx_nrc_create rejects a depth for which one of them exceeds the device's per-block limit.
constexpr uint32_t kMaxTcTrainHiddenLayers = 3; // deeper networks train on k_nrcTrain
static size_t nrcInferFusedSmem(uint32_t numMatrixWeights) { return kATileBytes + (size_t)numMatrixWeights * 2; }
template <uint32_t kEnc>
static size_t nrcInferMlpSmem(uint32_t numMatrixWeights) {
    return kATileBytes + 2 * sizeof(NrcTileStage<kEnc>) + 128 * kOutputDims * 4 + (size_t)numMatrixWeights * 2;
}
static size_t nrcTrainTcSmem(uint32_t numMatrixWeights, uint32_t numHiddenLayers) {
    return (size_t)numMatrixWeights * 4 + (size_t)(numHiddenLayers + 1) * kATileBytes + 3 * (size_t)kATileBytes;
}
static size_t nrcTrainSmem(uint32_t numMatrixWeights, uint32_t numHiddenLayers) {
    return ((size_t)numMatrixWeights + (size_t)(numHiddenLayers + 2) * 128 * kRowStride) * 2;
}

} // namespace gfx

using namespace gfx;

struct NrcKernelSmem { const void* kernel; const char* name; size_t dynamicBytes; };
template <uint32_t kEnc>
static void nrcKernelSmem(uint32_t M, uint32_t H, NrcKernelSmem (&kernels)[4]) {
    kernels[0] = { (const void*)k_nrcInfer<kEnc>, "k_nrcInfer", nrcInferFusedSmem(M) };
    kernels[1] = { (const void*)k_nrcInferMlp<kEnc>, "k_nrcInferMlp", nrcInferMlpSmem<kEnc>(M) };
    kernels[2] = { (const void*)k_nrcTrainTc<kEnc>, "k_nrcTrainTc", H <= kMaxTcTrainHiddenLayers ? nrcTrainTcSmem(M, H) : 0 };
    kernels[3] = { (const void*)k_nrcTrain<kEnc>, "k_nrcTrain", nrcTrainSmem(M, H) };
}

// every kernel that can train or infer a network of this depth and encoding fits in one block's shared memory (dynamic + static)
static int nrcCheckSharedMemory(gfx_ctx* ctx, const gfx_nrc* n) {
    int limit = 0;
    GFX_CUDA(ctx, cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    const uint32_t M = n->numMatrixWeights, H = n->numHiddenLayers;
    NrcKernelSmem kernels[4];
    if (n->positionEncoding == GFX_NRC_POSITION_ENCODING_HASH_GRID)
        nrcKernelSmem<kEncHashGrid>(M, H, kernels);
    else
        nrcKernelSmem<kEncTriangleWave>(M, H, kernels);
    for (const auto &k : kernels) {
        cudaFuncAttributes attr;
        GFX_CUDA(ctx, cudaFuncGetAttributes(&attr, k.kernel));
        const size_t need = k.dynamicBytes + attr.sharedSizeBytes;
        if (need > (size_t)limit) {
            char msg[256];
            snprintf(msg, sizeof(msg), "gfx_nrc_create: %u hidden layers need %zu bytes of shared memory per block in %s, "
                     "more than the device's limit of %d bytes", H, need, k.name, limit);
            ctx->setError(msg);
            return GFX_ERR_UNSUPPORTED;
        }
    }
    return GFX_OK;
}

#define NRC_CUDA(nrc, call) GFX_CUDA((nrc)->ctx, call)

extern "C" {

int gfx_nrc_train(gfx_nrc* n, void* stream, const float* inputData, const float* targetData, uint32_t numData, float* lossOnHost);
int gfx_nrc_reset(gfx_nrc* n, uint32_t seed);
void gfx_nrc_destroy(gfx_nrc* n);

int gfx_nrc_create(gfx_ctx* ctx, uint32_t numHiddenLayers, float learningRate, gfx_nrc** out) {
    return gfx_nrc_create_with_encoding(ctx, GFX_NRC_POSITION_ENCODING_HASH_GRID, numHiddenLayers, learningRate, out);
}

int gfx_nrc_create_with_encoding(gfx_ctx* ctx, int positionEncoding, uint32_t numHiddenLayers, float learningRate,
                                 gfx_nrc** out) {
    if (!ctx || !out)
        return GFX_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (positionEncoding != GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE && positionEncoding != GFX_NRC_POSITION_ENCODING_HASH_GRID) {
        ctx->setError("gfx_nrc_create: positionEncoding must be GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE or _HASH_GRID");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    if (numHiddenLayers < 1 || numHiddenLayers > 8) {
        ctx->setError("gfx_nrc_create: numHiddenLayers must be in 1..8");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    GFX_CUDA(ctx, cudaSetDevice(ctx->device));
    gfx_nrc* n = new gfx_nrc();
    n->ctx = ctx;
    n->positionEncoding = positionEncoding;
    n->numHiddenLayers = numHiddenLayers;
    n->learningRate = learningRate;
    n->adamEpsilon = positionEncoding == GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE ? 1e-8f : 1e-15f;
    setupLevels(n);
    const int fits = nrcCheckSharedMemory(ctx, n);
    if (fits != GFX_OK) {
        delete n;
        return fits;
    }
    const size_t P = n->numParams;
    GFX_CUDA(ctx, cudaMalloc(&n->params, P * 2));
    GFX_CUDA(ctx, cudaMalloc(&n->paramsEma, P * 2));
    GFX_CUDA(ctx, cudaMalloc(&n->master, P * 4));
    GFX_CUDA(ctx, cudaMalloc(&n->m1, P * 4));
    GFX_CUDA(ctx, cudaMalloc(&n->m2, P * 4));
    GFX_CUDA(ctx, cudaMalloc(&n->steps, P * 4));
    GFX_CUDA(ctx, cudaMalloc(&n->grads, P * 8));
    GFX_CUDA(ctx, cudaMalloc(&n->loss, 16));
    GFX_CUDA(ctx, cudaMalloc(&n->ummaWeights, (size_t)n->numMatrixWeights * 2));
    GFX_CUDA(ctx, cudaMalloc(&n->trainBlobFwd, (size_t)n->numMatrixWeights * 2));
    GFX_CUDA(ctx, cudaMalloc(&n->trainBlobT, (size_t)n->numMatrixWeights * 2));
    GFX_CUDA(ctx, cudaMemset(n->params, 0, P * 2));
    GFX_CUDA(ctx, cudaMemset(n->paramsEma, 0, P * 2));
    GFX_CUDA(ctx, cudaMemset(n->master, 0, P * 4));
    GFX_CUDA(ctx, cudaMemset(n->m1, 0, P * 4));
    GFX_CUDA(ctx, cudaMemset(n->m2, 0, P * 4));
    GFX_CUDA(ctx, cudaMemset(n->steps, 0, P * 4));
    GFX_CUDA(ctx, cudaMemset(n->grads, 0, P * 8));
    const int rc = gfx_nrc_reset(n, 1337u); // tcnn::Trainer's default seed: a fresh cache equals the reference's fresh cache
    if (rc != GFX_OK) {
        gfx_nrc_destroy(n);
        return rc;
    }
    *out = n;
    return GFX_OK;
}

int gfx_nrc_reset(gfx_nrc* n, uint32_t seed) {
    if (!n)
        return GFX_ERR_INVALID_ARGUMENT;
    const size_t P = n->numParams;
    std::vector<float> master;
    tcnnInitialParams(seed, n->numHiddenLayers, n->numMatrixWeights, n->numParams, &master);
    NRC_CUDA(n, cudaMemcpy(n->master, master.data(), P * 4, cudaMemcpyHostToDevice));
    k_nrcFloatToHalf<<<(n->numParams + 255) / 256, 256>>>(n->numParams, n->master, n->params); // trainer.h:104-107
    n->ctx->launches++;
    NRC_CUDA(n, cudaMemset(n->paramsEma, 0, P * 2)); // EmaOptimizer::allocate zeroes the inference weights (ema.h:88-100)
    NRC_CUDA(n, cudaMemset(n->m1, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->m2, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->steps, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->grads, 0, P * 8));
    n->globalStep = 0;
    n->ummaDirty = true;
    NRC_CUDA(n, cudaDeviceSynchronize());
    return GFX_OK;
}

int gfx_nrc_keep_gradients(gfx_nrc* n, int on) {
    if (!n)
        return GFX_ERR_INVALID_ARGUMENT;
    if (on && !n->gradsFloat)
        NRC_CUDA(n, cudaMalloc(&n->gradsFloat, (size_t)n->numParams * 4));
    n->keepGradients = on != 0;
    return GFX_OK;
}

int gfx_nrc_read(gfx_nrc* n, int which, void* hostOut, size_t bytes) {
    if (!n || !hostOut)
        return GFX_ERR_INVALID_ARGUMENT;
    const size_t P = n->numParams;
    const void* src = nullptr;
    size_t need = P * 2;
    switch (which) {
    case GFX_NRC_READ_MASTER: src = n->master; need = P * 4; break;
    case GFX_NRC_READ_TRAINING: src = n->params; break;
    case GFX_NRC_READ_INFERENCE: src = n->paramsEma; break;
    case GFX_NRC_READ_GRADIENTS: src = n->gradsFloat; need = P * 4; break;
    default: return GFX_ERR_INVALID_ARGUMENT;
    }
    if (!src)
        return GFX_ERR_NOT_READY;
    if (bytes != need)
        return GFX_ERR_INVALID_ARGUMENT;
    NRC_CUDA(n, cudaDeviceSynchronize());
    NRC_CUDA(n, cudaMemcpy(hostOut, src, need, cudaMemcpyDeviceToHost));
    return GFX_OK;
}

void gfx_nrc_destroy(gfx_nrc* n) {
    if (!n)
        return;
    cudaFree(n->params); cudaFree(n->paramsEma); cudaFree(n->master); cudaFree(n->m1); cudaFree(n->m2);
    cudaFree(n->steps); cudaFree(n->grads); cudaFree(n->loss); cudaFree(n->ummaWeights); cudaFree(n->trainBlobFwd); cudaFree(n->trainBlobT); cudaFree(n->gradsFloat); cudaFree(n->positions); cudaFree(n->features);
    delete n;
}

uint32_t gfx_nrc_num_params(gfx_nrc* n) { return n ? n->numParams : 0; }

int gfx_nrc_set_params(gfx_nrc* n, const void* hostHalfParams, size_t bytes) {
    if (!n || !hostHalfParams || bytes != (size_t)n->numParams * 2)
        return GFX_ERR_INVALID_ARGUMENT;
    const size_t P = n->numParams;
    NRC_CUDA(n, cudaMemcpy(n->params, hostHalfParams, bytes, cudaMemcpyHostToDevice));
    NRC_CUDA(n, cudaMemcpy(n->paramsEma, n->params, bytes, cudaMemcpyDeviceToDevice));
    k_nrcHalfToFloat<<<(n->numParams + 255) / 256, 256>>>(n->numParams, n->params, n->master);
    n->ctx->launches++;
    NRC_CUDA(n, cudaMemset(n->m1, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->m2, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->steps, 0, P * 4));
    NRC_CUDA(n, cudaMemset(n->grads, 0, P * 8));
    n->globalStep = 0;
    n->ummaDirty = true;
    NRC_CUDA(n, cudaDeviceSynchronize());
    return GFX_OK;
}

int gfx_nrc_get_params(gfx_nrc* n, void* hostHalfParams, size_t bytes) {
    if (!n || !hostHalfParams || bytes != (size_t)n->numParams * 2)
        return GFX_ERR_INVALID_ARGUMENT;
    NRC_CUDA(n, cudaMemcpy(hostHalfParams, n->paramsEma, bytes, cudaMemcpyDeviceToHost));
    return GFX_OK;
}

static int nrcEnsureScratch(gfx_nrc* n, uint32_t numQueries) {
    if (numQueries <= n->scratchQueries)
        return GFX_OK;
    cudaFree(n->positions);
    cudaFree(n->features);
    n->positions = nullptr;
    n->features = nullptr;
    n->scratchQueries = 0;
    NRC_CUDA(n, cudaMalloc(&n->positions, (size_t)numQueries * 16));
    NRC_CUDA(n, cudaMalloc(&n->features, (size_t)numQueries * kLevels * 4));
    n->scratchQueries = numQueries;
    return GFX_OK;
}

static uint32_t nrcSmCount() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return (uint32_t)sms;
}

// pack + grid encode of the inference weights' hash grid (the two kernels in front of k_nrcInferMlp); numData (or *numDataPtr)
// is a multiple of 128
static int nrcGridEncodeLaunch(gfx_nrc* n, cudaStream_t s, const float* inputData, uint32_t numData, const uint32_t* numDataPtr) {
    int rc = nrcEnsureScratch(n, numData);
    if (rc != GFX_OK)
        return rc;
    const uint32_t sms = nrcSmCount();
    { GFX_TIMED(n->ctx, s, "nrc_pack_positions");
    k_nrcPackPositions<<<sms * 4, 256, 0, s>>>(inputData, n->positions, numData, numDataPtr); }
    n->ctx->launches++;
    const uint32_t replicas = sms / kLevels > 0 ? sms / kLevels : 1u;
    const size_t smem = (size_t)(1u << kLog2HashmapSize) * 4;
    NRC_CUDA(n, cudaFuncSetAttribute(k_nrcGridEncode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    { GFX_TIMED(n->ctx, s, "nrc_grid_encode");
    k_nrcGridEncode<<<kLevels * replicas, kEncodeThreads, smem, s>>>(n->levels, n->paramsEma + n->numMatrixWeights, n->positions,
                                                                     n->features, replicas, numData, numDataPtr); }
    n->ctx->launches++;
    NRC_CUDA(n, cudaGetLastError());
    return GFX_OK;
}

static int nrcInferLaunch(gfx_nrc* n, cudaStream_t s, const float* inputData, float* predictionData, uint32_t numData,
                          const uint32_t* numDataPtr) {
    if (n->ummaDirty) {
        k_nrcPrepWeights<<<32, 256, 0, s>>>(n->paramsEma, n->numHiddenLayers, reinterpret_cast<__half*>(n->ummaWeights), nullptr);
        n->ctx->launches++;
        n->ummaDirty = false;
    }
    const uint32_t sms = nrcSmCount();
    const uint32_t numTiles = numData / kTileRows; // upper bound when numDataPtr is given
    // buffers the TMA bulk copies cannot take (not 16-byte aligned) go through the one-kernel form, which encodes by L2 gathers
    // inside the MLP kernel
    const bool hashGrid = n->positionEncoding == GFX_NRC_POSITION_ENCODING_HASH_GRID;
    const bool aligned = (reinterpret_cast<uintptr_t>(inputData) & 15u) == 0 && (reinterpret_cast<uintptr_t>(predictionData) & 15u) == 0;
    if (!aligned) {
        const size_t smem = nrcInferFusedSmem(n->numMatrixWeights);
        auto kernel = hashGrid ? k_nrcInfer<kEncHashGrid> : k_nrcInfer<kEncTriangleWave>;
        NRC_CUDA(n, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const uint32_t grid = numTiles < sms * 6 ? numTiles : sms * 6;
        GFX_TIMED(n->ctx, s, "nrc_infer");
        kernel<<<grid, 128, smem, s>>>(n->levels, n->paramsEma + n->numMatrixWeights, n->ummaWeights, n->numHiddenLayers,
                                       inputData, predictionData, numData, numDataPtr);
        n->ctx->launches++;
        NRC_CUDA(n, cudaGetLastError());
        return GFX_OK;
    }
    // the triangle wave has nothing in front of the persistent MLP kernel
    if (hashGrid) {
        const int rc = nrcGridEncodeLaunch(n, s, inputData, numData, numDataPtr);
        if (rc != GFX_OK)
            return rc;
    }
    const size_t smem = hashGrid ? nrcInferMlpSmem<kEncHashGrid>(n->numMatrixWeights) : nrcInferMlpSmem<kEncTriangleWave>(n->numMatrixWeights);
    auto kernel = hashGrid ? k_nrcInferMlp<kEncHashGrid> : k_nrcInferMlp<kEncTriangleWave>;
    NRC_CUDA(n, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t ctasPerSm = (uint32_t)(220 * 1024 / (smem + 1024));
    const uint32_t maxGrid = sms * (ctasPerSm ? ctasPerSm : 1u);
    const uint32_t grid = numTiles < maxGrid ? numTiles : maxGrid;
    GFX_TIMED(n->ctx, s, "nrc_infer");
    kernel<<<grid, 128, smem, s>>>(n->ummaWeights, n->numHiddenLayers, inputData, n->features, predictionData, numData,
                                   numDataPtr);
    n->ctx->launches++;
    NRC_CUDA(n, cudaGetLastError());
    return GFX_OK;
}

// test hook (gfx_nrc_encode_debug): the encoded network input of numData queries, [numData][64] halves, through the split path
static int nrcEncodeDebug(gfx_nrc* n, cudaStream_t s, const float* inputData, uint32_t numData, void* outHalf) {
    const bool hashGrid = n->positionEncoding == GFX_NRC_POSITION_ENCODING_HASH_GRID;
    if (hashGrid) {
        const int rc = nrcGridEncodeLaunch(n, s, inputData, numData, nullptr);
        if (rc != GFX_OK)
            return rc;
    }
    auto kernel = hashGrid ? k_nrcAssembleEncoding<kEncHashGrid> : k_nrcAssembleEncoding<kEncTriangleWave>;
    kernel<<<(numData + 127) / 128, 128, 0, s>>>(inputData, n->features, numData, reinterpret_cast<__half*>(outHalf));
    n->ctx->launches++;
    NRC_CUDA(n, cudaGetLastError());
    return GFX_OK;
}

int gfx_nrc_infer(gfx_nrc* n, void* stream, const float* inputData, float* predictionData, uint32_t numData) {
    if (!n || (!inputData && numData) || (!predictionData && numData))
        return GFX_ERR_INVALID_ARGUMENT;
    if (numData & 0x7F) { // network_interface.cu:143 Assert((numData & 0x7F) == 0)
        n->ctx->setError("gfx_nrc_infer: numData must be a multiple of 128");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    if (numData == 0)
        return GFX_OK;
    return nrcInferLaunch(n, (cudaStream_t)stream, inputData, predictionData, numData, nullptr);
}

int gfx_nrc_encode_debug(gfx_nrc* n, void* stream, const float* inputData, uint32_t numData, void* outHalf) {
    if (!n || !inputData || !outHalf || (numData & 0x7F))
        return GFX_ERR_INVALID_ARGUMENT;
    if (numData == 0)
        return GFX_OK;
    return nrcEncodeDebug(n, (cudaStream_t)stream, inputData, numData, outHalf);
}

int gfx_nrc_frame_infer(gfx_ctx* ctx, gfx_nrc* n, void* stream) {
    if (!ctx || !n || n->ctx != ctx)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    const int rc = ensureNrcFrame(ctx);
    if (rc != GFX_OK)
        return rc;
    const FrameState::Nrc &N = ctx->frame.nrc;
    // numInferenceQueries = pad128(W*H + #tiles) was left in the state block by gfx_nrc_preprocess
    return nrcInferLaunch(n, (cudaStream_t)stream, N.inferenceQuery, N.inferredRadiance, N.queryCapacity, N.state + 26);
}

int gfx_nrc_frame_infer_rows(gfx_ctx* ctx, gfx_nrc* n, void* stream, uint32_t rowLo, uint32_t rowHi) {
    if (!ctx || !n || n->ctx != ctx)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    int rc = ensureNrcFrame(ctx);
    if (rc != GFX_OK)
        return rc;
    const FrameState::Nrc &N = ctx->frame.nrc;
    const uint32_t W = ctx->frame.W, H = ctx->frame.H;
    if (rowLo >= rowHi || rowHi > H)
        return GFX_ERR_INVALID_ARGUMENT;
    const size_t numPixels = (size_t)W * H, first = (size_t)rowLo * W;
    if ((first & 127u) || (numPixels & 127u)) {
        ctx->setError("gfx_nrc_frame_infer_rows: rowLo * width and width * height must be multiples of the 128-query tile");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    // the strip's terminal queries (one per pixel; the tail of the last 128-query tile reads into the next rows, whose
    // predictions this rank does not use) ...
    const uint32_t numRowQueries = (uint32_t)((((size_t)(rowHi - rowLo) * W + 127) / 128) * 128);
    const uint32_t rowQueries = (uint32_t)(first + numRowQueries <= N.queryCapacity ? numRowQueries : N.queryCapacity - first);
    rc = nrcInferLaunch(n, (cudaStream_t)stream, N.inferenceQuery + 14 * first, N.inferredRadiance + 3 * first, rowQueries, nullptr);
    if (rc != GFX_OK)
        return rc;
    // ... and the training-suffix queries of all tiles (slots of the other ranks' tiles hold stale queries: their
    // predictions are never read here, propagation only walks the suffixes this rank traced)
    const uint32_t suffixCapacity = (uint32_t)(N.queryCapacity - numPixels);
    return nrcInferLaunch(n, (cudaStream_t)stream, N.inferenceQuery + 14 * numPixels, N.inferredRadiance + 3 * numPixels, suffixCapacity,
                          N.state + 27);
}

int gfx_nrc_frame_train(gfx_ctx* ctx, gfx_nrc* n, void* stream, float* lossOnHost) {
    if (!ctx || !n || n->ctx != ctx)
        return GFX_ERR_INVALID_ARGUMENT;
    if (!ctx->frame.created)
        return GFX_ERR_NOT_READY;
    int rc = ensureNrcFrame(ctx);
    if (rc != GFX_OK)
        return rc;
    const FrameState::Nrc &N = ctx->frame.nrc;
    // neural_radiance_caching_main.cpp:2350-2365: four steps over quarters of the shuffled 65 536 records
    const uint32_t batchSize = 65536 / 4;
    for (uint32_t step = 0; step < 4 && rc == GFX_OK; ++step)
        rc = gfx_nrc_train(n, stream, N.trainQuery[1] + (size_t)step * batchSize * 14, N.trainTarget[1] + (size_t)step * batchSize * 3,
                           batchSize, step == 3 ? lossOnHost : nullptr);
    return rc;
}

int gfx_nrc_train(gfx_nrc* n, void* stream, const float* inputData, const float* targetData, uint32_t numData, float* lossOnHost) {
    if (!n || !inputData || !targetData)
        return GFX_ERR_INVALID_ARGUMENT;
    if (numData & 0x7F) {
        n->ctx->setError("gfx_nrc_train: numData must be a multiple of 128");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    if (numData == 0)
        return GFX_OK;
    cudaStream_t s = (cudaStream_t)stream;
    NRC_CUDA(n, cudaMemsetAsync(n->loss, 0, 4, s));
    // Fully-connected layers on wgmma (forward, data gradient and weight gradient); deeper networks, whose activation tiles do
    // not fit in shared memory, train on CUDA cores.
    const bool hashGrid = n->positionEncoding == GFX_NRC_POSITION_ENCODING_HASH_GRID;
    if (n->numHiddenLayers <= kMaxTcTrainHiddenLayers) {
        const size_t smem = nrcTrainTcSmem(n->numMatrixWeights, n->numHiddenLayers);
        auto kernel = hashGrid ? k_nrcTrainTc<kEncHashGrid> : k_nrcTrainTc<kEncTriangleWave>;
        NRC_CUDA(n, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        { GFX_TIMED(n->ctx, s, "nrc_train_prep_weights");
        k_nrcPrepWeights<<<32, 256, 0, s>>>(n->params, n->numHiddenLayers, reinterpret_cast<__half*>(n->trainBlobFwd),
                                            reinterpret_cast<__half*>(n->trainBlobT)); }
        n->ctx->launches++;
        { GFX_TIMED(n->ctx, s, "nrc_train_fwd_bwd");
        kernel<<<numData / 128, 128, smem, s>>>(n->levels, n->params, n->numMatrixWeights, n->numHiddenLayers, n->trainBlobFwd,
                                                n->trainBlobT, inputData, targetData, numData, n->grads, n->loss); }
    }
    else {
        const size_t smem = nrcTrainSmem(n->numMatrixWeights, n->numHiddenLayers);
        auto kernel = hashGrid ? k_nrcTrain<kEncHashGrid> : k_nrcTrain<kEncTriangleWave>;
        NRC_CUDA(n, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        { GFX_TIMED(n->ctx, s, "nrc_train_fwd_bwd");
        kernel<<<numData / 128, 128, smem, s>>>(n->levels, n->params, n->numMatrixWeights, n->numHiddenLayers, inputData,
                                                targetData, numData, n->grads, n->loss); }
    }
    n->ctx->launches++;
    if (n->keepGradients) {
        k_nrcKeepGradients<<<(n->numParams + 255) / 256, 256, 0, s>>>(n->numParams, n->grads, n->gradsFloat);
        n->ctx->launches++;
    }
    ++n->globalStep;
    const float emaDecay = 0.99f;
    const float emaDebiasOld = 1 - (float)pow((double)emaDecay, (double)(n->globalStep - 1));
    const float emaDebiasNew = 1.0f / (1 - (float)pow((double)emaDecay, (double)n->globalStep));
    { GFX_TIMED(n->ctx, s, "nrc_adam_ema");
    k_nrcAdamEma<<<(n->numParams + 255) / 256, 256, 0, s>>>(n->numParams, n->numMatrixWeights, n->learningRate, n->adamEpsilon,
                                                            emaDebiasOld, emaDebiasNew, n->grads, n->master, n->params, n->paramsEma,
                                                            n->m1, n->m2, n->steps); }
    n->ctx->launches++;
    n->ummaDirty = true;
    NRC_CUDA(n, cudaGetLastError());
    if (lossOnHost) { // network_interface.cu:155-156: optional blocking read-back
        NRC_CUDA(n, cudaMemcpyAsync(lossOnHost, n->loss, 4, cudaMemcpyDeviceToHost, s));
        NRC_CUDA(n, cudaStreamSynchronize(s));
    }
    return GFX_OK;
}

} // extern "C"
