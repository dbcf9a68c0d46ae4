// oracle/nrc_triwave.cpp — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// Scalar restatement of the NRC network the reference builds through tiny-cuda-nn with the TRIANGLE-WAVE position encoding
// (NeuralRadianceCache::initialize(PositionEncoding::TriangleWave, ...), neural_radiance_caching/network_interface.cu:48-121;
// network_interface.h:5-8; the app's -position-encoding tri, neural_radiance_caching_main.cpp:458, 755-766, 1996-2027;
// ext/tiny-cuda-nn @ be460660, vendored source).  The hash-grid network is oracle/nrc.cpp; the MLP, loss, Adam and EMA below
// follow it line for line, only the encoding, the backward's end and Adam's epsilon differ.  Built into
// oracle/liborc_nrc_triwave.so by oracle/Makefile.triwave (tests/oracle_nrc_triwave.py binds it).
//   Composite encoding       TriangleWave(3 dims, 12 frequencies) + OneBlob(5 dims x 4 bins) + Identity(6 dims): inputs 0..35 the
//                            triangle wave feature-major (12 d + f), 36..55 one-blob, 56..61 identity, 62..63 ones (Composite pads
//                            its last nested encoding to the MLP's alignment, composite.h:100-111, 231-237; OneBlob's
//                            min_alignment 4 divides 36, so nothing is padded in between)
//     triangle_wave_encoding encodings/triangle_wave.h:47-81
//     one-blob               TriangleWave prefers AoS, so the Composite runs every nested encoding in AoS (composite.h:253-262):
//                            kernel_one_blob oneblob.h:83-108 with one_blob_subwarp_aligned :47-69 (last bin closed by "bin 0's
//                            left CDF + 1"), quartic_cdf common_device.h:478-483 with the three FMAs the reference's own build
//                            contracts it into; identity.h:67 x * 1 + 0
//                            The encoding has no parameters: numParams = the matrix weights, and NetworkWithInputEncoding::backward
//                            computes no input gradient (network_with_input_encoding.h:92-99) - no data gradient through layer 0.
//   FullyFusedMLP            64 neurons, n hidden layers, ReLU, linear output 3 (padded 16)
//                            src/fully_fused_mlp.cu:47-129 (forward), :150-259,:499-557 (backward)
//   RelativeL2Luminance      losses/relative_l2_luminance.h:41-88, loss scale 128 (trainer.h:187)
//   Adam + EMA(0.99)         optimizers/adam.h:49-115 with epsilon 1e-8 (network_interface.cu:94), optimizers/ema.h:46-121
// Two accumulation modes for the fully-connected layers, as in oracle/nrc.cpp (orc_nrctw_set_accumulate_half): 0 = fp32 per
// 64-term dot product (this repo's wgmma kernels), 1 = tiny-cuda-nn's half accumulator fragments (rounded every 16-wide k step).
// Pinned against the reference's own code: tests/golden/tcnn_nrc_triwave.npz (tests/golden/make_golden_tcnn_triwave.py), compared
// on the CPU (tests/test_oracle_nrc_triwave.py: the encoding bit for bit) and on the GPU (tests/test_gpu_tcnn_nrc_triwave.py).
// Parameter layout (shared with the CUDA library): the MLP matrices [out][in] in layer order (64x64, ..., last 16x64).
#include <cstdint>
#include <cstring>
#include <cmath>
#include <vector>
#include <omp.h>

namespace {

typedef _Float16 half;
inline float h2f(half h) { return (float)h; }
inline half f2h(float f) { return (half)f; }

constexpr uint32_t kInputDims = 14, kOutputDims = 3, kWidth = 64, kPaddedOutput = 16;
constexpr float kLossScale = 128.0f;

// quartic_cdf (common_device.h:478-483) as the reference's build evaluates it: its polynomial contracted into three FMAs
inline float quarticCdfContracted(float x) {
    const float u = x * 4.0f, u2 = u * u, u4 = u2 * u2;
    const float inner = std::fma(1.0f / 5.0f, u4, std::fma(-(2.0f / 3.0f), u2, 1.0f));
    return std::fmax(0.0f, std::fmin(1.0f, std::fma((15.0f / 16.0f) * u, inner, 0.5f)));
}

// triangle_wave_encoding (triangle_wave.h:71-75) of position coordinate p at frequency f
inline float triangleWave(float p, uint32_t f) {
    const float x = std::scalbn(p, (int)f - 1);
    const float val = x + (float)f * 0.25f;
    return std::fabs(val - std::floor(val) - 0.5f) * 4 - 1;
}

} // namespace

struct orc_nrctw {
    uint32_t numHiddenLayers;
    float learningRate;
    uint32_t numParams;             // = the matrix weights
    std::vector<half> params;       // current fp16 weights
    std::vector<half> paramsEma;    // inference weights (EMA)
    std::vector<float> master;      // fp32 master weights
    std::vector<float> m1, m2;      // Adam moments
    std::vector<uint32_t> steps;    // per-parameter step counters (adam.h:108)
    uint32_t globalStep = 0;
    int accumulateHalf = 0;
    std::vector<float> lastGradients; // loss-scaled gradients of the last training step, rounded to half like tcnn's buffer
};

// one output of a fully-connected layer: sum_i w[i * stride] * x[i] (oracle/nrc.cpp dotLayer)
static inline float dotLayer(const orc_nrctw* n, const half* w, size_t stride, const half* x, uint32_t count) {
    if (!n->accumulateHalf) {
        float acc = 0.0f;
        for (uint32_t i = 0; i < count; ++i)
            acc += h2f(w[i * stride]) * h2f(x[i]);
        return acc;
    }
    half acc = f2h(0.0f);
    for (uint32_t c = 0; c < count; c += 16) {
        float partial = 0.0f;
        for (uint32_t i = c; i < c + 16 && i < count; ++i)
            partial += h2f(w[i * stride]) * h2f(x[i]);
        acc = f2h(h2f(acc) + partial);
    }
    return h2f(acc);
}

// the Composite encoding of one query into 64 halves
static void encode(const float* in, half* out) {
    for (uint32_t d = 0; d < 3; ++d) // TriangleWave, feature-major: input 12 d + f
        for (uint32_t f = 0; f < 12; ++f)
            out[12 * d + f] = f2h(triangleWave(in[d], f));
    for (uint32_t d = 0; d < 5; ++d) { // kernel_one_blob: the CDF at the four left boundaries k / 4, three periodic images
        const float x = in[3 + d];
        float left[4];
        for (uint32_t k = 0; k < 4; ++k) {
            const float b = std::scalbn((float)k, -2);
            left[k] = quarticCdfContracted(b - x) + quarticCdfContracted(b - x - 1.0f) + quarticCdfContracted(b - x + 1.0f);
        }
        for (uint32_t k = 0; k < 4; ++k)
            out[36 + d * 4 + k] = f2h((k < 3 ? left[k + 1] : left[0] + 1.0f) - left[k]);
    }
    for (uint32_t d = 0; d < 6; ++d) // identity.h:67: x * scale + offset, scale 1, offset 0
        out[56 + d] = f2h(in[8 + d] * 1.0f + 0.0f);
    out[62] = out[63] = f2h(1.0f);
}

// forward through the MLP; acts[layer] receives the post-activation halves of every hidden layer
static void mlpForward(const orc_nrctw* n, const half* w, const half* x, half* acts /*numHidden*64*/, half* out /*16*/) {
    const half* in = x;
    for (uint32_t layer = 0; layer < n->numHiddenLayers; ++layer) {
        const half* W = w + (size_t)layer * kWidth * kWidth;
        half* o = acts + (size_t)layer * kWidth;
        for (uint32_t j = 0; j < kWidth; ++j)
            o[j] = f2h(std::fmax(dotLayer(n, W + j * kWidth, 1, in, kWidth), 0.0f)); // ReLU, stored as half
        in = o;
    }
    const half* W = w + (size_t)n->numHiddenLayers * kWidth * kWidth;
    for (uint32_t j = 0; j < kPaddedOutput; ++j)
        out[j] = f2h(dotLayer(n, W + j * kWidth, 1, in, kWidth));
}

extern "C" {

orc_nrctw* orc_nrctw_create(uint32_t numHiddenLayers, float learningRate) {
    orc_nrctw* n = new orc_nrctw();
    n->numHiddenLayers = numHiddenLayers;
    n->learningRate = learningRate;
    n->numParams = kWidth * kWidth * numHiddenLayers + kPaddedOutput * kWidth;
    n->params.assign(n->numParams, f2h(0.0f));
    n->paramsEma.assign(n->numParams, f2h(0.0f));
    n->master.assign(n->numParams, 0.0f);
    n->m1.assign(n->numParams, 0.0f);
    n->m2.assign(n->numParams, 0.0f);
    n->steps.assign(n->numParams, 0u);
    return n;
}
void orc_nrctw_destroy(orc_nrctw* n) { delete n; }
uint32_t orc_nrctw_num_params(orc_nrctw* n) { return n->numParams; }

// installs the same fp16 values as current, EMA (inference) and fp32 master weights; resets the optimizer state
void orc_nrctw_set_params(orc_nrctw* n, const uint16_t* halfBits) {
    std::memcpy(n->params.data(), halfBits, (size_t)n->numParams * 2);
    n->paramsEma = n->params;
    for (uint32_t i = 0; i < n->numParams; ++i)
        n->master[i] = h2f(n->params[i]);
    std::fill(n->m1.begin(), n->m1.end(), 0.0f);
    std::fill(n->m2.begin(), n->m2.end(), 0.0f);
    std::fill(n->steps.begin(), n->steps.end(), 0u);
    n->globalStep = 0;
}
void orc_nrctw_set_accumulate_half(orc_nrctw* n, int on) { n->accumulateHalf = on; }
void orc_nrctw_get_master(orc_nrctw* n, float* out) { std::memcpy(out, n->master.data(), (size_t)n->numParams * 4); }
int orc_nrctw_get_gradients(orc_nrctw* n, float* out) {
    if (n->lastGradients.size() != n->numParams)
        return 1;
    std::memcpy(out, n->lastGradients.data(), (size_t)n->numParams * 4);
    return 0;
}
void orc_nrctw_get_params(orc_nrctw* n, uint16_t* out, int ema) {
    std::memcpy(out, ema ? n->paramsEma.data() : n->params.data(), (size_t)n->numParams * 2);
}

void orc_nrctw_encode(orc_nrctw*, const float* in, uint32_t num, uint16_t* outHalfBits) {
#pragma omp parallel for schedule(static)
    for (int64_t q = 0; q < (int64_t)num; ++q)
        encode(in + (size_t)q * kInputDims, reinterpret_cast<half*>(outHalfBits) + (size_t)q * 64);
}

// NeuralRadianceCache::infer (network_interface.cu:141-147): inference runs on the EMA weights (trainer.h:89-93)
void orc_nrctw_infer(orc_nrctw* n, const float* in, float* out, uint32_t num) {
    const half* w = n->paramsEma.data();
#pragma omp parallel for schedule(static)
    for (int64_t q = 0; q < (int64_t)num; ++q) {
        half x[64], acts[64 * 8], o[16];
        encode(in + (size_t)q * kInputDims, x);
        mlpForward(n, w, x, acts, o);
        for (uint32_t k = 0; k < kOutputDims; ++k)
            out[(size_t)q * kOutputDims + k] = h2f(o[k]); // trim_and_cast_from
    }
}

// Trainer::training_step (trainer.h:178-197): forward, RelativeL2Luminance, backward, Adam, EMA. Returns the loss.
float orc_nrctw_train(orc_nrctw* n, const float* in, const float* target, uint32_t num) {
    const uint32_t H = n->numHiddenLayers;
    std::vector<float> grad(n->numParams, 0.0f);
    double lossSum = 0.0;
    const half* w = n->params.data();
    const int nt = omp_get_max_threads();
    std::vector<std::vector<float>> tgrad(nt);
#pragma omp parallel
    {
        std::vector<float> &g = tgrad[omp_get_thread_num()];
        g.assign(n->numParams, 0.0f);
        double localLoss = 0.0;
#pragma omp for schedule(static)
        for (int64_t q = 0; q < (int64_t)num; ++q) {
            half x[64], acts[64 * 8], o[16];
            encode(in + (size_t)q * kInputDims, x);
            mlpForward(n, w, x, acts, o);
            // relative_l2_luminance_loss (relative_l2_luminance.h:41-88), stride 16, dims 3
            const uint32_t nTotal = num * kOutputDims;
            const float r = h2f(o[0]), gch = h2f(o[1]), b = h2f(o[2]);
            const float luminance = 0.299f * r + 0.587f * gch + 0.114f * b;
            const float denom = luminance * luminance + 0.01f;
            half dOut[16];
            for (uint32_t k = 0; k < kPaddedOutput; ++k) {
                if (k >= kOutputDims) {
                    dOut[k] = f2h(0.0f);
                    continue;
                }
                const float difference = h2f(o[k]) - target[(size_t)q * kOutputDims + k];
                localLoss += difference * difference / denom / nTotal;
                dOut[k] = f2h(kLossScale * (2 * difference / denom) / nTotal);
            }
            // backward through the layers (fully_fused_mlp.cu:150-259, 773-900): dW = dY^T X, dX = W^T dY
            half dCur[64];
            {
                const half* W = w + (size_t)H * kWidth * kWidth;
                const half* hin = acts + (size_t)(H - 1) * kWidth; // H >= 1
                float* gW = g.data() + (size_t)H * kWidth * kWidth;
                for (uint32_t j = 0; j < kPaddedOutput; ++j) {
                    const float dj = h2f(dOut[j]);
                    if (dj != 0.0f)
                        for (uint32_t i = 0; i < kWidth; ++i)
                            gW[j * kWidth + i] += dj * h2f(hin[i]);
                }
                for (uint32_t i = 0; i < kWidth; ++i) {
                    const float acc = dotLayer(n, W + i, kWidth, dOut, kPaddedOutput);
                    dCur[i] = !(h2f(hin[i]) > 0.0f) ? f2h(0.0f) : f2h(acc); // ReLU backward (fully_fused_mlp.cu:163-176)
                }
            }
            for (int layer = (int)H - 1; layer >= 0; --layer) {
                const half* W = w + (size_t)layer * kWidth * kWidth;
                const half* hin = layer > 0 ? acts + (size_t)(layer - 1) * kWidth : x;
                float* gW = g.data() + (size_t)layer * kWidth * kWidth;
                for (uint32_t j = 0; j < kWidth; ++j) {
                    const float dj = h2f(dCur[j]);
                    if (dj != 0.0f)
                        for (uint32_t i = 0; i < kWidth; ++i)
                            gW[j * kWidth + i] += dj * h2f(hin[i]);
                }
                if (layer == 0)
                    break; // no input gradient for an encoding without parameters
                half dNext[64];
                for (uint32_t i = 0; i < kWidth; ++i) {
                    const float acc = dotLayer(n, W + i, kWidth, dCur, kWidth);
                    dNext[i] = !(h2f(hin[i]) > 0.0f) ? f2h(0.0f) : f2h(acc);
                }
                std::memcpy(dCur, dNext, sizeof(dCur));
            }
        }
#pragma omp critical
        lossSum += localLoss;
    }
    for (int t = 0; t < nt; ++t)
        for (uint32_t i = 0; i < n->numParams; ++i)
            grad[i] += tgrad[t][i];

    n->lastGradients.resize(n->numParams);
    for (uint32_t i = 0; i < n->numParams; ++i)
        n->lastGradients[i] = h2f(f2h(grad[i]));
    // Adam (adam.h:49-115) on half gradients, every parameter a matrix weight (L2 regularised), then EMA (ema.h:61-77,103-121)
    ++n->globalStep;
    const float beta1 = 0.9f, beta2 = 0.99f, epsilon = 1e-8f, l2Reg = 1e-6f;
    const float emaDecay = 0.99f;
    const float emaDebiasOld = 1 - (float)std::pow(emaDecay, (double)(n->globalStep - 1));
    const float emaDebiasNew = 1.0f / (1 - (float)std::pow(emaDecay, (double)n->globalStep));
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n->numParams; ++i) {
        const float weightFp = n->master[i];
        const float gradient = h2f(f2h(grad[i])) / kLossScale + l2Reg * weightFp;
        const float gradientSq = gradient * gradient;
        const float firstMoment = n->m1[i] = beta1 * n->m1[i] + (1 - beta1) * gradient;
        const float secondMoment = n->m2[i] = beta2 * n->m2[i] + (1 - beta2) * gradientSq;
        float lr = n->learningRate;
        const uint32_t currentStep = ++n->steps[i];
        lr *= std::sqrt(1 - std::pow(beta2, (float)currentStep)) / (1 - std::pow(beta1, (float)currentStep));
        const float effectiveLr = std::fmin(std::fmax(lr / (std::sqrt(secondMoment) + epsilon), 0.0f), 3.402823466e+38f);
        const float newWeight = weightFp - effectiveLr * firstMoment;
        n->master[i] = newWeight;
        n->params[i] = f2h(newWeight);
        const float filtered = (h2f(n->paramsEma[i]) * emaDecay * emaDebiasOld + h2f(n->params[i]) * (1 - emaDecay)) * emaDebiasNew;
        n->paramsEma[i] = f2h(filtered);
    }
    return (float)lossSum;
}

} // extern "C"
