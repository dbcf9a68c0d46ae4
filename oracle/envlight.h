// oracle/envlight.h — environment light of the CPU oracle (TEST INFRASTRUCTURE, see oracle.h).
//
// Restates, for the hot path's use of it:
//   - loadEnvironmentalTexture (common/common_host.cpp:2658-2711): texels clamped to [0, 65504], importance = luminance * sin(theta)
//     of the texel centre;
//   - RegularConstantContinuousDistribution1D/2D: host construction (common_host.cpp:292-357, non-alias branch: compensated sum of
//     PDF[i] / N into the CDF, normalisation by the integral) and device sampling / evaluation (common_shared.h:283-386);
//   - tex2DLod<float4>(envLightTexture, u, v, 0) with the sampler of :2664-2669 (linear filter, clamp addressing, normalised
//     coordinates).  The texture unit computes xB = u * W - 0.5, i = floor(xB), alpha = frac(xB) kept with 8 fractional bits
//     (CUDA programming guide, texture fetching: linear filtering) and blends the four texels; that arithmetic is restated in
//     software (weights rounded to 1/256, blend in fp32 in the order (1-a)(1-b) T00 + a(1-b) T10 + (1-a)b T01 + ab T11).
#ifndef ORACLE_ENVLIGHT_H
#define ORACLE_ENVLIGHT_H
#include "shading.h"
#include <vector>

namespace orc {

struct CompensatedSum { // basic_types.h:5427-5452
    float result = 0.0f, comp = 0.0f;
    void add(float value) {
        const float cInput = value - comp;
        const float sumTemp = result + cInput;
        comp = (sumTemp - result) - cInput;
        result = sumTemp;
    }
};

struct RegularConstantContinuousDistribution1D { // common_shared.h:283-354
    const float* PDF = nullptr;
    const float* CDF = nullptr;
    float integral = 0.0f;
    uint32_t numValues = 0;
    float sample(float u, float* probDensity) const { // :316-343
        int idx = 0;
        uint32_t pow2 = 1;
        while (pow2 < numValues)
            pow2 <<= 1;
        for (int d = (int)(pow2 >> 1); d >= 1; d >>= 1) {
            if (idx + d >= (int)numValues)
                continue;
            if (CDF[idx + d] <= u)
                idx += d;
        }
        const float t = (u - CDF[idx]) / (CDF[idx + 1] - CDF[idx]);
        *probDensity = PDF[idx];
        return (idx + t) / numValues;
    }
    float evaluatePDF(float smp) const { // :344-348
        const uint32_t idx = std::min(numValues - 1, (uint32_t)(smp * numValues));
        return PDF[idx];
    }
};

inline uint32_t mapPrimarySampleToDiscrete(float u01, uint32_t numValues) { // common_shared.h:142-152
    return std::min((uint32_t)(u01 * numValues), numValues - 1);
}

struct EnvLight {
    uint32_t W = 0, H = 0;
    std::vector<float> texels;      // RGBA, clamped
    std::vector<float> pdf, cdf;    // H rows of W and W + 1 values
    std::vector<float> rowIntegral; // H
    std::vector<float> topPdf, topCdf;
    float topIntegral = 0.0f;
    bool present() const { return W != 0; }

    RegularConstantContinuousDistribution1D row(uint32_t y) const {
        return RegularConstantContinuousDistribution1D{ pdf.data() + (size_t)y * W, cdf.data() + (size_t)y * (W + 1), rowIntegral[y], W };
    }
    RegularConstantContinuousDistribution1D top() const {
        return RegularConstantContinuousDistribution1D{ topPdf.data(), topCdf.data(), topIntegral, H };
    }
    // RegularConstantContinuousDistribution2D::sample / evaluatePDF (common_shared.h:371-383)
    void sample(float u0, float u1, float* d0, float* d1, float* probDensity) const {
        float topPDF;
        *d1 = top().sample(u1, &topPDF);
        const uint32_t idx1D = mapPrimarySampleToDiscrete(*d1, H);
        *d0 = row(idx1D).sample(u0, probDensity);
        *probDensity *= topPDF;
    }
    float evaluatePDF(float d0, float d1) const {
        const uint32_t idx1D = mapPrimarySampleToDiscrete(d1, H);
        return top().evaluatePDF(d1) * row(idx1D).evaluatePDF(d0);
    }
    // tex2DLod<float4>(envLightTexture, u, v, 0.0f).xyz, see the header comment
    float3 fetch(float u, float v) const {
        const float xB = u * W - 0.5f, yB = v * H - 0.5f;
        const float fx = std::floor(xB), fy = std::floor(yB);
        const float a = std::floor((xB - fx) * 256.0f + 0.5f) * (1.0f / 256.0f);
        const float b = std::floor((yB - fy) * 256.0f + 0.5f) * (1.0f / 256.0f);
        auto clampi = [](float f, uint32_t n) { return (uint32_t)std::min(std::max(f, 0.0f), (float)(n - 1)); };
        const uint32_t x0 = clampi(fx, W), x1 = clampi(fx + 1.0f, W), y0 = clampi(fy, H), y1 = clampi(fy + 1.0f, H);
        auto T = [&](uint32_t x, uint32_t y) {
            const float* t = texels.data() + 4 * ((size_t)y * W + x);
            return float3(t[0], t[1], t[2]);
        };
        const float w00 = (1 - a) * (1 - b), w10 = a * (1 - b), w01 = (1 - a) * b, w11 = a * b;
        return w00 * T(x0, y0) + w10 * T(x1, y0) + w01 * T(x0, y1) + w11 * T(x1, y1);
    }
};

// RegularConstantContinuousDistribution1DTemplate::initialize, non-alias branch (common_host.cpp:292-312).  Departure: with
// integral 0 (a black row or map) the reference's lines compute 0 / 0 = NaN for every entry; here PDF = 0 and CDF = i / n
// (DESIGN.md, "Environment maps with black rows").
inline float buildRegularDistribution1D(const float* values, uint32_t n, float* PDF, float* CDF) {
    CompensatedSum sum;
    for (uint32_t i = 0; i < n; ++i) {
        PDF[i] = values[i];
        CDF[i] = sum.result;
        sum.add(PDF[i] / n);
    }
    const float integral = sum.result;
    for (uint32_t i = 0; i < n; ++i) {
        if (integral > 0.0f) {
            PDF[i] /= integral;
            CDF[i] /= integral;
        }
        else {
            PDF[i] = 0.0f;
            CDF[i] = (float)i / (float)n;
        }
    }
    CDF[n] = 1.0f;
    return integral;
}

// false for a map with a NaN texel, which the clamp would pass into every pdf (the library refuses it the same way)
inline bool buildEnvLight(EnvLight* e, const float* rgba, uint32_t width, uint32_t height) {
    *e = EnvLight();
    if (!rgba || !width || !height)
        return true;
    for (size_t i = 0; i < (size_t)width * height; ++i)
        if (std::isnan(rgba[4 * i]) || std::isnan(rgba[4 * i + 1]) || std::isnan(rgba[4 * i + 2]))
            return false;
    e->W = width;
    e->H = height;
    e->texels.assign(rgba, rgba + 4 * (size_t)width * height);
    std::vector<float> importance((size_t)width * height);
    for (uint32_t y = 0; y < height; ++y) {
        const float theta = kPi * (y + 0.5f) / height;
        const float sinTheta = std::sin(theta);
        for (uint32_t x = 0; x < width; ++x) {
            float* t = e->texels.data() + 4 * ((size_t)y * width + x);
            for (int c = 0; c < 3; ++c)
                t[c] = std::min(std::max(t[c], 0.0f), 65504.0f);
            importance[(size_t)y * width + x] = sRGB_calcLuminance(float3(t[0], t[1], t[2])) * sinTheta;
        }
    }
    e->pdf.resize((size_t)width * height);
    e->cdf.resize((size_t)(width + 1) * height);
    e->rowIntegral.resize(height);
    for (uint32_t y = 0; y < height; ++y)
        e->rowIntegral[y] = buildRegularDistribution1D(importance.data() + (size_t)y * width, width,
                                                       e->pdf.data() + (size_t)y * width, e->cdf.data() + (size_t)y * (width + 1));
    e->topPdf.resize(height);
    e->topCdf.resize(height + 1);
    e->topIntegral = buildRegularDistribution1D(e->rowIntegral.data(), height, e->topPdf.data(), e->topCdf.data());
    return true;
}

// one image texture of a material and tex2DLod<float4>(tex, u, v, 0) with the reference's material samplers
// (common_host.cpp:1462-1481: linear filter, repeat addressing): the arithmetic of EnvLight::fetch with wrapped indices
struct ImageTexture {
    uint32_t W = 0, H = 0;
    std::vector<float> texels; // RGBA
    void fetch(float u, float v, float out[4]) const {
        const float xB = (u - std::floor(u)) * W - 0.5f, yB = (v - std::floor(v)) * H - 0.5f;
        const float fx = std::floor(xB), fy = std::floor(yB);
        const float a = std::floor((xB - fx) * 256.0f + 0.5f) * (1.0f / 256.0f);
        const float b = std::floor((yB - fy) * 256.0f + 0.5f) * (1.0f / 256.0f);
        const int ix = (int)fx, iy = (int)fy; // -1 .. W - 1
        const uint32_t x0 = ix < 0 ? W - 1 : (uint32_t)ix, x1 = (uint32_t)(ix + 1) >= W ? 0u : (uint32_t)(ix + 1);
        const uint32_t y0 = iy < 0 ? H - 1 : (uint32_t)iy, y1 = (uint32_t)(iy + 1) >= H ? 0u : (uint32_t)(iy + 1);
        const float* t00 = texels.data() + 4 * ((size_t)y0 * W + x0);
        const float* t10 = texels.data() + 4 * ((size_t)y0 * W + x1);
        const float* t01 = texels.data() + 4 * ((size_t)y1 * W + x0);
        const float* t11 = texels.data() + 4 * ((size_t)y1 * W + x1);
        const float w00 = (1 - a) * (1 - b), w10 = a * (1 - b), w01 = (1 - a) * b, w11 = a * b;
        for (int c = 0; c < 4; ++c)
            out[c] = w00 * t00[c] + w10 * t10[c] + w01 * t01[c] + w11 * t11[c];
    }
};

constexpr float kProbToSampleEnvLight = 0.25f; // restir_di_shared.h:6 (and the other apps' *_shared.h:6)

} // namespace orc

#endif
