// oracle/shading.h — TEST INFRASTRUCTURE (CPU oracle).  Not part of the product path.
//
// CPU restatement of the device helpers every ReSTIR/PT kernel of the reference shares:
//   PCG32RNG                       common/common_shared.h:116-138
//   DiscreteDistribution1D         common/common_shared.h:175-276
//   polar encoders / frames        common/common_device.cuh:14-140,149-203
//   Lambert / DiffuseAndSpecular / SimplePBR BRDFs   common/common_device.cuh:335-385,443-826
// Transcendentals go through gfxexp_b200/csrc/detmath.h (the same header the CUDA kernels
// use) so that host and device round identically; everything else is IEEE +,-,*,/,sqrt.
#pragma once
#include "vecmath.h"
#include "../gfxexp_b200/csrc/detmath.h"

namespace orc {

constexpr float kPi = 3.14159265358979323846f;

struct PCG32RNG { // common_shared.h:116-138
    uint64_t state;
    uint32_t next() {
        const uint64_t oldstate = state;
        state = oldstate * 6364136223846793005ULL + 1;
        const uint32_t xorshifted = (uint32_t)(((oldstate >> 18u) ^ oldstate) >> 27u);
        const uint32_t rot = (uint32_t)(oldstate >> 59u);
        return (xorshifted >> rot) | (xorshifted << ((-(int32_t)rot) & 31));
    }
    float getFloat0cTo1o() {
        const uint32_t fractionBits = (next() >> 9) | 0x3f800000u;
        return u2f(fractionBits) - 1.0f;
    }
};

struct DiscreteDistribution1D { // common_shared.h:175-276 (CDF variant, USE_WALKER_ALIAS_METHOD off)
    const float* weights = nullptr;
    const float* cdf = nullptr;
    float integral = 0.0f;
    uint32_t numValues = 0;

    uint32_t sample(float u, float* prob, float* remapped = nullptr) const { // :209-246
        u *= integral;
        int idx = 0;
        for (int d = (int)(nextPowerOf2(numValues) >> 1); d >= 1; d >>= 1) {
            if (idx + d >= (int)numValues)
                continue;
            if (cdf[idx + d] <= u)
                idx += d;
        }
        if (remapped) {
            const float lCDF = cdf[idx];
            float rCDF = integral;
            if (idx < (int)numValues - 1)
                rCDF = cdf[idx + 1];
            *remapped = (u - lCDF) / (rCDF - lCDF);
        }
        *prob = weights[idx] / integral;
        return (uint32_t)idx;
    }
    float evaluatePMF(uint32_t idx) const { // :248-253
        if (!weights || integral == 0.0f)
            return 0.0f;
        return weights[idx] / integral;
    }
};

// ---- polar encoders (common_device.cuh:14-79) --------------------------------------------
inline float3 fromPolarYUp(float phi, float theta) { // :14-20
    float sinPhi, cosPhi, sinTheta, cosTheta;
    dm_sincos(phi, &sinPhi, &cosPhi);
    dm_sincos(theta, &sinTheta, &cosTheta);
    return float3(-sinPhi * sinTheta, cosTheta, cosPhi * sinTheta);
}
inline void toPolarYUp(const float3 &v, float* phi, float* theta) { // :21-25
    *theta = dm_acos(std::fmin(std::fmax(v.y, -1.0f), 1.0f));
    // fmod(atan2 + 2pi, 2pi): atan2 is in [-pi, pi], so one conditional subtraction is exact.
    float t = dm_atan2(-v.x, v.z) + 2 * kPi;
    if (t >= 2 * kPi)
        t = t - 2 * kPi;
    *phi = t;
}
inline uint16_t encodeBarycentric(float bc) { // :27-29
    return (uint16_t)std::min(dm_f2uint(bc * 65535u), 65535u);
}
inline float decodeBarycentric(uint16_t qbc) { return qbc / 65535.0f; } // :31-33
inline uint32_t encodeVector(const float3 &v) { // :35-41 (encodeNormal :51-57 is identical)
    float phi, theta;
    toPolarYUp(v, &phi, &theta);
    const uint32_t qPhi = std::min(dm_f2uint((phi / (2 * kPi)) * 65535u), 65535u);
    const uint32_t qTheta = std::min(dm_f2uint((theta / kPi) * 65535u), 65535u);
    return (qTheta << 16) | qPhi;
}
inline float3 decodeVector(uint32_t qv) { // :43-49 (decodeNormal :59-65)
    const uint32_t qPhi = qv & 0xFFFF;
    const uint32_t qTheta = qv >> 16;
    const float phi = 2 * kPi * (qPhi / 65535.0f);
    const float theta = kPi * (qTheta / 65535.0f);
    return fromPolarYUp(phi, theta);
}
inline uint32_t encodeTexCoords(const float2 &tc) { // :67-71
    const uint32_t q0 = std::min(dm_f2uint((tc.x - std::floor(tc.x)) * 65535u), 65535u);
    const uint32_t q1 = std::min(dm_f2uint((tc.y - std::floor(tc.y)) * 65535u), 65535u);
    return (q1 << 16) | q0;
}
inline float2 decodeTexCoords(uint32_t qtc) { // :73-79
    return float2((qtc & 0xFFFF) / 65535.0f, (qtc >> 16) / 65535.0f);
}

inline void makeCoordinateSystem(const float3 &normal, float3* tangent, float3* bitangent) { // :92-100
    const float sign = normal.z >= 0 ? 1.0f : -1.0f;
    const float a = -1 / (sign + normal.z);
    const float b = normal.x * normal.y * a;
    *tangent = float3(1 + sign * normal.x * normal.x * a, sign * b, -sign * normal.x);
    *bitangent = float3(b, sign + normal.y * normal.y * a, -normal.y);
}

inline float3 offsetRayOrigin(const float3 &p, const float3 &geometricNormal) { // :114-143
    constexpr float kOrigin = 1.0f / 32.0f;
    constexpr float kFloatScale = 1.0f / 65536.0f;
    constexpr float kIntScale = 256.0f;
    const int32_t offsetInInt[3] = {
        dm_f2int(kIntScale * geometricNormal.x),
        dm_f2int(kIntScale * geometricNormal.y),
        dm_f2int(kIntScale * geometricNormal.z) };
    const float3 newP1(
        u2f((uint32_t)((int32_t)f2u(p.x) + (p.x < 0 ? -1 : 1) * offsetInInt[0])),
        u2f((uint32_t)((int32_t)f2u(p.y) + (p.y < 0 ? -1 : 1) * offsetInInt[1])),
        u2f((uint32_t)((int32_t)f2u(p.z) + (p.z < 0 ? -1 : 1) * offsetInInt[2])));
    const float3 newP2 = p + kFloatScale * geometricNormal;
    return float3(std::fabs(p.x) < kOrigin ? newP2.x : newP1.x,
                  std::fabs(p.y) < kOrigin ? newP2.y : newP1.y,
                  std::fabs(p.z) < kOrigin ? newP2.z : newP1.z);
}

struct ReferenceFrame { // :151-176
    float3 tangent, bitangent, normal;
    ReferenceFrame() {}
    ReferenceFrame(const float3 &_normal, const float3 &_tangent) : tangent(_tangent), normal(_normal) {
        bitangent = cross(normal, tangent);
    }
    float3 toLocal(const float3 &v) const { return float3(dot(tangent, v), dot(bitangent, v), dot(normal, v)); }
    float3 fromLocal(const float3 &v) const {
        return float3(dot(float3(tangent.x, bitangent.x, normal.x), v),
                      dot(float3(tangent.y, bitangent.y, normal.y), v),
                      dot(float3(tangent.z, bitangent.z, normal.z), v));
    }
};

inline void concentricSampleDisk(float u0, float u1, float* dx, float* dy) { // :285-317
    float r, theta;
    const float sx = 2 * u0 - 1;
    const float sy = 2 * u1 - 1;
    if (sx == 0 && sy == 0) {
        *dx = 0;
        *dy = 0;
        return;
    }
    if (sx >= -sy) {
        if (sx > sy) { r = sx; theta = sy / sx; }
        else { r = sy; theta = 2 - sx / sy; }
    }
    else {
        if (sx > sy) { r = -sy; theta = 6 + sx / sy; }
        else { r = -sx; theta = 4 + sy / sx; }
    }
    theta *= kPi / 4;
    float s, c;
    dm_sincos(theta, &s, &c);
    *dx = r * c;
    *dy = r * s;
}
inline float3 cosineSampleHemisphere(float u0, float u1) { // :319-323
    float x, y;
    concentricSampleDisk(u0, u1, &x, &y);
    return float3(x, y, std::sqrt(std::fmax(0.0f, 1.0f - x * x - y * y)));
}

// ---- BSDFs ------------------------------------------------------------------------------
// One tagged body instead of the reference's 16 direct-callable programs: same arithmetic
// (the author's USE_HARD_CODED_BSDF_FUNCTIONS path, common_device.cuh:890-963).
struct BSDF {
    uint32_t type; // 0 Lambert, 1 DiffuseAndSpecular (also SimplePBR after setup)
    float3 diffuseColor;   // Lambert: reflectance
    float3 specularF0Color;
    float roughness;

    // setupBSDFBody<...> (common_device.cuh:376-385, 778-826) with 1x1 textures.  REGULARIZE = BSDFFlags::Regularize
    // (:795-797, :821-823): the smoothness is halved, for DiffuseAndSpecular before the 0.999 clamp, for SimplePBR after it;
    // Lambert ignores the flag.
    template <bool REGULARIZE = false>
    void setup(uint32_t bsdfType, const float* p0, const float* p1, float p2) {
        if (bsdfType == 0) {
            type = 0;
            diffuseColor = float3(p0[0], p0[1], p0[2]);
            specularF0Color = float3(0.0f);
            roughness = 1.0f;
        }
        else if (bsdfType == 1) {
            type = 1;
            float smoothness = p2;
            if (REGULARIZE)
                smoothness *= 0.5f;
            smoothness = std::fmin(smoothness, 0.999f);
            diffuseColor = float3(p0[0], p0[1], p0[2]);
            specularF0Color = float3(p1[0], p1[1], p1[2]);
            roughness = 1 - smoothness;
        }
        else { // SimplePBR_BRDF(baseColor, 0.5f, smoothness, metallic) :767-776, :806-826
            type = 1;
            const float3 baseColor(p0[0], p0[1], p0[2]);
            float smoothness = std::fmin(1.0f - p1[1], 0.999f);
            if (REGULARIZE)
                smoothness *= 0.5f;
            const float metallic = p1[2];
            const float reflectance = 0.5f;
            diffuseColor = baseColor * (1 - metallic);
            specularF0Color = float3(0.16f * pow2(reflectance) * (1 - metallic)) + baseColor * metallic;
            roughness = 1 - smoothness;
        }
    }

    // GGXMicrofacetDistribution (:444-508)
    static float ggxEvaluate(float alpha_g, const float3 &m) {
        if (m.z <= 0.0f)
            return 0.0f;
        const float temp = pow2(m.x) + pow2(m.y) + pow2(m.z * alpha_g);
        return pow2(alpha_g) / (kPi * pow2(temp));
    }
    static float ggxSmithG1(float alpha_g, const float3 &v, const float3 &m) {
        if (dot(v, m) * v.z <= 0)
            return 0.0f;
        const float temp = pow2(alpha_g) * (pow2(v.x) + pow2(v.y)) / pow2(v.z);
        return 2 / (1 + std::sqrt(1 + temp));
    }
    static float ggxHeightCorrelatedSmithG(float alpha_g, const float3 &v1, const float3 &v2, const float3 &m) {
        const float t1 = pow2(alpha_g) * (pow2(v1.x) + pow2(v1.y)) / pow2(v1.z);
        const float t2 = pow2(alpha_g) * (pow2(v2.x) + pow2(v2.y)) / pow2(v2.z);
        const float Lambda1 = (-1 + std::sqrt(1 + t1)) / 2;
        const float Lambda2 = (-1 + std::sqrt(1 + t2)) / 2;
        const float chi1 = (dot(v1, m) / v1.z) > 0 ? 1.0f : 0.0f;
        const float chi2 = (dot(v2, m) / v2.z) > 0 ? 1.0f : 0.0f;
        return chi1 * chi2 / (1 + Lambda1 + Lambda2);
    }
    static float ggxEvaluatePDF(float alpha_g, const float3 &v, const float3 &m) {
        return ggxSmithG1(alpha_g, v, m) * std::fabs(dot(v, m)) * ggxEvaluate(alpha_g, m) / std::fabs(v.z);
    }
    static float ggxSample(float alpha_g, const float3 &v, float u0, float u1, float3* m, float* mPDensity) { // :470-504
        const float3 sv = normalize(float3(alpha_g * v.x, alpha_g * v.y, v.z));
        const float distIn2D = std::sqrt(sv.x * sv.x + sv.y * sv.y);
        const float recDistIn2D = 1.0f / distIn2D;
        const float3 T1 = (sv.z < 0.9999f) ? float3(sv.y * recDistIn2D, -sv.x * recDistIn2D, 0) : float3(1, 0, 0);
        const float3 T2(T1.y * sv.z, -T1.x * sv.z, distIn2D);
        const float a = 1.0f / (1.0f + sv.z);
        const float r = std::sqrt(u0);
        const float phi = kPi * ((u1 < a) ? u1 / a : 1 + (u1 - a) / (1.0f - a));
        float sinPhi, cosPhi;
        dm_sincos(phi, &sinPhi, &cosPhi);
        const float P1 = r * cosPhi;
        const float P2 = r * sinPhi * ((u1 < a) ? 1.0f : sv.z);
        *m = P1 * T1 + P2 * T2 + std::sqrt(1.0f - P1 * P1 - P2 * P2) * sv;
        *m = normalize(float3(alpha_g * m->x, alpha_g * m->y, m->z));
        const float D = ggxEvaluate(alpha_g, *m);
        *mPDensity = ggxSmithG1(alpha_g, v, *m) * std::fabs(dot(v, *m)) * D / std::fabs(v.z);
        return D;
    }

    float3 evaluate(const float3 &vGiven, const float3 &vSampled) const {
        if (type == 0) { // LambertBRDF::evaluate :358-363
            if (vGiven.z * vSampled.z > 0)
                return diffuseColor / kPi;
            return float3(0.0f);
        }
        // DiffuseAndSpecularBRDF::evaluate :648-690
        const float alpha_g = roughness * roughness;
        if (vSampled.z * vGiven.z <= 0)
            return float3(0.0f);
        const bool entering = vGiven.z >= 0.0f;
        const float3 dirV = entering ? vGiven : -vGiven;
        const float3 dirL = entering ? vSampled : -vSampled;
        const float3 m = normalize(dirL + dirV);
        const float dotLH = dot(dirL, m);
        const float oneMinusDotLH5 = pow5(1 - dotLH);
        const float D = ggxEvaluate(alpha_g, m);
        const float G = ggxHeightCorrelatedSmithG(alpha_g, dirL, dirV, m);
        const float3 F = lerp3(specularF0Color, float3(1.0f), oneMinusDotLH5);
        const float microfacetDenom = 4 * dirL.z * dirV.z;
        float3 specularValue = F * ((D * G) / microfacetDenom);
        if (G == 0)
            specularValue = float3(0.0f);
        const float F_D90 = 0.5f * roughness + 2 * roughness * dotLH * dotLH;
        const float oneMinusDotVN5 = pow5(1 - dirV.z);
        const float oneMinusDotLN5 = pow5(1 - dirL.z);
        const float diffuseFresnelOut = lerpf(1.0f, F_D90, oneMinusDotVN5);
        const float diffuseFresnelIn = lerpf(1.0f, F_D90, oneMinusDotLN5);
        const float3 diffuseValue = diffuseColor *
            (diffuseFresnelOut * diffuseFresnelIn * lerpf(1.0f, 1.0f / 1.51f, roughness) / kPi);
        return diffuseValue + specularValue;
    }

    float3 evaluateDHReflectanceEstimate(const float3 &vGiven) const {
        if (type == 0) // :372-374
            return diffuseColor;
        // :736-764
        const bool entering = vGiven.z >= 0.0f;
        const float3 dirV = entering ? vGiven : -vGiven;
        const float expectedCosTheta_d = dirV.z;
        const float expectedF_D90 = 0.5f * roughness + 2 * roughness * pow2(expectedCosTheta_d);
        const float oneMinusDotVN5 = pow5(1 - dirV.z);
        const float expectedDiffFGiven = lerpf(1.0f, expectedF_D90, oneMinusDotVN5);
        const float expectedDiffFSampled = 1.0f;
        const float3 diffuseDHR = diffuseColor * expectedDiffFGiven * expectedDiffFSampled * lerpf(1.0f, 1.0f / 1.51f, roughness);
        const float expectedOneMinusDotVH5 = pow5(1 - dirV.z) * (1 - roughness);
        const float3 specularDHR = lerp3(specularF0Color, float3(1.0f), expectedOneMinusDotVH5);
        return min3(diffuseDHR + specularDHR, float3(1.0f));
    }

    float3 sampleThroughput(const float3 &vGiven, float uDir0, float uDir1, float3* vSampled, float* dirPDensity) const {
        if (type == 0) { // :348-357
            *vSampled = cosineSampleHemisphere(uDir0, uDir1);
            *dirPDensity = vSampled->z / kPi;
            if (vGiven.z <= 0.0f)
                vSampled->z *= -1;
            return diffuseColor;
        }
        // :532-647
        const float alpha_g = roughness * roughness;
        const bool entering = vGiven.z >= 0.0f;
        float3 dirL;
        const float3 dirV = entering ? vGiven : -vGiven;
        const float oneMinusDotVN5 = pow5(1 - dirV.z);
        const float expectedF_D90 = 0.5f * roughness + 2 * roughness * vGiven.z * vGiven.z;
        const float expectedDiffuseFresnel = lerpf(1.0f, expectedF_D90, oneMinusDotVN5);
        const float iBaseColor = sRGB_calcLuminance(diffuseColor) * pow2(expectedDiffuseFresnel) *
            lerpf(1.0f, 1.0f / 1.51f, roughness);
        const float expectedOneMinusDotVH5 = pow5(1 - dirV.z);
        const float iSpecularF0 = sRGB_calcLuminance(specularF0Color);
        const float diffuseWeight = iBaseColor;
        const float specularWeight = lerpf(iSpecularF0, 1.0f, expectedOneMinusDotVH5);
        const float sumWeights = diffuseWeight + specularWeight;
        if (sumWeights == 0.0f) {
            *dirPDensity = 0.0f;
            return float3(0.0f);
        }
        const float uComponent = uDir1;
        float diffuseDirPDF, specularDirPDF;
        float3 m;
        float dotLH;
        float D;
        if (sumWeights * uComponent < diffuseWeight) {
            uDir1 = (sumWeights * uComponent - 0) / diffuseWeight;
            dirL = cosineSampleHemisphere(uDir0, uDir1);
            diffuseDirPDF = dirL.z / kPi;
            m = normalize(dirL + dirV);
            dotLH = std::fmin(dot(dirL, m), 1.0f);
            const float commonPDFTerm = 1.0f / (4 * dotLH);
            specularDirPDF = commonPDFTerm * ggxEvaluatePDF(alpha_g, dirV, m);
            D = ggxEvaluate(alpha_g, m);
        }
        else {
            uDir1 = (sumWeights * uComponent - diffuseWeight) / specularWeight;
            float mPDF;
            D = ggxSample(alpha_g, dirV, uDir0, uDir1, &m, &mPDF);
            const float dotVH = std::fmin(dot(dirV, m), 1.0f);
            dotLH = dotVH;
            dirL = 2 * dotVH * m - dirV;
            if (dirL.z * dirV.z <= 0) {
                *dirPDensity = 0.0f;
                return float3(0.0f);
            }
            const float commonPDFTerm = 1.0f / (4 * dotLH);
            specularDirPDF = commonPDFTerm * mPDF;
            diffuseDirPDF = dirL.z / kPi;
        }
        const float oneMinusDotLH5 = pow5(1 - dotLH);
        const float G = ggxHeightCorrelatedSmithG(alpha_g, dirL, dirV, m);
        const float3 F = lerp3(specularF0Color, float3(1.0f), oneMinusDotLH5);
        const float microfacetDenom = 4 * dirL.z * dirV.z;
        float3 specularValue = F * ((D * G) / microfacetDenom);
        if (G == 0)
            specularValue = float3(0.0f);
        const float F_D90 = 0.5f * roughness + 2 * roughness * dotLH * dotLH;
        const float oneMinusDotLN5 = pow5(1 - dirL.z);
        const float diffuseFresnelOut = lerpf(1.0f, F_D90, oneMinusDotVN5);
        const float diffuseFresnelIn = lerpf(1.0f, F_D90, oneMinusDotLN5);
        const float3 diffuseValue = diffuseColor *
            (diffuseFresnelOut * diffuseFresnelIn * lerpf(1.0f, 1.0f / 1.51f, roughness) / kPi);
        float3 ret = diffuseValue + specularValue;
        *vSampled = entering ? dirL : -dirL;
        *dirPDensity = (diffuseDirPDF * diffuseWeight + specularDirPDF * specularWeight) / sumWeights;
        ret *= dirL.z / *dirPDensity;
        return ret;
    }

    float evaluatePDF(const float3 &vGiven, const float3 &vSampled) const {
        if (type == 0) { // :364-369
            if (vGiven.z * vSampled.z > 0)
                return std::fabs(vSampled.z) / kPi;
            return 0.0f;
        }
        // :691-734
        const float alpha_g = roughness * roughness;
        const bool entering = vGiven.z >= 0.0f;
        const float3 dirV = entering ? vGiven : -vGiven;
        const float3 dirL = entering ? vSampled : -vSampled;
        const float3 m = normalize(dirL + dirV);
        const float dotLH = dot(dirL, m);
        const float commonPDFTerm = 1.0f / (4 * dotLH);
        const float expectedF_D90 = 0.5f * roughness + 2 * roughness * vGiven.z * vGiven.z;
        const float oneMinusDotVN5 = pow5(1 - dirV.z);
        const float expectedDiffuseFresnel = lerpf(1.0f, expectedF_D90, oneMinusDotVN5);
        const float iBaseColor = sRGB_calcLuminance(diffuseColor) * pow2(expectedDiffuseFresnel) *
            lerpf(1.0f, 1.0f / 1.51f, roughness);
        const float expectedOneMinusDotVH5 = pow5(1 - dirV.z);
        const float iSpecularF0 = sRGB_calcLuminance(specularF0Color);
        const float diffuseWeight = iBaseColor;
        const float specularWeight = lerpf(iSpecularF0, 1.0f, expectedOneMinusDotVH5);
        const float sumWeights = diffuseWeight + specularWeight;
        if (sumWeights == 0.0f)
            return 0.0f;
        const float diffuseDirPDF = dirL.z / kPi;
        const float specularDirPDF = commonPDFTerm * ggxEvaluatePDF(alpha_g, dirV, m);
        return (diffuseDirPDF * diffuseWeight + specularDirPDF * specularWeight) / sumWeights;
    }
};

} // namespace orc
