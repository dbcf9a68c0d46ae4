// oracle/shading_export.cpp — TEST INFRASTRUCTURE: orc_shading_debug, the op table of gfx_shading_debug
// (gfxexp_b200/csrc/shading_debug.cuh) over this oracle's restatement in shading.h, so that tests/test_shading_host.py can
// hold the device header's CPU build against it bit for bit at inputs no scene reaches.
//
// material: 9 floats {bsdfType, p0[3], p1[3], p2, regularize != 0}; every record is 8 floats in and out, unused output
// slots 0, integer codes as their bits.  Ops: 0 evaluate, 1 evaluatePDF, 2 sampleThroughput, 3 evaluateDHReflectanceEstimate,
// 4 concentricSampleDisk, 5 cosineSampleHemisphere, 6 toPolarYUp, 7 fromPolarYUp, 8 encodeVector, 9 decodeVector,
// 10 encodeBarycentric, 11 decodeBarycentric, 12 encodeTexCoords, 13 decodeTexCoords, 14 makeCoordinateSystem,
// 15 offsetRayOrigin.
#include "shading.h"
#include <cstddef>

namespace {

using namespace orc;

void shadingOp(int op, const float* mat, const float* a, float* o) {
    for (int k = 0; k < 8; ++k)
        o[k] = 0.0f;
    if (op <= 3) {
        BSDF bsdf;
        const uint32_t bsdfType = (uint32_t)mat[0];
        if (mat[8] != 0.0f)
            bsdf.setup<true>(bsdfType, mat + 1, mat + 4, mat[7]);
        else
            bsdf.setup<false>(bsdfType, mat + 1, mat + 4, mat[7]);
        const float3 vGiven(a[0], a[1], a[2]);
        if (op == 0) {
            const float3 f = bsdf.evaluate(vGiven, float3(a[3], a[4], a[5]));
            o[0] = f.x; o[1] = f.y; o[2] = f.z;
        }
        else if (op == 1) {
            o[0] = bsdf.evaluatePDF(vGiven, float3(a[3], a[4], a[5]));
        }
        else if (op == 2) {
            float3 vSampled(0.0f);
            float pdf = 0.0f;
            const float3 t = bsdf.sampleThroughput(vGiven, a[3], a[4], &vSampled, &pdf);
            o[0] = t.x; o[1] = t.y; o[2] = t.z;
            o[3] = vSampled.x; o[4] = vSampled.y; o[5] = vSampled.z;
            o[6] = pdf;
        }
        else {
            const float3 r = bsdf.evaluateDHReflectanceEstimate(vGiven);
            o[0] = r.x; o[1] = r.y; o[2] = r.z;
        }
        return;
    }
    switch (op) {
    case 4: concentricSampleDisk(a[0], a[1], &o[0], &o[1]); break;
    case 5: { const float3 v = cosineSampleHemisphere(a[0], a[1]); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 6: toPolarYUp(float3(a[0], a[1], a[2]), &o[0], &o[1]); break;
    case 7: { const float3 v = fromPolarYUp(a[0], a[1]); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 8: o[0] = u2f(encodeVector(float3(a[0], a[1], a[2]))); break;
    case 9: { const float3 v = decodeVector(f2u(a[0])); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 10: o[0] = u2f((uint32_t)encodeBarycentric(a[0])); break;
    case 11: o[0] = decodeBarycentric((uint16_t)(f2u(a[0]) & 0xFFFFu)); break;
    case 12: o[0] = u2f(encodeTexCoords(float2(a[0], a[1]))); break;
    case 13: { const float2 t = decodeTexCoords(f2u(a[0])); o[0] = t.x; o[1] = t.y; break; }
    case 14: {
        float3 t, b;
        makeCoordinateSystem(float3(a[0], a[1], a[2]), &t, &b);
        o[0] = t.x; o[1] = t.y; o[2] = t.z;
        o[3] = b.x; o[4] = b.y; o[5] = b.z;
        break;
    }
    case 15: { const float3 p = offsetRayOrigin(float3(a[0], a[1], a[2]), float3(a[3], a[4], a[5])); o[0] = p.x; o[1] = p.y; o[2] = p.z; break; }
    default: break;
    }
}

} // namespace

extern "C" int orc_shading_debug(int op, const float* material, const float* in, size_t n, float* out) {
    if (op < 0 || op > 15)
        return 1;
    for (size_t i = 0; i < n; ++i)
        shadingOp(op, material, in + 8 * i, out + 8 * i);
    return 0;
}
