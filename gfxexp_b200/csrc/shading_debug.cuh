// shading_debug.cuh — the op table of the shading test hook (gfx_shading_debug): one record of the shading layer of
// shading.cuh per call, so that tests can run the BSDFs, warps, encoders and frames on arrays.  The same function runs in
// the device kernel (lights.cu, k_shadingDebug) and in the CPU build of these headers (tests/cpp/shading_host.cpp); the
// oracle's orc_shading_debug (oracle/shading_export.cpp) keeps the same table over oracle/shading.h.
//
// material: 9 floats {bsdfType, p0[3], p1[3], p2, regularize != 0} as setupBSDFBody reads a material with 1x1 textures.
// Every record is kShadingDebugStride floats in and out; unused output slots are 0, integer codes travel as their bits.
//   op  in                                  out
//   0   vGiven, vSampled                    evaluate (rgb)
//   1   vGiven, vSampled                    evaluatePDF
//   2   vGiven, u0, u1                      sampleThroughput (rgb), vSampled, dirPDensity
//   3   vGiven                              evaluateDHReflectanceEstimate (rgb)
//   4   u0, u1                              concentricSampleDisk (dx, dy)
//   5   u0, u1                              cosineSampleHemisphere
//   6   v                                   toPolarYUp (phi, theta)
//   7   phi, theta                          fromPolarYUp
//   8   v                                   encodeVector (code bits)
//   9   code bits                           decodeVector
//   10  bc                                  encodeBarycentric (code bits)
//   11  code bits (low 16 used)             decodeBarycentric
//   12  u, v                                encodeTexCoords (code bits)
//   13  code bits                           decodeTexCoords
//   14  normal                              makeCoordinateSystem (tangent, bitangent)
//   15  p, geometric normal                 offsetRayOrigin
#pragma once
#include "shading.cuh"

namespace gfx {

constexpr int kShadingDebugNumOps = 16;
constexpr int kShadingDebugStride = 8;

GFX_D void shadingDebugOp(int op, const float* mat, const float* a, float* o) {
    for (int k = 0; k < kShadingDebugStride; ++k)
        o[k] = 0.0f;
    if (op <= 3) {
        BSDF bsdf;
        const uint32_t bsdfType = (uint32_t)mat[0];
        if (mat[8] != 0.0f)
            bsdf.setup<true>(bsdfType, mat + 1, mat + 4, mat[7]);
        else
            bsdf.setup<false>(bsdfType, mat + 1, mat + 4, mat[7]);
        const f3 vGiven(a[0], a[1], a[2]);
        if (op == 0) {
            const f3 f = bsdf.evaluate(vGiven, f3(a[3], a[4], a[5]));
            o[0] = f.x; o[1] = f.y; o[2] = f.z;
        }
        else if (op == 1) {
            o[0] = bsdf.evaluatePDF(vGiven, f3(a[3], a[4], a[5]));
        }
        else if (op == 2) {
            f3 vSampled(0.0f);
            float pdf = 0.0f;
            const f3 t = bsdf.sampleThroughput(vGiven, a[3], a[4], &vSampled, &pdf);
            o[0] = t.x; o[1] = t.y; o[2] = t.z;
            o[3] = vSampled.x; o[4] = vSampled.y; o[5] = vSampled.z;
            o[6] = pdf;
        }
        else {
            const f3 r = bsdf.evaluateDHReflectanceEstimate(vGiven);
            o[0] = r.x; o[1] = r.y; o[2] = r.z;
        }
        return;
    }
    switch (op) {
    case 4: concentricSampleDisk(a[0], a[1], &o[0], &o[1]); break;
    case 5: { const f3 v = cosineSampleHemisphere(a[0], a[1]); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 6: toPolarYUp(f3(a[0], a[1], a[2]), &o[0], &o[1]); break;
    case 7: { const f3 v = fromPolarYUp(a[0], a[1]); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 8: o[0] = __uint_as_float(encodeVector(f3(a[0], a[1], a[2]))); break;
    case 9: { const f3 v = decodeVector(__float_as_uint(a[0])); o[0] = v.x; o[1] = v.y; o[2] = v.z; break; }
    case 10: o[0] = __uint_as_float((uint32_t)encodeBarycentric(a[0])); break;
    case 11: o[0] = decodeBarycentric((uint16_t)(__float_as_uint(a[0]) & 0xFFFFu)); break;
    case 12: o[0] = __uint_as_float(encodeTexCoords(f2(a[0], a[1]))); break;
    case 13: { const f2 t = decodeTexCoords(__float_as_uint(a[0])); o[0] = t.x; o[1] = t.y; break; }
    case 14: {
        f3 t, b;
        makeCoordinateSystem(f3(a[0], a[1], a[2]), &t, &b);
        o[0] = t.x; o[1] = t.y; o[2] = t.z;
        o[3] = b.x; o[4] = b.y; o[5] = b.z;
        break;
    }
    case 15: { const f3 p = offsetRayOrigin(f3(a[0], a[1], a[2]), f3(a[3], a[4], a[5])); o[0] = p.x; o[1] = p.y; o[2] = p.z; break; }
    default: break;
    }
}

} // namespace gfx
