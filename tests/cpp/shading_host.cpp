// shading_host.cpp — the device shading layer of gfxexp_b200/csrc/shading.cuh (BSDFs, sampling warps, polar / barycentric /
// texture-coordinate encoders, makeCoordinateSystem, offsetRayOrigin), compiled for the CPU without changes.
//
// Shims stand in for the three device intrinsics the header uses and for the device's unsigned min; with -ffp-contract=off
// (the host counterpart of nvcc's -fmad=false) every float operation rounds as on sm_90a.  The entry point runs the op table
// of shading_debug.cuh (the one gfx_shading_debug runs on the device) over n records.
#include <cmath>
#include <cstdint>
#include <cstring>

#include <cuda_runtime.h>

static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline int __clz(uint32_t x) { return x ? __builtin_clz(x) : 32; }
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }

#include "../../gfxexp_b200/csrc/shading_debug.cuh"

extern "C" int shading_host(int op, const float* material, const float* in, uint32_t n, float* out) {
    if (op < 0 || op >= gfx::kShadingDebugNumOps)
        return 1;
    for (uint32_t i = 0; i < n; ++i)
        gfx::shadingDebugOp(op, material, in + gfx::kShadingDebugStride * (size_t)i, out + gfx::kShadingDebugStride * (size_t)i);
    return 0;
}
