// restir_common.cuh — reservoir storage, neighbour test and visibility-ray requests shared by the original
// (restir.cu) and the rearchitected (restir_rearch.cu) ReSTIR DI kernels.
#pragma once
#include "lighting.cuh"
#include "context.h"

namespace gfx {

struct Reservoir { // restir_di_shared.h:106-139
    LightSample sample;
    float sumWeights;
    uint32_t streamLength;
    GFX_D void initialize(const LightSample &s) { sample = s; sumWeights = 0; streamLength = 0; }
    GFX_D bool update(const LightSample &newSample, float weight, float u) {
        sumWeights += weight;
        const bool accepted = u < weight / sumWeights;
        if (accepted)
            sample = newSample;
        ++streamLength;
        return accepted;
    }
};


GFX_D Reservoir loadReservoir(const DevFrame &f, uint32_t idx, size_t pix) {
    const size_t n = (size_t)f.W * f.H;
    const float4 a = f.reservoir[idx][pix], b = f.reservoir[idx][n + pix], c = f.reservoir[idx][2 * n + pix];
    Reservoir r;
    r.sample.emittance = f3(a.x, a.y, a.z);
    r.sumWeights = a.w;
    r.sample.position = f3(b.x, b.y, b.z);
    const uint32_t m = __float_as_uint(b.w);
    r.streamLength = m & 0x7FFFFFFFu;
    r.sample.atInfinity = m >> 31;
    r.sample.normal = f3(c.x, c.y, c.z);
    return r;
}
GFX_D void storeReservoir(const DevFrame &f, uint32_t idx, size_t pix, const Reservoir &r) {
    const size_t n = (size_t)f.W * f.H;
    f.reservoir[idx][pix] = make_float4(r.sample.emittance.x, r.sample.emittance.y, r.sample.emittance.z, r.sumWeights);
    f.reservoir[idx][n + pix] = make_float4(r.sample.position.x, r.sample.position.y, r.sample.position.z,
                                            __uint_as_float((r.streamLength & 0x7FFFFFFFu) | (r.sample.atInfinity << 31)));
    f.reservoir[idx][2 * n + pix] = make_float4(r.sample.normal.x, r.sample.normal.y, r.sample.normal.z, 0.0f);
}

// M is kept in 31 bits next to atInfinity.  Spatial passes add up to 16 stream lengths per pass and any number of passes may
// run, so the sum saturates at 2^31 - 1 instead of wrapping into atInfinity (the reference keeps a full uint32_t, which
// wraps at 2^32).  Both inputs are at most 2^31 - 1, so the 32-bit sum cannot wrap.
GFX_D uint32_t saturatedStreamLength(uint32_t a, uint32_t b) { return min(a + b, 0x7FFFFFFFu); }

template <bool testGeometry>
GFX_D bool testNeighbor(const DevFrame &f, const DevCamera &camera, uint32_t nbBufIdx, int nbx, int nby, float dist,
                        const f3 &normalInWorld) { // restir_di_shared.h:747-771
    if (nbx < 0 || nbx >= (int)f.W || nby < 0 || nby >= (int)f.H)
        return false;
    const size_t nbPix = (size_t)nby * f.W + nbx;
    if (f.gb0[nbBufIdx][nbPix].x == 0xFFFFFFFFu)
        return false;
    if (testGeometry) {
        const float4 g2 = f.gb2[nbBufIdx][nbPix];
        const uint4 g3 = f.gb3[nbBufIdx][nbPix];
        const f3 nbPositionInWorld(g2.x, g2.y, g2.z);
        const f3 nbNormalInWorld = decodeVector(g3.x);
        const float nbDist = length(camera.position - nbPositionInWorld);
        if (fabsf(nbDist - dist) / dist > 0.1f || dot(normalInWorld, nbNormalInWorld) < 0.9f)
            return false;
    }
    return true;
}


// ---------------------------------------------------------------------------------------------
// A visibility ray requested by a pixel (wavefront mode): appended to the frame's queue with one atomic per
// warp (ballot compaction), traced by trace.cu's persistent kernel, answered in f.visibility[pixel].
struct RayRequest {
    f3 org, dir;
    float tmax;
    uint32_t pixel;
};
GFX_D void enqueueRay(const DevFrame &f, unsigned long long* rayCounter, bool want, const RayRequest &r) {
    const uint32_t lane = (threadIdx.x + threadIdx.y * blockDim.x) & 31u;
    const uint32_t mask = __ballot_sync(0xFFFFFFFFu, want);
    if (mask == 0)
        return;
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if ((int)lane == leader) {
        base = atomicAdd(f.rayCounters, (uint32_t)__popc(mask));
        atomicAdd(rayCounter, (unsigned long long)__popc(mask));
    }
    base = __shfl_sync(0xFFFFFFFFu, base, leader);
    if (want) {
        const uint32_t slot = base + __popc(mask & ((1u << lane) - 1u));
        f.rayQueue[2 * (size_t)slot] = make_float4(r.org.x, r.org.y, r.org.z, 0.0f);
        f.rayQueue[2 * (size_t)slot + 1] = make_float4(r.dir.x, r.dir.y, r.dir.z, r.tmax);
        f.rayPixel[slot] = r.pixel;
    }
}
GFX_D void visibilityRay(const f3 &shadingPoint, const LightSample &ls, uint32_t pixel, RayRequest* r) {
    // the ray of evaluateVisibility / performDirectLighting<..., true> (restir_di_shared.h:518-582)
    f3 shadowRayDir = ls.atInfinity ? ls.position : (ls.position - shadingPoint);
    const float dist2 = sqLength(shadowRayDir);
    float dist = sqrtf(dist2);
    shadowRayDir /= dist;
    if (ls.atInfinity)
        dist = 1e+10f;
    r->org = shadingPoint;
    r->dir = shadowRayDir;
    r->tmax = dist * 0.9999f;
    r->pixel = pixel;
}

} // namespace gfx
