// pathtrace.cu — the unidirectional path tracer as a wavefront pipeline on sm_90a.
//
// Replaces pathTracing.optixPipeline.launch(W, H, 1) (path_tracing/path_tracing_main.cpp:1780-1789) and its
// programs pathTrace_rayGen_generic / pathTrace_closestHit_generic / miss / performNextEventEstimation
// (path_tracing/gpu_kernels/optix_pathtracing_kernels.cu:18-71, 73-216, 218-300, 310-341) with
// computeSurfacePoint<> (path_tracing/path_tracing_shared.h:484-621); compile-time switches as in :12-16
// (area sampling, implicit + explicit light sampling, MIS).
//
// OptiX runs this as a per-pixel megakernel that recurses into closest-hit programs.  Here a path is a
// record in HBM and one frame is
//     k_ptFirstHit                          shade the G-buffer hit: emission, NEE (shadow ray request), BSDF sample
//     for pathLength = 2 .. maxPathLength
//         k_traceWavefront<any>             shadow rays of the previous vertex; the writer adds the unoccluded
//                                           NEE contribution to the path's radiance (keeps the reference's
//                                           summation order: NEE of vertex k before the emission of vertex k+1)
//         k_traceWavefront<closest>         extension rays -> (geometry, primitive, barycentrics) per queue slot
//         k_ptBounce                        closest-hit program on the compacted queue of live paths
//     k_ptAccumulate                        running mean into the beauty buffer
// Queues are compacted with one atomic per warp (ballot), each round has its own counters (one memset per
// frame) and the trace kernel is the persistent-thread kernel of wavefront.cuh, so lanes that finish early or
// whose path died do not idle.  Per-path state: rng (frame.rng), alpha|prevDirPDensity and radiance as two
// float4 planes indexed by pixel.  The RNG draw order of every pixel is the reference's.
#include "pathtrace.cuh"

namespace gfx {

// One path vertex: NEE + next direction.  The ReGIR variant (regir/gpu_kernels/optix_pathtracing_kernels.cu) draws its
// light sample from the cell reservoirs and runs the length limit and a Russian roulette of the ray-generation
// loop *before* the extension ray is traced (:254-263, `if constexpr (useReGIR || ...)`), in addition to the
// roulette of the closest-hit program.
template <bool REGIR>
GFX_D void shadeVertexVariant(const DevScene &s, const DevRegir &rg, const DevFrameParams &p, const f3 &positionInWorld,
                              const f3 &vOutLocal, const ReferenceFrame &shadingFrame, const BSDF &bsdf, PCG32RNG &rng, f3 alpha,
                              uint32_t pathLength, f3* radiance, VertexOutput* out) {
    if (REGIR) {
        neeRegir(s, rg, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, alpha, radiance, out);
        sampleNextDirection(vOutLocal, shadingFrame, bsdf, rng, alpha, out);
        if (out->wantExtension) {
            if (pathLength + 1 >= p.maxPathLength) {
                out->wantExtension = false;
            }
            else {
                const float continueProb = fminf(sRGB_calcLuminance(out->alpha) / sRGB_calcLuminance(f3(1.0f)), 1.0f);
                if (rng.getFloat0cTo1o() >= continueProb)
                    out->wantExtension = false;
                else
                    out->alpha /= continueProb;
            }
        }
    }
    else {
        shadeVertex(s, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, alpha, radiance, out);
    }
}

// the bounce kernel's variants: GFX_PT_BASELINE, GFX_PT_REGIR, and GFX_PT_SVGF without and with GFX_SVGF_MOLLIFY_SPECULAR
enum class PtVariant { Baseline, Regir, Svgf, SvgfMollify };

// pathTrace_rayGen_generic up to the path extension loop (:73-160).  BUMP: GfxFrameParams::enableBumpMapping (a kernel of its own,
// so that the frames without it run the code they ran before it existed; likewise k_ptBounce)
template <bool REGIR, bool BUMP>
__global__ void GFX_BOUNCE_BOUNDS k_ptFirstHit(DevScene s, DevFrame f, DevFrameParams p, DevPathState ps, DevRegir rg) {
    const uint32_t x = blockIdx.x * 8 + threadIdx.x;
    const uint32_t y = p.y0 + blockIdx.y * 8 + threadIdx.y;
    const uint32_t lane = (threadIdx.x + threadIdx.y * blockDim.x) & 31u;
    const bool inside = x < f.W && y < p.y1;
    const uint32_t pix = inside ? y * f.W + x : 0u;

    bool alive = false;
    f3 positionInWorld(0.0f);
    VertexOutput v;
    v.wantShadow = v.wantExtension = false;
    if (inside) {
        const uint4 gb0 = f.gb0[p.bufferIndex][pix];
        f3 radiance(0.001f, 0.001f, 0.001f);
        if (gb0.x != 0xFFFFFFFFu) {
            GBufferHit h;
            decodeGBufferHit(s, gb0, &h);
            const f3 alpha(1.0f);
            PCG32RNG rng{ f.rng[pix] };
            const GfxMaterialDesc* mat = s.materials + h.mesh.materialSlot;
            const f3 vOut = normalize(p.camera.position - h.sp.positionInWorld);
            const float frontHit = dot(vOut, h.sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            positionInWorld = offsetRayOrigin(h.sp.positionInWorld, frontHit * h.sp.geometricNormalInWorld);
            ReferenceFrame shadingFrame(h.sp.shadingNormalInWorld, h.sp.texCoord0DirInWorld);
            if (BUMP) // path_tracing :117-121, regir :200-203
                shadingFrame = bumpShadingFrameAtHit(s, h.mesh, gb0.z, h.bcB, h.bcC, shadingFrame);
            const f3 vOutLocal = shadingFrame.toLocal(vOut);

            radiance = f3(0.0f);
            if (vOutLocal.z > 0 && mat->hasEmittance)
                radiance += alpha * f3(mat->emittance[0], mat->emittance[1], mat->emittance[2]) / kPi;
            const BSDF bsdf = setupBsdfAtHit(s, h.mesh, gb0.z, h.bcB, h.bcC);
            shadeVertexVariant<REGIR>(s, rg, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, alpha, 1u, &radiance, &v);
            f.rng[pix] = rng.state;
            ps.alphaPdf[pix] = make_float4(v.alpha.x, v.alpha.y, v.alpha.z, v.dirPDensity);
            alive = true;
        }
        else if (s.env.enabled) { // :200-207: the environment seen directly; the miss program left (u, v) in the barycentrics
            radiance = s.env.powerCoeff * envFetch(s.env, decodeBarycentric((uint16_t)(gb0.w & 0xFFFFu)), decodeBarycentric((uint16_t)(gb0.w >> 16)));
        }
        ps.radiance[pix] = make_float4(radiance.x, radiance.y, radiance.z, 0.0f);
    }
    emitRays(s, ps, ps.counters, 0u, lane, pix, positionInWorld, v, alive);
}

// pathTrace_closestHit_generic (:218-300) + the bookkeeping of the path extension loop (:161-194) for the
// compacted queue of live paths; `round` = pathLength - 2 selects the queue parity and the counters.  The SVGF app's
// closest-hit program (svgf :381-468) and miss program (:482-513) are the baseline's but for two differences: no Russian
// roulette at pathLength 2 (round 0), whose random number is still drawn (:438-441), and with SvgfMollify the BSDF set up with
// BSDFFlags::Regularize (:446-450).
template <PtVariant V, bool BUMP>
__global__ void GFX_BOUNCE_BOUNDS k_ptBounce(DevScene s, DevFrame f, DevFrameParams p, DevPathState ps, DevRegir rg, uint32_t round,
                                             uint32_t maxLengthTerminate) {
    constexpr bool REGIR = V == PtVariant::Regir, SVGF = V == PtVariant::Svgf || V == PtVariant::SvgfMollify;
    const uint32_t curQueue = round & 1u, nextQueue = curQueue ^ 1u;
    const uint32_t* roundCounters = ps.counters + 4 * round;
    uint32_t* nextCounters = ps.counters + 4 * (round + 1);
    const uint32_t count = roundCounters[0];
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warpsPerGrid = gridDim.x * (blockDim.x >> 5);
    const uint32_t warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const float initImportance = sRGB_calcLuminance(f3(1.0f));

    for (uint32_t base = warp * 32u; base < count; base += warpsPerGrid * 32u) {
        const uint32_t slot = base + lane;
        bool alive = false;
        uint32_t pix = 0;
        f3 positionInWorld(0.0f);
        VertexOutput v;
        v.wantShadow = v.wantExtension = false;
        if (slot < count) {
            const uint4 hit = ps.extHits[slot];
            if (hit.y != 0xFFFFFFFFu) { // miss program: no environment light, the path ends
                pix = ps.extPixel[curQueue][slot];
                const float4 r0 = ps.extRays[curQueue][2 * (size_t)slot];
                const float4 r1 = ps.extRays[curQueue][2 * (size_t)slot + 1];
                const f3 rayOrigin(r0.x, r0.y, r0.z), rayDir(r1.x, r1.y, r1.z);
                const float4 ap = ps.alphaPdf[pix];
                f3 alpha(ap.x, ap.y, ap.z);
                const float prevDirPDensity = ap.w;
                const float4 rad = ps.radiance[pix];
                f3 radiance(rad.x, rad.y, rad.z);
                PCG32RNG rng{ f.rng[pix] };

                HitVertex h;
                setupHitVertex<BUMP>(s, hit, rayDir, &h);
                positionInWorld = h.positionInWorld;
                const GfxMaterialDesc* mat = s.materials + h.mesh.materialSlot;

                // implicit light sampling, MIS against the hypothetical NEE density (:262-275)
                if (h.vOutLocal.z > 0 && mat->hasEmittance) {
                    const f3 emittance(mat->emittance[0], mat->emittance[1], mat->emittance[2]);
                    const float dist2 = sqLength(positionInWorld - rayOrigin);
                    // regir's closest-hit program never computes the density (uninitialised in the reference): defined as 0
                    const float hypAreaPDensity = REGIR ? 0.0f : h.sp.hypAreaPDensity;
                    radiance += alpha * emittance * implicitEmissionWeight(hypAreaPDensity, dist2, h.vOutLocal.z, prevDirPDensity);
                }

                // Russian roulette (:277-281)
                const float continueProb = SVGF && round == 0 ? 1.0f : fminf(sRGB_calcLuminance(alpha) / initImportance, 1.0f);
                if (!(rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate)) {
                    alpha /= continueProb;
                    const BSDF bsdf = setupBsdfAtHit<V == PtVariant::SvgfMollify>(s, h.mesh, hit.y, __uint_as_float(hit.z),
                                                                                  __uint_as_float(hit.w));
                    shadeVertexVariant<REGIR>(s, rg, p, positionInWorld, h.vOutLocal, h.shadingFrame, bsdf, rng, alpha, round + 2,
                                              &radiance, &v);
                    ps.alphaPdf[pix] = make_float4(v.alpha.x, v.alpha.y, v.alpha.z, v.dirPDensity);
                    alive = true;
                }
                f.rng[pix] = rng.state;
                ps.radiance[pix] = make_float4(radiance.x, radiance.y, radiance.z, 0.0f);
            }
            else if (!REGIR && s.env.enabled) { // miss program (:310-341); the ReGIR ray type's miss program is empty
                addEnvLightOnMiss(s, ps, curQueue, slot, ps.extPixel[curQueue][slot], false);
            }
        }
        emitRays(s, ps, nextCounters, nextQueue, lane, pix, positionInWorld, v, alive);
    }
}

// ray-gen epilogue (:202-215)
__global__ void __launch_bounds__(256) k_ptAccumulate(DevFrame f, DevFrameParams p, DevPathState ps) {
    const uint32_t n = (p.y1 - p.y0) * f.W;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const size_t pix = (size_t)p.y0 * f.W + i;
    const float4 rad = ps.radiance[pix];
    const f3 contribution(rad.x, rad.y, rad.z);
    f3 prevColorResult(0.0f);
    if (p.numAccumFrames > 0) {
        const float4 b = f.beauty[pix];
        prevColorResult = f3(b.x, b.y, b.z);
    }
    const float curWeight = 1.0f / (1 + p.numAccumFrames);
    const f3 colorResult = (1 - curWeight) * prevColorResult + curWeight * contribution;
    f.beauty[pix] = make_float4(colorResult.x, colorResult.y, colorResult.z, 1.0f);
}

int ensurePathTraceBuffers(gfx_ctx* ctx) {
    FrameState &F = ctx->frame;
    const size_t n = (size_t)F.W * F.H;
    if (F.ptAlphaPdf)
        return GFX_OK;
    GFX_CUDA(ctx, cudaMalloc(&F.ptAlphaPdf, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.ptRadiance, n * 16));
    for (int i = 0; i < 2; ++i) {
        GFX_CUDA(ctx, cudaMalloc(&F.ptExtRays[i], n * 32));
        GFX_CUDA(ctx, cudaMalloc(&F.ptExtPixel[i], n * 4));
    }
    GFX_CUDA(ctx, cudaMalloc(&F.ptExtHits, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.ptShadowPending, n * 16));
    GFX_CUDA(ctx, cudaMalloc(&F.ptCounters, (kMaxPathRounds + 1) * 16));
    return GFX_OK;
}

DevPathState makePathState(const gfx_ctx* ctx) {
    const FrameState &F = ctx->frame;
    DevPathState ps;
    ps.alphaPdf = F.ptAlphaPdf;
    ps.radiance = F.ptRadiance;
    for (int i = 0; i < 2; ++i) {
        ps.extRays[i] = F.ptExtRays[i];
        ps.extPixel[i] = F.ptExtPixel[i];
    }
    ps.extHits = F.ptExtHits;
    ps.shadowRays = F.rayQueue;
    ps.shadowPixel = F.rayPixel;
    ps.shadowPending = F.ptShadowPending;
    ps.counters = F.ptCounters;
    return ps;
}

// ---- the SVGF app's path tracer (GFX_PT_SVGF) ----------------------------------------------------------------
// svgf/gpu_kernels/optix_pathtracing_kernels.cu:193-337 up to the temporal accumulation, which GFX_SVGF_TEMPORAL_ACCUMULATE
// runs.  The first vertex is the raster G-buffer's: position, interpolated and normalised shading normal, texture
// coordinate.  The geometric normal is that shading normal (:237), the frame is ReferenceFrame(normal) (no texture-coordinate
// tangent) and the origin is offset naively (:242).  Miss pixels return at once (:213-219): no RNG draw, no environment.
// The bounces are k_ptBounce<PtVariant::Svgf / SvgfMollify>.
__global__ void GFX_BOUNCE_BOUNDS k_ptSvgfFirstHit(DevScene s, DevFrame f, DevFrameParams p, DevPathState ps) {
    const uint32_t x = blockIdx.x * 8 + threadIdx.x;
    const uint32_t y = p.y0 + blockIdx.y * 8 + threadIdx.y;
    const uint32_t lane = (threadIdx.x + threadIdx.y * blockDim.x) & 31u;
    const bool inside = x < f.W && y < p.y1;
    const uint32_t pix = inside ? y * f.W + x : 0u;

    bool alive = false;
    f3 positionInWorld(0.0f);
    VertexOutput v;
    v.wantShadow = v.wantExtension = false;
    if (inside) {
        const uint4 gb0 = f.gb0[p.bufferIndex][pix];
        f3 radiance(0.0f);
        float4 albedo = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (gb0.x != 0xFFFFFFFFu) {
            GBufferHit h;
            decodeGBufferHit(s, gb0, &h);
            const f3 alpha(1.0f);
            PCG32RNG rng{ f.rng[pix] };
            const GfxMaterialDesc* mat = s.materials + h.mesh.materialSlot;
            const f3 shadingNormalInWorld = h.sp.shadingNormalInWorld;
            const f3 vOut = normalize(p.camera.position - h.sp.positionInWorld);
            const float frontHit = dot(vOut, shadingNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
            const ReferenceFrame shadingFrame(shadingNormalInWorld);
            positionInWorld = offsetRayOriginNaive(h.sp.positionInWorld, frontHit * shadingNormalInWorld);
            const f3 vOutLocal = shadingFrame.toLocal(vOut);

            if (vOutLocal.z > 0 && mat->hasEmittance)
                radiance += alpha * f3(mat->emittance[0], mat->emittance[1], mat->emittance[2]) / kPi;
            const BSDF bsdf = setupBsdfAtHit(s, h.mesh, gb0.z, h.bcB, h.bcC);
            const f3 dhReflectance = bsdf.evaluateDHReflectanceEstimate(vOutLocal); // :256; the 0.001 threshold is the temporal pass's
            albedo = make_float4(dhReflectance.x, dhReflectance.y, dhReflectance.z, 1.0f);
            shadeVertex(s, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, alpha, &radiance, &v);
            f.rng[pix] = rng.state;
            ps.alphaPdf[pix] = make_float4(v.alpha.x, v.alpha.y, v.alpha.z, v.dirPDensity);
            alive = true;
        }
        ps.radiance[pix] = make_float4(radiance.x, radiance.y, radiance.z, 0.0f);
        f.albedo[pix] = albedo;
    }
    emitRays(s, ps, ps.counters, 0u, lane, pix, positionInWorld, v, alive);
}

// :318-319: contribution = max(contribution, RGB(0.0f)), component-wise std::fmax: a NaN component becomes 0.  The single-spp
// result goes to the beauty buffer as it is (no running mean: the temporal pass accumulates).
__global__ void __launch_bounds__(256) k_ptSvgfEpilogue(DevFrame f, DevFrameParams p, DevPathState ps) {
    const uint32_t n = (p.y1 - p.y0) * f.W;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const size_t pix = (size_t)p.y0 * f.W + i;
    const float4 rad = ps.radiance[pix];
    f.beauty[pix] = make_float4(rad.x > 0.0f ? rad.x : 0.0f, rad.y > 0.0f ? rad.y : 0.0f, rad.z > 0.0f ? rad.z : 0.0f, 1.0f);
}

template <PtVariant V, bool BUMP>
static int launchPathTraceVariant(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params) {
    constexpr bool REGIR = V == PtVariant::Regir, SVGF = V == PtVariant::Svgf || V == PtVariant::SvgfMollify;
    const int rc = ensurePathTraceBuffers(ctx);
    if (rc != GFX_OK)
        return rc;
    DevFrameParams p = makeDevParams(ctx, params);
    if (p.y1 <= p.y0)
        return GFX_OK;
    p.maxPathLength = params->maxPathLength ? params->maxPathLength : 5u; // 0 = the hosts' default (svgf_main.cpp:1729)
    const DevScene s = ctx->devScene(params);
    const DevFrame f = ctx->devFrame();
    const DevPathState ps = makePathState(ctx);
    DevRegir rg = {};
    if (REGIR)
        rg = makeDevRegir(ctx, params);

    const uint32_t maxPathLength = p.maxPathLength;
    const uint32_t numRounds = min(max(maxPathLength, 2u) - 1u, kMaxPathRounds); // pathLength = 2 .. maxPathLength
    const WavefrontLabels labels = SVGF ? WavefrontLabels{ "pt_svgf_first_hit", "pt_trace_shadow", "pt_trace_extension", "pt_svgf_bounce", "pt_svgf_epilogue" }
                                        : WavefrontLabels{ "pt_first_hit", "pt_trace_shadow", "pt_trace_extension", "pt_bounce", "pt_accumulate" };
    // the last round requests no rays (maxLengthTerminate), nothing is left in flight
    return launchWavefrontFrame(
        ctx, stream, p, s, ps, numRounds, labels, ShadowAccumulateWriter{ ps.shadowPixel, ps.shadowPending, ps.radiance }, false,
        [&](dim3 grid, dim3 block) {
            if constexpr (SVGF)
                k_ptSvgfFirstHit<<<grid, block, 0, stream>>>(s, f, p, ps);
            else
                k_ptFirstHit<REGIR, BUMP><<<grid, block, 0, stream>>>(s, f, p, ps, rg);
        },
        [&](uint32_t blocks, uint32_t round) {
            const uint32_t maxLengthTerminate = (round + 2 >= maxPathLength || round + 1 == numRounds) ? 1u : 0u;
            k_ptBounce<V, BUMP><<<blocks, 64, 0, stream>>>(s, f, p, ps, rg, round, maxLengthTerminate);
        },
        [] {},
        [&](uint32_t blocks) {
            if constexpr (SVGF)
                k_ptSvgfEpilogue<<<blocks, 256, 0, stream>>>(f, p, ps);
            else
                k_ptAccumulate<<<blocks, 256, 0, stream>>>(f, p, ps);
        });
}

int launchPathTrace(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params, int variant) {
    if (params->enableBumpMapping && variant != GFX_PT_SVGF) {
        const int rc = ensureBumpTable(ctx);
        if (rc != GFX_OK)
            return rc;
    }
    if (variant == GFX_PT_NRC || variant == GFX_PT_NRC_INDIRECT)
        return launchPathTraceNrc(ctx, stream, params, variant == GFX_PT_NRC_INDIRECT);
    if (variant == GFX_PT_NRC_VISUALIZE_PREDICTION)
        return launchNrcVisualizePrediction(ctx, stream, params);
    if (variant == GFX_PT_SVGF) { // the SVGF app has no bump mapping
        if (params->svgfFlags & GFX_SVGF_MOLLIFY_SPECULAR)
            return launchPathTraceVariant<PtVariant::SvgfMollify, false>(ctx, stream, params);
        return launchPathTraceVariant<PtVariant::Svgf, false>(ctx, stream, params);
    }
    if (variant != GFX_PT_BASELINE && variant != GFX_PT_REGIR) {
        ctx->setError("gfx_pathtrace_launch: unknown variant");
        return GFX_ERR_INVALID_ARGUMENT;
    }
    const bool bump = params->enableBumpMapping != 0;
    if (variant == GFX_PT_BASELINE)
        return bump ? launchPathTraceVariant<PtVariant::Baseline, true>(ctx, stream, params)
                    : launchPathTraceVariant<PtVariant::Baseline, false>(ctx, stream, params);
    if (!ctx->frame.regir.created) {
        ctx->setError("gfx_pathtrace_launch(GFX_PT_REGIR): call gfx_regir_build_cells first");
        return GFX_ERR_NOT_READY;
    }
    return bump ? launchPathTraceVariant<PtVariant::Regir, true>(ctx, stream, params)
                : launchPathTraceVariant<PtVariant::Regir, false>(ctx, stream, params);
}

} // namespace gfx
