// regir.cu — ReGIR: world-space grid of light reservoirs, built every frame on sm_90a.
//
// Replaces kernelBuildCellReservoirs / kernelBuildCellReservoirsAndTemporalReuse / kernelUpdateLastAccessFrameIndices
// (regir/regir_main.cpp:2033-2068; regir/gpu_kernels/build_cell_reservoirs.cu:6-69, 71-233, 235-248) and the host-side
// grid set-up initializeReservoirs (regir/regir_main.cpp:1073-1109).  The lookup side (sampleFromCell) lives with
// the path tracer in pathtrace.cuh.
//
// Layout: a light slot is ONE aligned 64-byte record (Reservoir<LightSample> 48 B + ReservoirInfo 8 B of the
// reference, which keeps them in two arrays): the build writes it with four coalesced 16-byte stores per thread,
// the path tracer fetches a random slot with one 64-byte (two-sector) access instead of touching two arrays.
// One thread per slot, 512 slots per cell, so the four 128-thread blocks of an idle cell exit on one load.
#include "pathtrace.cuh"
#include <random>
#include <vector>

namespace gfx {

DevRegir makeDevRegir(const gfx_ctx* ctx, const GfxFrameParams* p) {
    const FrameState::Regir &R = ctx->frame.regir;
    DevRegir d;
    d.slots[0] = R.slots[0];
    d.slots[1] = R.slots[1];
    d.slotRngs = R.slotRngs;
    d.perCellNumAccesses = R.perCellNumAccesses;
    d.lastAccessFrameIndices = R.lastAccessFrameIndices;
    d.numActiveCells = R.numActiveCells;
    d.dimX = R.dim[0];
    d.dimY = R.dim[1];
    d.dimZ = R.dim[2];
    d.numCells = R.numCells;
    d.gridOrigin = f3(R.gridOrigin[0], R.gridOrigin[1], R.gridOrigin[2]);
    d.gridCellSize = f3(R.gridCellSize[0], R.gridCellSize[1], R.gridCellSize[2]);
    d.log2NumCandidatesPerLightSlot = p->regirLog2NumCandidatesPerLightSlot;
    d.log2NumCandidatesPerCell = p->regirLog2NumCandidatesPerCell;
    d.enableCellRandomization = p->regirEnableCellRandomization;
    d.bufferIndex = p->bufferIndex & 1;
    return d;
}

void releaseRegir(gfx_ctx* ctx) {
    FrameState::Regir &R = ctx->frame.regir;
    cudaFree(R.slots[0]); cudaFree(R.slots[1]); cudaFree(R.slotRngs); cudaFree(R.perCellNumAccesses);
    cudaFree(R.lastAccessFrameIndices); cudaFree(R.numActiveCells);
    R = FrameState::Regir();
}

// the cell grid over the scene's box (regir_main.cpp:1109, 1012)
void regirGrid(const GfxFrameParams* p, uint32_t dim[3], float origin[3], float cellSize[3]) {
    for (int c = 0; c < 3; ++c)
        dim[c] = p->regirGridDim[c];
    if (dim[0] == 0 || dim[1] == 0 || dim[2] == 0) {
        dim[0] = 32; dim[1] = 8; dim[2] = 32;
    }
    for (int c = 0; c < 3; ++c) {
        origin[c] = p->sceneAabbMin[c];
        cellSize[c] = (p->sceneAabbMax[c] - p->sceneAabbMin[c]) / (float)dim[c];
    }
}

// initializeReservoirs (regir_main.cpp:1073-1112), run by the build of frame `frameIndex` whenever the grid is new: the
// frame's first build, a build after gfx_frame_create, or a new regirGridDim
static int ensureRegir(gfx_ctx* ctx, const GfxFrameParams* p, uint32_t frameIndex) {
    FrameState::Regir &R = ctx->frame.regir;
    uint32_t dim[3];
    float origin[3], cellSize[3];
    regirGrid(p, dim, origin, cellSize);
    if (R.created && R.dim[0] == dim[0] && R.dim[1] == dim[1] && R.dim[2] == dim[2])
        return GFX_OK;
    releaseRegir(ctx);
    memcpy(R.dim, dim, sizeof(dim));
    R.numCells = dim[0] * dim[1] * dim[2];
    R.numSlots = R.numCells * kNumLightSlotsPerCell;
    memcpy(R.gridOrigin, origin, sizeof(origin));
    memcpy(R.gridCellSize, cellSize, sizeof(cellSize));
    for (int i = 0; i < 2; ++i) {
        GFX_CUDA(ctx, cudaMalloc(&R.slots[i], (size_t)R.numSlots * 64));
        GFX_CUDA(ctx, cudaMemset(R.slots[i], 0, (size_t)R.numSlots * 64));
    }
    GFX_CUDA(ctx, cudaMalloc(&R.slotRngs, (size_t)R.numSlots * 8));
    GFX_CUDA(ctx, cudaMalloc(&R.perCellNumAccesses, (size_t)R.numCells * 4));
    GFX_CUDA(ctx, cudaMalloc(&R.lastAccessFrameIndices, (size_t)R.numCells * 4));
    GFX_CUDA(ctx, cudaMalloc(&R.numActiveCells, 8));
    GFX_CUDA(ctx, cudaMemset(R.perCellNumAccesses, 0, (size_t)R.numCells * 4));
    GFX_CUDA(ctx, cudaMemset(R.numActiveCells, 0, 8));
    // the reference fills with -1 at startup (frame 0); frameIndex - 1 keeps that there and, for a grid created later, keeps
    // every cell built for the next 8 frames as well instead of idle from the start (DESIGN.md)
    const std::vector<uint32_t> lastAccess(R.numCells, frameIndex - 1u);
    GFX_CUDA(ctx, cudaMemcpy(R.lastAccessFrameIndices, lastAccess.data(), lastAccess.size() * 4, cudaMemcpyHostToDevice));
    std::vector<unsigned long long> states(R.numSlots);
    std::mt19937_64 rngSeed(591842031321323413ull);
    for (auto &st : states)
        st = rngSeed();
    GFX_CUDA(ctx, cudaMemcpy(R.slotRngs, states.data(), states.size() * 8, cudaMemcpyHostToDevice));
    R.created = true;
    return GFX_OK;
}

// build_cell_reservoirs.cu:6-69
GFX_D f3 sampleIntensity(const DevScene &s, const f3 &cellCenter, const f3 &halfCellSize, float minSquaredDistance, float uLight,
                         bool sampleEnv, float uPos0, float uPos1, LightSample* lightSample, float* probDensity) {
    if (sampleEnv)
        sampleEnvLight(s, uPos0, uPos1, lightSample, probDensity);
    else
        sampleLight(s, uLight, uPos0, uPos1, lightSample, probDensity);
    float dist2 = minSquaredDistance;
    float lpCos = 1;
    const bool isOutsideCell =
        lightSample->atInfinity ||
        lightSample->position.x < cellCenter.x - halfCellSize.x ||
        lightSample->position.x > cellCenter.x + halfCellSize.x ||
        lightSample->position.y < cellCenter.y - halfCellSize.y ||
        lightSample->position.y > cellCenter.y + halfCellSize.y ||
        lightSample->position.z < cellCenter.z - halfCellSize.z ||
        lightSample->position.z > cellCenter.z + halfCellSize.z;
    if (isOutsideCell) {
        const f3 shadowRayDir = lightSample->atInfinity ? lightSample->position : (lightSample->position - cellCenter);
        const float perpDistance = dot(-shadowRayDir, lightSample->normal);
        dist2 = sqLength(shadowRayDir);
        const float dist = sqrtf(dist2);
        // as written in the reference (:54-55): lpCos is still 1 here
        const bool cellIsInValidHalfSpace = lpCos > minSquaredDistance || lightSample->atInfinity;
        const bool cellIsInInvalidHalfSpace = lpCos < -minSquaredDistance;
        if (cellIsInValidHalfSpace)
            lpCos = perpDistance / dist;
        else if (cellIsInInvalidHalfSpace)
            lpCos = 0.0f;
    }
    if (lpCos > 0.0f) {
        const f3 Le = lightSample->emittance / kPi;
        return Le * (lpCos / dist2);
    }
    return f3(0.0f);
}

struct SlotReservoir { // Reservoir<LightSample> (regir_shared.h:95-132)
    LightSample sample;
    float sumWeights;
    uint32_t streamLength;
    GFX_D void initialize() {
        sample = emptyLightSample();
        sumWeights = 0;
        streamLength = 0;
    }
    GFX_D bool update(const LightSample &newSample, float weight, float u) {
        sumWeights += weight;
        const bool accepted = u < weight / sumWeights;
        if (accepted)
            sample = newSample;
        ++streamLength;
        return accepted;
    }
};

template <bool useTemporalReuse>
__global__ void __launch_bounds__(128) k_regirBuildCells(DevScene s, DevRegir rg, uint32_t frameIndex) {
    const uint32_t bufferIndex = rg.bufferIndex;
    const uint32_t linearThreadIndex = blockDim.x * blockIdx.x + threadIdx.x;
    const uint32_t cellLinearIndex = linearThreadIndex / kNumLightSlotsPerCell;
    if (cellLinearIndex >= rg.numCells)
        return;
    const uint32_t lastAccessFrameIndex = rg.lastAccessFrameIndices[cellLinearIndex];
    if (linearThreadIndex == 0)
        rg.numActiveCells[bufferIndex] = 0;
    if (linearThreadIndex % kNumLightSlotsPerCell == 0)
        rg.perCellNumAccesses[cellLinearIndex] = 0;
    if (frameIndex - lastAccessFrameIndex > 8)
        return;

    const uint32_t iz = cellLinearIndex / (rg.dimX * rg.dimY);
    const uint32_t iy = (cellLinearIndex % (rg.dimX * rg.dimY)) / rg.dimX;
    const uint32_t ix = cellLinearIndex % rg.dimX;
    const f3 cellCenter = rg.gridOrigin + f3((ix + 0.5f) * rg.gridCellSize.x, (iy + 0.5f) * rg.gridCellSize.y, (iz + 0.5f) * rg.gridCellSize.z);
    const f3 halfCellSize = 0.5f * rg.gridCellSize;
    const float minSquaredDistance = sqLength(0.5f * rg.gridCellSize);

    PCG32RNG rng{ rg.slotRngs[linearThreadIndex] };
    float selectedTargetPDensity = 0.0f;
    SlotReservoir reservoir;
    reservoir.initialize();

    // streaming RIS, target = luminous intensity reaching the cell's representative point
    const uint32_t numCandidates = 1u << rg.log2NumCandidatesPerLightSlot;
    for (uint32_t candIdx = 0; candIdx < numCandidates; ++candIdx) {
        float uLight = rng.getFloat0cTo1o();
        float probToSampleCurLightType;
        const bool sampleEnv = chooseEnvForCandidate(s, candIdx, numCandidates, &uLight, &probToSampleCurLightType); // :120-139
        LightSample lightSample = emptyLightSample();
        float areaPDensity = 0.0f;
        const float uPos0 = rng.getFloat0cTo1o();
        const float uPos1 = rng.getFloat0cTo1o();
        const f3 cont = sampleIntensity(s, cellCenter, halfCellSize, minSquaredDistance, uLight, sampleEnv, uPos0, uPos1, &lightSample, &areaPDensity);
        areaPDensity *= probToSampleCurLightType;
        const float targetPDensity = convertToWeight(cont);
        // a sample its sampler cannot produce (the environment's poles, areaPDensity = 0) weighs 0 rather than the
        // reference's 0 / 0 = NaN, which the temporal merge would carry in sumWeights forever (DESIGN.md)
        const float weight = areaPDensity > 0.0f ? targetPDensity / areaPDensity : 0.0f;
        if (reservoir.update(lightSample, weight, rng.getFloat0cTo1o()))
            selectedTargetPDensity = targetPDensity;
    }
    float recPDFEstimate = reservoir.sumWeights / (selectedTargetPDensity * reservoir.streamLength);
    if (!isfinite(recPDFEstimate)) {
        recPDFEstimate = 0.0f;
        selectedTargetPDensity = 0.0f;
    }

    if (useTemporalReuse) { // merge with the slot's accumulated reservoir of the previous frame, M capped at 20x
        const uint32_t prevBufferIndex = (bufferIndex + 1) % 2;
        const uint32_t selfStreamLength = reservoir.streamLength;
        if (recPDFEstimate == 0.0f)
            reservoir.initialize();
        uint32_t combinedStreamLength = selfStreamLength;
        const uint32_t maxNumPrevSamples = 20 * selfStreamLength;
        const float4* prev = rg.slots[prevBufferIndex] + 4 * (size_t)linearThreadIndex;
        const float4 p0 = prev[0], p1 = prev[1], p2 = prev[2], p3 = prev[3];
        LightSample prevLightSample;
        prevLightSample.emittance = f3(p0.x, p0.y, p0.z);
        prevLightSample.position = f3(p1.x, p1.y, p1.z);
        prevLightSample.normal = f3(p2.x, p2.y, p2.z);
        const uint32_t pm = __float_as_uint(p1.w);
        prevLightSample.atInfinity = pm >> 31;
        const uint32_t prevM = pm & 0x7FFFFFFFu;
        const float prevTargetDensity = p3.x;
        const uint32_t prevStreamLength = min(prevM, maxNumPrevSamples);
        const float lengthCorrection = static_cast<float>(prevStreamLength) / prevM;
        // a slot that was never built (M = 0) weighs 0 rather than the reference's 0 / 0 = NaN (DESIGN.md)
        const float weight = prevM > 0 ? lengthCorrection * p0.w : 0.0f;
        if (reservoir.update(prevLightSample, weight, rng.getFloat0cTo1o()))
            selectedTargetPDensity = prevTargetDensity;
        combinedStreamLength += prevStreamLength;
        reservoir.streamLength = combinedStreamLength;
        const float weightForEstimate = 1.0f / reservoir.streamLength;
        recPDFEstimate = weightForEstimate * reservoir.sumWeights / selectedTargetPDensity;
        if (!isfinite(recPDFEstimate)) {
            recPDFEstimate = 0.0f;
            selectedTargetPDensity = 0.0f;
        }
    }

    rg.slotRngs[linearThreadIndex] = rng.state;
    float4* cur = rg.slots[bufferIndex] + 4 * (size_t)linearThreadIndex;
    cur[0] = make_float4(reservoir.sample.emittance.x, reservoir.sample.emittance.y, reservoir.sample.emittance.z, reservoir.sumWeights);
    cur[1] = make_float4(reservoir.sample.position.x, reservoir.sample.position.y, reservoir.sample.position.z,
                         __uint_as_float((reservoir.streamLength & 0x7FFFFFFFu) | (reservoir.sample.atInfinity << 31)));
    cur[2] = make_float4(reservoir.sample.normal.x, reservoir.sample.normal.y, reservoir.sample.normal.z, recPDFEstimate);
    cur[3] = make_float4(selectedTargetPDensity, 0.0f, 0.0f, 0.0f);
}

// build_cell_reservoirs.cu:235-248
__global__ void k_regirUpdateAccess(DevRegir rg, uint32_t frameIndex) {
    const uint32_t cellLinearIndex = blockDim.x * blockIdx.x + threadIdx.x;
    const uint32_t perCellNumAccesses = cellLinearIndex < rg.numCells ? rg.perCellNumAccesses[cellLinearIndex] : 0u;
    if (perCellNumAccesses > 0)
        rg.lastAccessFrameIndices[cellLinearIndex] = frameIndex;
    const uint32_t numActiveCellsInGroup = __popc(__ballot_sync(0xFFFFFFFFu, perCellNumAccesses > 0));
    if ((threadIdx.x & 31u) == 0 && numActiveCellsInGroup > 0)
        atomicAdd(rg.numActiveCells + rg.bufferIndex, numActiveCellsInGroup);
}

int launchRegirBuildCells(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params, uint32_t frameIndex, int useTemporalReuse) {
    const int rc = ensureRegir(ctx, params, frameIndex);
    if (rc != GFX_OK)
        return rc;
    if (!ctx->scene.uploaded) {
        ctx->setError("gfx_regir_build_cells: no scene");
        return GFX_ERR_NOT_READY;
    }
    const DevRegir rg = makeDevRegir(ctx, params);
    const DevScene s = ctx->devScene(params);
    const uint32_t grid = (ctx->frame.regir.numSlots + 127) / 128;
    GFX_TIMED(ctx, stream, "regir_build_cells");
    if (useTemporalReuse)
        k_regirBuildCells<true><<<grid, 128, 0, stream>>>(s, rg, frameIndex);
    else
        k_regirBuildCells<false><<<grid, 128, 0, stream>>>(s, rg, frameIndex);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

int launchRegirUpdateAccess(gfx_ctx* ctx, cudaStream_t stream, const GfxFrameParams* params, uint32_t frameIndex) {
    if (!ctx->frame.regir.created) {
        ctx->setError("gfx_regir_update_access: call gfx_regir_build_cells first");
        return GFX_ERR_NOT_READY;
    }
    const DevRegir rg = makeDevRegir(ctx, params);
    k_regirUpdateAccess<<<(rg.numCells + 127) / 128, 128, 0, stream>>>(rg, frameIndex);
    ctx->launches++;
    GFX_CUDA(ctx, cudaGetLastError());
    return GFX_OK;
}

} // namespace gfx
