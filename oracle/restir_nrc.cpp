// oracle/restir_nrc.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of GFX_PT_NRC_INDIRECT and of the additive
// gfx_nrc_accumulate that follows it: ReSTIR DI + NRC as one estimator, ReSTIR DI's direct light at the primary vertex plus the NRC
// path tracer's light beyond it.  No counterpart in the reference, whose NRC app lists the combination as an open item.
//
// The restatement is nrc_pathtrace.inl's (through bump.cpp's copy, which tilts the shading frames when
// GfxFrameParams::enableBumpMapping is set and is nrc_pathtrace.inl's path tracer otherwise) with one switch, `indirect`, that only
// changes what enters the rendering radiance (st.contribution):
//   ray generation (:95-283):   no emission of the primary hit, no environment seen directly (a miss renders 0), no NEE term; the
//                               NEE draws stay, so every later vertex is the same; the shadow ray is traced for a training path
//                               only (its NEE target), so a non-training primary hit traces one ray fewer
//   pathLength 2 (:417-445, miss :625-672): the implicit emitter and environment terms go to the training target only
//   pathLength >= 3:            as GFX_PT_NRC
// gfx_nrc_accumulate after it adds: beauty += w * (contribution + alpha * cache), w = 1 / (1 + numAccumFrames).
// Like views.cpp and bump.cpp this file compiles the oracle renderer into its own library, liborc_restir_nrc.so
// (Makefile.restir_nrc, bound by tests/oracle_restir_nrc.py).
#include "bump.cpp"

// whether the light sample that performNextEventEstimation draws from `rng` has a non-zero unshadowed contribution: the library's
// path tracers queue a shadow ray only then (pathtrace.cuh neeBaseline), where the oracle traces one for every sample of positive
// density
static bool neeSampleContributes(const orc_scene* s, const GfxFrameParams* p, const float3 &shadingPoint, const float3 &vOutLocal,
                                 const ReferenceFrame &shadingFrame, const BSDF &bsdf, PCG32RNG rng) {
    float uLight = rng.getFloat0cTo1o();
    float probToSampleCurLightType;
    const bool selectEnvLight = chooseEnvForNee(s, p, &uLight, &probToSampleCurLightType);
    LightSample lightSample;
    float areaPDensity = 0.0f;
    const float u0 = rng.getFloat0cTo1o();
    const float u1 = rng.getFloat0cTo1o();
    sampleLight(s, p, uLight, selectEnvLight, u0, u1, &lightSample, &areaPDensity);
    if (!(areaPDensity * probToSampleCurLightType > 0.0f))
        return false;
    const float3 value = performDirectLighting<false>(s, shadingPoint, vOutLocal, shadingFrame, bsdf, lightSample);
    return value.x != 0.0f || value.y != 0.0f || value.z != 0.0f;
}

// skipped[0]: primary vertices whose shadow ray is not traced; skipped[1]: those of them whose light sample contributes
static void rncRayGen(orc_frame* f, orc_nrc_frame* n, const GfxFrameParams* p, const Camera &camera, uint32_t x, uint32_t y,
                      PathTraceCounters* counters, bool indirect, uint64_t* skipped) {
    const orc_scene* s = f->scene;
    const size_t pix = (size_t)y * f->W + x;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const GB0 gb0 = f->gb0[bufIdx][pix];
    const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
    const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
    NrcPathState &st = n->paths[pix];
    st = NrcPathState();

    const uint32_t tileSizeX = n->state[NRC_TILE_SIZE + 2 * bufIdx], tileSizeY = n->state[NRC_TILE_SIZE + 2 * bufIdx + 1];
    const uint32_t numPixelsInTile = tileSizeX * tileSizeY;
    const uint32_t localLinearIndex = (y % tileSizeY) * tileSizeX + (x % tileSizeX);
    st.isTrainingPath = (localLinearIndex + n->state[NRC_OFFSET_TRAINING_PATH]) % numPixelsInTile == 0;
    const uint32_t numTilesX = (f->W + tileSizeX - 1) / tileSizeX;
    const uint32_t tileX = x / tileSizeX, tileY = y / tileSizeY;
    st.linearTileIndex = tileY * numTilesX + tileX;
    const uint32_t localLinearTileIndex = (tileY % 4) * 4 + (tileX % 4);
    st.isUnbiasedTrainingTile = (localLinearTileIndex + n->state[NRC_OFFSET_UNBIASED_TILE]) % 16 == 0;

    st.contribution = indirect ? float3(0.0f) : float3(0.001f, 0.001f, 0.001f);
    st.renderingPathEndsWithCache = false;
    st.trainingSuffixEndsWithCache = false;
    st.pathLength = 1;
    if (gb0.instSlot == 0xFFFFFFFFu) {
        if (!indirect && useEnvLight(s, p)) // :323-331: the environment seen directly
            st.contribution = p->envLightPowerCoeff * s->env.fetch(bcB, bcC);
        return;
    }

    const InstData &inst = s->instances[gb0.instSlot];
    const MeshData &mesh = s->meshes[gb0.geomInstSlot];
    SurfacePoint sp;
    computeSurfacePointFromGBuffer(s, inst, mesh, gb0.primIndex, bcB, bcC, &sp);

    float3 alpha(1.0f);
    PCG32RNG rng{ f->rng[pix] };
    const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];

    float3 vOut = camera.position - sp.positionInWorld;
    const float primaryDist2 = sqLength(vOut);
    vOut /= std::sqrt(primaryDist2);
    const float primaryDotVN = dot(vOut, sp.geometricNormalInWorld);
    const float frontHit = primaryDotVN >= 0.0f ? 1.0f : -1.0f;
    const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
    st.primaryPathSpread = primaryDist2 / (4 * kPi * std::fabs(primaryDotVN));

    const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh.materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
    const float3 vOutLocal = shadingFrame.toLocal(vOut);

    float3 contribution(0.0f);
    if (!indirect && vOutLocal.z > 0 && mat.hasEmittance) {
        const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
        contribution += alpha * emittance / kPi;
    }
    const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);
    const uint64_t visibilityRaysBefore = counters->visibilityRays;
    const bool contributes = indirect && !st.isTrainingPath && neeSampleContributes(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng);
    const float3 directContNEE = performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, rng, counters);
    if (!indirect) {
        contribution += alpha * directContNEE;
    }
    else if (!st.isTrainingPath && counters->visibilityRays != visibilityRaysBefore) {
        counters->visibilityRays = visibilityRaysBefore;
        ++skipped[0];
        skipped[1] += contributes ? 1 : 0;
    }

    float3 vInLocal;
    float dirPDensity;
    const float uDir0 = rng.getFloat0cTo1o();
    const float uDir1 = rng.getFloat0cTo1o();
    const float3 localThroughput = bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
    alpha *= localThroughput;

    st.prevTrainDataIndex = kInvalidVertexDataIndex;
    if (st.isTrainingPath) {
        NrcStagedVertex &sv = n->staged[st.linearTileIndex];
        sv.want = true;
        sv.fromRayGen = true;
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, sv.query);
        sv.localThroughput = localThroughput;
        sv.directContNEE = directContNEE;
        sv.pathLength = st.pathLength;
    }

    st.active = true;
    st.rng = rng;
    st.alpha = alpha;
    st.contribution = contribution;
    st.prevDirPDensity = dirPDensity;
    st.curSqrtPathSpread = 0.0f;
    st.prevLocalThroughput = localThroughput;
    st.rayOrg = positionInWorld;
    st.rayDir = shadingFrame.fromLocal(vInLocal);
}

// one iteration of the path extension loop (:285-311) with the closest-hit program (:363-623) inlined
static void rncExtend(orc_frame* f, orc_nrc_frame* n, const GfxFrameParams* p, size_t pix, PathTraceCounters* counters, bool indirect) {
    const orc_scene* s = f->scene;
    NrcPathState &st = n->paths[pix];
    const bool isValidSampling = st.prevDirPDensity > 0.0f && std::isfinite(st.prevDirPDensity);
    if (!isValidSampling) {
        st.active = false;
        return;
    }
    ++st.pathLength;
    const bool maxLengthTerminate = (st.pathLength >= p->maxPathLength && p->maxPathLength > 0) || st.pathLength >= kMaxNrcRounds;
    // the implicit light of the primary vertex's BSDF sample: ReSTIR DI's part of the estimate
    const bool renderImplicit = !(indirect && st.pathLength == 2);
    st.active = false; // rwPayload.terminate = true

    ++counters->closestRays;
    const HitObject hit = traverseCanonical(s->bvh, st.rayOrg, st.rayDir, 0.0f, std::numeric_limits<float>::max());
    if (hit.primIndex == UINT32_MAX) { // pathTrace_miss_generic (:625-672)
        if (useEnvLight(s, p)) {
            const float3 directContImplicit = evaluateEnvLightOnMiss(s, p, st.rayDir, st.prevDirPDensity, true);
            if (renderImplicit && !st.renderingPathEndsWithCache)
                st.contribution += st.alpha * directContImplicit;
            if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
                float* tgt = &n->trainTarget[0][3 * (size_t)st.prevTrainDataIndex];
                const float3 add = st.prevLocalThroughput * directContImplicit;
                tgt[0] += add.x; tgt[1] += add.y; tgt[2] += add.z;
            }
        }
        return;
    }

    const InstData &inst = s->instances[s->geomToInst[hit.geomIndex]];
    const MeshData &mesh = s->meshes[s->geomToMesh[hit.geomIndex]];
    SurfacePoint sp;
    computeSurfacePointAtHit(s, p, inst, mesh, hit.primIndex, hit.bcB, hit.bcC, &sp);
    const GfxMaterialDesc &mat = s->materials[mesh.materialSlot];

    const float3 vOut = normalize(-st.rayDir);
    const float frontHit = dot(vOut, sp.geometricNormalInWorld) >= 0.0f ? 1.0f : -1.0f;
    const ReferenceFrame shadingFrame = shadingFrameAt(s, p, mesh.materialSlot, sp.texCoord, sp.shadingNormalInWorld, sp.texCoord0DirInWorld);
    const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
    const float3 vOutLocal = shadingFrame.toLocal(vOut);

    const float dist2 = sqLength(positionInWorld - st.rayOrg);
    st.curSqrtPathSpread += std::sqrt(dist2 / (st.prevDirPDensity * std::fabs(vOutLocal.z)));

    // implicit light sampling (:417-445)
    if (vOutLocal.z > 0 && mat.hasEmittance) {
        const float3 emittance(mat.emittance[0], mat.emittance[1], mat.emittance[2]);
        const float lightPDensity = sp.hypAreaPDensity * dist2 / vOutLocal.z;
        const float bsdfPDensity = st.prevDirPDensity;
        const float misWeight = pow2(bsdfPDensity) / (pow2(bsdfPDensity) + pow2(lightPDensity));
        const float3 directContImplicit = emittance * (misWeight / kPi);
        if (renderImplicit && !st.renderingPathEndsWithCache)
            st.contribution += st.alpha * directContImplicit;
        if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
            float* tgt = &n->trainTarget[0][3 * (size_t)st.prevTrainDataIndex];
            const float3 add = st.prevLocalThroughput * directContImplicit;
            tgt[0] += add.x; tgt[1] += add.y; tgt[2] += add.z;
        }
    }

    // Russian roulette (:447-469)
    bool performRR = true;
    bool terminatedByRR = false;
    float recContinueProb = 1.0f;
    if (st.isTrainingPath)
        performRR = st.pathLength > 2;
    if (performRR) {
        const float continueProb = std::fmin(sRGB_calcLuminance(st.alpha) / sRGB_calcLuminance(float3(1.0f)), 1.0f);
        if (st.rng.getFloat0cTo1o() >= continueProb || maxLengthTerminate) {
            if (st.renderingPathEndsWithCache && st.isTrainingPath && st.isUnbiasedTrainingTile)
                return;
            terminatedByRR = true;
        }
        recContinueProb = 1.0f / continueProb;
    }

    const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);

    // path termination by the spread heuristic (:474-531)
    bool endsWithCache = pow2(st.curSqrtPathSpread) > kPathTerminationFactor * st.primaryPathSpread;
    if (st.renderingPathEndsWithCache && st.isTrainingPath && st.isUnbiasedTrainingTile)
        endsWithCache = false;
    if (endsWithCache) {
        float query[14];
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, query);
        if (!st.renderingPathEndsWithCache) {
            std::memcpy(&n->inferenceQuery[14 * pix], query, sizeof(query));
            writeTerminalInfo(n, pix, st.alpha, st.pathLength, true, st.isTrainingPath, st.isUnbiasedTrainingTile);
            st.renderingPathEndsWithCache = true;
            if (st.isTrainingPath)
                st.curSqrtPathSpread = 0;
            else
                return;
        }
        else {
            if (!st.trainingSuffixEndsWithCache) {
                const size_t offset = (size_t)f->W * f->H;
                std::memcpy(&n->inferenceQuery[14 * (offset + st.linearTileIndex)], query, sizeof(query));
                n->suffixTerminal[st.linearTileIndex] = packSuffixTerminal(st.prevTrainDataIndex, true, st.pathLength);
                st.trainingSuffixEndsWithCache = true;
            }
            return;
        }
    }

    if (terminatedByRR)
        return;
    st.alpha *= recContinueProb;
    if (st.isTrainingPath && !st.trainingSuffixEndsWithCache && st.prevTrainDataIndex != kInvalidVertexDataIndex) {
        uint32_t* vi = &n->trainVertexInfo[4 * (size_t)st.prevTrainDataIndex];
        for (int c = 0; c < 3; ++c)
            vi[c] = f2u(u2f(vi[c]) * recContinueProb);
    }

    const float3 directContNEE = performNextEventEstimation(s, p, positionInWorld, vOutLocal, shadingFrame, bsdf, st.rng, counters);
    if (!st.renderingPathEndsWithCache)
        st.contribution += st.alpha * directContNEE;

    float3 vInLocal;
    float dirPDensity;
    const float uDir0 = st.rng.getFloat0cTo1o();
    const float uDir1 = st.rng.getFloat0cTo1o();
    const float3 localThroughput = bsdf.sampleThroughput(vOutLocal, uDir0, uDir1, &vInLocal, &dirPDensity);
    st.alpha *= localThroughput;
    st.rayOrg = positionInWorld;
    st.rayDir = shadingFrame.fromLocal(vInLocal);
    st.prevDirPDensity = dirPDensity;
    st.prevLocalThroughput = localThroughput;
    st.active = true; // rwPayload.terminate = false

    if (st.isTrainingPath && !st.trainingSuffixEndsWithCache) {
        NrcStagedVertex &sv = n->staged[st.linearTileIndex];
        sv.want = true;
        sv.fromRayGen = false;
        createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, sv.query);
        sv.localThroughput = localThroughput;
        sv.directContNEE = directContNEE;
        sv.pathLength = st.pathLength;
    }
}

// the variant of each frame's last NRC path trace, which selects the accumulation
static std::mutex g_lastTraceMutex;
static std::map<const orc_frame*, bool> g_lastTraceIndirect;

// gfx_pathtrace_launch(GFX_PT_NRC or GFX_PT_NRC_INDIRECT) on the rows params->tileOriginY / tileRows; returns the rays traced and,
// in skippedShadowRays[0], the primary vertices that drew a light sample but traced no shadow ray (GFX_PT_NRC_INDIRECT's
// non-training primary hits; 0 for GFX_PT_NRC), in skippedShadowRays[1] those of them whose sample contributes (the rays the
// library's GFX_PT_NRC traces and GFX_PT_NRC_INDIRECT does not)
extern "C" uint64_t orc_rnc_pathtrace(orc_frame* f, const GfxFrameParams* p, int variant, int numThreads, uint64_t* skippedShadowRays) {
    if (numThreads <= 0) numThreads = omp_get_max_threads();
    const bool indirect = variant == GFX_PT_NRC_INDIRECT;
    {
        std::lock_guard<std::mutex> lock(g_lastTraceMutex);
        g_lastTraceIndirect[f] = indirect;
    }
    orc_nrc_frame* n = nrcFrame(f);
    const Camera camera = makeCamera(p->camera);
    const uint32_t W = f->W, H = f->H;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const uint32_t tileSizeX = n->state[NRC_TILE_SIZE + 2 * bufIdx], tileSizeY = n->state[NRC_TILE_SIZE + 2 * bufIdx + 1];
    const uint32_t numTilesX = (W + tileSizeX - 1) / tileSizeX, numTilesY = (H + tileSizeY - 1) / tileSizeY;
    std::vector<uint32_t> tileToPixel((size_t)numTilesX * numTilesY, 0u);
    for (auto &sv : n->staged)
        sv.want = false;

    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    for (size_t pix = 0; pix < (size_t)W * H; ++pix)
        if (pix < (size_t)y0 * W || pix >= (size_t)y1 * W)
            n->paths[pix].active = false;
    uint64_t rays = 0, skipped = 0, skippedContributing = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays, skipped, skippedContributing)
    for (int64_t y = y0; y < (int64_t)y1; ++y) {
        PathTraceCounters counters;
        uint64_t rowSkipped[2] = { 0, 0 };
        for (uint32_t x = 0; x < W; ++x) {
            rncRayGen(f, n, p, camera, x, (uint32_t)y, &counters, indirect, rowSkipped);
            const NrcPathState &st = n->paths[(size_t)y * W + x];
            if (st.isTrainingPath)
                tileToPixel[st.linearTileIndex] = (uint32_t)(y * W + x);
        }
        rays += counters.closestRays + counters.visibilityRays;
        skipped += rowSkipped[0];
        skippedContributing += rowSkipped[1];
    }
    nrcCommitStagedVertices(f, n, p, tileToPixel);

    for (uint32_t round = 0; round < kMaxNrcRounds; ++round) {
        uint64_t numActive = 0;
#pragma omp parallel for schedule(dynamic, 2) num_threads(numThreads) reduction(+ : rays, numActive)
        for (int64_t y = y0; y < (int64_t)y1; ++y) {
            PathTraceCounters counters;
            for (uint32_t x = 0; x < W; ++x) {
                const size_t pix = (size_t)y * W + x;
                if (!n->paths[pix].active)
                    continue;
                rncExtend(f, n, p, pix, &counters, indirect);
                numActive += n->paths[pix].active ? 1 : 0;
            }
            rays += counters.closestRays + counters.visibilityRays;
        }
        if (!nrcCommitStagedVertices(f, n, p, tileToPixel, numActive != 0))
            break;
    }

    // ray-gen epilogue (:312-360)
    for (size_t pix = (size_t)y0 * W; pix < (size_t)y1 * W; ++pix) {
        const NrcPathState &st = n->paths[pix];
        if (f->gb0[bufIdx][pix].instSlot != 0xFFFFFFFFu) {
            f->rng[pix] = st.rng.state;
            if (st.isTrainingPath && !st.trainingSuffixEndsWithCache)
                n->suffixTerminal[st.linearTileIndex] = packSuffixTerminal(st.prevTrainDataIndex, false, st.pathLength);
        }
        if (!st.renderingPathEndsWithCache)
            writeTerminalInfo(n, pix, float3(0.0f), st.pathLength, false, st.isTrainingPath, st.isUnbiasedTrainingTile);
        n->frameContribution[3 * pix + 0] = st.contribution.x;
        n->frameContribution[3 * pix + 1] = st.contribution.y;
        n->frameContribution[3 * pix + 2] = st.contribution.z;
    }
    if (skippedShadowRays) {
        skippedShadowRays[0] = skipped;
        skippedShadowRays[1] = skippedContributing;
    }
    return rays;
}

// gfx_nrc_accumulate: nrc_pathtrace.inl's blend (nrc_setup_kernels.cu:51-92), or after GFX_PT_NRC_INDIRECT the addition to this
// frame's ReSTIR DI beauty
extern "C" void orc_rnc_nrc_accumulate(orc_frame* f, const GfxFrameParams* p) {
    bool indirect = false;
    {
        std::lock_guard<std::mutex> lock(g_lastTraceMutex);
        const auto it = g_lastTraceIndirect.find(f);
        indirect = it != g_lastTraceIndirect.end() && it->second;
    }
    if (!indirect) {
        orc_nrc_accumulate(f, p);
        return;
    }
    orc_nrc_frame* n = nrcFrame(f);
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(f->H, p->tileOriginY + p->tileRows) : f->H;
    for (size_t i = (size_t)y0 * f->W; i < (size_t)y1 * f->W; ++i) {
        const uint32_t* t = &n->terminalInfo[4 * i];
        const float3 alpha(u2f(t[0]), u2f(t[1]), u2f(t[2]));
        const float3 directCont(n->frameContribution[3 * i], n->frameContribution[3 * i + 1], n->frameContribution[3 * i + 2]);
        float3 radiance(0.0f);
        if (t[3] & 1u) {
            radiance = max3(float3(n->inferredRadiance[3 * i], n->inferredRadiance[3 * i + 1], n->inferredRadiance[3 * i + 2]), float3(0.0f));
            if (p->radianceScale > 0)
                radiance /= p->radianceScale;
            const float* q = &n->inferenceQuery[14 * i];
            radiance *= (float3(q[8], q[9], q[10]) + float3(q[11], q[12], q[13]));
        }
        const float3 contribution = directCont + alpha * radiance;
        const float curWeight = 1.0f / (1 + p->numAccumFrames);
        const float3 colorResult = float3(f->beauty[i].x, f->beauty[i].y, f->beauty[i].z) + curWeight * contribution;
        f->beauty[i] = F4{ colorResult.x, colorResult.y, colorResult.z, 1.0f };
    }
}

// the frame is going away: forget its variant (orc_frame_destroy is render.cpp's)
extern "C" void orc_rnc_frame_destroy(orc_frame* f) {
    {
        std::lock_guard<std::mutex> lock(g_lastTraceMutex);
        g_lastTraceIndirect.erase(f);
    }
    orc_frame_destroy(f);
}
