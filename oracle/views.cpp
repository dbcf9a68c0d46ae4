// oracle/views.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of the debug views of the NRC and ReGIR apps:
//   visualizePrediction                            neural_radiance_caching/gpu_kernels/optix_pathtracing_kernels.cu:702-778
//   visualizeToOutputBuffer                        neural_radiance_caching/gpu_kernels/copy_buffers.cu:32-130
//   calcCellLinearIndex / getFNV1Hash32 / calcCellColor / visualizeToOutputBuffer
//                                                  regir/gpu_kernels/copy_buffers.cu:30-76, 95-108
//   HSVtoRGB                                       common/basic_types.h:5365-5388
// The visualizePrediction pass builds its queries from the oracle renderer's scene, G-buffer and NRC buffers, whose types
// are private to render.cpp: this file compiles render.cpp into its own library, liborc_views.so (Makefile.views, bound by
// tests/oracle_views.py), so the pass runs on a frame of that library.  The views end in orc_present (present.cpp, linked
// in): the view's float4 value of every pixel goes through the same alpha override, tone map, gamma and packing as a plain
// COLOR present, as the reference tints in visualizeToOutputBuffer and tone-maps in its display shader afterwards.
// The ReGIR grid is the one regir.inl builds from the frame parameters (regir_main.cpp:1109, 0 = 32 x 8 x 32).
#include "render.cpp"

extern "C" {
/* the buffers gfx_present_launch reads for the views, as host copies in their download layouts; NULL = not read */
typedef struct OrcViewInputs {
    const uint32_t* terminalInfo;     /* 4 x W*H */
    const float* inferredRadiance;    /* 3 x at least W*H */
    const float* inferenceQuery;      /* 14 x at least W*H */
    const float* gbuffer1;            /* 2 x W*H: motion vectors of frame->bufferIndex */
    const float* gbuffer2;            /* 4 x W*H: position, qGeometricNormal */
} OrcViewInputs;
}

struct ViewGrid {
    uint32_t dim[3];
    float3 origin, cellSize;
};

static ViewGrid viewGrid(const GfxFrameParams* p) {
    ViewGrid g;
    for (int c = 0; c < 3; ++c)
        g.dim[c] = p->regirGridDim[c];
    if (g.dim[0] == 0 || g.dim[1] == 0 || g.dim[2] == 0) {
        g.dim[0] = 32; g.dim[1] = 8; g.dim[2] = 32;
    }
    const float3 minP(p->sceneAabbMin[0], p->sceneAabbMin[1], p->sceneAabbMin[2]);
    const float3 maxP(p->sceneAabbMax[0], p->sceneAabbMax[1], p->sceneAabbMax[2]);
    g.origin = minP;
    g.cellSize = (maxP - minP) / float3((float)g.dim[0], (float)g.dim[1], (float)g.dim[2]);
    return g;
}

static uint32_t getFNV1Hash32(uint32_t x) { // the 4 bytes of x in memory order (little endian)
    uint32_t hash = 2166136261u;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(&x);
    for (int i = 0; i < 4; ++i)
        hash = (16777619u * hash) ^ bytes[i];
    return hash;
}

static float3 HSVtoRGB(float h, float s, float v) {
    if (s == 0)
        return float3(v, v, v);
    const float hm = h - std::floor(h);
    const int32_t hi = static_cast<int32_t>(hm * 6);
    const float f = hm * 6 - hi;
    const float m = v * (1 - s);
    const float n = v * (1 - s * f);
    const float k = v * (1 - s * (1 - f));
    if (hi == 0) return float3(v, k, m);
    if (hi == 1) return float3(n, v, m);
    if (hi == 2) return float3(m, v, k);
    if (hi == 3) return float3(m, n, v);
    if (hi == 4) return float3(k, m, v);
    if (hi == 5) return float3(v, m, n);
    return float3(0.0f);
}

static float3 calcCellColor(const ViewGrid &g, const float3 &positionInWorld) {
    // calcCellLinearIndex; float -> uint32 saturates like cvt.rzi.u32.f32 (as in regir.inl)
    const float3 relPos = positionInWorld - g.origin;
    const uint32_t ix = std::min(dm_f2uint(relPos.x / g.cellSize.x), g.dim[0] - 1);
    const uint32_t iy = std::min(dm_f2uint(relPos.y / g.cellSize.y), g.dim[1] - 1);
    const uint32_t iz = std::min(dm_f2uint(relPos.z / g.cellSize.z), g.dim[2] - 1);
    const uint32_t cellLinearIndex = iz * g.dim[0] * g.dim[1] + iy * g.dim[0] + ix;
    PCG32RNG rng;
    rng.state = (static_cast<uint64_t>(getFNV1Hash32(cellLinearIndex)) << 32) | 3018421212u; // setState
    const float h = rng.getFloat0cTo1o();
    const float s = 0.5f + 0.5f * rng.getFloat0cTo1o();
    const float v = 0.5f + 0.5f * rng.getFloat0cTo1o();
    return HSVtoRGB(h, s, v);
}

extern "C" void orc_regir_cell_color(const GfxFrameParams* p, const float* positions, uint32_t n, float* rgb) {
    const ViewGrid g = viewGrid(p);
    for (uint32_t i = 0; i < n; ++i) {
        const float3 c = calcCellColor(g, float3(positions[3 * i], positions[3 * i + 1], positions[3 * i + 2]));
        rgb[3 * i] = c.x; rgb[3 * i + 1] = c.y; rgb[3 * i + 2] = c.z;
    }
}

// the view's value of pixel i before alpha override / tone map / gamma; src = the source pixel (COLOR / NORMAL modes)
static void viewValue(const GfxPresentParams* config, const OrcViewInputs* in, const ViewGrid &grid, size_t i, float src[4]) {
    const GfxFrameParams* p = config->frame;
    const uint32_t* t = in->terminalInfo ? in->terminalInfo + 4 * i : nullptr;
    if (config->mode == GFX_PRESENT_NRC_PREDICTION) {                                 // copy_buffers.cu:52-67
        float3 radiance(0.0f);
        if (t[3] & 1u) {
            const float* r = in->inferredRadiance + 3 * i;
            radiance = max3(float3(r[0], r[1], r[2]), float3(0.0f));
            if (p->radianceScale > 0)
                radiance /= p->radianceScale;
            const float* q = in->inferenceQuery + 14 * i;
            radiance *= (float3(q[8], q[9], q[10]) + float3(q[11], q[12], q[13])); // useReflectanceFactorization
        }
        const float3 c = float3(u2f(t[0]), u2f(t[1]), u2f(t[2])) * radiance;
        src[0] = c.x; src[1] = c.y; src[2] = c.z; src[3] = 1.0f;
    }
    else if (config->mode == GFX_PRESENT_FLOW) {                                      // copy_buffers.cu:87-94
        const float* mv = in->gbuffer1 + 2 * i;
        src[0] = std::fmin(std::fmax(config->motionVectorScale * mv[0] + config->motionVectorOffset, 0.0f), 1.0f);
        src[1] = std::fmin(std::fmax(config->motionVectorScale * mv[1] + config->motionVectorOffset, 0.0f), 1.0f);
        src[2] = config->motionVectorOffset;
        src[3] = 1.0f;
    }
    else if (config->mode == GFX_PRESENT_NRC_PATH_LENGTH) {                           // copy_buffers.cu:96-112
        const int32_t pathLength = (int32_t)((t[3] >> 1) & 0xFFu);                    // an 8-bit field promotes to int
        const float tl = std::fmin((pathLength - 1) / 5.0f, 1.0f);
        const float3 R(1.0f, 0.0f, 0.0f), G(0.0f, 1.0f, 0.0f), B(0.0f, 0.0f, 1.0f);
        float3 v;
        if (tl < 0.5f) {
            const float tt = 2 * tl;
            v = B * (1.0f - tt) + G * tt;
        }
        else {
            const float tt = 2 * (tl - 0.5f);
            v = G * (1.0f - tt) + R * tt;
        }
        src[0] = v.x; src[1] = v.y; src[2] = v.z; src[3] = 1.0f;
    }
    else if (config->mode == GFX_PRESENT_COLOR && (config->flags & GFX_PRESENT_REGIR_CELLS)) { // regir copy_buffers.cu:99-107
        const float* g = in->gbuffer2 + 4 * i;
        const float3 cellColor = calcCellColor(grid, float3(g[0], g[1], g[2]));
        src[0] *= cellColor.x;
        src[1] *= cellColor.y;
        src[2] *= cellColor.z;
    }
    if (config->flags & GFX_PRESENT_NRC_TRAINING_PATHS) {                            // copy_buffers.cu:118-127
        if ((t[3] >> 9) & 1u) {
            src[0] *= 1.0f; src[1] *= 0.25f; src[2] *= 1.0f; src[3] *= 1.0f;
        }
        else if ((t[3] >> 10) & 1u) {
            src[0] *= 0.25f; src[1] *= 1.0f; src[2] *= 0.25f; src[3] *= 1.0f;
        }
    }
}

extern "C" void orc_present_views(const float* srcRGBA, uint32_t width, uint32_t height, const GfxPresentParams* config,
                                  const OrcViewInputs* in, uint32_t* image) {
    const ViewGrid grid = viewGrid(config->frame);
    const size_t n = (size_t)width * height;
    std::vector<float> view(4 * n);
    for (size_t i = 0; i < n; ++i) {
        float src[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
        if (config->mode == GFX_PRESENT_COLOR || config->mode == GFX_PRESENT_NORMAL) {
            const float* s = srcRGBA + 4 * i;
            src[0] = s[0]; src[1] = s[1]; src[2] = s[2]; src[3] = s[3];
        }
        if (config->mode == GFX_PRESENT_NORMAL) {                                       // copy_buffers.cu:22-25, 59-66
            float3 normal(src[0], src[1], src[2]);
            if (normal.x != 0 || normal.y != 0 || normal.z != 0)
                normal = normalize(normal);
            src[0] = 0.5f + 0.5f * normal.x;
            src[1] = 0.5f + 0.5f * normal.y;
            src[2] = 0.5f + 0.5f * normal.z;
            src[3] = 1.0f;
        }
        viewValue(config, in, grid, i, src);
        std::copy(src, src + 4, &view[4 * i]);
    }
    GfxPresentParams plain = *config;
    plain.mode = GFX_PRESENT_COLOR;
    plain.flags &= GFX_PRESENT_TONE_MAP | GFX_PRESENT_SRGB_GAMMA | GFX_PRESENT_FLIP_Y;
    orc_present(view.data(), width, height, &plain, image);
}

// visualizePrediction: the radiance query of every primary hit, built like nrcRayGen builds it, at row y * W + x (a miss
// leaves its row as it was); terminal info alpha 1, pathLength 1, hasQuery = hit; the host then infers W*H queries
// (neural_radiance_caching_main.cpp:2376-2384), pad128 like every inference launch here
extern "C" void orc_nrc_visualize_prediction(orc_frame* f, const GfxFrameParams* p) {
    orc_nrc_frame* n = nrcFrame(f);
    const orc_scene* s = f->scene;
    const Camera camera = makeCamera(p->camera);
    const uint32_t bufIdx = p->bufferIndex & 1;
    for (size_t pix = 0; pix < (size_t)f->W * f->H; ++pix) {
        const GB0 gb0 = f->gb0[bufIdx][pix];
        const bool hit = gb0.instSlot != 0xFFFFFFFFu;
        if (hit) {
            const float bcB = decodeBarycentric((uint16_t)(gb0.qbc & 0xFFFFu));
            const float bcC = decodeBarycentric((uint16_t)(gb0.qbc >> 16));
            const InstData &inst = s->instances[gb0.instSlot];
            const MeshData &mesh = s->meshes[gb0.geomInstSlot];
            SurfacePoint sp;
            computeSurfacePointFromGBuffer(s, inst, mesh, gb0.primIndex, bcB, bcC, &sp);
            float3 vOut = camera.position - sp.positionInWorld;
            const float primaryDist2 = sqLength(vOut);
            vOut /= std::sqrt(primaryDist2);
            const float primaryDotVN = dot(vOut, sp.geometricNormalInWorld);
            const float frontHit = primaryDotVN >= 0.0f ? 1.0f : -1.0f;
            const float3 positionInWorld = offsetRayOrigin(sp.positionInWorld, frontHit * sp.geometricNormalInWorld);
            const ReferenceFrame shadingFrame(sp.shadingNormalInWorld, sp.texCoord0DirInWorld); // no bump mapping here
            const BSDF bsdf = setupBsdf(s, mesh.materialSlot, sp.texCoord);
            createRadianceQuery(p, positionInWorld, shadingFrame.normal, vOut, bsdf, &n->inferenceQuery[14 * pix]);
        }
        writeTerminalInfo(n, pix, float3(1.0f), 1, hit, false, false);
    }
    n->state[NRC_NUM_INFERENCE_QUERIES] = (f->W * f->H + 127) / 128 * 128;
}
