// oracle/svgf_views.cpp — TEST INFRASTRUCTURE (CPU oracle).  CPU restatement of the SVGF app's "Buffer to Display" debug
// views, gfx_svgf_debug_visualize:
//   debugVisualize           svgf/gpu_kernels/visualize.cu:6-87 (the per-view arithmetic :27-83)
//   launch sites             svgf/svgf_main.cpp:2138-2145 (Noisy Beauty, Variance), :2175-2185 (the others)
// The app reads the lighting, albedo and moment planes at the launch index, its G-buffers at glPix(launch index), and writes
// the view at glPix(launch index), the indexing of applyAlbedoModulationAndTemporalAntiAliasing (svgf.cu:555, 610); every
// plane here is top-down like the final image, so pixel (x, y) of each plane is pixel (x, y) of the view.
//
// This file compiles the SVGF app's oracle with its TAA jitter (svgf_taa_jitter.cpp, which compiles svgf_app.cpp and
// render.cpp) into its own library, liborc_svgf_views.so (Makefile.svgf_views, bound by tests/oracle_svgf_views.py), and links
// denoise.o, so the views read the planes of that library's SVGF passes: lighting 0 and 1, albedo and moments through
// orc_svgf_buffer_ptr.  The oracle's SVGF state keeps no normal plane and does not export its prevScreenPos, so
// orc_svgf_view_inputs restates the two from the frame as the passes write them: the shading normal the temporal pass decodes
// (0 at background pixels) and prevScreenPos = ((x, y) + 0.5 - motion vector) / (W, H) at hits, fillBackground's reprojected
// pixel-centre direction at background pixels (denoise.cpp, svgf.cu:443-449).  Both are the values of the frame's last
// temporal pass and background fill, which is where the app launches the views that read them.
#include "svgf_taa_jitter.cpp"

// the planes a view reads (tests/oracle_svgf_views.py mirrors the struct)
struct OrcSvgfViewPlanes {
    const float* lighting[2];      // float4 per pixel: lighting rgb + variance, planes 0 and 1
    const float* albedo;           // float4: the SVGF albedo
    const float* normal;           // float4: the decoded shading normal
    const float* prevScreenPos;    // float2
    const uint32_t* moments;       // uint32 x4: the moments of the current temporal set, z = sampleInfo
};

// debugVisualize on rows [y0, y1) of `in`; out: float4 per pixel.  -1 for a view outside 0..6.
extern "C" int orc_svgf_view_planes(const OrcSvgfViewPlanes* in, uint32_t W, uint32_t H, uint32_t y0, uint32_t y1, int view,
                                    int modulateAlbedo, float motionVectorOffset, float motionVectorScale,
                                    uint32_t numFilteringStages, float* out) {
    if (view < GFX_SVGF_VIEW_NOISY_BEAUTY || view > GFX_SVGF_VIEW_SAMPLE_COUNT)
        return -1;
    for (uint32_t y = y0; y < std::min(y1, H); ++y) {
        for (uint32_t x = 0; x < W; ++x) {
            const size_t pix = (size_t)y * W + x;
            float c[4] = { 0.0f, 0.0f, 0.0f, 1.0f };
            switch (view) {
            case GFX_SVGF_VIEW_NOISY_BEAUTY: { // :28-38
                const float* l = in->lighting[0] + 4 * pix;
                c[0] = l[0]; c[1] = l[1]; c[2] = l[2];
                if (modulateAlbedo) {
                    const float* a = in->albedo + 4 * pix;
                    c[0] *= a[0]; c[1] *= a[1]; c[2] *= a[2];
                }
            } break;
            case GFX_SVGF_VIEW_VARIANCE: // :39-45
                c[0] = c[1] = c[2] = std::sqrt(in->lighting[0][4 * pix + 3]);
                break;
            case GFX_SVGF_VIEW_FILTERED_VARIANCE: // :46-52
                c[0] = c[1] = c[2] = std::sqrt(in->lighting[numFilteringStages % 2][4 * pix + 3]);
                break;
            case GFX_SVGF_VIEW_ALBEDO: { // :53-57
                const float* a = in->albedo + 4 * pix;
                c[0] = a[0]; c[1] = a[1]; c[2] = a[2];
            } break;
            case GFX_SVGF_VIEW_NORMAL: { // :58-62, 0.5 * n + Normal3D(0.5)
                const float* n = in->normal + 4 * pix;
                c[0] = 0.5f * n[0] + 0.5f; c[1] = 0.5f * n[1] + 0.5f; c[2] = 0.5f * n[2] + 0.5f;
            } break;
            case GFX_SVGF_VIEW_MOTION_VECTOR: { // :63-73
                const float* psp = in->prevScreenPos + 2 * pix;
                const float curX = (x + 0.5f) / W, curY = (y + 0.5f) / H;
                const float mvX = (float)W * (curX - psp[0]), mvY = (float)H * (curY - psp[1]);
                c[0] = std::fmin(std::fmax(motionVectorScale * mvX + motionVectorOffset, 0.0f), 1.0f);
                c[1] = std::fmin(std::fmax(motionVectorScale * mvY + motionVectorOffset, 0.0f), 1.0f);
                c[2] = motionVectorOffset;
            } break;
            default: { // GFX_SVGF_VIEW_SAMPLE_COUNT, :74-80: sampleInfo.count is the low 24 bits
                const uint32_t count = in->moments[4 * pix + 2] & 0xFFFFFFu;
                c[0] = c[1] = c[2] = std::fmin(count / 255.0f, 1.0f);
            } break;
            }
            std::memcpy(out + 4 * pix, c, 16);
        }
    }
    return 0;
}

// the shading normal (float4, w = 0) and prevScreenPos (float2) of rows [tileOriginY, +tileRows) of the oracle frame `f`, as
// GFX_SVGF_TEMPORAL_ACCUMULATE and GFX_SVGF_FILL_BACKGROUND of the frame params `p` write them
extern "C" void orc_svgf_view_inputs(orc_frame* f, const GfxFrameParams* p, float* normal, float* prevScreenPos) {
    const uint32_t W = f->W, H = f->H;
    const uint32_t bufIdx = p->bufferIndex & 1;
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    const auto camera = [](const GfxCamera &c, Mat3* orientation, float* vw, float* vh) {
        std::memcpy(orientation->m, c.orientation, 36);
        *vh = 2 * std::tan(c.fovY * 0.5f);
        *vw = c.aspect * *vh;
    };
    Mat3 orientation, prevOrientation;
    float vw, vh, prevVw, prevVh;
    camera(p->camera, &orientation, &vw, &vh);
    camera(p->prevCamera, &prevOrientation, &prevVw, &prevVh);
    for (uint32_t y = y0; y < y1; ++y) {
        for (uint32_t x = 0; x < W; ++x) {
            const size_t pix = (size_t)y * W + x;
            float2 psp(0.0f, 0.0f);
            float3 n(0.0f);
            if (f->gb0[bufIdx][pix].instSlot != 0xFFFFFFFFu) { // temporal pass
                n = decodeVector(f->gb3[bufIdx][pix].qShadingNormal);
                const GB1 mv = f->gb1[bufIdx][pix];
                psp = float2((x + 0.5f - mv.mvx) / W, (y + 0.5f - mv.mvy) / H);
            }
            else { // fillBackground: the pixel centre's direction in the previous camera's frame
                const float fx = (x + 0.5f) / W;
                const float fy = (y + 0.5f) / H;
                float3 direction = normalize(orientation.mul(float3(vw * (0.5f - fx), vh * (0.5f - fy), 1)));
                const float* o = prevOrientation.m;
                direction = float3(o[0] * direction.x + o[3] * direction.y + o[6] * direction.z,
                                   o[1] * direction.x + o[4] * direction.y + o[7] * direction.z,
                                   o[2] * direction.x + o[5] * direction.y + o[8] * direction.z);
                direction /= direction.z;
                psp = float2(0.5f - direction.x / prevVw, 0.5f - direction.y / prevVh);
            }
            normal[4 * pix + 0] = n.x; normal[4 * pix + 1] = n.y; normal[4 * pix + 2] = n.z; normal[4 * pix + 3] = 0.0f;
            prevScreenPos[2 * pix + 0] = psp.x; prevScreenPos[2 * pix + 1] = psp.y;
        }
    }
}

// gfx_svgf_debug_visualize on the oracle's SVGF state `s` of frame `f`: the rows of `p` of `out` (float4 per pixel); -1 for a
// view outside 0..6
extern "C" int orc_svgf_debug_visualize(orc_svgf* s, orc_frame* f, const GfxFrameParams* p, int view, float motionVectorOffset,
                                        float motionVectorScale, uint32_t numFilteringStages, float* out) {
    const uint32_t W = f->W, H = f->H;
    const size_t n = (size_t)W * H;
    std::vector<float> normal(4 * n, 0.0f), prevScreenPos(2 * n, 0.0f);
    orc_svgf_view_inputs(f, p, normal.data(), prevScreenPos.data());
    OrcSvgfViewPlanes in;
    for (uint32_t i = 0; i < 2; ++i)
        in.lighting[i] = (const float*)orc_svgf_buffer_ptr(s, GFX_BUF_SVGF_LIGHTING_VARIANCE, i, nullptr);
    in.albedo = (const float*)orc_svgf_buffer_ptr(s, GFX_BUF_SVGF_ALBEDO, 0, nullptr);
    in.normal = normal.data();
    in.prevScreenPos = prevScreenPos.data();
    in.moments = (const uint32_t*)orc_svgf_buffer_ptr(s, GFX_BUF_SVGF_MOMENTS, p->bufferIndex & 1, nullptr);
    const uint32_t y0 = p->tileOriginY, y1 = p->tileRows ? std::min(H, p->tileOriginY + p->tileRows) : H;
    return orc_svgf_view_planes(&in, W, H, y0, y1, view, (p->svgfFlags & GFX_SVGF_MODULATE_ALBEDO) != 0, motionVectorOffset,
                                motionVectorScale, numFilteringStages, out);
}
