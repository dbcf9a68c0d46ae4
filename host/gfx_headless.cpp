// gfx_headless.cpp — a headless C++ host on top of the C ABI of include/gfxb200.h.
//
// The reference hosts are C++ programs (restir_di/restir_di_main.cpp, path_tracing/path_tracing_main.cpp,
// regir/regir_main.cpp, neural_radiance_caching/neural_radiance_caching_main.cpp, svgf/svgf_main.cpp) whose frame loops end in OptiX /
// CUDA launches.  This file is those frame loops with the window, UI and asset import removed and every launch line
// replaced by the gfx_* call that INTEGRATION.md names for it; it exists to show (and to test, see
// tests/test_gpu_host_cpp.py) that the boundary is a plain C ABI: nothing here knows about Python, torch or CUDA
// types.  Scene and default parameters come from a flat binary file written by gfxexp_b200/scenes.py::save_scene_bin.
//
//   gfx_headless <scene.bin> <renderer> <width> <height> <frames> <out.raw> [nrc_params.f16] [-position-encoding tri|hash]
//                [-view prediction|pathlength|flow|cells|noisy|variance|filtered-variance|albedo|normal|motion|samples]
//                [-taa-jitter] [-bump-mapping]
//   -bump-mapping (every renderer but svgf): the apps' "Enable Bump Mapping" checkbox, GfxFrameParams::enableBumpMapping.  The
//   scene file carries no textures, so every material reads the reference's default 1x1 bump texel.
//   -position-encoding: the NRC network's position encoding, as the reference app's command line takes it
//   (neural_radiance_caching_main.cpp:458, 755-766); hash grid by default.  nrc_params.f16 must hold that network's
//   gfx_nrc_num_params halves.
//   renderer: restir | restir_unbiased | rearch | rearch_unbiased | pathtrace | regir | nrc | restir_nrc | restir_nrc_unbiased | svgf
//   restir_nrc[_unbiased]: ReSTIR DI + NRC as one estimator - the restir[_unbiased] frame, then the nrc frame's launches on the same
//   G-buffer with GFX_PT_NRC_INDIRECT, whose gfx_nrc_accumulate adds the light beyond the primary vertex to ReSTIR DI's image.
//   svgf: the SVGF app's frame (svgf_main.cpp:1980-2172) with its defaults - its own path tracer with specular mollification,
//   temporal accumulation, variance, 5 a-trous stages, background, albedo modulation + TAA; its output is the filtered image
//   GFX_BUF_SVGF_FINAL of the last frame instead of the beauty buffer.
//   -taa-jitter (svgf): the app's TAA sub-pixel jitter, GFX_SVGF_SUBPIXEL_JITTER; the app sets it whenever enableTemporalAA is on
//   (svgf_main.cpp:2005-2008), the library computes the offsets.
//   -view (with a .png output): write a debug view after the last frame instead of the beauty, as the reference apps'
//   "buffer to display" choices show it (gfx_present_launch): prediction = "Directly Visualized Prediction" (nrc: the
//   visualizePrediction pass + inference of the primary hits, neural_radiance_caching_main.cpp:2371-2387), pathlength =
//   "Rendering Path Length" (nrc), flow = "Motion Vector" (any renderer), cells = "Visualize Cells" (regir).
//   The SVGF app's views (svgf only): noisy, variance, filtered-variance, albedo, normal, motion and samples = "Noisy Beauty",
//   "Variance", "Filtered Variance", "Albedo", "Normal", "Motion Vector" and "Sample Count" (svgf_main.cpp:1823-1839): every
//   frame launches gfx_svgf_debug_visualize where the app does (:2138-2145, 2175-2185), and the last one is presented with the
//   app's display flags (:1907-1911).
// Output: the accumulated beauty buffer (svgf: the filtered image) (float4 per pixel, row-major) after <frames> frames, plus one line of JSON
// with the mean milliseconds per frame (wall clock around a synchronised loop).
#include "gfxb200.h"
#include "png_writer.h"

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

void check(gfx_ctx* ctx, int rc, const char* what) {
    if (rc != GFX_OK)
        throw std::runtime_error(std::string(what) + " failed (" + std::to_string(rc) + "): " +
                                 (ctx ? gfx_last_error_string(ctx) : "no context"));
}

struct SceneFile {
    std::vector<std::vector<float>> positions, normals, tangents, texcoords;
    std::vector<std::vector<uint32_t>> triangles;
    std::vector<GfxMeshDesc> meshes;
    std::vector<GfxMaterialDesc> materials;
    std::vector<GfxInstanceDesc> instances;
    std::vector<uint32_t> slots;
    GfxFrameParams defaults;
    GfxSceneDesc desc = {};
};

template <typename T>
void readInto(FILE* f, T* dst, size_t count) {
    if (count && fread(dst, sizeof(T), count, f) != count)
        throw std::runtime_error("scene file truncated");
}

void loadScene(const char* path, uint32_t width, uint32_t height, SceneFile* s) {
    FILE* f = fopen(path, "rb");
    if (!f)
        throw std::runtime_error(std::string("cannot open ") + path);
    char magic[4];
    uint32_t hdr[5];
    readInto(f, magic, 4);
    readInto(f, hdr, 5);
    if (memcmp(magic, "GFXS", 4) != 0 || hdr[4] != sizeof(GfxFrameParams))
        throw std::runtime_error("not a GFXS scene file of this ABI version");
    const uint32_t numMeshes = hdr[0], numMaterials = hdr[1], numInstances = hdr[2], numSlots = hdr[3];
    s->positions.resize(numMeshes); s->normals.resize(numMeshes); s->tangents.resize(numMeshes);
    s->texcoords.resize(numMeshes); s->triangles.resize(numMeshes); s->meshes.resize(numMeshes);
    for (uint32_t m = 0; m < numMeshes; ++m) {
        uint32_t mh[3];
        readInto(f, mh, 3);
        s->positions[m].resize(3 * (size_t)mh[0]); s->normals[m].resize(3 * (size_t)mh[0]);
        s->tangents[m].resize(3 * (size_t)mh[0]); s->texcoords[m].resize(2 * (size_t)mh[0]);
        s->triangles[m].resize(3 * (size_t)mh[1]);
        readInto(f, s->positions[m].data(), s->positions[m].size());
        readInto(f, s->normals[m].data(), s->normals[m].size());
        readInto(f, s->tangents[m].data(), s->tangents[m].size());
        readInto(f, s->texcoords[m].data(), s->texcoords[m].size());
        readInto(f, s->triangles[m].data(), s->triangles[m].size());
        GfxMeshDesc &d = s->meshes[m];
        d.positions = s->positions[m].data(); d.normals = s->normals[m].data(); d.tangents = s->tangents[m].data();
        d.texcoords = s->texcoords[m].data(); d.triangles = s->triangles[m].data();
        d.numVertices = mh[0]; d.numTriangles = mh[1]; d.materialSlot = mh[2];
    }
    s->materials.resize(numMaterials); s->instances.resize(numInstances); s->slots.resize(numSlots);
    readInto(f, s->materials.data(), numMaterials);
    readInto(f, s->instances.data(), numInstances);
    readInto(f, s->slots.data(), numSlots);
    readInto(f, &s->defaults, 1);
    fclose(f);
    // the file carries the parameter defaults for a square image; aspect follows the requested size
    s->defaults.camera.aspect = (float)width / (float)height;
    s->defaults.prevCamera.aspect = s->defaults.camera.aspect;
    s->desc.meshes = s->meshes.data(); s->desc.materials = s->materials.data(); s->desc.instances = s->instances.data();
    s->desc.instanceMeshSlots = s->slots.data();
    s->desc.numMeshes = numMeshes; s->desc.numMaterials = numMaterials; s->desc.numInstances = numInstances;
    s->desc.numInstanceMeshSlots = numSlots;
}

} // namespace

int main(int argc, char** argv) {
    if (argc < 7) {
        fprintf(stderr, "usage: %s <scene.bin> <renderer> <width> <height> <frames> <out.raw | out.png> [nrc_params.f16] "
                "[-position-encoding tri|hash] [-view prediction|pathlength|flow|cells|noisy|variance|filtered-variance|albedo|"
                "normal|motion|samples] [-taa-jitter] [-bump-mapping]\n", argv[0]);
        return 2;
    }
    const char* nrcParamsPath = nullptr;
    int positionEncoding = GFX_NRC_POSITION_ENCODING_HASH_GRID;
    std::string view;
    int svgfView = -1; // GfxSVGFView of an SVGF app view
    bool taaJitter = false;
    bool bumpMapping = false;
    for (int i = 7; i < argc; ++i) {
        const std::string arg = argv[i];
        if (arg == "-position-encoding" && i + 1 < argc) {
            const std::string v = argv[++i];
            if (v == "tri")
                positionEncoding = GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE;
            else if (v == "hash")
                positionEncoding = GFX_NRC_POSITION_ENCODING_HASH_GRID;
            else {
                fprintf(stderr, "-position-encoding takes tri or hash, not %s\n", v.c_str());
                return 2;
            }
        }
        else if (arg == "-view" && i + 1 < argc) {
            view = argv[++i];
            static const char* const svgfViews[] = { "noisy", "variance", "filtered-variance", "albedo", "normal", "motion", "samples" };
            for (int v = 0; v < 7; ++v)
                if (view == svgfViews[v])
                    svgfView = v; // GFX_SVGF_VIEW_NOISY_BEAUTY + v
            if (view != "prediction" && view != "pathlength" && view != "flow" && view != "cells" && svgfView < 0) {
                fprintf(stderr, "-view takes prediction, pathlength, flow, cells, noisy, variance, filtered-variance, albedo, "
                        "normal, motion or samples, not %s\n", view.c_str());
                return 2;
            }
        }
        else if (arg == "-taa-jitter")
            taaJitter = true;
        else if (arg == "-bump-mapping") // the apps' "Enable Bump Mapping" checkbox (perFramePlp.enableBumpMapping)
            bumpMapping = true;
        else if (!nrcParamsPath && arg[0] != '-')
            nrcParamsPath = argv[i];
        else {
            fprintf(stderr, "unexpected argument %s\n", argv[i]);
            return 2;
        }
    }
    const std::string renderer = argv[2];
    const std::string outPath = argv[6];
    const bool pngOut = outPath.size() > 4 && outPath.compare(outPath.size() - 4, 4, ".png") == 0;
    if (!view.empty() && (!pngOut || ((view == "prediction" || view == "pathlength") && renderer != "nrc") ||
                          (view == "cells" && renderer != "regir") || (svgfView >= 0 && renderer != "svgf"))) {
        fprintf(stderr, "-view %s needs a .png output and %s\n", view.c_str(),
                view == "cells" ? "the regir renderer" : view == "flow" ? "nothing else" : svgfView >= 0 ? "the svgf renderer" :
                "the nrc renderer");
        return 2;
    }
    if (taaJitter && renderer != "svgf") {
        fprintf(stderr, "-taa-jitter needs the svgf renderer\n");
        return 2;
    }
    if (bumpMapping && renderer == "svgf") { // the SVGF app has no bump mapping
        fprintf(stderr, "-bump-mapping does not apply to the svgf renderer\n");
        return 2;
    }
    const uint32_t width = (uint32_t)atoi(argv[3]), height = (uint32_t)atoi(argv[4]);
    const int frames = atoi(argv[5]);
    gfx_ctx* gfx = nullptr;
    gfx_nrc* nrc = nullptr;
    try {
        SceneFile scene;
        loadScene(argv[1], width, height, &scene);
        check(nullptr, gfx_ctx_create(0, &gfx), "gfx_ctx_create");                        // GPUEnvironment::initialize
        check(gfx, gfx_scene_upload(gfx, &scene.desc), "gfx_scene_upload");                // Scene::initialize + create*
        check(gfx, gfx_bvh_build(gfx, nullptr, 0), "gfx_bvh_build");                       // Scene::updateASs
        check(gfx, gfx_frame_create(gfx, width, height), "gfx_frame_create");
        check(gfx, gfx_rng_seed(gfx, 591842031321323413ull), "gfx_rng_seed");              // restir_di_main.cpp:1309-1321
        check(gfx, gfx_restir_setup_neighbor_table(gfx), "gfx_restir_setup_neighbor_table");

        const bool restirNrc = renderer == "restir_nrc" || renderer == "restir_nrc_unbiased";
        const bool unbiased = renderer == "restir_unbiased" || renderer == "rearch_unbiased" || renderer == "restir_nrc_unbiased";
        if (renderer == "nrc" || restirNrc) {
            check(gfx, gfx_nrc_create_with_encoding(gfx, positionEncoding, 2, 1e-2f, &nrc),  // neuralRadianceCache.initialize
                  "gfx_nrc_create_with_encoding");
            if (nrcParamsPath) {
                FILE* pf = fopen(nrcParamsPath, "rb");
                if (!pf)
                    throw std::runtime_error("cannot open the NRC parameter file");
                std::vector<uint16_t> halfParams(gfx_nrc_num_params(nrc));
                const size_t got = fread(halfParams.data(), 2, halfParams.size(), pf);
                const bool longer = fgetc(pf) != EOF;
                fclose(pf);
                if (got != halfParams.size() || longer)
                    throw std::runtime_error("the NRC parameter file does not hold this network's " +
                                             std::to_string(halfParams.size()) + " halves");
                check(gfx, gfx_nrc_set_params(nrc, halfParams.data(), halfParams.size() * 2), "gfx_nrc_set_params");
            }
        }
        std::mt19937 perFrameRng(72139121);                                                // neural_radiance_caching_main.cpp:1602

        GfxFrameParams fp = scene.defaults;
        fp.enableBumpMapping = bumpMapping ? 1u : 0u;
        // the NRC frame after its G-buffer pass (neural_radiance_caching_main.cpp:2270-2368)
        auto nrcFrame = [&](bool newSequence, int variant) {
            const uint32_t offsetToSelectUnbiasedTile = perFrameRng();
            const uint32_t offsetToSelectTrainingPath = perFrameRng();
            check(gfx, gfx_nrc_preprocess(gfx, nullptr, &fp, offsetToSelectUnbiasedTile, offsetToSelectTrainingPath, newSequence),
                  "preprocessNRC");
            check(gfx, gfx_pathtrace_launch(gfx, nullptr, &fp, variant), "pathTraceNRC");
            check(gfx, gfx_nrc_frame_infer(gfx, nrc, nullptr), "neuralRadianceCache.infer");
            check(gfx, gfx_nrc_accumulate(gfx, nullptr, &fp), "accumulateInferredRadianceValues");
            check(gfx, gfx_nrc_propagate(gfx, nullptr, &fp), "propagateRadianceValues");
            check(gfx, gfx_nrc_shuffle(gfx, nullptr, &fp), "shuffleTrainingData");
            check(gfx, gfx_nrc_frame_train(gfx, nrc, nullptr, nullptr), "neuralRadianceCache.train");
        };
        uint32_t lastSpatialNeighborBaseIndex = 0, lastReservoirIndex = 1;                 // restir_di_main.cpp:1685-1686
        const uint32_t numSpatialReusePasses = 1;
        double totalMs = 0.0;
        for (int frameIndex = 0; frameIndex < frames; ++frameIndex) {
            check(gfx, gfx_synchronize(gfx, nullptr), "gfx_synchronize");
            const auto t0 = std::chrono::steady_clock::now();
            const bool newSequence = frameIndex == 0;
            const uint32_t bufferIndex = frameIndex % 2;
            fp.numAccumFrames = (uint32_t)frameIndex;
            fp.frameIndex = (uint32_t)frameIndex;
            fp.bufferIndex = bufferIndex;
            fp.resetFlowBuffer = newSequence;
            fp.useUnbiasedEstimator = unbiased;
            check(gfx, gfx_light_dist_build(gfx, nullptr, bufferIndex), "gfx_light_dist_build");

            if (renderer == "restir" || renderer == "restir_unbiased" || restirNrc) {      // restir_di_main.cpp:2352-2421
                uint32_t currentReservoirIndex = (lastReservoirIndex + 1) % 2;
                fp.currentReservoirIndex = currentReservoirIndex;
                fp.spatialNeighborBaseIndex = lastSpatialNeighborBaseIndex;
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                const int entry = (fp.enableTemporalReuse && !newSequence)
                    ? (unbiased ? GFX_RESTIR_INITIAL_AND_TEMPORAL_UNBIASED : GFX_RESTIR_INITIAL_AND_TEMPORAL_BIASED)
                    : GFX_RESTIR_INITIAL_RIS;
                check(gfx, gfx_restir_launch(gfx, nullptr, &fp, entry), "performInitialAndTemporalRIS");
                if (fp.enableSpatialReuse) {
                    for (uint32_t i = 0; i < numSpatialReusePasses; ++i) {
                        fp.spatialNeighborBaseIndex = lastSpatialNeighborBaseIndex + fp.numSpatialNeighbors * i;
                        check(gfx, gfx_restir_launch(gfx, nullptr, &fp, unbiased ? GFX_RESTIR_SPATIAL_UNBIASED : GFX_RESTIR_SPATIAL_BIASED),
                              "performSpatialRIS");
                        currentReservoirIndex = (currentReservoirIndex + 1) % 2;
                        fp.currentReservoirIndex = currentReservoirIndex;
                    }
                    lastSpatialNeighborBaseIndex += fp.numSpatialNeighbors * numSpatialReusePasses;
                }
                check(gfx, gfx_restir_launch(gfx, nullptr, &fp, GFX_RESTIR_SHADING), "shading");
                lastReservoirIndex = currentReservoirIndex;
                if (restirNrc)
                    nrcFrame(newSequence, GFX_PT_NRC_INDIRECT);
            }
            else if (renderer == "rearch" || renderer == "rearch_unbiased") {              // restir_di_main.cpp:2423-2493
                const uint32_t currentReservoirIndex = (lastReservoirIndex + 1) % 2;
                fp.currentReservoirIndex = currentReservoirIndex;
                fp.spatialNeighborBaseIndex = lastSpatialNeighborBaseIndex;
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                check(gfx, gfx_restir_launch(gfx, nullptr, &fp, GFX_RESTIR_PRESAMPLE_LIGHTS), "performLightPreSampling");
                check(gfx, gfx_restir_launch(gfx, nullptr, &fp, GFX_RESTIR_PER_PIXEL_RIS), "performPerPixelRIS");
                GfxFrameParams launch = fp;
                if (newSequence)
                    launch.enableTemporalReuse = launch.enableSpatialReuse = 0;            // plain entry points on a new sequence
                check(gfx, gfx_restir_launch(gfx, nullptr, &launch, GFX_RESTIR_TRACE_SHADOW_RAYS), "traceShadowRays");
                check(gfx, gfx_restir_launch(gfx, nullptr, &launch, GFX_RESTIR_SHADE_AND_RESAMPLE), "shadeAndResample");
                ++lastSpatialNeighborBaseIndex;
                lastReservoirIndex = currentReservoirIndex;
            }
            else if (renderer == "pathtrace") {                                            // path_tracing_main.cpp:1771-1789
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                check(gfx, gfx_pathtrace_launch(gfx, nullptr, &fp, GFX_PT_BASELINE), "pathTraceBaseline");
            }
            else if (renderer == "regir") {                                                // regir_main.cpp:2022-2068
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                check(gfx, gfx_regir_build_cells(gfx, nullptr, &fp, (uint32_t)frameIndex, !newSequence), "buildCellReservoirs");
                check(gfx, gfx_pathtrace_launch(gfx, nullptr, &fp, GFX_PT_REGIR), "pathTraceReGIR");
                check(gfx, gfx_regir_update_access(gfx, nullptr, &fp, (uint32_t)frameIndex), "updateLastAccessFrameIndices");
            }
            else if (renderer == "nrc") {                                                  // neural_radiance_caching_main.cpp:2256-2368
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                nrcFrame(newSequence, GFX_PT_NRC);
            }
            else if (renderer == "svgf") {                                                 // svgf_main.cpp:1980-2172
                constexpr uint32_t numFilteringStages = 5;
                fp.svgfFlags |= GFX_SVGF_ENABLE_TEMPORAL_ACCUMULATION | GFX_SVGF_MOLLIFY_SPECULAR;  // the app's defaults (:1729-1733)
                if (taaJitter)
                    fp.svgfFlags |= GFX_SVGF_SUBPIXEL_JITTER;  // :2005-2008, with enableTemporalAA (on in the scene file's defaults)
                if (newSequence)
                    fp.svgfFlags |= GFX_SVGF_IS_FIRST_FRAME;
                else
                    fp.svgfFlags &= ~(uint32_t)GFX_SVGF_IS_FIRST_FRAME;
                check(gfx, gfx_gbuffer_launch(gfx, nullptr, &fp), "gfx_gbuffer_launch");
                check(gfx, gfx_pathtrace_launch(gfx, nullptr, &fp, GFX_PT_SVGF), "pathTraceWithTemporalAccumulation");
                check(gfx, gfx_svgf_launch(gfx, nullptr, &fp, GFX_SVGF_TEMPORAL_ACCUMULATE, 0), "temporal accumulation");
                check(gfx, gfx_svgf_launch(gfx, nullptr, &fp, GFX_SVGF_ESTIMATE_VARIANCE, 0), "estimateVariance");
                if (svgfView == GFX_SVGF_VIEW_NOISY_BEAUTY || svgfView == GFX_SVGF_VIEW_VARIANCE)  // :2138-2145
                    check(gfx, gfx_svgf_debug_visualize(gfx, nullptr, &fp, svgfView, 0.5f, 0.1f, numFilteringStages), "debugVisualize");
                for (uint32_t stage = 0; stage < numFilteringStages; ++stage)
                    check(gfx, gfx_svgf_launch(gfx, nullptr, &fp, GFX_SVGF_ATROUS, stage), "applyATrousFilter_box3x3");
                check(gfx, gfx_svgf_launch(gfx, nullptr, &fp, GFX_SVGF_FILL_BACKGROUND, numFilteringStages), "fillBackground");
                check(gfx, gfx_svgf_launch(gfx, nullptr, &fp, GFX_SVGF_MODULATE_TAA, numFilteringStages),
                      "applyAlbedoModulationAndTemporalAntiAliasing");
                if (svgfView > GFX_SVGF_VIEW_VARIANCE)  // :2175-2185; offset 0.5, scale 10^-1 (:1724, 2143)
                    check(gfx, gfx_svgf_debug_visualize(gfx, nullptr, &fp, svgfView, 0.5f, 0.1f, numFilteringStages), "debugVisualize");
            }
            else {
                throw std::runtime_error("unknown renderer " + renderer);
            }
            check(gfx, gfx_synchronize(gfx, nullptr), "gfx_synchronize");
            totalMs += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        }

        // the svgf renderer shows the filtered image of the last frame's temporal set
        const int outBuffer = renderer == "svgf" ? GFX_BUF_SVGF_FINAL : GFX_BUF_BEAUTY_ACCUM;
        const uint32_t outIndex = renderer == "svgf" ? fp.bufferIndex : 0u;
        if (pngOut) {
            // the reference's screenshot: tone map + sRGB gamma on the accumulated beauty (saveImage with
            // SDRImageSaverConfig, common_host.cpp:2859-2897; brightness 0 -> scale 10^0), written as PNG
            GfxPresentParams pp = { outBuffer, outIndex, GFX_PRESENT_COLOR, GFX_PRESENT_TONE_MAP | GFX_PRESENT_SRGB_GAMMA, 1.0f, 1.0f,
                                    &fp, 0.1f, 0.5f };  // motion vectors x 10^-1 + 0.5 (neural_radiance_caching_main.cpp:2462)
            if (view == "prediction") {                                                    // :2371-2387
                check(gfx, gfx_pathtrace_launch(gfx, nullptr, &fp, GFX_PT_NRC_VISUALIZE_PREDICTION), "visualizePrediction");
                check(gfx, gfx_nrc_frame_infer(gfx, nrc, nullptr), "neuralRadianceCache.infer");
                pp.mode = GFX_PRESENT_NRC_PREDICTION;
            }
            else if (view == "pathlength")
                pp.mode = GFX_PRESENT_NRC_PATH_LENGTH;
            else if (view == "flow")
                pp.mode = GFX_PRESENT_FLOW;
            else if (view == "cells")
                pp.flags |= GFX_PRESENT_REGIR_CELLS;
            else if (svgfView >= 0) {                                                     // svgf_main.cpp:1907-1911
                pp.sourceBuffer = GFX_BUF_SVGF_DEBUG_VISUALIZE;
                pp.sourceIndex = 0;
                pp.flags = svgfView <= GFX_SVGF_VIEW_FILTERED_VARIANCE ? GFX_PRESENT_TONE_MAP | GFX_PRESENT_SRGB_GAMMA : 0u;
            }
            check(gfx, gfx_present_launch(gfx, nullptr, &pp), "gfx_present_launch");
            std::vector<uint32_t> image((size_t)width * height);
            check(gfx, gfx_buffer_download(gfx, nullptr, GFX_BUF_PRESENT_RGBA8, 0, image.data(), image.size() * 4), "gfx_buffer_download");
            if (!gfxhost::writePng(outPath.c_str(), width, height, image.data()))
                throw std::runtime_error("cannot write the output image");
        }
        else {
            std::vector<float> beauty((size_t)width * height * 4);
            check(gfx, gfx_buffer_download(gfx, nullptr, outBuffer, outIndex, beauty.data(), beauty.size() * 4), "gfx_buffer_download");
            FILE* of = fopen(outPath.c_str(), "wb");
            if (!of || fwrite(beauty.data(), 4, beauty.size(), of) != beauty.size())
                throw std::runtime_error("cannot write the output image");
            fclose(of);
        }
        printf("{\"renderer\": \"%s\", \"width\": %u, \"height\": %u, \"frames\": %d, \"ms_per_frame\": %.4f, \"kernel_launches\": %llu}\n",
               renderer.c_str(), width, height, frames, totalMs / frames, (unsigned long long)gfx_kernel_launch_count(gfx));
    }
    catch (const std::exception &e) {
        fprintf(stderr, "gfx_headless: %s\n", e.what());
        if (nrc) gfx_nrc_destroy(nrc);
        if (gfx) gfx_ctx_destroy(gfx);
        return 1;
    }
    if (nrc) gfx_nrc_destroy(nrc);
    gfx_ctx_destroy(gfx);
    return 0;
}
