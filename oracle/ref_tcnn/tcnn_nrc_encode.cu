// oracle/ref_tcnn/tcnn_nrc_encode.cu — TEST INFRASTRUCTURE: the input encoding of the reference's NRC network, as tiny-cuda-nn's
// NetworkWithInputEncoding runs it, built from the reference's own (vendored) tiny-cuda-nn sources where they lie (recipe:
// oracle/ref_tcnn/Makefile.encode -> oracle/_ref/libtcnn_nrc_encode.so, linked against the objects oracle/ref_tcnn/Makefile
// compiles; nothing of tiny-cuda-nn is copied into this repo).
//
// tcnn_nrc_encode builds NetworkWithInputEncoding from the encoding and network parts of NeuralRadianceCache::initialize's config
// (neural_radiance_caching/network_interface.cu:48-121, key for key, as oracle/ref_tcnn/tcnn_nrc.cu does) - the network part
// sets the alignment the Composite pads its last nested encoding to - and runs the network's own encoding
// (NetworkWithInputEncoding::encoding()) the way inference_mixed_precision_impl does (network_with_input_encoding.h:59-63), in
// the encoding's preferred layout.  tests/golden/make_golden_tcnn_triwave.py stores what it computes.
//
// C ABI (host pointers; returns 0 on success, the message on stderr otherwise).
#include <tiny-cuda-nn/config.h>
#include <tiny-cuda-nn/network_with_input_encoding.h>

#include <cstdint>
#include <cstdio>
#include <vector>

using namespace tcnn;
using precision_t = network_precision_t;

namespace {

constexpr uint32_t kNumInputDims = 14, kNumOutputDims = 3; // network_interface.cu:21-23

json encodingConfig(uint32_t posEnc) {
    json oneBlob = {{"n_dims_to_encode", 5}, {"otype", "OneBlob"}, {"n_bins", 4}};
    json identity = {{"n_dims_to_encode", 6}, {"otype", "Identity"}};
    json pos = posEnc == 0 ? json{{"n_dims_to_encode", 3}, {"otype", "TriangleWave"}, {"n_frequencies", 12}}
                           : json{{"n_dims_to_encode", 3}, {"otype", "HashGrid"}, {"per_level_scale", 2.0f},
                                  {"log2_hashmap_size", 15}, {"base_resolution", 16}, {"n_levels", 16}, {"n_features_per_level", 2}};
    return {{"otype", "Composite"}, {"nested", json::array({pos, oneBlob, identity})}};
}

} // namespace

extern "C" {

// posEnc: PositionEncoding (0 = TriangleWave, 1 = HashGrid); hostIn [numData][14]; hostOutHalf receives
// [numData][padded_output_width()] halves row-major whatever the encoding's layout; *width = padded_output_width() (64).
// A hash-grid encoding runs on the parameters its fresh network holds.
int tcnn_nrc_encode(uint32_t posEnc, uint32_t numHiddenLayers, const float* hostIn, uint32_t numData, uint16_t* hostOutHalf,
                    uint32_t* width) {
    try {
        if (numData & 0x7F)
            throw std::runtime_error{"numData must be a multiple of 128."};
        json network = {{"otype", "FullyFusedMLP"}, {"n_neurons", 64}, {"n_hidden_layers", numHiddenLayers},
                        {"activation", "ReLU"}, {"output_activation", "None"}};
        NetworkWithInputEncoding<precision_t> net{kNumInputDims, kNumOutputDims, encodingConfig(posEnc), network};
        GPUMemory<float> params(net.n_params());
        GPUMemory<precision_t> paramsHalf(net.n_params());
        pcg32 rng{1337};
        net.initialize_params(rng, params.data(), paramsHalf.data(), paramsHalf.data(), paramsHalf.data(), paramsHalf.data());
        const auto& encoding = net.encoding();
        const uint32_t w = encoding->padded_output_width();
        GPUMemory<float> dIn((size_t)numData * kNumInputDims);
        CUDA_CHECK_THROW(cudaMemcpy(dIn.data(), hostIn, dIn.get_bytes(), cudaMemcpyHostToDevice));
        GPUMatrix<float> inputs(dIn.data(), kNumInputDims, numData);
        GPUMatrixDynamic<precision_t> encoded{w, numData, nullptr, encoding->preferred_output_layout()};
        encoding->inference_mixed_precision(nullptr, inputs, encoded, true);
        CUDA_CHECK_THROW(cudaDeviceSynchronize());
        std::vector<uint16_t> raw((size_t)w * numData);
        CUDA_CHECK_THROW(cudaMemcpy(raw.data(), encoded.data(), raw.size() * sizeof(uint16_t), cudaMemcpyDeviceToHost));
        const bool columnMajor = encoded.layout() == CM; // CM: one sample's features contiguous
        for (uint32_t q = 0; q < numData; ++q)
            for (uint32_t k = 0; k < w; ++k)
                hostOutHalf[(size_t)q * w + k] = columnMajor ? raw[(size_t)q * w + k] : raw[(size_t)k * numData + q];
        *width = w;
        return 0;
    }
    catch (const std::exception& e) {
        fprintf(stderr, "tcnn_nrc_encode: %s\n", e.what());
        return 1;
    }
}

} // extern "C"
