// wavenet_infer.cu -- the reference's C-ABI (include/wavenet_infer.h) on top of the engine.
// Replaces pytorch/wavenet_infer.cu:40-149 of the reference; semantics documented in the header.
#include "../../include/wavenet_infer.h"
#include "../../include/nvwn_b200.h"

#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace {
// must match the wavenet channels (pytorch/wavenet_infer.cu:34-37)
const int A = 256;
const int R = 64;
const int S = 256;

// error convention of the reference: print "GPUassert: ..." and exit (nv_wavenet_util.cuh:34-40)
void check(int rc, const char* what)
{
    if (rc != 0) {
        fprintf(stderr, "GPUassert: %s (%s) %s %d\n", nvwn_last_error(), what, __FILE__, rc);
        exit(rc > 0 ? rc : 1);
    }
}

void infer_impl(int dtype, int sample_count, int batch_size, float* embedding_prev, float* embedding_curr,
                int num_layers, int max_dilation,
                float** in_layer_weights_prev, float** in_layer_weights_curr, float** in_layer_biases,
                float** res_layer_weights, float** res_layer_biases,
                float** skip_layer_weights, float** skip_layer_biases,
                float* conv_out_weight, float* conv_end_weight, int use_embed_tanh,
                float* cond_input, int implementation, int* samples)
{
    if (!samples) { fprintf(stderr, "wavenet_infer: samples must not be NULL\n"); abort(); }   // assert(samples), wavenet_infer.cu:142
    nvwn_engine* e = nullptr;
    check(nvwn_create(&e, dtype, R, S, A, num_layers, max_dilation, batch_size, sample_count,
                      (implementation >= 0 && implementation <= 4) ? NVWN_KERNEL_AUTO : implementation, use_embed_tanh),
          "create");
    check(nvwn_set_embeddings(e, embedding_prev, embedding_curr), "setEmbeddings");
    for (int l = 0; l < num_layers; l++) {
        check(nvwn_set_layer_weights(e, l, in_layer_weights_prev[l], in_layer_weights_curr[l], in_layer_biases[l],
                                     res_layer_weights[l], res_layer_biases[l], skip_layer_weights[l], skip_layer_biases[l]),
              "setLayerWeights");
    }
    // "We didn't use biases on our outputs" (wavenet_infer.cu:75-82)
    std::vector<float> zero_bias(A, 0.f);
    check(nvwn_set_out_weights(e, conv_out_weight, zero_bias.data(), conv_end_weight, zero_bias.data()), "setOutWeights");

    // Matrix outputSelectors(batch_size, sample_count); outputSelectors.randomize(0.5, 1.0)  (wavenet_infer.cu:92-93): libc rand()
    std::vector<float> selectors((size_t)sample_count * batch_size);
    check(nvwn_libc_selectors(selectors.data(), batch_size, sample_count), "selectors");
    check(nvwn_set_inputs(e, cond_input, selectors.data()), "setInputs");
    check(nvwn_run(e, sample_count, batch_size, samples, /*dumpActivations=*/1, nullptr), "run");
    cudaError_t ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) {
        fprintf(stderr, "GPUassert: %s %s %d\n", cudaGetErrorString(ce), __FILE__, __LINE__);
        exit(ce);
    }
    nvwn_destroy(e);
}
}  // namespace

extern "C" {

void wavenet_infer(int sample_count, int batch_size, float* embedding_prev, float* embedding_curr, int num_layers, int max_dilation,
                   float** in_layer_weights_prev, float** in_layer_weights_curr, float** in_layer_biases, float** res_layer_weights,
                   float** res_layer_biases, float** skip_layer_weights, float** skip_layer_biases, float* conv_out_weight,
                   float* conv_end_weight, int use_embed_tanh, float* cond_input, int implementation, int* samples)
{
    infer_impl(NVWN_FP32, sample_count, batch_size, embedding_prev, embedding_curr, num_layers, max_dilation, in_layer_weights_prev,
               in_layer_weights_curr, in_layer_biases, res_layer_weights, res_layer_biases, skip_layer_weights, skip_layer_biases,
               conv_out_weight, conv_end_weight, use_embed_tanh, cond_input, implementation, samples);
}

// same arguments, fp16 arithmetic (T_data = half build of the reference: README.md:24-25, a second .so there; a second symbol here)
void wavenet_infer_fp16(int sample_count, int batch_size, float* embedding_prev, float* embedding_curr, int num_layers, int max_dilation,
                        float** in_layer_weights_prev, float** in_layer_weights_curr, float** in_layer_biases, float** res_layer_weights,
                        float** res_layer_biases, float** skip_layer_weights, float** skip_layer_biases, float* conv_out_weight,
                        float* conv_end_weight, int use_embed_tanh, float* cond_input, int implementation, int* samples)
{
    infer_impl(NVWN_FP16, sample_count, batch_size, embedding_prev, embedding_curr, num_layers, max_dilation, in_layer_weights_prev,
               in_layer_weights_curr, in_layer_biases, res_layer_weights, res_layer_biases, skip_layer_weights, skip_layer_biases,
               conv_out_weight, conv_end_weight, use_embed_tanh, cond_input, implementation, samples);
}

int get_R(void) { return R; }
int get_S(void) { return S; }
int get_A(void) { return A; }

}  // extern "C"
