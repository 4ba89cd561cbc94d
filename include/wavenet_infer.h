/*
 * wavenet_infer.h -- the reference's C-ABI for the WaveNet inference hot path, kept verbatim
 * in meaning so that libwavenet_infer.so built from this repo is a drop-in for the one built
 * by the reference (replaces pytorch/wavenet_infer.h:28-58 / pytorch/wavenet_infer.cu:105-149).
 *
 * Semantics kept from the reference (pytorch/wavenet_infer.cu:40-145):
 *   - R/S/A are fixed at build time: R=64, S=256, A=256, arithmetic in fp32
 *     (typedef nvWavenetInfer<float,float,R,S,A>, wavenet_infer.cu:35-38);
 *   - every float* may point to host or device memory and is copied before return;
 *     the float** arguments are host arrays of num_layers pointers;
 *   - all matrices fp32 column-major M x K (README.md:38); embeddings A x R as emb[a*R + r];
 *   - cond_input is float[sample_count][num_layers][batch_size][2R];
 *   - output-layer biases are zero (wavenet_infer.cu:75-82);
 *   - output selectors are drawn on the host with libc rand(), two draws per element,
 *     batch-major, value = rand()/RAND_MAX  (Matrix::randomize(0.5, 1.0), wavenet_infer.cu:92-93,
 *     matrix.cpp:38-56) -- so a caller that seeds srand() gets the reference's selectors;
 *   - samples is caller-allocated int[batch_size][sample_count], host OR device;
 *   - synchronous; CUDA failures print "GPUassert: ..." to stderr and exit(code)
 *     (nv_wavenet_util.cuh:34-40);
 *   - `implementation` 0..4 (AUTO, SINGLE_BLOCK, DUAL_BLOCK, PERSISTENT, MANYBLOCK) is accepted
 *     and ignored: one sm_90a kernel family replaces all four.
 *
 * The arithmetic of this entry point is bit-exact fp32 (DESIGN.md §4).  wavenet_infer_fp16 (below) takes the same arguments
 * and runs the fp16 kernels (the reference builds a second library with T_data = half for that, README.md:24-25).
 */
#ifndef WAVENET_INFER_H
#define WAVENET_INFER_H

#ifdef __cplusplus
extern "C" {
#endif

/* Argument order and types are the ABI (pytorch/wavenet_infer.h:34-52); the reference's parameter names are given in
 * the comments.  L = n_layers; every matrix fp32 column-major. */
void wavenet_infer(int n_samples,                 /* sample_count */
                   int n_utterances,              /* batch_size */
                   float* emb_prev,               /* embedding_prev  [A][R] */
                   float* emb_cur,                /* embedding_curr  [A][R] */
                   int n_layers,                  /* num_layers */
                   int max_dilation,
                   float** w_prev,                /* in_layer_weights_prev  L x (2R x R), the x[t-d] half of the dilated conv */
                   float** w_cur,                 /* in_layer_weights_curr  L x (2R x R), the x[t] half */
                   float** b_gate,                /* in_layer_biases        L x 2R */
                   float** w_res,                 /* res_layer_weights      L x (R x R) */
                   float** b_res,                 /* res_layer_biases       L x R */
                   float** w_skip,                /* skip_layer_weights     L x (S x R) */
                   float** b_skip,                /* skip_layer_biases      L x S */
                   float* w_zs,                   /* conv_out_weight        A x S */
                   float* w_za,                   /* conv_end_weight        A x A */
                   int tanh_on_embedding,         /* use_embed_tanh */
                   float* conditioning,           /* cond_input  [n_samples][L][n_utterances][2R] */
                   int implementation,
                   int* samples_out);             /* samples     [n_utterances][n_samples] */

/* Same arguments and semantics, fp16 arithmetic (weights, conditioning and GEMM inputs rounded to fp16, fp32 accumulation). */
void wavenet_infer_fp16(int n_samples, int n_utterances, float* emb_prev, float* emb_cur, int n_layers, int max_dilation,
                        float** w_prev, float** w_cur, float** b_gate, float** w_res, float** b_res, float** w_skip, float** b_skip,
                        float* w_zs, float* w_za, int tanh_on_embedding, float* conditioning, int implementation, int* samples_out);

/* channel counts of this build (pytorch/wavenet_infer.h:54-57) */
int get_R(void);
int get_S(void);
int get_A(void);

#ifdef __cplusplus
}
#endif
#endif
