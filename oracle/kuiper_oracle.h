/* kuiper_oracle.h -- CPU restatement of the KuiperLLama decode hot path.
 *
 * TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may build, load or call this.  The product library
 * (kuiperllama_b200/) never links it and has no CPU fallback.
 *
 * Every function restates one piece of the reference (paths relative to its root) in
 * plain C with fp32 arithmetic in the reference's CPU order.  The reference's CPU matmul
 * delegates to Armadillo 14.0.1 -> OpenBLAS sgemv (un-vendored, version unpinned;
 * kuiper/source/op/kernels/cpu/matmul_kernel.cpp:37-40), whose summation order is not part
 * of the reference; the restatement uses a strict left-to-right fp32 dot product
 * (KO_MATMUL_STRICT) and, for the timed baseline only, an optional BLAS/OpenMP path.
 *
 * Pinning (SURVEY.md section 8c): tests/test_oracle_golden.py checks this file against every
 * known-answer vector the reference's own tests hold for the path (test_load.cpp:102-105,
 * test_cu_matmul.cpp:55-75, test_cu_emb.cpp:28-57, test_cu_add.cpp:24) and against fixtures
 * produced by importing the reference's PyTorch model + exporter (tools/model.py,
 * tools/export.py) -- see tests/golden/make_golden.py.
 */
#ifndef KUIPER_ORACLE_H_
#define KUIPER_ORACLE_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* RoPE / eps flavour = the reference's compile-time build flags (CMakeLists.txt:16-25). */
enum {
  KO_FLAVOUR_LLAMA2 = 0,
  KO_FLAVOUR_LLAMA3 = 1,
  KO_FLAVOUR_QWEN2 = 2,
  /* test-only: Qwen2 FILE LAYOUT (qkv bias interleaved, export_qwen2.py:103-110) with Llama-2
   * arithmetic -- what tools/model_qwen2.py actually computes; pins the layout against it. */
  KO_FLAVOUR_QWEN2FILE = 3
};
enum { KO_MATMUL_STRICT = 0, KO_MATMUL_FAST = 1 };

void ko_set_matmul_mode(int mode);       /* default KO_MATMUL_STRICT */
int ko_set_blas_library(const char* so); /* dlopen an OpenBLAS for KO_MATMUL_FAST; 0 = ok */
int ko_num_threads(void);                /* threads KO_MATMUL_FAST will use */
int ko_set_num_threads(int n);           /* OpenMP + loaded BLAS, via their APIs; returns the BLAS's count (0: none) */

float ko_flavour_eps(int flavour);   /* rmsnorm_kernel.cpp:20-24 */
float ko_flavour_theta(int flavour); /* rope_kernel.cpp:8,48,88 */

/* cpu/matmul_kernel.cpp:5-41: out[K] = (W[K,M] . x[M]) * scale, W row-major [out,in]. */
void ko_matmul_f32(const float* x, const float* w, float* out, int M, int K, float scale);
/* cuda/matmul_kernel.cu:68-74 (no CPU version exists): sum_i x[i]*scales[(p*M+i)/g]*(float)w. */
void ko_matmul_w8(const float* x, const int8_t* w, const float* scales, float* out, int M, int K,
                  int group_size);
/* Same, but in the CUDA kernel's exact reduction order (128 strided lanes, cub warp-shuffle
 * tree, sequential add of 4 warp aggregates) -- the bit-exact target for the int8 path. */
void ko_matmul_w8_cuda_order(const float* x, const int8_t* w, const float* scales, float* out,
                             int M, int K, int group_size);
/* fp32 GEMV in the CUDA kernel's exact order (cuda/matmul_kernel.cu:6-54). */
void ko_matmul_f32_cuda_order(const float* x, const float* w, float* out, int M, int K);

void ko_rmsnorm(const float* x, const float* w, float* out, int n, float eps);
void ko_add(const float* a, const float* b, float* out, int n);
void ko_swiglu(const float* x1, const float* x3, float* out, int n);
void ko_softmax_inplace(float* x, int n);
void ko_scale_sum(const float* value, const float* score, float* out, int pos, int size,
                  int stride);
void ko_embedding(const int32_t* tokens, int n_tokens, const float* table, float* out, int dim,
                  int vocab);
int64_t ko_argmax(const float* logits, int64_t n);
void ko_sincos(int head_size, int seq_len, float theta, float* sin_cache, float* cos_cache);
void ko_rope(int flavour, int dim, int kv_dim, int head_size, float* q, float* k, int pos,
             const float* sin_cache, const float* cos_cache);
void ko_mha(int pos, int head_num, int layer_index, int seq_len, int kv_dim, int kv_mul,
            int head_size, float* out, const float* q, float* score, const float* key_cache,
            const float* value_cache);

/* export.py:49-73 quantize_q80: symmetric int8, groups of g consecutive elements. */
void ko_quantize_q80(const float* w, int64_t n, int group_size, int8_t* q, float* scales);

/* ---- whole model: model.cpp:41-151 (file), llama3.cpp:147-167,600-745 (forward) -------- */
typedef struct ko_model ko_model;

typedef struct {
  int32_t dim, hidden_dim, layer_num, head_num, kv_head_num, vocab_size, seq_len;
  int32_t kv_dim, kv_mul, head_size;
  int32_t shared_classifier, is_quant, group_size, flavour;
} ko_config;

ko_model* ko_model_open(const char* path, int is_quant, int flavour);
void ko_model_close(ko_model* m);
const ko_config* ko_model_config(const ko_model* m);
/* One position; returns greedy id (std::max_element = first maximum).  logits may be NULL. */
int ko_model_step(ko_model* m, int token, int pos, float* logits_out);
/* Pointers into the mmap for tests (NULL if absent). name in {tok_emb, wq, wk, wv, wo, w1, w2,
 * w3, wcls, attn_norm, ffn_norm, final_norm, bq, bk, bv}; scales_out gets the fp32 scale block
 * for quantised tensors. */
const void* ko_model_tensor(const ko_model* m, const char* name, int layer,
                            const float** scales_out);
const float* ko_model_key_cache(const ko_model* m);
const float* ko_model_value_cache(const ko_model* m);

#ifdef __cplusplus
}
#endif
#endif /* KUIPER_ORACLE_H_ */
