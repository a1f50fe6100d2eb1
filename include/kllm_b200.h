/* kllm_b200.h -- C-ABI of the H100-native KuiperLLama decode path (libkllm_b200.so).
 *
 * This is the drop-in boundary: plain pointers, ints and an opaque stream, no C++ or torch
 * types.  Every entry point names the reference interface it replaces (paths relative to the
 * zjhellofss/KuiperLLama tree).  The C++ adapters that keep the reference's
 * `kernel::get_*_kernel(DeviceType)` registry signatures verbatim live in
 * kuiperllama_b200/kuiper/source/op/kernels/ and only translate tensor::Tensor -> pointers.
 *
 * Conventions
 *   - all data pointers are DEVICE pointers unless the parameter name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream), exactly as
 *     the reference passes `void* stream` / `CudaConfig::stream`;
 *   - functions enqueue work and return without synchronising unless documented otherwise;
 *   - return value: 0 = ok, >0 = cudaError_t from the launch, <0 = KLLM_E_* argument error
 *     (the reference CHECK-aborts instead; the C++ adapters turn non-zero into LOG(FATAL));
 *   - there is NO CPU fallback: without a CUDA device every call returns an error.
 *
 * Arithmetic contract: fp32 throughout, each kernel reproduces the reference CUDA kernel's
 * floating-point operation order (see DESIGN.md "Bit-exactness"), so results are bit-identical
 * to the reference's own CUDA path compiled for sm_90a, not merely within tolerance.
 */
#ifndef KLLM_B200_H_
#define KLLM_B200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KLLM_OK 0
#define KLLM_E_INVALID (-1)     /* bad argument (null pointer, non-positive size, ...) */
#define KLLM_E_UNSUPPORTED (-2) /* shape outside what the kernels handle */
#define KLLM_E_STATE (-3)       /* decoder used before/after its valid life cycle */
#define KLLM_E_NODEVICE (-4)    /* no usable CUDA device */
#define KLLM_E_COMM (-5)        /* tensor-parallel transport unavailable / collective failed */

/* RoPE pairing / constants = the reference's compile-time flavour (CMakeLists.txt:16-25). */
#define KLLM_FLAVOUR_LLAMA2 0 /* interleaved pairs, theta 1e4, eps 1e-5 */
#define KLLM_FLAVOUR_LLAMA3 1 /* half-split pairs, theta 5e5, eps 1e-5 */
#define KLLM_FLAVOUR_QWEN2 2  /* half-split pairs, theta 1e6, eps 1e-6, qkv bias */

const char* kllm_version(void);
const char* kllm_error_string(int code);
/* Number of kernel launches issued through this library since load (bench.py's gpu_launches). */
uint64_t kllm_launch_count(void);

/* ---- registry-level ops ---------------------------------------------------------------
 * One per `kernel::get_*_kernel(kDeviceCUDA)` entry (kernels_interface.h:6-68).            */

/* MatmulKernel  -> matmul_kernel_cu, cuda/matmul_kernel.cu:89-109.
 * out[out_dim] = W[out_dim,in_dim] . x[in_dim], W row-major. */
int kllm_gemv_f32(const float* x, const float* w, float* out, int in_dim, int out_dim,
                  void* stream);

/* MatmulKernelQuant -> matmul_kernel_cu_qint8, cuda/matmul_kernel.cu:111-134.
 * out[p] = sum_i x[i] * scales[(p*in_dim+i)/group_size] * (float)w[p*in_dim+i]. */
int kllm_gemv_w8(const float* x, const int8_t* w, const float* scales, float* out, int in_dim,
                 int out_dim, int group_size, void* stream);

/* kllm_gemv_f32 over bf16 weights (the decoder's KLLM_WEIGHTS_BF16): w[out_dim, in_dim] holds bf16 bit patterns,
 * each widened exactly to fp32 before the same fp32 arithmetic, so out is bit-identical to kllm_gemv_f32 over the
 * widened matrix.  Any in_dim; rows need not be aligned. */
int kllm_gemv_bf16(const float* x, const uint16_t* w, float* out, int in_dim, int out_dim, void* stream);

/* RMSNormKernel -> rmsnorm_kernel_cu, cuda/rmsnorm_kernel.cu:52-78 (eps is the flavour
 * constant there; here it is an argument). In-place (out == x) is allowed. */
int kllm_rmsnorm_f32(const float* x, const float* w, float* out, int n, float eps, void* stream);

/* AddKernel -> add_kernel_cu, cuda/add_kernel.cu:14-32. */
int kllm_add_f32(const float* a, const float* b, float* out, int n, void* stream);

/* SwigluKernel -> swiglu_kernel_cu, cuda/swiglu_kernel.cu:24-47: out = (x1*sigmoid(x1))*x3. */
int kllm_swiglu_f32(const float* x1, const float* x3, float* out, int n, void* stream);

/* sin_cos_cache_calc_cu, cuda/rope_kernel.cu:138-151: tables [seq_len, head_size]. */
int kllm_sincos_init(int head_size, int seq_len, int flavour, float* sin_cache, float* cos_cache,
                     void* stream);

/* RoPEKernel -> rope_kernel_cu, cuda/rope_kernel.cu:153-170. q[dim], k[kv_dim] rotated in
 * place.  `pos` by value (the reference dereferences a host int32 tensor, :157).  Unlike the
 * reference's half-split kernels (:13,:59 `idx > total_pairs`) nothing is touched out of
 * bounds. */
int kllm_rope_f32(int flavour, int dim, int kv_dim, int head_size, float* q, float* k, int pos,
                  const float* sin_cache, const float* cos_cache, void* stream);

/* MHAKernel -> mha_kernel_cu, cuda/mha_kernel.cu:112-130.  key/value cache layout
 * [layer][seq_len][kv_dim] fp32; score is the [head_num, seq_len] workspace the reference
 * also takes (left holding the softmax probabilities, as the reference leaves it). */
int kllm_mha_decode_f32(int pos, int head_num, int layer_index, int seq_len, int kv_dim,
                        int kv_mul, int head_size, float* mha_out, const float* query,
                        float* score, const float* key_cache, const float* value_cache,
                        void* stream);

/* EmbeddingKernel -> emb_kernel_cu, cuda/emb_kernel.cu:23-48.  tokens are DEVICE int32 here
 * (the reference does a blocking H2D copy of a host tensor per call, :25-29). Tokens outside
 * [0, vocab) leave their output row untouched, as the reference does. */
int kllm_embedding_f32(const int32_t* tokens, int n_tokens, const float* table, float* out,
                       int dim, int vocab, void* stream);

/* argmax_kernel_cu, cuda/argmax_kernel.cu:73-87: greedy id, lowest index on ties.
 * Result goes to *out_index (device, int64); no allocation, no synchronisation. */
int kllm_argmax_f32(const float* logits, int64_t n, int64_t* out_index, void* stream);
/* Convenience with the reference's blocking semantics: returns the index or <0 on error. */
int64_t kllm_argmax_f32_sync(const float* logits, int64_t n, void* stream);

/* The sampling counterpart of kllm_argmax_f32 (what sampler::ArgmaxSampler calls): the id drawn from
 * logits[0..n) of position `pos` by the sampling rule of DESIGN.md "Sampling" (temperature, top_k,
 * Philox4x32-10 Gumbel noise keyed by seed and indexed by (pos, i)).  temperature == 0 is the greedy
 * argmax; top_k <= 0 or >= n keeps every logit.  The id is a pure function of (logits, temperature,
 * top_k, seed, pos).  Result to *out_index (device, int64); no synchronisation.  KLLM_E_INVALID for NULL
 * pointers, n outside [1, 2^31), pos < 0, or a temperature that is negative or not finite. */
int kllm_sample_f32(const float* logits, int64_t n, float temperature, int32_t top_k, uint64_t seed, int32_t pos,
                    int64_t* out_index, void* stream);
/* kllm_sample_f32 with nucleus (top-p) sampling after top-k, as in HF's TopPLogitsWarper: a token of the
 * top-k set is dropped once the probability mass strictly above it reaches top_p; equal logits are kept or
 * dropped together, and the maximum is always kept.  The mass is an exact integer sum (DESIGN.md
 * "Sampling", step 3b), so the id stays a pure function of (logits, temperature, top_k, top_p, seed, pos).
 * top_p == 1 is off: the id is then exactly kllm_sample_f32's.  Flat distributions whose nucleus does not fit
 * the block's shared memory take a slower path over the whole vector.  KLLM_E_INVALID as kllm_sample_f32,
 * and for top_p that is NaN, <= 0 or > 1. */
int kllm_sample_top_p_f32(const float* logits, int64_t n, float temperature, int32_t top_k, float top_p,
                          uint64_t seed, int32_t pos, int64_t* out_index, void* stream);
/* The repetition penalty of HF's RepetitionPenaltyLogitsProcessor (DESIGN.md "Sampling", step 0b), what a
 * caller of the per-op path runs before kllm_sample_top_p_f32 or an argmax: out[0..n) = logits[0..n), except
 * out[i] = logits[i] < 0 ? logits[i] * penalty : logits[i] / penalty (one fp32 IEEE operation) for every i
 * listed in ids[0..n_ids) (device).  An id listed more than once is penalised once; ids outside [0, n) are
 * ignored.  `out` must not overlap `logits`.  penalty == 1 copies the logits.  No synchronisation.
 * KLLM_E_INVALID for NULL pointers (ids may be NULL when n_ids == 0), out == logits, n outside [1, 2^31),
 * n_ids < 0, or a penalty that is not finite or <= 0. */
int kllm_repetition_penalty_f32(const float* logits, float* out, int64_t n, const int32_t* ids, int32_t n_ids,
                                float penalty, void* stream);
/* The whole of step 0 (DESIGN.md 5.9) over explicit id lists: out[0..n) = logits[0..n) (device) with, in order,
 * the logit bias of the map bias_ids_host[k] -> bias_host[k], k < n_bias (HOST arrays: the map is validated here;
 * n_bias == 0 skips the step), the repetition penalty over rep_ids[0..n_rep) (device, as
 * kllm_repetition_penalty_f32), then l_i - frequency * c_i and l_i - presence for every i with c_i > 0
 * occurrences in count_ids[0..n_count) (device).  Ids outside [0, n) in rep_ids / count_ids are ignored.  With
 * n_bias == 0 and frequency == presence == 0 it equals kllm_repetition_penalty_f32 bit for bit.  Enqueued on
 * `stream` with a stream-ordered scratch [n] (two with a bias); staging the bias table synchronises the stream.
 * KLLM_E_INVALID for NULL pointers where the count is > 0, out == logits, n outside [1, 2^31), a negative count
 * or n_count >= 2^30, a penalty that is not finite or <= 0, an alpha that is not finite, and a bias id outside
 * [0, n), a repeated bias id or a bias that is not finite. */
int kllm_logit_penalties_f32(const float* logits, float* out, int64_t n, const int32_t* bias_ids_host,
                             const float* bias_host, int32_t n_bias, float penalty, const int32_t* rep_ids,
                             int32_t n_rep, float frequency, float presence, const int32_t* count_ids,
                             int32_t n_count, void* stream);
/* Log-probabilities of logits[0..n) (device) by the rule of DESIGN.md 5.8: out_lp[j] = log softmax(logits)[ids[j]]
 * for j < n_ids, NaN for an id outside [0, n); out_top_ids / out_top_lp[0..top_n) = the top_n largest logits in
 * descending order, lowest index on ties, with their log-probabilities (index -1, lp -inf past the n-th).  All
 * outputs device memory; ids may be NULL when n_ids == 0, the top arrays when top_n == 0.  One block of one
 * launch; no synchronisation.  The ids are exact; each lp is within the bound of DESIGN.md 5.8 of the fp64
 * log_softmax of the same fp32 logits.  KLLM_E_INVALID for NULL pointers, n outside [1, 2^31), n_ids < 0 or
 * top_n outside [0, KLLM_MAX_TOP_LOGPROBS]. */
#define KLLM_MAX_TOP_LOGPROBS 20
int kllm_logprobs_f32(const float* logits, int64_t n, const int32_t* ids, int32_t n_ids, int32_t top_n, float* out_lp,
                      int32_t* out_top_ids, float* out_top_lp, void* stream);

/* ---- fused per-layer entry points -------------------------------------------------------
 * What LLama2Model::forward (llama3.cpp:147-167) calls instead of 15 launches per layer.
 * All are compositions of the ops above with identical arithmetic.                          */

typedef struct {
  const void* w;       /* fp32 or int8 [rows, in_dim] row-major */
  const float* scales; /* int8 only: fp32 [rows*in_dim/group_size] */
  const float* bias;   /* optional [rows] (Qwen2 q/k/v), added after the dot product */
  float* out;          /* [rows] */
  int rows;
} kllm_gemv_seg;

typedef struct {
  const float* x;       /* [in_dim] input activation */
  const float* norm_w;  /* optional: RMSNorm weight applied to x first (attention_rms /
                           ffn rmsnorm, llama3.cpp:600-609,687-691) */
  float norm_eps;
  float* norm_out;      /* optional: where the normalised x is also written (the reference
                           keeps it in kOutputRMSNorm) */
  int in_dim;
  int group_size;       /* 0 = fp32 weights, else int8 group size */
  int n_seg;            /* 1..3 row segments sharing x (q|k|v, or w1|w3) */
  kllm_gemv_seg seg[3];
  /* epilogue */
  const float* residual; /* optional: out[p] = residual[p] + dot (VecAdd, llama3.cpp:683,719) */
  int swiglu_pair;       /* 1: n_seg==2, seg[0]=w1, seg[1]=w3, seg[0].out = swiglu(d1, d3) */
} kllm_gemv_job;

int kllm_gemv_fused(const kllm_gemv_job* job, void* stream);

/* ---- batched prompt GEMM on the Hopper tensor cores (TOLERANCED: TF32 multiply, fp32 accumulate) ----
 * out[n_tokens, out_dim] = x[n_tokens, in_dim] . w[out_dim, in_dim]^T, all fp32 row-major device memory.
 * Replaces the n_tokens single-row GEMVs the reference issues for a prompt, one full forward per
 * prompt token (demo/main.cpp:18-23 -> LLama2Model::predict, llama3.cpp:147-167; MatmulLayer::forward,
 * matmul.cpp:57-80): the weight matrix is streamed once per 256 tokens instead of once per token.
 * TMA tensor-map loads (cp.async.bulk.tensor, 128-byte swizzle) feed wgmma.mma_async (tf32) with the
 * accumulators in registers.  Results agree with the fp32 GEMV to ~1e-3 relative (10-bit mantissas), NOT
 * bit for bit: the decode path never uses it.  in_dim % 4 == 0, 16-byte aligned x and w. */
int kllm_gemm_tf32(const float* x, const float* w, float* out, int n_tokens, int in_dim, int out_dim,
                   void* stream);
/* The same GEMM for int8 group-quantised weights (export.py --version 3):
 *   out[n_tokens, out_dim] = x[n_tokens, in_dim] . (s (.) w)[out_dim, in_dim]^T,
 *   s[n, k] = scales[(n * in_dim + k) / group_size]  -- the weight kllm_gemv_w8 dequantises.
 * x, out fp32; w int8 row-major; scales fp32; all device memory.  The weight tile is dequantised in
 * shared memory (scale * w in fp32, rounded to the nearest tf32) and multiplied on the same wgmma
 * tf32 path, so the error is that of kllm_gemm_tf32: per element within
 * 4e-3 * sqrt(in_dim) * rms(x row) * rms(dequantised w row) of the exact product
 * (tests/test_prefill_int8_gpu.py).  KLLM_E_INVALID for NULL pointers or non-positive sizes;
 * KLLM_E_UNSUPPORTED unless in_dim % 16 == 0, in_dim % group_size == 0, group_size % 32 == 0 and
 * x, w are 16-byte aligned. */
int kllm_gemm_w8_tf32(const float* x, const int8_t* w, const float* scales, float* out, int n_tokens, int in_dim,
                      int out_dim, int group_size, void* stream);
/* The same GEMM for bf16 weights (the decoder's KLLM_WEIGHTS_BF16): w[out_dim, in_dim] holds bf16 bit patterns.  The
 * weight tile is loaded as bf16 and widened into the fp32 tile; a bf16 value is exact in tf32, so out is bit-identical
 * to kllm_gemm_tf32 over the widened matrix.  KLLM_E_INVALID for NULL pointers or non-positive sizes;
 * KLLM_E_UNSUPPORTED unless in_dim % 8 == 0 and x, w are 16-byte aligned. */
int kllm_gemm_bf16_tf32(const float* x, const uint16_t* w, float* out, int n_tokens, int in_dim, int out_dim,
                        void* stream);

/* ---- tensor-parallel exchange --------------------------------------------------------------
 * Not in the reference (single GPU: llama3.cpp:118 pins device 0); SURVEY.md section 8e.  One
 * process per GPU; each owns a kllm_comm.  The decoder issues exactly two all-reduces per layer:
 * after o_proj (before the residual add of llama3.cpp:683-684) and after down_proj (:719).
 *   KLLM_COMM_PEER: one-shot all-reduce over NVLink peer memory (CUDA IPC), rank-ordered sum,
 *                   residual add fused; set up = create on every rank, exchange the 64-byte IPC
 *                   handles out of band, connect, barrier.
 *   KLLM_COMM_NCCL: ncclAllReduce on the decoder's stream (libnccl dlopen'ed at run time);
 *                   set up = unique_id on rank 0, broadcast the 128 bytes, create everywhere.  */
#define KLLM_COMM_PEER 0
#define KLLM_COMM_NCCL 1
typedef struct kllm_comm kllm_comm;
int kllm_comm_unique_id(unsigned char* out128);
/* max_count: largest vector (floats, multiple of 4) ever reduced = the model dim. */
int kllm_comm_create(int world, int rank, int backend, int max_count, const unsigned char* nccl_id128,
                     kllm_comm** out);
int kllm_comm_ipc_handle(kllm_comm* comm, unsigned char* out64);
/* handles: world x 64 bytes, rank-ordered (own entry ignored).  Every rank must have connected
 * (caller barrier) before the first all-reduce, and must stop reducing before any rank destroys. */
int kllm_comm_connect(kllm_comm* comm, const unsigned char* handles);
/* out = (residual ? residual : 0) + sum over ranks of `partial`, summed in rank order; all
 * device pointers, 16-byte aligned, count a multiple of 4.  `partial` is clobbered (NCCL). */
int kllm_comm_allreduce_residual(kllm_comm* comm, const float* partial, const float* residual, float* out,
                                 int count, void* stream);
/* In-place sum; signature of kllm_decoder_desc.allreduce (ctx = the kllm_comm). */
int kllm_comm_allreduce(void* comm, float* buf, int count, void* stream);
int kllm_comm_info(const kllm_comm* comm, int* world, int* rank, int* backend);
void kllm_comm_destroy(kllm_comm* comm);

/* ---- whole decoder ------------------------------------------------------------------------
 * Device-resident model: replaces Model::{init_mem,forward,predict,post_processing,embedding,
 * fill_input} (llama3.cpp:425-500,147-167,642-650,733-745,578-598; model.cpp:245-263) for the
 * per-token loop of demo/main.cpp:18-41.  Weights stay where the caller put them (device);
 * the decoder owns activations, KV cache, sin/cos tables and a captured CUDA graph.        */

typedef struct {
  int32_t dim, hidden_dim, layer_num, head_num, kv_head_num, vocab_size, seq_len;
  int32_t flavour;     /* KLLM_FLAVOUR_* */
  int32_t group_size;  /* 0 = fp32 weights; 64 = export.py --version 3 int8 */
  /* device pointers, reference checkpoint order (SURVEY.md Appendix A); per-layer arrays are
   * HOST arrays of layer_num device pointers. */
  const float* tok_emb;               /* [vocab, dim] */
  const float* const* attn_norm;      /* [L] -> [dim] */
  const float* const* ffn_norm;       /* [L] -> [dim] */
  const float* final_norm;            /* [dim] */
  const void* const* wq; const void* const* wk; const void* const* wv; const void* const* wo;
  const void* const* w1; const void* const* w2; const void* const* w3;
  const void* wcls;                   /* [vocab, dim] (== tok_emb when shared, fp32 only) */
  /* int8 only: fp32 scale blocks, same shapes / group_size */
  const float* const* sq; const float* const* sk; const float* const* sv; const float* const* so;
  const float* const* s1; const float* const* s2; const float* const* s3;
  const float* scls;
  /* Qwen2 only (may be NULL): */
  const float* const* bq; const float* const* bk; const float* const* bv;
  /* tensor parallel: this rank's shard description (tp_size 1 = single GPU).  With tp_size>1
   * wq/wk/wv/w1/w3 hold this rank's ROWS, wo/w2 this rank's input COLUMNS (repacked
   * contiguous), head_num/kv_head_num/hidden_dim above are the LOCAL counts and `dim` is the
   * full model dim.  allreduce is called after o_proj and after down_proj. */
  int32_t tp_size, tp_rank;
  int (*allreduce)(void* ctx, float* buf, int count, void* stream);
  void* allreduce_ctx;
  /* preferred over the callback when set: the decoder then uses the fused
   * all-reduce + residual add of kllm_comm_allreduce_residual */
  kllm_comm* comm;
  /* Numerics of the persistent engine.  KLLM_NUMERICS_EXACT (0, the default of a zeroed struct): every
   * reduction in the reference's order -- logits and ids bit-identical to the reference's CUDA path
   * (the verification mode).  KLLM_NUMERICS_FAST (1): free summation order where it buys speed --
   * int8 rows as fixed-point activations x int8 weights on dp4a, attention as flash-decoding (split by
   * timestep, online softmax) -- within the north-star tolerance (|dlogit| <= 1e-4, same greedy ids
   * where the top-2 margin exceeds 2e-4; tests/test_decoder_gpu.py).  Environment KLLM_MODE=exact|fast
   * overrides this field at create time. */
  int32_t numerics;
  /* Precision of the KV cache (DESIGN.md 5.10).  KLLM_KV_F32 (0, the default of a zeroed struct): fp32 rows.
   * KLLM_KV_BF16 (1): an opt-in toleranced variant of the fast numerics for long contexts -- half the cache
   * memory and half the attention's cache reads.  Rounding rule: each K row (after RoPE) and each V row is
   * rounded to bf16, round to nearest even, when it is written to the cache.  A decode step at position
   * pos attends over rows < pos as read from the cache (bf16, widened exactly to fp32) and over row pos
   * in fp32 from registers; the batched prefill (kllm_decoder_prefill_tf32 / _w8) reads every row it
   * attends over from the cache, those of its own block included, so all of them as bf16.  All arithmetic
   * stays fp32.  Every decoder entry keeps its semantics; kllm_decoder_read_kv returns the widened bf16
   * values.  kllm_decoder_create returns KLLM_E_INVALID for any other value and KLLM_E_UNSUPPORTED, creating
   * nothing, when KLLM_KV_BF16 cannot be honoured: exact numerics (after the KLLM_MODE override), the graph
   * engine (KLLM_ENGINE=graph, or a shape only it takes), tp_size > 1, or head_size % 32 != 0.
   * kllm_decoder_profile returns KLLM_E_UNSUPPORTED on a bf16 decoder.
   * KLLM_KV_FP8 (2, DESIGN.md 5.12): both caches hold fp8 e4m3 codes (__nv_fp8_e4m3, torch.float8_e4m3fn) with a
   * static scale per (layer, KV head) from kv_scales (required) -- a quarter of the fp32 cache's memory and reads.  An element x
   * of a K row (after RoPE) or a V row at layer l, KV head h is cached as code = e4m3(fp32(x * inv)), round to nearest
   * even and saturated to +-448, with inv = 1.0f / s (one fp32 division per scale, at create); the code stands for
   * value(code) * s.  The positions are as for KLLM_KV_BF16: a decode step reads rows < pos from the cache and row pos
   * unrounded from registers, the batched prefill reads every row from the cache.  All arithmetic stays fp32 (the
   * kernels may fold s into the score scale and the merged output).  kllm_decoder_read_kv returns fp32(value * s).
   * The refusals are KLLM_KV_BF16's, with head_size % 64 != 0 in place of % 32; fp32, int8 and bf16 weights all
   * take it. */
  int32_t kv_cache;
  /* Storage of the weight matrices (DESIGN.md 5.11).  KLLM_WEIGHTS_F32 (0, the default of a zeroed struct): as
   * group_size says.  KLLM_WEIGHTS_BF16 (1): wq wk wv wo w1 w2 w3 and wcls are device arrays of bf16 (uint16 bit
   * patterns), each the caller's fp32 tensor rounded to nearest even (torch.Tensor.to(torch.bfloat16)); half the
   * bytes every decode step streams.  tok_emb, the norms and the Qwen2 biases stay fp32; with a shared classifier
   * wcls is a separate bf16 copy of the embedding (the row gather keeps reading the fp32 tok_emb).  All arithmetic
   * stays fp32: a bf16 value widens exactly, so every entry's ids, logits and KV cache are bit for bit those of the
   * same decoder with KLLM_WEIGHTS_F32 over the rounded weights widened back to fp32, in either numerics at the same
   * ring geometry (KLLM_STAGE_BYTES / KLLM_ATTN_SPLIT: bf16 rows pick their own default stage), and with either
   * kv_cache.  Shapes the persistent engine does not take (dim, hidden_dim or the query rows not multiples of 8) run
   * on the graph engine.  kllm_decoder_create returns KLLM_E_INVALID for any other value or for bf16 with
   * group_size > 0, and KLLM_E_UNSUPPORTED, creating nothing, for tp_size > 1.  kllm_decoder_prefill_w8 and
   * kllm_decoder_profile return KLLM_E_UNSUPPORTED on a bf16-weight decoder. */
  int32_t weights;
  /* The fp8 KV cache's scales (kv_cache KLLM_KV_FP8), a host array [2][layer_num][kv_head_num]: first the K scales
   * s_k[l][h], then the V scales s_v[l][h] (kv_head_num as given here, this rank's).  Copied at create.  Required
   * with KLLM_KV_FP8 and NULL (the default of a zeroed struct) with every other cache: kllm_decoder_create returns
   * KLLM_E_INVALID for KLLM_KV_FP8 without scales (a description written before the fp8 cache existed, whose value 2
   * was refused, stays refused), for scales with another cache, and for a scale that is not finite and > 0.  Unit
   * scales are an array of ones; the Python and C++ front ends pass one when no scales are given. */
  const float* kv_scales;
} kllm_decoder_desc;
#define KLLM_NUMERICS_EXACT 0
#define KLLM_NUMERICS_FAST 1
#define KLLM_KV_F32 0
#define KLLM_KV_BF16 1
#define KLLM_KV_FP8 2
#define KLLM_WEIGHTS_F32 0
#define KLLM_WEIGHTS_BF16 1

typedef struct kllm_decoder kllm_decoder;

/* `stream`: the cudaStream_t every launch and copy of this decoder is ordered on.  NULL = the decoder
 * creates a private non-blocking stream and device-synchronises once here, so weights uploaded on
 * any other stream before this call are complete; with a caller's stream the caller orders its
 * uploads before the first step (same stream, or an event). */
int kllm_decoder_create(const kllm_decoder_desc* desc, void* stream, kllm_decoder** out);
void kllm_decoder_destroy(kllm_decoder* dec);

/* One position through the reference-facing path with HOST buffers: copies the token id
 * host->device, runs the captured forward for `pos`, copies the greedy id device->host and
 * synchronises (predict + post_processing semantics, llama3.cpp:642-650,733-745).
 * is_prompt != 0 mirrors predict(..., is_prompt=true): the forward runs, *next_host = -1. */
int kllm_decoder_step(kllm_decoder* dec, int32_t token_host, int32_t pos, int is_prompt,
                      int32_t* next_host);

/* The whole prompt in one call: positions start_pos .. start_pos + n_tokens - 1 take tokens_host[i] as
 * input, fill the KV cache, and *next_host is the greedy id after the LAST prompt token (what
 * demo/main.cpp:18-41 obtains by calling predict() once per prompt position with is_prompt = true and
 * discarding every result but the last).  Persistent engine: one launch, and the classifier pass --
 * which the reference runs and throws away for every prompt position (llama3.cpp:642-650, 738-739) --
 * is skipped for all but the last position.  Bit-identical KV cache and next id to stepping. */
int kllm_decoder_prompt(kllm_decoder* dec, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                        int32_t* next_host);
/* TOLERANCED batched prefill: the same contract as kllm_decoder_prompt, but the prompt positions go
 * through every layer together -- each projection one GEMM [n, in] x [out, in]^T on the wgmma
 * tensor cores (TF32 multiply, fp32 accumulate, kllm_gemm_tf32), the weights streamed once per 256
 * positions instead of once per position; classifier only for the last position.  KV-cache rows and
 * logits agree with the position-by-position path to ~1e-3 relative, NOT bit for bit (TF32 keeps 10
 * mantissa bits).  fp32 checkpoints on one GPU, their weights held in fp32 or, KLLM_WEIGHTS_BF16, in bf16
 * (kllm_gemm_bf16_tf32: bit for bit the fp32-weight decoder's result over the widened weights; dim, hidden_dim and
 * head_num * head_size must then be multiples of 8); KLLM_E_UNSUPPORTED otherwise (use kllm_decoder_prompt),
 * checked before any launch, so a refused call leaves the cache, the history and the logits as they were.
 * A token id outside [0, vocab_size) is refused with KLLM_E_INVALID before any launch. */
int kllm_decoder_prefill_tf32(kllm_decoder* dec, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                              int32_t* next_host);
/* The batched prefill for int8 checkpoints: the contract and the tolerance of kllm_decoder_prefill_tf32
 * (KV-cache rows within 5e-2 * (row rms + 1e-3), last logits within 2e-2 * max|logit| of the
 * position-by-position path; tests/test_prefill_int8_gpu.py), each projection one kllm_gemm_w8_tf32.
 * int8 checkpoints on one GPU whose projections the GEMM accepts (dim, hidden_dim % 16 == 0, both
 * multiples of group_size, group_size % 32 == 0); KLLM_E_UNSUPPORTED otherwise -- fp32 checkpoints
 * take kllm_decoder_prefill_tf32, anything else kllm_decoder_prompt. */
int kllm_decoder_prefill_w8(kllm_decoder* dec, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                            int32_t* next_host);
/* Device-resident greedy loop: positions start_pos .. start_pos+n_steps-1, each step feeding
 * the previous argmax back without leaving the GPU; ids copied to out_tokens_host at the end
 * (one synchronisation).  teacher_host (optional, n_steps ids) forces the inputs instead. */
int kllm_decoder_generate(kllm_decoder* dec, int32_t first_token, int32_t start_pos,
                          int32_t n_steps, const int32_t* teacher_host,
                          int32_t* out_tokens_host);

/* The generate loop that stops at a stop id and streams its ids to the host while it runs.
 *  - Step i feeds token t_i at position start_pos + i and produces id_i; t_0 = first_token, t_i = id_{i-1}
 *    (kllm_decoder_generate without a teacher).  Ids are drawn by the decoder's sampling settings (greedy by
 *    default), so a stop applies to the drawn id.
 *  - The loop ends after the first step whose id is in stop_ids[0 .. n_stop), or after max_steps steps.
 *  - *n_out is the number of ids produced, counting the stop id; out_tokens_host (capacity max_steps)
 *    receives them.
 *  - On return the KV cache holds positions start_pos .. start_pos + *n_out - 1 and kllm_decoder_logits returns
 *    the logits of the last step that ran: a later call may continue at start_pos + *n_out with
 *    id_{n_out-1} as its input.
 *  - Every id reaches on_tokens (if non-null) exactly once, in order, before the call returns: the callbacks'
 *    concatenation equals out_tokens_host[0 .. *n_out).  The callback runs on the calling thread and must not
 *    call into the same decoder.
 *  - With n_stop == 0 and no callback the result equals kllm_decoder_generate(..., n_steps = max_steps,
 *    teacher = NULL) bit for bit: ids, logits and KV cache.
 *  - KLLM_E_INVALID, before any launch, for: n_stop outside [0, KLLM_MAX_STOP_IDS]; a stop id outside
 *    [0, vocab); start_pos + max_steps > seq_len; max_steps <= 0; a null out_tokens_host or n_out; n_stop > 0
 *    with a null stop_ids.
 * Persistent engine: one launch; every CTA of every rank computes the same id, so each decides the stop by
 * itself.  Graph engine: one captured step per launch, and the host waits for each id before it launches the
 * next step (a host turnaround per token, as with kllm_decoder_step).  Ids reach the host through mapped
 * pinned memory either way, while the loop is still running. */
#define KLLM_MAX_STOP_IDS 16
typedef void (*kllm_token_callback)(void* ctx, const int32_t* ids, int32_t n_ids);
int kllm_decoder_generate_until(kllm_decoder* dec, int32_t first_token, int32_t start_pos, int32_t max_steps,
                                const int32_t* stop_ids, int32_t n_stop,
                                kllm_token_callback on_tokens, void* ctx,
                                int32_t* out_tokens_host, int32_t* n_out);

/* Speculative decoding's verify pass (DESIGN.md 5.13): tokens_host[0] is the id fed at start_pos, tokens_host[1 ..
 * n_tokens) are drafts for the positions after it, and all n_tokens positions run through every layer in ONE pass
 * over the weights.
 *  - At each position start_pos + i the id id_i is drawn by the settings in force (greedy, sampling, top-p,
 *    penalties, logit bias), over the history as fed, and recorded as any entry records it.
 *  - a = the number of leading drafts with tokens_host[i] == id_{i-1}.  out_ids_host (capacity n_tokens) receives
 *    id_0 .. id_a, and *n_accepted = a.
 *  - The result is bit for bit that of kllm_decoder_generate(dec, tokens_host[0], start_pos, a + 1, NULL, ...) on a
 *    decoder with the same description and state: the ids, kllm_decoder_logits (the logits of start_pos + a), the KV
 *    rows of positions <= start_pos + a, the history and the log-probability record.  One exception: on the
 *    persistent engine a record entry's log-probabilities may differ from that engine's own in the last bits
 *    (DESIGN.md 5.13); its ids are the same.
 *  - Past the frontier, at start_pos + a + 1 .. start_pos + n_tokens - 1, the history and the record hold what they
 *    held before the call; the KV rows there are unspecified (at most n_tokens - 1 rows, none read by an entry that
 *    does not feed its position first).  A call continues at start_pos + a + 1 with id_a as its input.
 * Refusals, before any launch, leave the cache, the history, the record and the logits as they were:
 * KLLM_E_UNSUPPORTED for the fast numerics (after KLLM_MODE; so also the bf16 and fp8 KV caches) and for
 * tp_size > 1; KLLM_E_INVALID for n_tokens outside [1, KLLM_MAX_VERIFY_TOKENS], a token outside [0, vocab),
 * start_pos < 0, start_pos + n_tokens > seq_len and NULL pointers.  fp32, int8 and bf16 weights, either engine.
 * Each length's chain is captured as a CUDA graph on first use: one graph launch and one synchronisation per call. */
#define KLLM_MAX_VERIFY_TOKENS 8
int kllm_decoder_verify(kllm_decoder* dec, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                        int32_t* out_ids_host, int32_t* n_accepted);

/* Speculative decoding with prompt-lookup drafts: kllm_decoder_generate_until's arguments and semantics, each round
 * drafting from the decoder's history and checking the draft with kllm_decoder_verify.
 * Drafting rule (kuiperllama_b200/speculative.py lookup_draft mirrors it): let p be the next position, t the id fed
 * there, c = history[0 .. p) followed by t, L = p + 1.  For n = ngram_max down to 1, skip n when the suffix
 * c[L-n .. L) has fewer than n ids or contains -1; else take the LARGEST s with s + n <= L - 1 and
 * c[s .. s+n) == c[L-n .. L).  The draft is c[s+n ..], cut at the first -1 and after
 * m = min(draft_len, max_steps - produced - 1, seq_len - p - 1) ids.  The first n with a non-empty draft wins; with
 * none the round is one plain step on the decoder's engine.
 *  - Each round streams its accepted ids to on_tokens.  A stop id ends the loop at its position; ids a round drew
 *    past a stop are rejected as wrong drafts are, with the history and the record put back.
 *  - The ids, *n_out, the callbacks' concatenation, kllm_decoder_logits, the history, the record and the KV rows
 *    below start_pos + *n_out are bit for bit those of kllm_decoder_generate_until with the same arguments (the
 *    record with kllm_decoder_verify's exception).  first_token must lie in [0, vocab).
 *  - stats (optional): rounds (verify passes and plain steps), drafted (draft ids verified), accepted (draft ids
 *    accepted); speculative.py simulate_rounds predicts them from the ids.
 * KLLM_E_INVALID for draft_len outside [1, KLLM_MAX_VERIFY_TOKENS - 1] and ngram_max outside [1, 8], with
 * kllm_decoder_generate_until's refusals and kllm_decoder_verify's KLLM_E_UNSUPPORTED cases, all before any launch. */
typedef struct {
  int32_t rounds;
  int32_t drafted;
  int32_t accepted;
} kllm_spec_stats;
int kllm_decoder_generate_speculative(kllm_decoder* dec, int32_t first_token, int32_t start_pos, int32_t max_steps,
                                      const int32_t* stop_ids, int32_t n_stop, int32_t draft_len, int32_t ngram_max,
                                      kllm_token_callback on_tokens, void* ctx, int32_t* out_tokens_host,
                                      int32_t* n_out, kllm_spec_stats* stats);

/* A batch of decoders sharing one model (DESIGN.md 5.14): up to KLLM_MAX_BATCH sequences decoded in ONE pass over
 * the weights per step.  Member b is row b; each member has its own position, so sequences of different lengths
 * share a pass, and its own history, draw settings, log-probability record, logits and cache.
 *  - kllm_batch_step / kllm_batch_generate leave every member bit for bit as its own kllm_decoder_step (is_prompt
 *    0) / kllm_decoder_generate (teacher NULL) with the same arguments would: the ids, kllm_decoder_logits (the
 *    logits of its last position), the KV rows of the positions fed, the history, the log-probability record and
 *    the state its own next entry continues from.  Every draw uses that member's settings in force.  One exception,
 *    kllm_decoder_verify's: on the persistent engine a record entry's log-probabilities may differ from that
 *    engine's own in the last bits; the ids and top-N ids are exact.
 *  - Members may be used on their own between batch calls and may belong to several batches; calls must not overlap.
 *    A batch is destroyed before its members.
 *  - Each call synchronises every member's stream, runs on the batch's stream (NULL at create: a private
 *    non-blocking one) and returns after a synchronisation.  The chain of one step is captured as a CUDA graph at
 *    create; generate launches it n_steps times, each member's id fed back on the device.
 * kllm_batch_create refuses, before any launch and leaving every member unchanged: KLLM_E_INVALID for n outside
 * [1, KLLM_MAX_BATCH], NULL pointers and the same decoder twice; KLLM_E_UNSUPPORTED for a member
 * kllm_decoder_verify refuses (the fast numerics, so the bf16 and fp8 caches, and tp_size > 1) and for members
 * that do not describe the same model: the same shape, flavour, group size, weight format and weight device
 * pointers, on one engine with one cache layout (so one KLLM_ATTN_SPLIT). */
#define KLLM_MAX_BATCH 8
typedef struct kllm_batch kllm_batch;
int kllm_batch_create(kllm_decoder* const* members, int32_t n, void* stream, kllm_batch** out);
void kllm_batch_destroy(kllm_batch* batch);
/* One step of every member: tokens_host[b] fed at pos_host[b]; next_host[b] receives member b's id.
 * KLLM_E_INVALID, before any launch and leaving every member unchanged, for NULL pointers, a token outside
 * [0, vocab), pos < 0 and pos >= seq_len. */
int kllm_batch_step(kllm_batch* batch, const int32_t* tokens_host, const int32_t* pos_host, int32_t* next_host);
/* n_steps steps of every member from first_tokens_host[b] at start_pos_host[b]; out_tokens_host [n][n_steps]
 * receives member b's ids in row b.  KLLM_E_INVALID, before any launch and leaving every member unchanged, for
 * NULL pointers, n_steps <= 0, a token outside [0, vocab), start_pos < 0 and start_pos + n_steps > seq_len. */
int kllm_batch_generate(kllm_batch* batch, const int32_t* first_tokens_host, const int32_t* start_pos_host,
                        int32_t n_steps, int32_t* out_tokens_host);
/* Every member generates on its own terms in one loop (DESIGN.md 5.15): member b from first_tokens_host[b] at
 * start_pos_host[b] until the first of its n_stop_host[b] stop ids (row b of stop_ids_host [n][KLLM_MAX_STOP_IDS])
 * or max_steps_host[b] ids, whichever comes first.
 *  - Member b ends bit for bit as its own kllm_decoder_generate_until(first_tokens_host[b], start_pos_host[b],
 *    max_steps_host[b], its stop ids, n_stop_host[b], ...) would leave it: the ids, n_out_host[b],
 *    kllm_decoder_logits, the history, the log-probability record and the state its own next entry continues from.
 *    The record has kllm_batch_generate's exception: on the persistent engine a record entry's log-probabilities
 *    may differ from that engine's own in the last bits.
 *  - Nothing past a member's end is written: once member b has produced its stop id or its max_steps_host[b]-th
 *    id, no later pass touches its cache, history, record, logits or state.
 *  - Row b of out_tokens_host [n][M], M = max_b max_steps_host[b], receives member b's n_out_host[b] ids, the stop
 *    id included; the rest of the row is not written.
 *  - Every id of member b reaches on_tokens(ctx, b, ...) (if non-null) exactly once, in order, while the loop runs
 *    and before the call returns.  The order across members is not specified.  The callback runs on the calling
 *    thread and must not call into the batch or its members.
 *  - Each pass carries only the members still running: stats (optional) receives passes = max_b n_out_host[b] and
 *    rows = sum_b n_out_host[b], the rows summed over the passes.
 *  - kllm_batch_step and kllm_batch_generate behave as before afterwards.
 * KLLM_E_INVALID, before any launch and leaving every member unchanged, for NULL pointers (on_tokens and stats may
 * be NULL), max_steps <= 0, start_pos < 0, start_pos + max_steps > seq_len, n_stop outside [0, KLLM_MAX_STOP_IDS],
 * and a first token or stop id outside [0, vocab).
 * The host drives the loop: after each pass it waits for the pass's ids through each member's mapped memory and
 * decides the stops, then launches the next pass.  The step of k rows is captured as a CUDA graph on first use and
 * kept; the n-row step is the one kllm_batch_create captured. */
typedef void (*kllm_batch_token_callback)(void* ctx, int32_t member, const int32_t* ids, int32_t n_ids);
typedef struct {
  int32_t passes;
  int32_t rows;
} kllm_batch_stats;
int kllm_batch_generate_until(kllm_batch* batch, const int32_t* first_tokens_host, const int32_t* start_pos_host,
                              const int32_t* max_steps_host, const int32_t* stop_ids_host, const int32_t* n_stop_host,
                              kllm_batch_token_callback on_tokens, void* ctx, int32_t* out_tokens_host,
                              int32_t* n_out_host, kllm_batch_stats* stats);

/* Beam search of one prompt with B = the batch's member count beams (DESIGN.md 5.16): transformers'
 * generate(num_beams=B, do_sample=False, length_penalty, early_stopping, num_return_sequences=n_return) with no
 * logits processors, every running beam a row of one pass over the weights.  kuiperllama_b200/beam.py states the
 * rule; early_stopping is one of the KLLM_BEAM_EARLY_* codes.
 *  - The caller has filled member 0's cache for positions [0, start_pos) with any entry; first_token is fed at
 *    start_pos.  The call copies member 0's rows [0, start_pos] into the other members; their earlier contents at
 *    positions below start_pos + max_new_tokens are overwritten.
 *  - The results are bit for bit those of beam.py run over each member's own logits, with lp by rule L1-L3 over the
 *    one-block partition (kllm_logprobs_f32's).  Hypothesis i (h descending) has out_len_host[i] ids in row i of
 *    out_ids_host [n_return][max_new_tokens] (an eos id that ended it included; the rest of the row is not written),
 *    its score h = fp32(S / fp32(t ^ length_penalty)) at out_score_host[i] and its sum of log-probabilities S at
 *    out_sum_host[i].  stats (optional) receives the passes, the cache forks and fork_rows = the positions they
 *    copied, summed over the forks.
 *  - Afterwards member 0's rows below start_pos are unchanged; everything else the members hold at or past
 *    start_pos (K/V rows, position, history, record and logits) is unspecified.  kllm_batch_step,
 *    kllm_batch_generate and kllm_batch_generate_until behave as before.
 * Before any launch, leaving every member unchanged: KLLM_E_INVALID for NULL outputs, a first token or eos id outside
 * [0, vocab), start_pos < 0, max_new_tokens <= 0, start_pos + max_new_tokens > seq_len, n_eos outside
 * [0, KLLM_MAX_BEAM_EOS] (or n_eos > 0 with NULL ids), n_return outside [1, B], a length_penalty that is not finite
 * and early_stopping outside {0, 1, 2}; KLLM_E_UNSUPPORTED for a member whose draw settings are not a new
 * decoder's (greedy, no repetition, frequency or presence penalty, no logit bias; the logprob setting does not
 * matter) and for vocab < max(2, 1 + n_eos) * B.
 * Each pass runs the batch's embedding and layer chain over the running beams, then one block per row takes the
 * row's top B + KLLM_MAX_BEAM_EOS ids and their lp into mapped host memory; the host applies the rule, and a beam
 * that shares its parent with an earlier one takes a dropped beam's member, whose rows one kernel per pass copies
 * from the parent's.  The passes of 1 and of B rows are captured as CUDA graphs on first use and kept. */
#define KLLM_MAX_BEAM_EOS 8
#define KLLM_BEAM_EARLY_HEURISTIC 0 /* transformers early_stopping=False */
#define KLLM_BEAM_EARLY_ALL_DONE 1  /* early_stopping=True */
#define KLLM_BEAM_EARLY_NEVER 2     /* early_stopping="never" */
typedef struct {
  int32_t passes;
  int32_t forks;
  int64_t fork_rows;
} kllm_beam_stats;
int kllm_batch_beam_search(kllm_batch* batch, int32_t first_token, int32_t start_pos, int32_t max_new_tokens,
                           const int32_t* eos_ids, int32_t n_eos, float length_penalty, int32_t early_stopping,
                           int32_t n_return, int32_t* out_ids_host, int32_t* out_len_host, float* out_score_host,
                           float* out_sum_host, kllm_beam_stats* stats);

/* Copies into dst what src holds for positions [0, n_pos): the K/V rows (cache elements as stored: fp32, bf16, or
 * fp8 codes at equal scales, in any layout), the history and the log-probability record entries.  Afterwards any
 * entry on dst that continues at a position <= n_pos returns what it would on src, bit for bit; dst keeps its own
 * draw settings, so forks of one prompt can sample with different seeds.  One prefill and n - 1 copies give n
 * sequences of one prompt to batch.
 * KLLM_E_INVALID for NULL pointers, src == dst and n_pos outside [0, seq_len]; KLLM_E_UNSUPPORTED unless both
 * describe the same model (as kllm_batch_create), on the same engine with the same cache layout, kv_cache and fp8
 * scales, with tp_size 1; both before any launch, with nothing copied.  Runs on dst's stream after synchronising
 * src's, one kernel over the layout's indices, and returns after a synchronisation. */
int kllm_decoder_copy_prefix(kllm_decoder* dst, const kllm_decoder* src, int32_t n_pos);

/* Sampling instead of the greedy id, from this call on, for every id the decoder returns: kllm_decoder_step
 * (non-prompt), _prompt, _prefill_tf32 / _w8 and _generate, including the ids generate feeds back on the
 * device.  Each id is the rule of kllm_sample_f32 applied to the logits of the position just processed,
 * with that position as `pos`: the same seed gives the same ids on either engine and on every
 * tensor-parallel rank.  temperature 0 restores the exact greedy behaviour (a new decoder is greedy).
 * The parameters live in device memory: no engine or graph is rebuilt.  Synchronises the decoder's
 * stream.  KLLM_E_INVALID for a temperature that is negative or not finite. */
int kllm_decoder_set_sampling(kllm_decoder* dec, float temperature, int32_t top_k, uint64_t seed);
/* kllm_decoder_set_sampling with nucleus sampling: each id is then the rule of kllm_sample_top_p_f32, in
 * every entry that kllm_decoder_set_sampling covers (step, prompt, both batched prefills, generate and
 * generate_until), on either engine and every tensor-parallel rank.  top_p == 1 is exactly
 * kllm_decoder_set_sampling, which itself sets top_p back to 1.  KLLM_E_INVALID, with the settings in force
 * left unchanged, for a temperature that is negative or not finite and for top_p that is NaN, <= 0 or > 1. */
int kllm_decoder_set_sampling_top_p(kllm_decoder* dec, float temperature, int32_t top_k, float top_p, uint64_t seed);
/* Repetition penalty before the draw, from this call on, in every entry that kllm_decoder_set_sampling covers,
 * on either engine and every tensor-parallel rank, greedy or sampled: each id is drawn from the logits with
 * kllm_repetition_penalty_f32's step applied to the ids fed at positions [lo, pos] (lo = 0 for last_n == 0,
 * the whole sequence; else max(0, pos - last_n + 1)), as recorded by the decoder (kllm_decoder_read_history).
 * penalty < 1 raises those logits instead.  penalty == 1 is off (a new decoder's setting): the ids are then
 * exactly those without it.  Independent of the sampling settings: neither call changes the other's.
 * kllm_decoder_logits keeps returning the raw logits.  Synchronises the decoder's stream.  KLLM_E_INVALID,
 * with the settings in force left unchanged, for a penalty that is not finite or <= 0 and for last_n < 0. */
int kllm_decoder_set_repetition_penalty(kllm_decoder* dec, float penalty, int32_t last_n);
/* Frequency and presence penalties before the draw (DESIGN.md 5.9, OpenAI's frequency_penalty /
 * presence_penalty), from this call on, in every entry that kllm_decoder_set_sampling covers, on either engine and
 * every tensor-parallel rank: with c_i the number of times id i was fed at positions [from_pos, pos] (the
 * decoder's history), every i with c_i > 0 gets l_i - frequency * c_i, then l_i - presence, after the repetition
 * penalty.  from_pos is absolute: the prompt's length counts only the generated ids (the draw after the prompt
 * counts none), 0 the prompt too.  frequency == presence == 0 is off (a new decoder's setting).  Negative values
 * raise the counted ids.  Independent of the other setters.  kllm_decoder_logits keeps returning the raw logits
 * and kllm_decoder_score ignores it.  Synchronises the decoder's stream.  KLLM_E_INVALID, with the settings in
 * force left unchanged, for a value that is not finite and for from_pos < 0. */
int kllm_decoder_set_frequency_presence(kllm_decoder* dec, float frequency, float presence, int32_t from_pos);
/* Logit bias before the draw (DESIGN.md 5.9, OpenAI's logit_bias), from this call on, in the same entries:
 * l_i + bias of i, before the penalties, for every id of the map ids_host[k] -> bias_host[k], k < n (host
 * arrays).  Each call replaces the whole map; n == 0 clears it (a new decoder's setting).  A large negative bias
 * bans an id, a large positive one forces it.  Independent of the other setters.  Synchronises the decoder's
 * stream.  KLLM_E_INVALID, with the map in force left unchanged, for NULL arrays with n > 0, n < 0, an id
 * outside [0, vocab_size), a repeated id, or a bias that is not finite. */
int kllm_decoder_set_logit_bias(kllm_decoder* dec, const int32_t* ids_host, const float* bias_host, int32_t n);
/* Log-probabilities of the returned ids, from this call on (DESIGN.md 5.8): whenever a position's classifier runs,
 * the decoder records, at that position, the id it returns with its log-probability and, for top_n > 0, the
 * top_n largest logits with theirs.  Log-probabilities are taken over the RAW logits (kllm_decoder_logits),
 * before the repetition penalty, temperature, top-k and top-p, so they mean the same whatever the sampling
 * settings.  Entries are written by kllm_decoder_step (non-prompt), the last position of _prompt /
 * _prefill_tf32 / _prefill_w8, every position of _generate (with or without a teacher: the entry holds the
 * drawn id) and the positions of _generate_until that ran; prompt positions whose classifier is skipped write
 * nothing, and processing a position again overwrites its entry.  top_n -1 is off (a new decoder's setting),
 * 0 records the id's log-probability only, 1..KLLM_MAX_TOP_LOGPROBS also the top_n.  Ids, logits, KV cache and
 * history are bit-identical with and without it.  Clears the record (every id -1) and synchronises the stream.
 * KLLM_E_INVALID, with the setting in force left unchanged, for top_n outside [-1, KLLM_MAX_TOP_LOGPROBS]. */
int kllm_decoder_set_logprobs(kllm_decoder* dec, int32_t top_n);
/* The record of positions [start_pos, start_pos + n): ids_host / lp_host [n], and, when non-NULL,
 * top_ids_host / top_lp_host [n][top_n] with the top_n in force (nothing is written to them when it is <= 0).
 * An id of -1 marks a position without an entry.  Blocking.  KLLM_E_INVALID for a range outside [0, seq_len)
 * or NULL ids_host / lp_host. */
int kllm_decoder_read_logprobs(kllm_decoder* dec, int32_t start_pos, int32_t n, int32_t* ids_host, float* lp_host,
                               int32_t* top_ids_host, float* top_lp_host);
/* Teacher-forced scoring: feeds tokens_host[0 .. n_tokens - 2] at positions start_pos .. start_pos + n_tokens - 2,
 * running the classifier at every one, and writes lp_host[i] = log p(tokens_host[i + 1] | the tokens up to
 * position start_pos + i), n_tokens - 1 values, by the rule of kllm_decoder_set_logprobs.  The record of those
 * positions then holds the TARGET id tokens_host[i + 1] and its log-probability (with the top_n in force when
 * logprobs are on).  Afterwards the KV cache and the history hold those positions, so tokens_host[n_tokens - 1]
 * fed at start_pos + n_tokens - 1 continues the sequence.  Sampling and penalty settings do not change the
 * result.  Persistent engine: one launch.  KLLM_E_INVALID, before any launch, for n_tokens < 2, a token outside
 * [0, vocab_size), start_pos < 0, start_pos + n_tokens > seq_len (the position that continues the sequence must
 * exist) or NULL pointers. */
int kllm_decoder_score(kllm_decoder* dec, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                       float* lp_host);

/* Blocking copies for tests: logits of the last step [vocab]; the KV cache in the REFERENCE
 * layout [layer][seq_len][kv_dim] (llama3.cpp:469-475) whatever the engine keeps internally (a bf16
 * cache, KLLM_KV_BF16: its values widened exactly to fp32; an fp8 cache, KLLM_KV_FP8: fp32(value(code) * scale)). */
int kllm_decoder_logits(kllm_decoder* dec, float* logits_host);
/* Device pointer to the same logits [vocab] (what the reference keeps in
 * ModelBufferType::kForwardOutput, llama3.cpp:498-506); valid until the decoder is destroyed,
 * contents ordered after the last step on the decoder's stream. */
const float* kllm_decoder_logits_device(const kllm_decoder* dec);
int kllm_decoder_read_kv(kllm_decoder* dec, float* key_host, float* value_host);
/* The decoder's history [seq_len]: the id fed as input at each position by any entry (the id whose K/V rows
 * are that row of the cache), -1 where none was fed or the id was outside the vocabulary.  Feeding a
 * position again overwrites its entry. */
int kllm_decoder_read_history(kllm_decoder* dec, int32_t* ids_host);
/* Kernel launches one decode step issues (graph nodes; 1 for the persistent engine). */
int kllm_decoder_launches_per_step(const kllm_decoder* dec);
/* Classifier rows THIS rank streams per token: vocab_size, or vocab_size / tp_size when the
 * tensor-parallel persistent engine shards the classifier by vocabulary (cls_logits,
 * llama3.cpp:722-731, computed once across the ranks instead of once per rank).  That needs a
 * kllm_comm created with max_count >= max(dim, vocab_size / tp_size): the ranks publish their
 * logits rows through the same tagged exchange area as the o_proj / down_proj partials. */
int kllm_decoder_classifier_rows(const kllm_decoder* dec);
/* "persistent": one cooperative megakernel launch runs whole positions with a TMA-fed weight
 * ring; "graph": CUDA-graph chain of fused launches (shapes the ring does not handle, tensor
 * parallel).  Environment KLLM_ENGINE=graph|persistent forces a choice at create time. */
const char* kllm_decoder_engine(const kllm_decoder* dec);
/* Persistent engine only (KLLM_E_UNSUPPORTED on the graph engine): the attention geometry create chose.
 * tile: timesteps per K ring stage (the flash form's K and V tile); split: CTAs per query head (the
 * exact form splits the V dims into head_size / split slices, the flash form the timesteps);
 * tile_v: timesteps per V ring stage; stage_bytes: bytes per ring stage. */
int kllm_decoder_attention_geometry(const kllm_decoder* dec, int* tile, int* split, int* tile_v,
                                    int* stage_bytes);
/* Persistent engine only: run n_steps positions and record, for step `profiled_step`, sixteen
 * stamps per CTA per schedule phase into stamps_host[grid][phases][16] (capacity in uint64
 * elements).  Globaltimer ns: [0] phase entered, [1] input vector staged (+normalised), [2] last
 * ring stage consumed, [3] grid barrier passed, [10] input vector polled (before the norm).
 * SM cycles of warp 0: [4] addend prefetch, [5] dot products, [6] reductions, [7] epilogues,
 * [8] waiting for ring stages, [9] rows of a stage.  Measurement aid (tools/phase_timeline.py). */
int kllm_decoder_profile(kllm_decoder* dec, int32_t first_token, int32_t start_pos,
                         int32_t n_steps, int32_t profiled_step, uint64_t* stamps_host,
                         int32_t capacity, int32_t* grid_out, int32_t* phases_out);

#ifdef __cplusplus
}
#endif
#endif /* KLLM_B200_H_ */
