// Small per-token ops of the decode path, one C-ABI entry per reference registry op:
// rmsnorm, add, swiglu, rope (+ sin/cos table), embedding gather, greedy argmax.
// Reference: kuiper/source/op/kernels/cuda/{rmsnorm,add,swiglu,rope,emb,argmax}_kernel.cu.
// All are latency-bound (<= 600 KB touched); they exist for registry parity and for the
// pieces the fused GEMV prologue/epilogues do not absorb.  Arithmetic order follows the
// reference kernels bit for bit (DESIGN.md "Bit-exactness").
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"
#include "sampling.cuh"

namespace kllm {

std::atomic<uint64_t>& launch_counter() {
  static std::atomic<uint64_t> c{0};
  return c;
}

int smem_opt_in(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> granted;  // (device, kernel) -> the attribute's value
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return KLLM_E_NODEVICE;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = granted[{dev, kernel}];
  if (bytes <= have) return 0;
  const cudaError_t e =
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e != cudaSuccess) return static_cast<int>(e);
  have = bytes;
  return 0;
}

// ---- rmsnorm: rmsnorm_kernel.cu:4-50 (one 128-thread block there; one warp carrying the
// same 128 virtual threads here for the sum, the whole CTA for the scaling pass). ---------
__global__ void __launch_bounds__(256) rmsnorm_kernel(const float* __restrict__ x,
                                                      const float* __restrict__ w, float* out,
                                                      int n, float eps) {
  __shared__ float s_scale;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x < 32) {
    const int pack_num = n >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int base = 0; base < pack_num; base += 128) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int idx = base + 32 * j + lane;
        if (idx < pack_num) {
          const float4 v = x4[idx];
          float s = acc[j];
          s = __fmaf_rn(v.x, v.x, s);
          s = __fmaf_rn(v.y, v.y, s);
          s = __fmaf_rn(v.z, v.z, s);
          s = __fmaf_rn(v.w, v.w, s);
          acc[j] = s;
        }
      }
    }
    for (int i = (pack_num << 2) + lane; i < n; i += 128) acc[0] = __fmaf_rn(x[i], x[i], acc[0]);
    const float sum = block128_sum_vt(acc);
    if (lane == 0) s_scale = rsqrtf(__fadd_rn(__fdiv_rn(sum, static_cast<float>(n)), eps));
  }
  __syncthreads();
  const float sc = s_scale;
  const int pack_off = (n >> 2) << 2;
  // every element is read before it is written by the same thread: in-place safe
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float xi = x[i], wi = w[i];
    out[i] = (i < pack_off) ? __fmul_rn(__fmul_rn(sc, xi), wi) : __fmul_rn(__fmul_rn(wi, xi), sc);
  }
}

__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* out,
                           int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __fadd_rn(a[i], b[i]);
}

__global__ void swiglu_kernel(const float* __restrict__ x1, const float* __restrict__ x3,
                              float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = swiglu_ref(x1[i], x3[i]);
}

// rope_kernel.cu:38-49 / 84-95 / 124-135: same expression, same libdevice calls, and -- like the
// reference -- a LITERAL base per flavour so the compiler sees the same powf call site.
template <int kFlavour>
__global__ void sincos_kernel(int head_size, int seq_len, float* sin_cache, float* cos_cache) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= head_size * seq_len) return;
  const int pos = idx / head_size;
  const int head_dim = idx % head_size;
  float freq;
  if (kFlavour == KLLM_FLAVOUR_LLAMA3) {
    freq = 1.0f / pow(500000.0f, static_cast<float>(head_dim) / static_cast<float>(head_size));
  } else if (kFlavour == KLLM_FLAVOUR_QWEN2) {
    freq = 1.0f / pow(1000000.0f, static_cast<float>(head_dim) / static_cast<float>(head_size));
  } else {
    freq = 1.0f / pow(10000.0f, static_cast<float>(head_dim) / static_cast<float>(head_size));
  }
  float val = static_cast<float>(pos) * freq;
  float fcr = cosf(val);
  float fci = sinf(val);
  *(sin_cache + pos * head_size + head_dim) = fci;
  *(cos_cache + pos * head_size + head_dim) = fcr;
}

// rope_kernel.cu:97-122 (interleaved) as compiled:
//   x' = fma(fcr, x, -(fci*y));  y' = fma(fci, x, fcr*y)
__global__ void rope_interleaved_kernel(int pos, int dim, int kv_dim, int head_size, float* q, float* k,
                                        const float* __restrict__ sin_cache,
                                        const float* __restrict__ cos_cache) {
  const int idx = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (idx >= dim) return;
  const int head_dim = idx % head_size;
  const float fci = sin_cache[pos * head_size + head_dim];
  const float fcr = cos_cache[pos * head_size + head_dim];
  {
    const float2 v = *reinterpret_cast<float2*>(q + idx);
    float2 r;
    r.x = __fmaf_rn(fcr, v.x, -__fmul_rn(fci, v.y));
    r.y = __fmaf_rn(fci, v.x, __fmul_rn(fcr, v.y));
    *reinterpret_cast<float2*>(q + idx) = r;
  }
  if (idx < kv_dim) {
    const float2 v = *reinterpret_cast<float2*>(k + idx);
    float2 r;
    r.x = __fmaf_rn(fcr, v.x, -__fmul_rn(fci, v.y));
    r.y = __fmaf_rn(fci, v.x, __fmul_rn(fcr, v.y));
    *reinterpret_cast<float2*>(k + idx) = r;
  }
}

// rope_kernel.cu:5-36 / 51-82 (half-split) as compiled:
//   v0' = fma(fcr, v0, -(fci*v1));  v1' = fma(fci, v0, fcr*v1)
// One thread per pair; the reference's `idx > total_pairs` lets thread total_pairs run past
// the end of q -- here the bound is exact.
__global__ void rope_halfsplit_kernel(int pos, int dim, int kv_dim, int head_size, float* q, float* k,
                                      const float* __restrict__ sin_cache,
                                      const float* __restrict__ cos_cache) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = head_size / 2;
  const int total_pairs = (dim / head_size) * half;
  if (idx >= total_pairs) return;
  const int head_idx = idx / half;
  const int head_dim = idx % half;
  const int i = head_idx * head_size;
  const int v0_idx = i + head_dim;
  const int v1_idx = v0_idx + half;
  const float fci = sin_cache[pos * head_size + head_dim * 2];
  const float fcr = cos_cache[pos * head_size + head_dim * 2];
  const int rotn = i < kv_dim ? 2 : 1;
  for (int v = 0; v < rotn; ++v) {
    float* vec = v == 0 ? q : k;
    const float v0 = vec[v0_idx];
    const float v1 = vec[v1_idx];
    vec[v0_idx] = __fmaf_rn(fcr, v0, -__fmul_rn(fci, v1));
    vec[v1_idx] = __fmaf_rn(fci, v0, __fmul_rn(fcr, v1));
  }
}

// emb_kernel.cu:3-21: one CTA per token, row copy (128-bit when aligned).
__global__ void embedding_kernel(const int32_t* __restrict__ tokens, int n_tokens,
                                 const float* __restrict__ table, float* out, int dim,
                                 int vocab) {
  const int t = blockIdx.x;
  if (t >= n_tokens) return;
  const int32_t token = tokens[t];
  if (token < 0 || token >= vocab) return;
  const float* src = table + static_cast<size_t>(token) * dim;
  float* dst = out + static_cast<size_t>(t) * dim;
  if ((dim & 3) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int i = threadIdx.x; i < (dim >> 2); i += blockDim.x) d4[i] = s4[i];
  } else {
    for (int i = threadIdx.x; i < dim; i += blockDim.x) dst[i] = src[i];
  }
}

// argmax_kernel.cu:5-71: maximum value, lowest index among equals.  Two passes over
// gridDim.x partials keep it exact and order-independent: (value, index) pairs compared
// lexicographically form a total order, so any reduction tree gives the same answer.
struct ArgPair {
  float v;
  long long i;
};

__device__ __forceinline__ ArgPair arg_better(ArgPair a, ArgPair b) {
  if (b.i < 0) return a;
  if (a.i < 0) return b;
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}

__device__ __forceinline__ ArgPair arg_block_reduce(ArgPair p) {
  __shared__ float sv[32];
  __shared__ long long si[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    ArgPair o;
    o.v = __shfl_down_sync(kFull, p.v, off);
    o.i = __shfl_down_sync(kFull, p.i, off);
    p = arg_better(p, o);
  }
  if (lane == 0) {
    sv[warp] = p.v;
    si[warp] = p.i;
  }
  __syncthreads();
  if (warp == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    p.v = lane < nw ? sv[lane] : 0.f;
    p.i = lane < nw ? si[lane] : -1;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      ArgPair o;
      o.v = __shfl_down_sync(kFull, p.v, off);
      o.i = __shfl_down_sync(kFull, p.i, off);
      p = arg_better(p, o);
    }
  }
  return p;  // valid in thread 0
}

__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ x, long long n,
                                                      long long* out) {
  ArgPair best{0.f, -1};
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = x[i];
    if (best.i < 0 || v > best.v) best = ArgPair{v, i};
  }
  best = arg_block_reduce(best);
  if (threadIdx.x == 0) *out = best.i < 0 ? 0 : best.i;
}

// kllm_sample_f32: one block draws the id by the rule of sampling.cuh
__global__ void __launch_bounds__(1024) sample_kernel(const float* __restrict__ logits, int n, SampleParams sp, int pos,
                                                      long long* out_index) {
  constexpr int kScratch = sampling::kDrawScratchBytes;
  __shared__ __align__(16) unsigned char scratch[kScratch];
  const int i = sampling::draw_block<1024>(logits, n, sp, pos, nullptr, nullptr, 0, scratch, kScratch,
                                           [] { __syncthreads(); });
  if (threadIdx.x == 0) *out_index = i;
}

// kllm_repetition_penalty_f32: the raw logits, then step 0b of sampling.cuh over the ids.  The second kernel
// reads the raw logit, so an id listed twice writes the same value twice.
__global__ void copy_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[i];
}
__global__ void penalize_ids_kernel(const float* __restrict__ logits, float* __restrict__ out, int n,
                                    const int32_t* __restrict__ ids, int n_ids, float penalty) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_ids) return;
  const int id = ids[j];
  if (id >= 0 && id < n) out[id] = sampling::penalize(logits[id], penalty);
}

// kllm_logit_penalties_f32: step 0 of sampling.cuh over explicit id lists, block b over its own range of rows
__global__ void __launch_bounds__(256) logit_penalties_kernel(const float* __restrict__ logits, float* out, int n,
                                                              PenaltyParams pp, const int32_t* rep_ids, int n_rep,
                                                              const int32_t* count_ids, int n_count) {
  const int lo = static_cast<int>(static_cast<int64_t>(blockIdx.x) * n / gridDim.x);
  const int hi = static_cast<int>(static_cast<int64_t>(blockIdx.x + 1) * n / gridDim.x);
  sampling::step0_rows<256>(logits, out, lo, hi, pp, sampling::IdRange{rep_ids, 0, n_rep},
                            sampling::IdRange{count_ids, 0, n_count}, [] { __syncthreads(); });
}

// kllm_logprobs_f32: the logprob rule of sampling.cuh over one block (the graph engine's partition), then lp of
// every listed id
__global__ void __launch_bounds__(1024) logprobs_kernel(const float* __restrict__ logits, int n,
                                                        const int32_t* __restrict__ ids, int n_ids, int top_n,
                                                        float* out_lp, int32_t* out_top_ids, float* out_top_lp) {
  constexpr int kScratch = sampling::logprob_scratch_bytes(1024);
  __shared__ __align__(16) unsigned char scratch[kScratch];
  sampling::logprobs_block<1024>(logits, n, top_n, scratch, kScratch, [] { __syncthreads(); });
  const sampling::LogprobScratch& ls = *reinterpret_cast<const sampling::LogprobScratch*>(scratch);
  if (static_cast<int>(threadIdx.x) < top_n) {
    const int i = ls.top_i[threadIdx.x];
    out_top_ids[threadIdx.x] = i;
    out_top_lp[threadIdx.x] = i < 0 ? -INFINITY : sampling::logprob(ls.top_v[threadIdx.x], ls.m, ls.lse_off);
  }
  for (int j = threadIdx.x; j < n_ids; j += 1024) {
    const int id = ids[j];
    out_lp[j] = (id >= 0 && id < n) ? sampling::logprob(logits[id], ls.m, ls.lse_off) : __int_as_float(0x7fffffff);
  }
}

}  // namespace kllm

using namespace kllm;

extern "C" {

const char* kllm_version(void) { return "kllm_b200 0.1 (sm_90a)"; }

const char* kllm_error_string(int code) {
  switch (code) {
    case KLLM_OK: return "ok";
    case KLLM_E_INVALID: return "invalid argument";
    case KLLM_E_UNSUPPORTED: return "unsupported shape";
    case KLLM_E_STATE: return "invalid decoder state";
    case KLLM_E_NODEVICE: return "no CUDA device";
    case KLLM_E_COMM: return "tensor-parallel transport unavailable or failed";
    default: return code > 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : "unknown";
  }
}

uint64_t kllm_launch_count(void) { return launch_counter().load(); }

int kllm_rmsnorm_f32(const float* x, const float* w, float* out, int n, float eps, void* stream) {
  if (!x || !w || !out || n <= 0) return KLLM_E_INVALID;
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) return KLLM_E_UNSUPPORTED;
  rmsnorm_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, w, out, n, eps);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_add_f32(const float* a, const float* b, float* out, int n, void* stream) {
  if (!a || !b || !out || n <= 0) return KLLM_E_INVALID;
  add_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, b, out, n);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_swiglu_f32(const float* x1, const float* x3, float* out, int n, void* stream) {
  if (!x1 || !x3 || !out || n <= 0) return KLLM_E_INVALID;
  swiglu_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(x1, x3, out, n);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_sincos_init(int head_size, int seq_len, int flavour, float* sin_cache, float* cos_cache,
                     void* stream) {
  if (!sin_cache || !cos_cache || head_size <= 0 || seq_len <= 0) return KLLM_E_INVALID;
  const long long total = static_cast<long long>(head_size) * seq_len;
  if (total > 0x7fffffffLL) return KLLM_E_UNSUPPORTED;
  const int blocks = static_cast<int>((total + 255) / 256);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (flavour == KLLM_FLAVOUR_LLAMA2) {
    sincos_kernel<KLLM_FLAVOUR_LLAMA2><<<blocks, 256, 0, s>>>(head_size, seq_len, sin_cache, cos_cache);
  } else if (flavour == KLLM_FLAVOUR_LLAMA3) {
    sincos_kernel<KLLM_FLAVOUR_LLAMA3><<<blocks, 256, 0, s>>>(head_size, seq_len, sin_cache, cos_cache);
  } else if (flavour == KLLM_FLAVOUR_QWEN2) {
    sincos_kernel<KLLM_FLAVOUR_QWEN2><<<blocks, 256, 0, s>>>(head_size, seq_len, sin_cache, cos_cache);
  } else {
    return KLLM_E_INVALID;
  }
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_rope_f32(int flavour, int dim, int kv_dim, int head_size, float* q, float* k, int pos,
                  const float* sin_cache, const float* cos_cache, void* stream) {
  if (!q || !k || !sin_cache || !cos_cache || pos < 0 || dim <= 0 || kv_dim <= 0 || head_size <= 0 ||
      (head_size & 1) || dim % head_size != 0)
    return KLLM_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int pairs = dim / 2;
  if (flavour == KLLM_FLAVOUR_LLAMA2) {
    rope_interleaved_kernel<<<(pairs + 127) / 128, 128, 0, s>>>(pos, dim, kv_dim, head_size, q, k, sin_cache,
                                                                cos_cache);
  } else if (flavour == KLLM_FLAVOUR_LLAMA3 || flavour == KLLM_FLAVOUR_QWEN2) {
    rope_halfsplit_kernel<<<(pairs + 127) / 128, 128, 0, s>>>(pos, dim, kv_dim, head_size, q, k, sin_cache,
                                                              cos_cache);
  } else {
    return KLLM_E_INVALID;
  }
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_embedding_f32(const int32_t* tokens, int n_tokens, const float* table, float* out,
                       int dim, int vocab, void* stream) {
  if (!tokens || !table || !out || n_tokens <= 0 || dim <= 0 || vocab <= 0)
    return KLLM_E_INVALID;
  embedding_kernel<<<n_tokens, 128, 0, static_cast<cudaStream_t>(stream)>>>(tokens, n_tokens,
                                                                           table, out, dim, vocab);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_argmax_f32(const float* logits, int64_t n, int64_t* out_index, void* stream) {
  if (!logits || !out_index || n <= 0) return KLLM_E_INVALID;
  argmax_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, static_cast<long long>(n), reinterpret_cast<long long*>(out_index));
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_sample_f32(const float* logits, int64_t n, float temperature, int32_t top_k, uint64_t seed, int32_t pos,
                    int64_t* out_index, void* stream) {
  if (!logits || !out_index || n <= 0 || n > 0x7fffffffLL || pos < 0) return KLLM_E_INVALID;
  if (!std::isfinite(temperature) || temperature < 0.f) return KLLM_E_INVALID;
  sample_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(logits, static_cast<int>(n),
                                                                   SampleParams{temperature, top_k, seed}, pos,
                                                                   reinterpret_cast<long long*>(out_index));
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_sample_top_p_f32(const float* logits, int64_t n, float temperature, int32_t top_k, float top_p,
                          uint64_t seed, int32_t pos, int64_t* out_index, void* stream) {
  if (!logits || !out_index || n <= 0 || n > 0x7fffffffLL || pos < 0) return KLLM_E_INVALID;
  if (!std::isfinite(temperature) || temperature < 0.f) return KLLM_E_INVALID;
  if (!(top_p > 0.f && top_p <= 1.f)) return KLLM_E_INVALID;
  sample_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(logits, static_cast<int>(n),
                                                                   SampleParams{temperature, top_k, seed, top_p}, pos,
                                                                   reinterpret_cast<long long*>(out_index));
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int kllm_repetition_penalty_f32(const float* logits, float* out, int64_t n, const int32_t* ids, int32_t n_ids,
                                float penalty, void* stream) {
  if (!logits || !out || out == logits || n <= 0 || n > 0x7fffffffLL || n_ids < 0 || (n_ids > 0 && !ids))
    return KLLM_E_INVALID;
  if (!std::isfinite(penalty) || !(penalty > 0.f)) return KLLM_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int m = static_cast<int>(n);
  copy_f32_kernel<<<std::min(1024, (m + 255) / 256), 256, 0, s>>>(logits, out, m);
  count_launch();
  if (n_ids > 0) {  // after the copy, in stream order
    penalize_ids_kernel<<<static_cast<unsigned>((static_cast<int64_t>(n_ids) + 255) / 256), 256, 0, s>>>(logits, out, m, ids, n_ids, penalty);
    count_launch();
  }
  return static_cast<int>(cudaGetLastError());
}

int kllm_logit_penalties_f32(const float* logits, float* out, int64_t n, const int32_t* bias_ids_host,
                             const float* bias_host, int32_t n_bias, float penalty, const int32_t* rep_ids,
                             int32_t n_rep, float frequency, float presence, const int32_t* count_ids,
                             int32_t n_count, void* stream) {
  if (!logits || !out || out == logits || n <= 0 || n > 0x7fffffffLL || n_bias < 0 || n_rep < 0 || n_count < 0 ||
      n_count >= sampling::kInHistory || (n_bias > 0 && (!bias_ids_host || !bias_host)) || (n_rep > 0 && !rep_ids) ||
      (n_count > 0 && !count_ids))
    return KLLM_E_INVALID;
  if (!std::isfinite(penalty) || !(penalty > 0.f) || !std::isfinite(frequency) || !std::isfinite(presence))
    return KLLM_E_INVALID;
  const int m = static_cast<int>(n);
  std::vector<float> table;
  if (n_bias > 0) {
    std::vector<char> seen(m, 0);
    table.assign(m, 0.f);
    for (int32_t k = 0; k < n_bias; ++k) {
      const int32_t id = bias_ids_host[k];
      if (id < 0 || id >= m || seen[id] || !std::isfinite(bias_host[k])) return KLLM_E_INVALID;
      seen[id] = 1;
      table[id] = 0.f + bias_host[k];  // HF's table: 0 + b
    }
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // scratch: the mark words [n] (zeroed), then the dense bias table [n]
  int32_t* marks = nullptr;
  const size_t bytes = sizeof(int32_t) * m + (n_bias > 0 ? sizeof(float) * m : 0);
  if (cudaMallocAsync(reinterpret_cast<void**>(&marks), bytes, s) != cudaSuccess) return KLLM_E_NODEVICE;
  float* bias = n_bias > 0 ? reinterpret_cast<float*>(marks + m) : nullptr;
  int rc = static_cast<int>(cudaMemsetAsync(marks, 0, sizeof(int32_t) * m, s));
  // from pageable memory: returns once the table is staged, so `table` may go out of scope
  if (rc == 0 && bias) rc = static_cast<int>(cudaMemcpyAsync(bias, table.data(), sizeof(float) * m,
                                                             cudaMemcpyHostToDevice, s));
  if (rc == 0) {
    PenaltyParams pp{};
    pp.penalty = penalty, pp.frequency = frequency == 0.f ? 0.f : frequency;
    pp.presence = presence == 0.f ? 0.f : presence;
    pp.bias = bias, pp.marks = marks;
    const int rep_n = sampling::penalty_active(pp) ? n_rep : 0;
    const int cnt_n = sampling::counts_active(pp) ? n_count : 0;
    logit_penalties_kernel<<<std::max(1, std::min(64, (m + 4095) / 4096)), 256, 0, s>>>(logits, out, m, pp, rep_ids,
                                                                                        rep_n, count_ids, cnt_n);
    count_launch();
    rc = static_cast<int>(cudaGetLastError());
  }
  const int frc = static_cast<int>(cudaFreeAsync(marks, s));
  return rc != 0 ? rc : frc;
}

int kllm_logprobs_f32(const float* logits, int64_t n, const int32_t* ids, int32_t n_ids, int32_t top_n, float* out_lp,
                      int32_t* out_top_ids, float* out_top_lp, void* stream) {
  if (!logits || n <= 0 || n > 0x7fffffffLL || n_ids < 0 || (n_ids > 0 && (!ids || !out_lp))) return KLLM_E_INVALID;
  if (top_n < 0 || top_n > KLLM_MAX_TOP_LOGPROBS || (top_n > 0 && (!out_top_ids || !out_top_lp))) return KLLM_E_INVALID;
  logprobs_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(logits, static_cast<int>(n), ids, n_ids, top_n,
                                                                     out_lp, out_top_ids, out_top_lp);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int64_t kllm_argmax_f32_sync(const float* logits, int64_t n, void* stream) {
  static thread_local int64_t* d_idx = nullptr;
  if (d_idx == nullptr && cudaMalloc(&d_idx, sizeof(int64_t)) != cudaSuccess) return KLLM_E_NODEVICE;
  const int rc = kllm_argmax_f32(logits, n, d_idx, stream);
  if (rc != 0) return rc < 0 ? rc : -1000 - rc;
  int64_t h = -1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cudaMemcpyAsync(&h, d_idx, sizeof(h), cudaMemcpyDeviceToHost, s) != cudaSuccess) return -1000;
  if (cudaStreamSynchronize(s) != cudaSuccess) return -1000;
  return h;
}

}  // extern "C"
