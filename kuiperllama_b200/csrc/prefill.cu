// Batched prompt prefill around the wgmma GEMM (prefill_gemm.cu) -- the TOLERANCED alternative to
// feeding the prompt position by position (demo/main.cpp:18-23 calls LLama2Model::predict once per
// prompt token; llama3.cpp:147-167 then runs the whole single-token forward, classifier included).
//
// For a block of T prompt positions every projection is ONE GEMM [T, in] x [out, in]^T on the tensor
// cores (TF32 multiply, fp32 accumulate) instead of T GEMVs, so the weights are streamed once per
// 256 tokens; the small per-token operators (RMSNorm, RoPE, causal attention over the cache, SiLU*gate,
// residual adds) are plain fp32 CUDA kernels over the T rows; only the last position runs the
// classifier (the reference throws the others away, llama3.cpp:738-739).  The K / V rows land in the
// decoder's cache in the layout of the engine that will continue decoding.
//
// Because of TF32 (10 mantissa bits per operand) the cache rows and the final logits agree with the
// position-by-position path to ~1e-3 relative, not bit for bit; tests/test_prefill_gpu.py states the
// bound.  fp32 and int8 checkpoints (the int8 GEMM dequantises its weight tiles to TF32), single GPU.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>
#include <type_traits>

#include "../../include/kllm_b200.h"
#include "cache_layout.h"
#include "kllm_device.cuh"
#include "kllm_host.h"
#include "kv_fp8.cuh"

namespace kllm {
namespace prefill {

__global__ void embed_rows_kernel(const int32_t* __restrict__ tokens, const float* __restrict__ table,
                                  float* __restrict__ x, int dim, int vocab) {
  const int t = blockIdx.x;
  int tok = tokens[t];
  if (tok < 0 || tok >= vocab) tok = 0;
  const float4* src = reinterpret_cast<const float4*>(table + static_cast<size_t>(tok) * dim);
  float4* dst = reinterpret_cast<float4*>(x + static_cast<size_t>(t) * dim);
  for (int i = threadIdx.x; i < (dim >> 2); i += blockDim.x) dst[i] = src[i];
}

__device__ __forceinline__ float block_sum(float v, float* scratch) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float total = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) total += scratch[w];
  return total;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, off));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float m = -FLT_MAX;
  for (int w = 0; w < (blockDim.x >> 5); ++w) m = fmaxf(m, scratch[w]);
  return m;
}

// rmsnorm_kernel.cu:4-50 per row (summation order differs: toleranced path)
__global__ void rmsnorm_rows_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out,
                                    int dim, float eps) {
  __shared__ float scratch[32];
  const float* row = x + static_cast<size_t>(blockIdx.x) * dim;
  float* o = out + static_cast<size_t>(blockIdx.x) * dim;
  float ss = 0.f;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) ss += row[i] * row[i];
  const float total = block_sum(ss, scratch);
  const float sc = rsqrtf(total / static_cast<float>(dim) + eps);
  for (int i = threadIdx.x; i < dim; i += blockDim.x) o[i] = (sc * row[i]) * w[i];
}

__global__ void add_bias_rows_kernel(float* __restrict__ y, const float* __restrict__ b, int n) {
  float* row = y + static_cast<size_t>(blockIdx.x) * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) row[i] += b[i];
}
__global__ void add_rows_kernel(float* __restrict__ x, const float* __restrict__ y, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    x[i] = x[i] + y[i];  // llama3.cpp:683,719: x + out
}
__global__ void swiglu_rows_kernel(float* __restrict__ h1, const float* __restrict__ h3, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    h1[i] = swiglu_ref(h1[i], h3[i]);
}

// A cache element of type E (float, or __nv_bfloat16 for the bf16 KV cache: rounded to nearest even on the way
// in, widened exactly on the way out; or __nv_fp8_e4m3 for the fp8 one: encoded at the inverse `inv` of its scale on
// the way in, fp32(value(code) * s) on the way out).  The float and bf16 forms take no scale.
__device__ __forceinline__ void put(float* p, float v, float) { *p = v; }
__device__ __forceinline__ void put(__nv_bfloat16* p, float v, float) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void put(__nv_fp8_e4m3* p, float v, float inv) { p->__x = e4m3_encode(v, inv); }
__device__ __forceinline__ float get(const float* p, float) { return *p; }
__device__ __forceinline__ float get(const __nv_bfloat16* p, float) { return __bfloat162float(*p); }
__device__ __forceinline__ float get(const __nv_fp8_e4m3* p, float s) { return __fmul_rn(e4m3_value(p->__x), s); }
template <typename E>
constexpr bool kScaled = std::is_same_v<E, __nv_fp8_e4m3>;

// The fp8 cache's scales of one layer, [kv_head] each (null for the other caches): the K and V scales, or their
// inverses
struct KvScales {
  const float* k;
  const float* v;
};

// RoPE (rope_kernel.cu) on the T query rows in place, and on the T key rows while they are scattered,
// with the value rows, into the layer's cache (of element type E; fp8: at the inverses `inv` of the layer's scales):
// the layer at layer_off elements into kcache / vcache, row t at position at.first + t; or, with at.members (the
// batch, fp32 only), row t into the layer of members[t]'s cache at *members[t].pos.
// grid = (T, rope_blocks): one thread per rotation pair and per value element.
template <typename E>
__global__ void rope_scatter_kernel(float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                    const float* __restrict__ sin_t, const float* __restrict__ cos_t,
                                    E* kcache, E* vcache, size_t layer_off, CacheLayout c, int heads,
                                    int kv_heads, int flavour, ChainPos at, KvScales inv) {
  const int t = blockIdx.x, hs = c.head_size, half = hs >> 1;
  int pos = at.first.get() + t;
  if (at.members != nullptr) {
    const ChainMember& mb = at.members[t];
    pos = *mb.pos;
    kcache = reinterpret_cast<E*>(mb.key_cache), vcache = reinterpret_cast<E*>(mb.value_cache);
  }
  kcache += layer_off, vcache += layer_off;
  const int p0 = blockIdx.y * blockDim.x + threadIdx.x, stride = gridDim.y * blockDim.x;
  float* qrow = q + static_cast<size_t>(t) * heads * hs;
  const float* krow = k + static_cast<size_t>(t) * kv_heads * hs;
  const float* vrow = v + static_cast<size_t>(t) * kv_heads * hs;
  for (int p = p0; p < (heads + kv_heads) * half; p += stride) {
    const int h = p / half, j = p % half;
    int i0, i1;
    if (flavour == KLLM_FLAVOUR_LLAMA2) {
      i0 = 2 * j, i1 = 2 * j + 1;
    } else {
      i0 = j, i1 = j + half;
    }
    const float fci = sin_t[static_cast<size_t>(pos) * hs + 2 * j];
    const float fcr = cos_t[static_cast<size_t>(pos) * hs + 2 * j];
    if (h < heads) {
      float* qh = qrow + h * hs;
      const float a = qh[i0], b = qh[i1];
      qh[i0] = __fmaf_rn(fcr, a, -__fmul_rn(fci, b));
      qh[i1] = __fmaf_rn(fci, a, __fmul_rn(fcr, b));
    } else {
      const int kvh = h - heads;
      const float a = krow[kvh * hs + i0], b = krow[kvh * hs + i1];
      const float ik = kScaled<E> ? inv.k[kvh] : 1.f;
      put(kcache + k_index(c, pos, kvh, i0), __fmaf_rn(fcr, a, -__fmul_rn(fci, b)), ik);
      put(kcache + k_index(c, pos, kvh, i1), __fmaf_rn(fci, a, __fmul_rn(fcr, b)), ik);
    }
  }
  for (int p = p0; p < kv_heads * hs; p += stride)
    put(vcache + v_index(c, pos, p / hs, p % hs), vrow[p], kScaled<E> ? inv.v[p / hs] : 1.f);
}

// rope_scatter_kernel's grid of 256-thread blocks for T positions: the rotation pairs of one position over blocks
inline dim3 rope_grid(int T, int heads, int kv_heads, int head_size) {
  return dim3(T, ((heads + kv_heads) * (head_size >> 1) + 255) / 256);
}

// Causal attention of query (t, head) over cache positions 0 .. start_pos + t (mha_kernel.cu:47-110
// arithmetic, fp32, over cache elements of type E; fp8: at the layer's scales `sc`).  grid = (heads, T); scores in
// dynamic shared memory.
template <typename E>
__global__ void attn_rows_kernel(const float* __restrict__ q, const E* __restrict__ kcache,
                                 const E* __restrict__ vcache, float* __restrict__ out, CacheLayout c, int heads,
                                 int kv_mul, int start_pos, KvScales scales) {
  extern __shared__ float sc[];
  __shared__ float scratch[32];
  const int head = blockIdx.x, t = blockIdx.y, pos = start_pos + t, hs = c.head_size, kvh = head / kv_mul;
  const float s_k = kScaled<E> ? scales.k[kvh] : 1.f, s_v = kScaled<E> ? scales.v[kvh] : 1.f;
  const float* qh = q + (static_cast<size_t>(t) * heads + head) * hs;
  const float scale = 1.f / sqrtf(static_cast<float>(hs));
  float mx = -FLT_MAX;
  for (int j = threadIdx.x; j <= pos; j += blockDim.x) {
    float s = 0.f;
    for (int i = 0; i < hs; ++i) s = __fmaf_rn(get(kcache + k_index(c, j, kvh, i), s_k), qh[i], s);
    s *= scale;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_max(mx, scratch);
  float sum = 0.f;
  for (int j = threadIdx.x; j <= pos; j += blockDim.x) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = block_sum(sum, scratch);
  __syncthreads();
  for (int i = threadIdx.x; i < hs; i += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j <= pos; ++j) acc = __fmaf_rn(sc[j] / sum, get(vcache + v_index(c, j, kvh, i), s_v), acc);
    out[(static_cast<size_t>(t) * heads + head) * hs + i] = acc;
  }
}

}  // namespace prefill

using namespace prefill;

int prefill_block(const DecoderModel& dm, const DecoderCache& m, PrefillWorkspace& ws, const int32_t* tokens_dev, int T,
                  int start_pos, cudaStream_t s) {
  const int dim = dm.dim, hid = dm.hidden_dim, heads = dm.head_num, kvh = dm.kv_head_num;
  const int q_rows = dm.q_rows, kvd = dm.kv_dim;
  auto count = [&]() {
    count_launch();
    return static_cast<int>(cudaGetLastError());
  };
  // out[T, N] = x[T, K] . w^T (+ bias)
  auto gemm = [&](const float* x, const Matrix& w, float* out, int K, int N) {
    int rc;
    if (dm.format == WeightFormat::kInt8)
      rc = kllm_gemm_w8_tf32(x, static_cast<const int8_t*>(w.w), w.scales, out, T, K, N, dm.group_size, s);
    else if (dm.format == WeightFormat::kBf16)
      rc = kllm_gemm_bf16_tf32(x, static_cast<const uint16_t*>(w.w), out, T, K, N, s);
    else
      rc = kllm_gemm_tf32(x, static_cast<const float*>(w.w), out, T, K, N, s);
    if (rc != 0 || w.bias == nullptr) return rc;
    add_bias_rows_kernel<<<T, 256, 0, s>>>(out, w.bias, N);
    return count();
  };
  const int ew_grid = 528;  // 4 x 132 SMs for the grid-stride elementwise kernels
  embed_rows_kernel<<<T, 256, 0, s>>>(tokens_dev, dm.tok_emb, ws.x, dim, dm.vocab_size);
  KLLM_TRY(count());
  const CacheLayout& cl = m.cache;
  for (int l = 0; l < dm.layer_num; ++l) {
    const LayerWeights& lw = dm.layers[l];
    const size_t layer_off = static_cast<size_t>(l) * dm.seq_len * kvd;
    rmsnorm_rows_kernel<<<T, 256, 0, s>>>(ws.x, lw.attn_norm, ws.xn, dim, dm.eps);
    KLLM_TRY(count());
    KLLM_TRY(gemm(ws.xn, lw.q, ws.q, dim, q_rows));
    KLLM_TRY(gemm(ws.xn, lw.k, ws.k, dim, kvd));
    KLLM_TRY(gemm(ws.xn, lw.v, ws.v, dim, kvd));
    const size_t sc_bytes = static_cast<size_t>(start_pos + T) * sizeof(float);
    // the layer's cache, of element type E
    auto attend = [&](auto* kc, auto* vc, KvScales inv, KvScales sc) {
      rope_scatter_kernel<<<rope_grid(T, heads, kvh, dm.head_size), 256, 0, s>>>(
          ws.q, ws.k, ws.v, m.sin_cache, m.cos_cache, kc, vc, layer_off, cl, heads, kvh, dm.flavour,
          ChainPos{PosArg{nullptr, start_pos}, nullptr}, inv);
      KLLM_TRY(count());
      attn_rows_kernel<<<dim3(heads, T), 128, sc_bytes, s>>>(ws.q, kc + layer_off, vc + layer_off, ws.att, cl, heads,
                                                             dm.kv_mul, start_pos, sc);
      return 0;
    };
    if (cl.elem == KLLM_KV_FP8) {
      const size_t n = static_cast<size_t>(dm.layer_num) * kvh, h0 = static_cast<size_t>(l) * kvh;
      const float* ks = m.kv_scales;  // [4][L][kv_head]: s_k, s_v, 1 / s_k, 1 / s_v
      KLLM_TRY(attend(reinterpret_cast<__nv_fp8_e4m3*>(m.key_cache), reinterpret_cast<__nv_fp8_e4m3*>(m.value_cache),
                    KvScales{ks + 2 * n + h0, ks + 3 * n + h0}, KvScales{ks + h0, ks + n + h0}));
    } else if (cl.elem == KLLM_KV_BF16) {
      KLLM_TRY(attend(reinterpret_cast<__nv_bfloat16*>(m.key_cache), reinterpret_cast<__nv_bfloat16*>(m.value_cache),
                    KvScales{}, KvScales{}));
    } else {
      KLLM_TRY(attend(m.key_cache, m.value_cache, KvScales{}, KvScales{}));
    }
    KLLM_TRY(count());
    KLLM_TRY(gemm(ws.att, lw.o, ws.tmp, q_rows, dim));
    add_rows_kernel<<<ew_grid, 256, 0, s>>>(ws.x, ws.tmp, static_cast<size_t>(T) * dim);
    KLLM_TRY(count());
    rmsnorm_rows_kernel<<<T, 256, 0, s>>>(ws.x, lw.ffn_norm, ws.xn, dim, dm.eps);
    KLLM_TRY(count());
    KLLM_TRY(gemm(ws.xn, lw.w1, ws.h1, dim, hid));
    KLLM_TRY(gemm(ws.xn, lw.w3, ws.h3, dim, hid));
    swiglu_rows_kernel<<<ew_grid, 256, 0, s>>>(ws.h1, ws.h3, static_cast<size_t>(T) * hid);
    KLLM_TRY(count());
    KLLM_TRY(gemm(ws.h1, lw.w2, ws.tmp, hid, dim));
    add_rows_kernel<<<ew_grid, 256, 0, s>>>(ws.x, ws.tmp, static_cast<size_t>(T) * dim);
    KLLM_TRY(count());
  }
  return 0;
}

int launch_rope_scatter_f32(const DecoderModel& dm, const DecoderCache& c, int layer, float* q, const float* k,
                            const float* v, ChainPos at, int T, cudaStream_t s) {
  if (c.cache.elem != KLLM_KV_F32) return KLLM_E_UNSUPPORTED;
  const size_t layer_off = static_cast<size_t>(layer) * dm.seq_len * dm.kv_dim;
  rope_scatter_kernel<<<rope_grid(T, dm.head_num, dm.kv_head_num, dm.head_size), 256, 0, s>>>(
      q, k, v, c.sin_cache, c.cos_cache, c.key_cache, c.value_cache, layer_off, c.cache, dm.head_num,
      dm.kv_head_num, dm.flavour, at, KvScales{});
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int prefill_attention_smem_opt_in(size_t bytes) {
  if (bytes <= 48 * 1024) return 0;
  for (const void* k : {reinterpret_cast<const void*>(attn_rows_kernel<float>),
                        reinterpret_cast<const void*>(attn_rows_kernel<__nv_bfloat16>),
                        reinterpret_cast<const void*>(attn_rows_kernel<__nv_fp8_e4m3>)})
    if (int rc = smem_opt_in(k, bytes)) return rc;
  return 0;
}

}  // namespace kllm
