// Single-query (decode) attention over the fp32 KV cache: scores -> softmax -> weighted sum of
// values, one CTA per query head, GQA through head / kv_mul.
// Replaces multi_head_attention_kernel + softmax_gpu
// (kuiper/source/op/kernels/cuda/mha_kernel.cu:7-130).
//
// Arithmetic follows the reference kernel operation for operation so the output is
// bit-identical: each score is one left-to-right FFMA chain over head_size, softmax sums are
// taken by 256 strided lanes folded with the cub block-reduce tree, and out[i] is a single
// FFMA chain over t = 0..pos.  What changes is the memory side: q is staged in shared memory,
// value rows are streamed through a double-buffered shared-memory tile by all 256 threads
// (coalesced 128-bit loads) while the head_size chain-owning threads consume them, so the
// serial chain runs at shared-memory latency instead of L2 latency.
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"

namespace kllm {

constexpr int kMhaThreads = 256;
constexpr int kVTile = 32;  // timesteps per staged value tile

// cub::BlockReduce<float,256>::Sum (warp-reductions algorithm): per-warp shuffle tree, then
// thread 0 adds the 8 warp aggregates left to right.  Returns the total in thread 0 only.
__device__ __forceinline__ float block256_sum(float v, float* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_tree_sum(v);
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  float total = 0.f;
  if (threadIdx.x == 0) {
    total = s_warp[0];
#pragma unroll
    for (int w = 1; w < kMhaThreads / 32; ++w) total = __fadd_rn(total, s_warp[w]);
  }
  return total;
}

__device__ __forceinline__ float block256_max(float v, float* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, off));
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  float m = s_warp[0];
#pragma unroll
  for (int w = 1; w < kMhaThreads / 32; ++w) m = fmaxf(m, s_warp[w]);
  return m;  // every thread
}

// Query row blockIdx.y (one row of q, scores and output per row) at position `pos` over a cache in the graph
// engine's layout [seq][kv_dim], or with kTiled the persistent engine's exact-mode layout
// (prefill::CacheLayout: K [kv_head][head_size / 4][seq][4], V [kv_head][vsplit][seq][head_size / vsplit]).
// The layout, the row's position and its cache move addresses only; every operation is the same in each kernel
// below.
template <bool kTiled>
__device__ __forceinline__ void mha_decode_row(int pos, int seq_len, const float* __restrict__ query,
                                               float* score_ptr, float* output, const float* __restrict__ key_cache,
                                               const float* __restrict__ value_cache, int kv_dim, int kv_mul,
                                               int head_size, long long layer_offset, int vsplit) {
  extern __shared__ __align__(16) float smem[];
  float* q_s = smem;                           // [head_size]
  float* v_s = smem + head_size;               // [2][kVTile][head_size]
  __shared__ float s_warp[kMhaThreads / 32];
  __shared__ float s_bcast;

  const int head = blockIdx.x + blockIdx.y * gridDim.x;  // the (position, head) row of q, scores and output
  const int tid = threadIdx.x;
  const float scale = 1.f / sqrtf(static_cast<float>(head_size));
  const float* query_head = query + static_cast<size_t>(head) * head_size;
  float* score_head = score_ptr + static_cast<size_t>(head) * seq_len;
  const int kvh = blockIdx.x / kv_mul;
  // K row t: float4 chunk i at kbase + t * (4 or kv_dim) + 4 * i * k4_stride; V element (t, i) at vbase + (the tiled
  // or the flat index)
  const size_t kv_head_off = kTiled ? static_cast<size_t>(kvh) * head_size * seq_len : static_cast<size_t>(kvh) * head_size;
  const float* kbase = key_cache + layer_offset + kv_head_off;
  const float* vbase = value_cache + layer_offset + kv_head_off;
  const int k4_stride = kTiled ? seq_len : 1;
  const int dv = head_size / vsplit;

  for (int i = tid; i < head_size; i += kMhaThreads) q_s[i] = query_head[i];
  __syncthreads();

  // ---- scores: mha_kernel.cu:61-91 --------------------------------------------------
  const float4* q4 = reinterpret_cast<const float4*>(q_s);
  for (int t = tid; t <= pos; t += kMhaThreads) {
    const float4* k4 = reinterpret_cast<const float4*>(kbase + static_cast<size_t>(t) * (kTiled ? 4 : kv_dim));
    float score = 0.0f;
#pragma unroll 4
    for (int i = 0; i < (head_size >> 2); ++i) {
      const float4 kv = k4[static_cast<size_t>(i) * k4_stride];
      const float4 qv = q4[i];
      score = __fmaf_rn(kv.x, qv.x, score);
      score = __fmaf_rn(kv.y, qv.y, score);
      score = __fmaf_rn(kv.z, qv.z, score);
      score = __fmaf_rn(kv.w, qv.w, score);
    }
    score_head[t] = __fmul_rn(score, scale);
  }
  __syncthreads();

  // ---- softmax: mha_kernel.cu:7-45 ---------------------------------------------------
  const int size = pos + 1;
  float max_val = tid < size ? score_head[tid] : -FLT_MAX;
  for (int i = tid + kMhaThreads; i < size; i += kMhaThreads) max_val = fmaxf(max_val, score_head[i]);
  max_val = block256_max(max_val, s_warp);
  __syncthreads();

  float sum = 0.0f;
  for (int i = tid; i < size; i += kMhaThreads) {
    const float e = expf(score_head[i] - max_val);
    score_head[i] = e;
    sum += e;
  }
  sum = block256_sum(sum, s_warp);
  if (tid == 0) s_bcast = sum;
  __syncthreads();
  sum = s_bcast;
  for (int i = tid; i < size; i += kMhaThreads) score_head[i] = score_head[i] / sum;
  __syncthreads();

  // ---- weighted value sum: mha_kernel.cu:97-109 ----------------------------------------
  // All threads stage value tiles; threads < head_size own one output chain each.
  const int vec_per_row = head_size >> 2;
  const int n_tiles = (size + kVTile - 1) / kVTile;
  auto stage = [&](int tile, int buf) {
    const int t0 = tile * kVTile;
    float4* dst = reinterpret_cast<float4*>(v_s + static_cast<size_t>(buf) * kVTile * head_size);
    for (int e = tid; e < kVTile * vec_per_row; e += kMhaThreads) {
      const int tt = e / vec_per_row, c = e % vec_per_row;
      if (t0 + tt <= pos)
        dst[e] = *reinterpret_cast<const float4*>(
            vbase + (kTiled ? (static_cast<size_t>(4 * c / dv) * seq_len + t0 + tt) * dv + (4 * c) % dv
                            : static_cast<size_t>(t0 + tt) * kv_dim + 4 * c));
    }
  };
  float value = 0.0f;
  stage(0, 0);
  __syncthreads();
  for (int tile = 0; tile < n_tiles; ++tile) {
    const int buf = tile & 1;
    if (tile + 1 < n_tiles) stage(tile + 1, buf ^ 1);
    if (tid < head_size) {
      const float* vt = v_s + static_cast<size_t>(buf) * kVTile * head_size + tid;
      const int t0 = tile * kVTile;
      const int cnt = min(kVTile, size - t0);
#pragma unroll 8
      for (int tt = 0; tt < cnt; ++tt)
        value = __fmaf_rn(score_head[t0 + tt], vt[tt * head_size], value);
    }
    __syncthreads();
  }
  if (tid < head_size) output[static_cast<size_t>(head) * head_size + tid] = value;
}

// Position pos_arg + blockIdx.y of one cache
template <bool kTiled>
__global__ void __launch_bounds__(kMhaThreads)
mha_decode_kernel(PosArg pos_arg, int seq_len, const float* __restrict__ query, float* score_ptr,
                  float* output, const float* __restrict__ key_cache,
                  const float* __restrict__ value_cache, int kv_dim, int kv_mul, int head_size,
                  long long layer_offset, int vsplit) {
  mha_decode_row<kTiled>(pos_arg.get() + blockIdx.y, seq_len, query, score_ptr, output, key_cache, value_cache,
                         kv_dim, kv_mul, head_size, layer_offset, vsplit);
}

// A batch's row blockIdx.y: member blockIdx.y's cache at that member's position (kllm_batch, DESIGN.md 5.14)
template <bool kTiled>
__global__ void __launch_bounds__(kMhaThreads)
mha_members_kernel(const ChainMember* __restrict__ members, int seq_len, const float* __restrict__ query,
                   float* score_ptr, float* output, int kv_dim, int kv_mul, int head_size, long long layer_offset,
                   int vsplit) {
  const ChainMember& mb = members[blockIdx.y];
  mha_decode_row<kTiled>(*mb.pos, seq_len, query, score_ptr, output, mb.key_cache, mb.value_cache, kv_dim, kv_mul,
                         head_size, layer_offset, vsplit);
}

int launch_mha_rows(ChainPos at, int n_pos, const prefill::CacheLayout& c, int head_num, int layer_index,
                    int kv_mul, float* mha_out, const float* query, float* score, const float* key_cache,
                    const float* value_cache, cudaStream_t stream) {
  const int hs = c.head_size;
  if (!mha_out || !query || !score || n_pos <= 0) return KLLM_E_INVALID;
  if (at.members == nullptr && (!key_cache || !value_cache)) return KLLM_E_INVALID;
  if (c.elem != KLLM_KV_F32 || (hs & 3) != 0 || (c.kv_dim & 3) != 0 || hs > kMhaThreads) return KLLM_E_UNSUPPORTED;
  if (c.mega && (hs % c.split != 0 || (hs / c.split) % 4 != 0)) return KLLM_E_UNSUPPORTED;
  const long long layer_offset = static_cast<long long>(layer_index) * c.seq_len * c.kv_dim;
  // head_size 188 is the largest whose q row and two value tiles fit the default 48 KB; larger
  // heads (up to 256: 66 KB) opt in.  The tiling does not touch the arithmetic.
  const size_t smem = sizeof(float) * (hs + 2 * kVTile * hs);
  const dim3 grid(head_num, n_pos);
  const int vsplit = c.mega ? c.split : 1;
  auto launch = [&](auto one, auto rows) {
    const void* k = at.members ? reinterpret_cast<const void*>(rows) : reinterpret_cast<const void*>(one);
    if (smem > 48 * 1024) {
      if (const int rc = smem_opt_in(k, smem)) return rc;
    }
    if (at.members)
      rows<<<grid, kMhaThreads, smem, stream>>>(at.members, c.seq_len, query, score, mha_out, c.kv_dim, kv_mul, hs,
                                                layer_offset, vsplit);
    else
      one<<<grid, kMhaThreads, smem, stream>>>(at.first, c.seq_len, query, score, mha_out, key_cache, value_cache,
                                               c.kv_dim, kv_mul, hs, layer_offset, vsplit);
    return 0;
  };
  const int rc = c.mega ? launch(mha_decode_kernel<true>, mha_members_kernel<true>)
                        : launch(mha_decode_kernel<false>, mha_members_kernel<false>);
  if (rc != 0) return rc;
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace kllm

extern "C" int kllm_mha_decode_f32(int pos, int head_num, int layer_index, int seq_len, int kv_dim,
                                   int kv_mul, int head_size, float* mha_out, const float* query,
                                   float* score, const float* key_cache, const float* value_cache,
                                   void* stream) {
  if (pos < 0 || pos >= seq_len || head_num <= 0 || kv_mul <= 0 || head_size <= 0 || layer_index < 0)
    return KLLM_E_INVALID;
  const kllm::prefill::CacheLayout flat{0, seq_len, kv_dim, head_size, 1, KLLM_KV_F32};
  return kllm::launch_mha_rows(kllm::ChainPos{kllm::PosArg{nullptr, pos}, nullptr}, 1, flat, head_num, layer_index,
                               kv_mul, mha_out, query, score, key_cache, value_cache,
                               static_cast<cudaStream_t>(stream));
}
