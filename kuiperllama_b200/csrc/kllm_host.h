// Host-side plumbing shared by the translation units of libkllm_b200.so.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>

#include "../../include/kllm_b200.h"
#include "cache_layout.h"
#include "decoder_model.h"

namespace kllm {
// Launch accounting for bench.py's `gpu_launches` claim: every kernel<<<>>> issued by this
// library bumps the counter (graph replays add the node count of the replayed graph).
std::atomic<uint64_t>& launch_counter();
inline void count_launch(uint64_t n = 1) { launch_counter().fetch_add(n, std::memory_order_relaxed); }

// Opt `kernel` in to `bytes` of dynamic shared memory on the current device.  The attribute belongs to the kernel
// function, one value per device for the whole process, and every live decoder launches the same instantiations at
// its own size: so the value only ever rises, to the largest size any caller has asked for (a later decoder's smaller
// request must not refuse an earlier one's launches).  Each launch still passes its own size.  Thread-safe.
int smem_opt_in(const void* kernel, size_t bytes);

// A position that is either a host value or read from device memory at kernel run time; the
// decoder's CUDA graphs use the device form so ONE captured graph serves every position.
struct PosArg {
  const int* ptr;
  int val;
  __host__ __device__ int get() const { return ptr != nullptr ? *ptr : val; }
};

// One row of a batch's chain (kllm_batch, DESIGN.md 5.14): a member decoder's fp32 KV cache in its engine's layout,
// and the position word of its step state (mega::State::pos), read at run time so that one captured chain serves
// every position
struct ChainMember {
  float* key_cache;
  float* value_cache;
  const int* pos;
};

// Where the chain's n rows run: row i at first + i in one cache, or, with `members` (a device table of n rows, the
// batch), row i at *members[i].pos in members[i]'s cache
struct ChainPos {
  PosArg first;
  const ChainMember* members;
};

// Returns the first nonzero status of a call (a KLLM_E_* code or a cudaError_t)
#define KLLM_TRY(expr)                      \
  do {                                      \
    const int rc_ = static_cast<int>(expr); \
    if (rc_ != 0) return rc_;               \
  } while (0)

// The fused GEMV of `job` over nv <= 8 input vectors x[nv][in_dim] (nv > 1: kllm_decoder_verify's positions), each
// with the single vector's arithmetic, of weights in `format`: kInt8 with the job's group_size > 0, kF32 or kBf16
// with group_size 0.  Vector v's rows land at seg.out + v * seg.rows (SwiGLU: + v * rows of the pair) and its
// residual is residual + v * rows.
int gemv_dispatch(const kllm_gemv_job* job, WeightFormat format, cudaStream_t stream, int nv = 1);

// mha_decode_kernel for the n_pos query positions at.first, at.first + 1, .. (q, output
// [n_pos][head_num * head_size], scores [n_pos][head_num][seq_len]) over an fp32 cache in either engine's layout;
// with at.members, mha_members_kernel: row i over members[i]'s cache at its position (key_cache and value_cache unused)
int launch_mha_rows(ChainPos at, int n_pos, const prefill::CacheLayout& c, int head_num, int layer_index,
                    int kv_mul, float* mha_out, const float* query, float* score, const float* key_cache,
                    const float* value_cache, cudaStream_t stream);

// tp_comm.cu: exchange areas [2][world][stride] of 64-bit tagged words, one per rank (peer transport)
int comm_tagged_areas(kllm_comm* comm, unsigned long long** areas8, int* world, int* rank, int* stride);

// The decoder's KV cache, in the layout of its engine, and its RoPE tables: what the batched prefill (prefill.cu) and
// the decode chain (verify.cu) write and read
struct DecoderCache {
  prefill::CacheLayout cache;
  float* key_cache; float* value_cache;  // cache.elem: bf16 or fp8 elements behind these pointers
  const float* sin_cache; const float* cos_cache;
  const float* kv_scales;  // KLLM_KV_FP8: device [4][L][kv_head], s_k, s_v, 1 / s_k, 1 / s_v
};
struct PrefillWorkspace {  // [block, .] activations
  float *x, *xn, *q, *k, *v, *att, *h1, *h3, *tmp;
};
// prefill.cu: one block of T prompt positions of the model through every layer with batched wgmma GEMMs, into
// the caches in the layout of the engine that continues decoding
int prefill_block(const DecoderModel& dm, const DecoderCache& m, PrefillWorkspace& ws, const int32_t* tokens_dev, int T,
                  int start_pos, cudaStream_t stream);
int prefill_attention_smem_opt_in(size_t bytes);
// RoPE on T query rows [T][q_rows] in place and on T key rows [T][kv_dim], scattered with the value rows into layer
// `layer` of an fp32 cache at positions at.first .. at.first + T - 1 (or, with at.members, row t into members[t]'s
// cache at its position): kllm_rope_f32's arithmetic (prefill.cu)
int launch_rope_scatter_f32(const DecoderModel& dm, const DecoderCache& c, int layer, float* q, const float* k,
                            const float* v, ChainPos at, int T, cudaStream_t s);

inline float flavour_eps(int flavour) { return flavour == KLLM_FLAVOUR_QWEN2 ? 1e-6f : 1e-5f; }
}  // namespace kllm
