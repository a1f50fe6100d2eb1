// The KV cache layouts of one layer, as the batched prefill writes and reads them (prefill.cu) and
// kllm_decoder_read_kv converts them back to the graph engine's [seq][kv_dim].
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace kllm {
namespace prefill {  // the prefill's kernels take a CacheLayout by value

struct CacheLayout {
  int mega;  // 1: persistent engine K [kvh][hs/4][seq][4], V [kvh][split][seq][hs/split]; 0: [seq][kv_dim]
  int seq_len, kv_dim, head_size, split;
  int bf16;  // with mega: bf16 elements, K [kvh][hs/8][seq][8] (16-byte chunks of 8 dims), V split 1
};
__host__ __device__ __forceinline__ size_t k_index(const CacheLayout& c, int pos, int kvh, int i) {
  if (c.mega && c.bf16)
    return (static_cast<size_t>(kvh) * (c.head_size >> 3) + (i >> 3)) * c.seq_len * 8 + static_cast<size_t>(pos) * 8 + (i & 7);
  if (c.mega) return (static_cast<size_t>(kvh) * (c.head_size >> 2) + (i >> 2)) * c.seq_len * 4 + static_cast<size_t>(pos) * 4 + (i & 3);
  return static_cast<size_t>(pos) * c.kv_dim + kvh * c.head_size + i;
}
__host__ __device__ __forceinline__ size_t v_index(const CacheLayout& c, int pos, int kvh, int i) {
  if (c.mega) {
    const int dv = c.head_size / c.split;
    return ((static_cast<size_t>(kvh) * c.split + i / dv) * c.seq_len + pos) * dv + i % dv;
  }
  return static_cast<size_t>(pos) * c.kv_dim + kvh * c.head_size + i;
}

}  // namespace prefill
}  // namespace kllm
