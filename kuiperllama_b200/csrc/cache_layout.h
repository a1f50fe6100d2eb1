// The KV cache layouts of one layer, as the batched prefill writes and reads them (prefill.cu) and
// kllm_decoder_read_kv converts them back to the graph engine's [seq][kv_dim].
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/kllm_b200.h"

namespace kllm {
namespace prefill {  // the prefill's kernels take a CacheLayout by value

struct CacheLayout {
  int mega;  // 1: persistent engine K [kvh][hs/4][seq][4], V [kvh][split][seq][hs/split]; 0: [seq][kv_dim]
  int seq_len, kv_dim, head_size, split;
  // the element, a kllm_decoder_desc::kv_cache value.  With mega, K keeps 16-byte chunks: KLLM_KV_BF16 K
  // [kvh][hs/8][seq][8] bf16, KLLM_KV_FP8 K [kvh][hs/16][seq][16] e4m3 codes; both with V split 1
  int elem;
};
__host__ __device__ __forceinline__ int kv_elem_bytes(int elem) {
  return elem == KLLM_KV_FP8 ? 1 : elem == KLLM_KV_BF16 ? 2 : 4;
}
__host__ __device__ __forceinline__ size_t k_index(const CacheLayout& c, int pos, int kvh, int i) {
  if (c.mega) {  // w elements of a 16-byte chunk
    const int w = 16 / kv_elem_bytes(c.elem);
    return (static_cast<size_t>(kvh) * (c.head_size / w) + i / w) * c.seq_len * w + static_cast<size_t>(pos) * w + i % w;
  }
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
