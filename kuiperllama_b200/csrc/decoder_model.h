// The decoder's model as its three consumers read it -- the graph engine (decoder.cu), the persistent engine
// (megakernel.cu) and the batched prefill (prefill.cu): the shape, one weight format for every matrix, and each
// matrix with its scales and bias.  build_decoder_model is the one place a kllm_decoder_desc becomes a format.
// Only .cu files include it: the format and its element size are also the kernels' template parameter.
#pragma once
#include <cstddef>
#include <vector>

#include "../../include/kllm_b200.h"

namespace kllm {

enum class WeightFormat { kF32, kInt8, kBf16 };

constexpr __host__ __device__ int weight_bytes(WeightFormat f) {
  return f == WeightFormat::kInt8 ? 1 : f == WeightFormat::kBf16 ? 2 : 4;
}

// log2(group_size) for a power of two, else -1 (the kernels then divide)
inline int group_shift_of(int group_size) {
  if (group_size <= 0 || (group_size & (group_size - 1)) != 0) return -1;
  int s = 0;
  while ((1 << s) < group_size) ++s;
  return s;
}

// A weight matrix [rows, in_dim], row-major, in the model's format.
struct Matrix {
  const void* w;
  const float* scales;  // kInt8 only: the fp32 scale of each group_size weights
  const float* bias;    // Qwen2 q / k / v only: [rows], added after the dot product
};

struct LayerWeights {
  const float *attn_norm, *ffn_norm;
  Matrix q, k, v, o, w1, w2, w3;
};

// All pointers are device pointers.  Under tensor parallelism the counts are this rank's (kllm_decoder_desc), dim
// the full model's.
struct DecoderModel {
  int dim, hidden_dim, layer_num, head_num, kv_head_num, vocab_size, seq_len;
  int head_size, kv_dim, kv_mul, q_rows, flavour;
  float eps;
  WeightFormat format;
  int group_size, group_shift;  // kInt8: the scales' group and its log2 (-1: not a power of two); else 0, -1
  const float* tok_emb;
  const float* final_norm;
  Matrix cls;
  std::vector<LayerWeights> layers;

  // rows row0.. of `m`, a matrix of in_dim columns
  Matrix rows_from(const Matrix& m, size_t row0, int in_dim) const {
    return {static_cast<const unsigned char*>(m.w) + row0 * in_dim * weight_bytes(format),
            m.scales == nullptr ? nullptr : m.scales + row0 * (in_dim / group_size),
            m.bias == nullptr ? nullptr : m.bias + row0};
  }
};

// The model `desc` describes, or the KLLM_E_* code of its first broken rule (kllm_decoder_create's order).
int build_decoder_model(const kllm_decoder_desc& desc, DecoderModel* out);

}  // namespace kllm
