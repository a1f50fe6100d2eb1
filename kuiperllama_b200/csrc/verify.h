// The decode chain (verify.cu): n <= KLLM_MAX_VERIFY_TOKENS positions through every layer and the classifier in one
// pass over the weights.  The graph engine's step is the chain at n = 1; kllm_decoder_verify runs it at n positions.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/kllm_b200.h"
#include "kllm_host.h"
#include "megakernel.h"
#include "sampling.cuh"

namespace kllm {

// The chain's per-position rows, [n][.] each: x [dim] (the embeddings in, the residual stream), q and att
// [q_rows], k and v [kv_dim], h [hidden_dim], score [head_num][seq_len], logits [vocab_size]
struct ChainRows {
  float *x, *q, *k, *v, *att, *h, *score, *logits;
};

// Tensor parallelism (n = 1): the row-parallel matmuls Wo and W2 write this rank's partial sums to `partial` [dim],
// and x += their all-reduce over the description's transport
struct TpReduce {
  const kllm_decoder_desc* desc;
  float* partial;
};

// Enqueues, for the n rows at `at` (the positions at.first, at.first + 1, .. of the cache c, or a batch's members,
// each at its own position in its own cache), every layer (q|k|v GEMV, RoPE with the k and v rows written into the
// cache, attention, Wo with residual, W1|W3 SwiGLU, W2 with residual) and then the final-norm classifier.  With
// at.members, c gives the layout and the RoPE tables only.  tp: null on one GPU.
int enqueue_layers(const DecoderModel& m, const DecoderCache& c, const ChainRows& rows, int n, ChainPos at,
                   const TpReduce* tp, cudaStream_t s);

// The final RMSNorm and classifier of n rows x [n][dim] into logits [n][vocab_size]: the chain's last step
int enqueue_classifier(const DecoderModel& m, const float* x, float* logits, int n, cudaStream_t s);

// The call's arguments and result in device memory, so that one captured chain per block length serves every
// position: the host uploads the first part and reads `ids` and `accepted` back.
struct VerifyIo {
  int32_t tokens[KLLM_MAX_VERIFY_TOKENS];  // tokens[0] fed at start_pos, tokens[i] the draft for start_pos + i
  int32_t start_pos;
  int32_t n_stop;  // an id in stop[0 .. n_stop) ends the acceptance at its position
  int32_t stop[KLLM_MAX_STOP_IDS];
  int32_t ids[KLLM_MAX_VERIFY_TOKENS];  // id_i drawn at start_pos + i
  int32_t accepted;                     // a: id_0 .. id_a stand
};

// Per-position scratch [KLLM_MAX_VERIFY_TOKENS][.] and the saved history and record entries of the block
struct VerifyWorkspace {
  ChainRows rows;
  float* penalized;
  int32_t* marks;  // step 0's mark words, one row per position, zero between calls
  int32_t* saved_hist;
  sampling::LogprobRecord saved;  // indexed by the position's offset in the block
  VerifyIo* io;
};

// What the verify pass reads and writes of the decoder besides its cache
struct VerifyTarget {
  const DrawSettings* cfg;
  mega::State* state;  // left as kllm_decoder_generate of a + 1 steps leaves it
  int32_t* hist;
  sampling::LogprobRecord rec;
  float* logits;  // receives row a
};

// Enqueues the verify pass of n positions: the embeddings, the chain, a draw per position and the acceptance; every
// position is read from ws.io
int enqueue_verify(const DecoderModel& m, const DecoderCache& c, const VerifyTarget& t, const VerifyWorkspace& ws,
                   int n, cudaStream_t s);

}  // namespace kllm
