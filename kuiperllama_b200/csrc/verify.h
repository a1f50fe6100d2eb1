// kllm_decoder_verify's chain (verify.cu): a block of up to KLLM_MAX_VERIFY_TOKENS positions through every layer in one
// pass over the weights, each position's arithmetic that of the graph engine's step (decoder.cu enqueue_step).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/kllm_b200.h"
#include "kllm_host.h"
#include "megakernel.h"
#include "sampling.cuh"

namespace kllm {

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
  float *x, *q, *k, *v, *att, *h, *logits, *penalized, *score;
  int32_t* marks;  // step 0's mark words, one row per position, zero between calls
  int32_t* saved_hist;
  sampling::LogprobRecord saved;  // indexed by the position's offset in the block
  VerifyIo* io;
};

// What the chain reads and writes of the decoder
struct VerifyTarget {
  prefill::CacheLayout cache;
  float *key_cache, *value_cache;
  const float *sin_cache, *cos_cache;
  const DrawSettings* cfg;
  mega::State* state;  // left as kllm_decoder_generate of a + 1 steps leaves it
  int32_t* hist;
  sampling::LogprobRecord rec;
  float* logits;  // receives row a
};

// Enqueues the chain for n positions; every position is read from ws.io
int enqueue_verify(const DecoderModel& m, const VerifyTarget& t, const VerifyWorkspace& ws, int n, cudaStream_t s);

}  // namespace kllm
