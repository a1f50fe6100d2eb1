// kllm_decoder_verify: n <= KLLM_MAX_VERIFY_TOKENS positions through every layer in ONE pass over the weights, for
// speculative decoding (DESIGN.md 5.13).  Each position's arithmetic is the graph engine's step operation for
// operation (decoder.cu enqueue_step), so position start_pos + i yields the bits a step there yields on either engine
// in the exact numerics:
//
//   step (per position)                          here (per block of n positions)
//   embed_token_kernel                      ->   verify_embed_kernel: n rows; saves the history and record entries
//   gemv_fused(norm -> q | k@cache | v@cache) ->  gemv_multi(norm -> q | k | v), n vectors per weight pack
//   rope (in place in the cache row)         ->   rope_scatter: the same rotation, written through CacheLayout
//   mha                                      ->   mha over (heads, positions), the same kernel and order
//   gemv_fused(wo, + residual)               ->   gemv_multi(wo, + residual)
//   gemv_fused(norm -> w1|w3 -> silu*gate)   ->   gemv_multi(norm -> w1|w3 -> silu*gate)
//   gemv_fused(w2, + residual)               ->   gemv_multi(w2, + residual)
//   gemv_fused(norm -> cls), argmax+advance  ->   gemv_multi(norm -> cls), one draw block per position, accept
#include <cuda_runtime.h>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"
#include "verify.h"

namespace kllm {

// Block i: saves the history and record entries of position start_pos + i, records tokens[i] as the id fed there
// (the draws read the history as fed) and gathers its embedding row.  kllm_decoder_verify checked every token.
__global__ void verify_embed_kernel(VerifyIo* io, const float* __restrict__ table, float* x, int dim, int32_t* hist,
                                    sampling::LogprobRecord rec, int32_t* saved_hist, sampling::LogprobRecord saved) {
  const int i = blockIdx.x, pos = io->start_pos + i, token = io->tokens[i];
  constexpr int T = sampling::kMaxTopLogprobs;
  if (threadIdx.x == 0) {
    saved_hist[i] = hist[pos];
    hist[pos] = token;
    saved.id[i] = rec.id[pos];
    saved.lp[i] = rec.lp[pos];
  }
  if (threadIdx.x < T) {
    saved.top_ids[i * T + threadIdx.x] = rec.top_ids[static_cast<size_t>(pos) * T + threadIdx.x];
    saved.top_lp[i * T + threadIdx.x] = rec.top_lp[static_cast<size_t>(pos) * T + threadIdx.x];
  }
  const float4* s4 = reinterpret_cast<const float4*>(table + static_cast<size_t>(token) * dim);
  float4* d4 = reinterpret_cast<float4*>(x + static_cast<size_t>(i) * dim);
  for (int e = threadIdx.x; e < (dim >> 2); e += blockDim.x) d4[e] = s4[e];
}

// argmax_advance_kernel's draw and record entry at position start_pos + blockIdx.x, from that position's logits row,
// with its own step-0 marks and penalised row so that the blocks run at once
constexpr int kDrawScratchBytes = sampling::kDrawScratchBase + 2048 * 8;
static_assert(kDrawScratchBytes >= sampling::logprob_scratch_bytes(1024), "one scratch for the draw and the logprobs");

__global__ void __launch_bounds__(1024)
verify_draw_kernel(const float* __restrict__ logits_rows, float* penalized_rows, int32_t* marks_rows, int n,
                   const DrawSettings* cfg, VerifyIo* io, const int32_t* hist, sampling::LogprobRecord rec) {
  __shared__ __align__(16) unsigned char scratch[kDrawScratchBytes];
  const int i = blockIdx.x, pos = io->start_pos + i;
  const float* logits = logits_rows + static_cast<size_t>(i) * n;
  const float* l = logits;
  PenaltyParams pen = cfg->penalty;
  pen.marks = marks_rows + static_cast<size_t>(i) * n;
  if (sampling::step0_active(pen)) {
    float* penalized = penalized_rows + static_cast<size_t>(i) * n;
    sampling::step0_history<1024>(logits, penalized, 0, n, pen, hist, pos, [] { __syncthreads(); });
    l = penalized;
  }
  const int bi = sampling::draw_block<1024>(l, n, cfg->sample, pos, nullptr, nullptr, 0, scratch, kDrawScratchBytes,
                                            [] { __syncthreads(); });
  const int id = bi < 0 ? 0 : bi;
  const int top_n = cfg->lp_top_n;
  if (top_n >= 0) {
    sampling::logprobs_block<1024>(logits, n, top_n, scratch, kDrawScratchBytes, [] { __syncthreads(); });
    const size_t row = static_cast<size_t>(pos) * sampling::kMaxTopLogprobs;
    sampling::write_entry(logits, n, id, top_n, *reinterpret_cast<const sampling::LogprobScratch*>(scratch),
                          rec.id + pos, rec.lp + pos, rec.top_ids + row, rec.top_lp + row);
  }
  if (threadIdx.x == 0) io->ids[i] = id;
}

// a = the number of leading drafts equal to the id drawn before them, up to the first stop id; then the history and
// record entries of the rejected positions are put back, row a's logits become the decoder's, and the state is
// what kllm_decoder_generate of a + 1 steps leaves.
__global__ void verify_accept_kernel(VerifyIo* io, int n, const float* __restrict__ logits_rows, float* logits, int vocab,
                                     mega::State* st, int32_t* hist, sampling::LogprobRecord rec,
                                     const int32_t* saved_hist, sampling::LogprobRecord saved) {
  __shared__ int s_a;
  constexpr int T = sampling::kMaxTopLogprobs;
  if (threadIdx.x == 0) {
    int a = 0;
    for (; a + 1 < n && io->tokens[a + 1] == io->ids[a]; ++a) {
      bool stop = false;
      for (int j = 0; j < io->n_stop; ++j) stop |= io->stop[j] == io->ids[a];
      if (stop) break;
    }
    s_a = a;
    io->accepted = a;
    const int p = io->start_pos, id = io->ids[a];
    st->next = id;
    st->token = id;
    st->pos = p + a + 1;
    st->step = a + 1;
  }
  __syncthreads();
  const int a = s_a, p = io->start_pos;
  for (int i = a + 1; i < n; ++i) {
    const int pos = p + i;
    if (threadIdx.x == 0) {
      hist[pos] = saved_hist[i];
      rec.id[pos] = saved.id[i];
      rec.lp[pos] = saved.lp[i];
    }
    if (threadIdx.x < T) {
      rec.top_ids[static_cast<size_t>(pos) * T + threadIdx.x] = saved.top_ids[i * T + threadIdx.x];
      rec.top_lp[static_cast<size_t>(pos) * T + threadIdx.x] = saved.top_lp[i * T + threadIdx.x];
    }
  }
  const float* row = logits_rows + static_cast<size_t>(a) * vocab;
  for (int e = threadIdx.x; e < vocab; e += blockDim.x) logits[e] = row[e];
}

#define VF_TRY(expr)                        \
  do {                                      \
    const int rc_ = static_cast<int>(expr); \
    if (rc_ != 0) return rc_;               \
  } while (0)

int enqueue_verify(const DecoderModel& m, const VerifyTarget& t, const VerifyWorkspace& ws, int n, cudaStream_t s) {
  const int dim = m.dim, hid = m.hidden_dim, q_rows = m.q_rows, kvd = m.kv_dim;
  const PosArg first{&ws.io->start_pos, 0};
  GemvExtra wx;
  wx.format = m.format;
  auto job = [&](const float* x, int in_dim, int n_seg, const float* norm_w) {
    kllm_gemv_job j{};
    j.x = x;
    j.norm_w = norm_w;
    j.norm_eps = m.eps;
    j.in_dim = in_dim;
    j.group_size = m.group_size;
    j.n_seg = n_seg;
    return j;
  };
  auto seg = [](const Matrix& w, float* out, int rows) { return kllm_gemv_seg{w.w, w.scales, w.bias, out, rows}; };

  verify_embed_kernel<<<n, 256, 0, s>>>(ws.io, m.tok_emb, ws.x, dim, t.hist, t.rec, ws.saved_hist, ws.saved);
  count_launch();
  VF_TRY(cudaGetLastError());
  for (int l = 0; l < m.layer_num; ++l) {
    const LayerWeights& lw = m.layers[l];
    {
      kllm_gemv_job j = job(ws.x, dim, 3, lw.attn_norm);
      j.seg[0] = seg(lw.q, ws.q, q_rows);
      j.seg[1] = seg(lw.k, ws.k, kvd);
      j.seg[2] = seg(lw.v, ws.v, kvd);
      VF_TRY(gemv_dispatch(&j, wx, s, n));
    }
    VF_TRY(launch_rope_scatter_f32(m, t.cache, l, ws.q, ws.k, ws.v, t.sin_cache, t.cos_cache, t.key_cache,
                                   t.value_cache, first, n, s));
    VF_TRY(launch_mha_rows(first, n, t.cache, m.head_num, l, m.kv_mul, ws.att, ws.q, ws.score, t.key_cache,
                           t.value_cache, s));
    {
      kllm_gemv_job j = job(ws.att, q_rows, 1, nullptr);
      j.seg[0] = seg(lw.o, ws.x, dim);
      j.residual = ws.x;
      VF_TRY(gemv_dispatch(&j, wx, s, n));
    }
    {
      kllm_gemv_job j = job(ws.x, dim, 2, lw.ffn_norm);
      j.seg[0] = seg(lw.w1, ws.h, hid);
      j.seg[1] = seg(lw.w3, nullptr, hid);
      j.swiglu_pair = 1;
      VF_TRY(gemv_dispatch(&j, wx, s, n));
    }
    {
      kllm_gemv_job j = job(ws.h, hid, 1, nullptr);
      j.seg[0] = seg(lw.w2, ws.x, dim);
      j.residual = ws.x;
      VF_TRY(gemv_dispatch(&j, wx, s, n));
    }
  }
  {
    kllm_gemv_job j = job(ws.x, dim, 1, m.final_norm);
    j.seg[0] = seg(m.cls, ws.logits, m.vocab_size);
    VF_TRY(gemv_dispatch(&j, wx, s, n));
  }
  verify_draw_kernel<<<n, 1024, 0, s>>>(ws.logits, ws.penalized, ws.marks, m.vocab_size, t.cfg, ws.io, t.hist, t.rec);
  count_launch();
  VF_TRY(cudaGetLastError());
  verify_accept_kernel<<<1, 1024, 0, s>>>(ws.io, n, ws.logits, t.logits, m.vocab_size, t.state, t.hist, t.rec,
                                          ws.saved_hist, ws.saved);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace kllm
