// The decode chain: n <= KLLM_MAX_VERIFY_TOKENS positions through every layer in ONE pass over the weights.  The graph
// engine's step (decoder.cu enqueue_step) is the chain at n = 1 between its embedding and its draw, and
// kllm_decoder_verify (speculative decoding, DESIGN.md 5.13) runs it at n positions.  Each launch computes every
// position with the arithmetic of a single one, so position start_pos + i yields the bits a step there yields on
// either engine in the exact numerics:
//
//   reference, per layer (15-18 launches)          here (6 launches for n positions)
//   rmsnorm, wq, wk, wv [+3 bias adds]        ->   gemv(norm -> q | k | v [+bias]), n vectors per weight pack
//   rope (pos read on the host)               ->   rope_scatter: q in place, k and v into the cache rows
//   mha                                       ->   mha over (heads, positions)
//   wo, add                                   ->   gemv(wo, + residual)
//   rmsnorm, w1, w3, swiglu                   ->   gemv(norm -> w1|w3 -> silu*gate)
//   w2, add                                   ->   gemv(w2, + residual)
//   final: rmsnorm, cls                       ->   gemv(norm -> cls)
//
// The verify pass wraps the chain in verify_embed_kernel (n rows; saves the history and record entries), one draw
// block per position and verify_accept_kernel.  A batch of decoders (kllm_batch, decoder.cu) runs it at n members,
// each row over its own member's cache at that member's position (ChainPos::members); the GEMVs are the same.
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

// The draw and record entry at position start_pos + blockIdx.x from that position's logits row, with its own step-0
// marks and penalised row so that the blocks run at once
__global__ void __launch_bounds__(1024)
verify_draw_kernel(const float* __restrict__ logits_rows, float* penalized_rows, int32_t* marks_rows, int n,
                   const DrawSettings* cfg, VerifyIo* io, const int32_t* hist, sampling::LogprobRecord rec) {
  const int i = blockIdx.x, pos = io->start_pos + i;
  PenaltyParams pen = cfg->penalty;
  pen.marks = marks_rows + static_cast<size_t>(i) * n;
  const int id = sampling::draw_and_record(logits_rows + static_cast<size_t>(i) * n, n, cfg, pen,
                                           penalized_rows + static_cast<size_t>(i) * n, hist, pos, true, nullptr, rec);
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

namespace {

kllm_gemv_seg seg(const Matrix& w, float* out, int rows) { return {w.w, w.scales, w.bias, out, rows}; }

// A GEMV of the model's matrices over x, RMS-normalised first with norm_w when it is set
kllm_gemv_job job(const DecoderModel& m, const float* x, int in_dim, int n_seg, const float* norm_w = nullptr) {
  kllm_gemv_job j{};
  j.x = x;
  j.norm_w = norm_w;
  j.norm_eps = m.eps;
  j.in_dim = in_dim;
  j.group_size = m.group_size;
  j.n_seg = n_seg;
  return j;
}

// x += w . in (feed_forward's adds, llama3.cpp:683-684, 719): in the GEMV's residual epilogue, or under tensor
// parallelism x += all-reduce(this rank's partial sums) (SURVEY.md 8e)
int residual_gemv(const DecoderModel& m, const Matrix& w, const float* in, int in_dim, float* x, const TpReduce* tp,
                  int n, cudaStream_t s) {
  kllm_gemv_job j = job(m, in, in_dim, 1);
  j.seg[0] = seg(w, tp ? tp->partial : x, m.dim);
  j.residual = tp ? nullptr : x;
  KLLM_TRY(gemv_dispatch(&j, m.format, s, n));
  if (tp == nullptr) return 0;
  const kllm_decoder_desc& d = *tp->desc;
  if (d.comm != nullptr) return kllm_comm_allreduce_residual(d.comm, tp->partial, x, x, d.dim, s);
  KLLM_TRY(d.allreduce(d.allreduce_ctx, tp->partial, d.dim, s));
  return kllm_add_f32(x, tp->partial, x, d.dim, s);
}

}  // namespace

int enqueue_classifier(const DecoderModel& m, const float* x, float* logits, int n, cudaStream_t s) {
  kllm_gemv_job j = job(m, x, m.dim, 1, m.final_norm);
  j.seg[0] = seg(m.cls, logits, m.vocab_size);
  return gemv_dispatch(&j, m.format, s, n);
}

int enqueue_layers(const DecoderModel& m, const DecoderCache& c, const ChainRows& r, int n, ChainPos at,
                   const TpReduce* tp, cudaStream_t s) {
  const int dim = m.dim, hid = m.hidden_dim, q_rows = m.q_rows, kvd = m.kv_dim;  // q_rows == dim unless tensor-parallel
  for (int l = 0; l < m.layer_num; ++l) {
    const LayerWeights& lw = m.layers[l];
    // attention_rms + attention_qkv (llama3.cpp:600-640)
    {
      kllm_gemv_job j = job(m, r.x, dim, 3, lw.attn_norm);
      j.seg[0] = seg(lw.q, r.q, q_rows);
      j.seg[1] = seg(lw.k, r.k, kvd);
      j.seg[2] = seg(lw.v, r.v, kvd);
      KLLM_TRY(gemv_dispatch(&j, m.format, s, n));
    }
    KLLM_TRY(launch_rope_scatter_f32(m, c, l, r.q, r.k, r.v, at, n, s));
    // attention_mha (llama3.cpp:652-676)
    KLLM_TRY(launch_mha_rows(at, n, c.cache, m.head_num, l, m.kv_mul, r.att, r.q, r.score, c.key_cache,
                             c.value_cache, s));
    KLLM_TRY(residual_gemv(m, lw.o, r.att, q_rows, r.x, tp, n, s));
    // feed_forward (llama3.cpp:686-720)
    {
      kllm_gemv_job j = job(m, r.x, dim, 2, lw.ffn_norm);
      j.seg[0] = seg(lw.w1, r.h, hid);
      j.seg[1] = seg(lw.w3, nullptr, hid);
      j.swiglu_pair = 1;
      KLLM_TRY(gemv_dispatch(&j, m.format, s, n));
    }
    KLLM_TRY(residual_gemv(m, lw.w2, r.h, hid, r.x, tp, n, s));
  }
  // cls_logits (llama3.cpp:722-731)
  return enqueue_classifier(m, r.x, r.logits, n, s);
}

int enqueue_verify(const DecoderModel& m, const DecoderCache& c, const VerifyTarget& t, const VerifyWorkspace& ws,
                   int n, cudaStream_t s) {
  verify_embed_kernel<<<n, 256, 0, s>>>(ws.io, m.tok_emb, ws.rows.x, m.dim, t.hist, t.rec, ws.saved_hist, ws.saved);
  count_launch();
  KLLM_TRY(cudaGetLastError());
  KLLM_TRY(enqueue_layers(m, c, ws.rows, n, ChainPos{PosArg{&ws.io->start_pos, 0}, nullptr}, nullptr, s));
  verify_draw_kernel<<<n, 1024, 0, s>>>(ws.rows.logits, ws.penalized, ws.marks, m.vocab_size, t.cfg, ws.io, t.hist,
                                        t.rec);
  count_launch();
  KLLM_TRY(cudaGetLastError());
  verify_accept_kernel<<<1, 1024, 0, s>>>(ws.io, n, ws.rows.logits, t.logits, m.vocab_size, t.state, t.hist, t.rec,
                                          ws.saved_hist, ws.saved);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace kllm
