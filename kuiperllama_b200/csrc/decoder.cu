// Device-resident single-batch decoder: the per-token forward of LLama2Model / Qwen2Model
// (kuiper/source/model/llama3.cpp:147-167, 600-745; qwen2.cpp) on either engine.  The graph engine's step is a
// fixed chain of fused launches captured ONCE in a CUDA graph and replayed for every position:
//
//   embed_token_kernel -> the decode chain at one position (verify.cu enqueue_layers: 6 launches per layer and the
//   final-norm classifier) -> argmax_advance_kernel
//
// The position, the current token and the step counter live in device memory, so the
// captured graph is position independent and a whole greedy run needs no host round trip
// (reference: 2 blocking copies + 1 cudaMalloc per token, emb_kernel.cu:25-29,
// argmax_kernel.cu:73-87).  Buffer roles follow llama3.cpp:425-500.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <utility>
#include <vector>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"
#include "megakernel.h"
#include "sampling.cuh"
#include "verify.h"

namespace kllm {

constexpr int kStreamIds = 32;  // int32 offset of the streamed ids behind the count (kllm_decoder::stream_host)
static_assert(mega::kMaxStopIds == KLLM_MAX_STOP_IDS, "one stop-set capacity");

// Also records the fed id in the history (sampling.cuh step 0), -1 for an id outside the vocabulary.  Block b of nb
// copies its share of the embedding row into x.
__device__ __forceinline__ void embed_token(const mega::State* st, const float* __restrict__ table, float* x, int dim,
                                            int vocab, int32_t* hist, int b, int nb) {
  const int32_t token = st->token;
  const bool valid = token >= 0 && token < vocab;
  if (b == 0 && threadIdx.x == 0) hist[st->pos] = valid ? token : -1;
  if (!valid) return;
  const float4* s4 = reinterpret_cast<const float4*>(table + static_cast<size_t>(token) * dim);
  float4* d4 = reinterpret_cast<float4*>(x);
  for (int i = b * blockDim.x + threadIdx.x; i < (dim >> 2); i += nb * blockDim.x)
    d4[i] = s4[i];
}

__global__ void embed_token_kernel(const mega::State* st, const float* __restrict__ table,
                                   float* x, int dim, int vocab, int32_t* hist) {
  embed_token(st, table, x, dim, vocab, hist, blockIdx.x, gridDim.x);
}

// The id of the step (greedy, argmax_kernel.cu:49-71 semantics, or drawn by the sampling rule of
// sampling.cuh under the decoder's settings `cfg`) fused with the loop bookkeeping: record the id, feed it (or,
// with the state's `teacher` switch, the teacher's id) to the next step, pos += 1.  The settings and the entry's
// mode are read from device memory, so one captured graph serves every entry and setting.
// With the state's `streamed` switch (kllm_decoder_generate_until) the id is also published to mapped host memory:
// the id, then the count with release semantics at system scope, which the host polls.
// The draw and record entry (sampling.cuh draw_and_record, DESIGN.md 5.8): with logprobs on, from the state's step
// `lp_from` on, the entry of the drawn id, or of teacher[step + 1] in `lp_target` mode.
// One block of 1024 threads: argmax_advance_kernel, and each member's block of a batch's draw.
__device__ __forceinline__ void draw_advance(const float* __restrict__ logits, int n, const DrawSettings* cfg,
                                             mega::State* st, int32_t* out_tokens, const int32_t* teacher,
                                             int max_steps, int32_t* stream_ids, int32_t* stream_count,
                                             const int32_t* hist, float* penalized, sampling::LogprobRecord rec) {
  const int step0 = st->step;  // read by every thread before thread 0 advances the state
  const int next = sampling::draw_and_record(logits, n, cfg, cfg->penalty, penalized, hist, st->pos,
                                             step0 >= st->lp_from, st->lp_target ? teacher + step0 + 1 : nullptr, rec);
  if (threadIdx.x == 0) {
    const int step = st->step;
    st->next = next;
    if (out_tokens != nullptr && step < max_steps) out_tokens[step] = next;
    if (st->streamed) {
      stream_ids[step] = next;
      asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(stream_count), "r"(step + 1) : "memory");
    }
    st->token = (st->teacher && step + 1 < max_steps) ? teacher[step + 1] : next;
    st->pos = st->pos + 1;
    st->step = step + 1;
  }
}

__global__ void __launch_bounds__(1024)
argmax_advance_kernel(const float* __restrict__ logits, int n, const DrawSettings* cfg, mega::State* st,
                      int32_t* out_tokens, const int32_t* teacher, int max_steps, int32_t* stream_ids,
                      int32_t* stream_count, const int32_t* hist, float* penalized, sampling::LogprobRecord rec) {
  draw_advance(logits, n, cfg, st, out_tokens, teacher, max_steps, stream_ids, stream_count, hist, penalized, rec);
}

// What a batch's embedding and draw read and write of one member: the arguments of argmax_advance_kernel in the
// member's own step.  The streamed ids go to the member's own mapped area, as in its own kllm_decoder_generate_until.
struct BatchTarget {
  mega::State* st;
  const DrawSettings* cfg;
  int32_t* hist;
  float* penalized;
  sampling::LogprobRecord rec;
  int32_t* out_tokens;
  const int32_t* teacher;
  float* logits;  // receives the member's row of the batch's logits
  int32_t* stream_ids;
  int32_t* stream_count;
};

// grid (4, members): member blockIdx.y's embedding into row blockIdx.y, as embed_token_kernel's 4 blocks do it
__global__ void batch_embed_kernel(const BatchTarget* __restrict__ members, const float* __restrict__ table, float* x,
                                   int dim, int vocab) {
  const BatchTarget& mb = members[blockIdx.y];
  embed_token(mb.st, table, x + static_cast<size_t>(blockIdx.y) * dim, dim, vocab, mb.hist, blockIdx.x, gridDim.x);
}

// Block b: member b's step draw over row b of the batch's logits, then the row becomes the member's logits
__global__ void __launch_bounds__(1024)
batch_draw_kernel(const float* __restrict__ logits_rows, int n, const BatchTarget* __restrict__ members,
                  int max_steps) {
  const BatchTarget& mb = members[blockIdx.x];
  const float* row = logits_rows + static_cast<size_t>(blockIdx.x) * n;
  draw_advance(row, n, mb.cfg, mb.st, mb.out_tokens, mb.teacher, max_steps, mb.stream_ids, mb.stream_count, mb.hist,
               mb.penalized, mb.rec);
  for (int e = threadIdx.x; e < n; e += blockDim.x) mb.logits[e] = row[e];
}

// The K and V rows of position pos in one layer of a cache, element by element through the layout's own index, so
// any layout and element (T of its size: fp32, bf16 or fp8 codes) is copied as stored.  The block's threads share it.
template <typename T>
__device__ __forceinline__ void copy_kv_position(const T* __restrict__ ks, const T* __restrict__ vs, T* __restrict__ kd,
                                                 T* __restrict__ vd, const prefill::CacheLayout& c, int pos,
                                                 int layer_index) {
  const size_t layer = static_cast<size_t>(layer_index) * c.seq_len * c.kv_dim;
  for (int p = threadIdx.x; p < c.kv_dim; p += blockDim.x) {
    const int kvh = p / c.head_size, i = p % c.head_size;
    const size_t ki = layer + prefill::k_index(c, pos, kvh, i), vi = layer + prefill::v_index(c, pos, kvh, i);
    kd[ki] = ks[ki];
    vd[vi] = vs[vi];
  }
}

// One prefix of a cache: positions [0, gridDim.x) of every layer (blockIdx.y)
template <typename T>
__global__ void copy_prefix_kernel(const T* __restrict__ ks, const T* __restrict__ vs, T* __restrict__ kd,
                                   T* __restrict__ vd, prefill::CacheLayout c) {
  copy_kv_position(ks, vs, kd, vd, c, blockIdx.x, blockIdx.y);
}

// The (source, destination) caches of a beam-search pass's forks (kllm_batch_beam_search): fork f copies member
// src's rows into member dst's.  A batch's caches are fp32.
struct ForkTable {
  const float* ks[KLLM_MAX_BATCH];
  const float* vs[KLLM_MAX_BATCH];
  float* kd[KLLM_MAX_BATCH];
  float* vd[KLLM_MAX_BATCH];
};

// Every fork of a pass in one launch: grid (positions [lo, lo + gridDim.x), layers, forks).  Sources are surviving
// beams' members and destinations dropped ones', so no block reads what another writes.
__global__ void fork_rows_kernel(const __grid_constant__ ForkTable t, int lo, prefill::CacheLayout c) {
  const int f = blockIdx.z;
  copy_kv_position(t.ks[f], t.vs[f], t.kd[f], t.vd[f], c, lo + static_cast<int>(blockIdx.x), blockIdx.y);
}

// The ids a beam-search pass reads back per row: the top kBeamTop of the logprob rule and their lp, in the rule's
// order (logit descending, lowest id on ties).  B + KLLM_MAX_BEAM_EOS serves every eos count with one captured pass:
// a top-N selection is exact, so its first B + n_eos entries are those of top_n = B + n_eos.
constexpr int kBeamTop = KLLM_MAX_BATCH + KLLM_MAX_BEAM_EOS;
static_assert(kBeamTop <= sampling::kMaxTopLogprobs, "the logprob rule's top-N holds a pass's candidates");
struct BeamCandidates {
  int32_t ids[KLLM_MAX_BATCH][kBeamTop];
  float lp[KLLM_MAX_BATCH][kBeamTop];
};

// Block r: rule L1-L3 over row r of the batch's logits (one block, kllm_logprobs_f32's partition), its top top_n ids
// and their lp into row r of `out` (mapped host memory)
__global__ void __launch_bounds__(1024)
beam_candidates_kernel(const float* __restrict__ logits_rows, int n, int top_n, BeamCandidates* out) {
  constexpr int kScratch = sampling::logprob_scratch_bytes(1024);
  __shared__ __align__(16) unsigned char scratch[kScratch];
  const int r = blockIdx.x;
  sampling::logprobs_block<1024>(logits_rows + static_cast<size_t>(r) * n, n, top_n, scratch, kScratch,
                                 [] { __syncthreads(); });
  const sampling::LogprobScratch& ls = *reinterpret_cast<const sampling::LogprobScratch*>(scratch);
  if (static_cast<int>(threadIdx.x) < top_n) {
    const int i = ls.top_i[threadIdx.x];
    out->ids[r][threadIdx.x] = i;
    out->lp[r][threadIdx.x] = i < 0 ? -INFINITY : sampling::logprob(ls.top_v[threadIdx.x], ls.m, ls.lse_off);
  }
}

// value(code) of an e4m3 code (sign, 4 exponent bits of bias 7, 3 mantissa bits; no infinities, S.1111.111 is NaN)
float e4m3_value_host(uint8_t code) {
  const int e = (code >> 3) & 15, f = code & 7;
  float v;
  if (e == 15 && f == 7)
    v = NAN;
  else if (e == 0)
    v = std::ldexp(static_cast<float>(f), -9);  // subnormal: f / 8 * 2^-6
  else
    v = std::ldexp(static_cast<float>(8 + f), e - 10);
  return (code & 0x80) ? -v : v;
}

int build_decoder_model(const kllm_decoder_desc& d, DecoderModel* out) {
  if (d.dim <= 0 || d.hidden_dim <= 0 || d.layer_num <= 0 || d.head_num <= 0 ||
      d.kv_head_num <= 0 || d.vocab_size <= 0 || d.seq_len <= 0)
    return KLLM_E_INVALID;
  if (!d.tok_emb || !d.attn_norm || !d.ffn_norm || !d.final_norm || !d.wq || !d.wk || !d.wv ||
      !d.wo || !d.w1 || !d.w2 || !d.w3 || !d.wcls)
    return KLLM_E_INVALID;
  const bool int8 = d.group_size > 0;
  if (int8 && (!d.sq || !d.sk || !d.sv || !d.so || !d.s1 || !d.s2 || !d.s3 || !d.scls)) return KLLM_E_INVALID;
  const int tp = d.tp_size > 1 ? d.tp_size : 1;
  if (tp > 1 && d.allreduce == nullptr && d.comm == nullptr) return KLLM_E_INVALID;
  // head_size from the FULL model: dim / (head_num * tp)
  if (d.dim % (d.head_num * tp) != 0 || d.head_num % d.kv_head_num != 0) return KLLM_E_INVALID;
  if ((d.dim & 3) != 0 || (d.hidden_dim & 3) != 0) return KLLM_E_UNSUPPORTED;
  if (d.kv_cache != KLLM_KV_F32 && d.kv_cache != KLLM_KV_BF16 && d.kv_cache != KLLM_KV_FP8) return KLLM_E_INVALID;
  // the fp8 cache's scales: given for that cache and only for it, each finite and > 0.  A description with kv_cache 2
  // and no scales -- one written before the fp8 cache existed -- stays refused as it was.
  if ((d.kv_cache == KLLM_KV_FP8) != (d.kv_scales != nullptr)) return KLLM_E_INVALID;
  if (d.kv_scales != nullptr) {
    for (size_t i = 0; i < 2 * static_cast<size_t>(d.layer_num) * d.kv_head_num; ++i)
      if (!std::isfinite(d.kv_scales[i]) || !(d.kv_scales[i] > 0.f)) return KLLM_E_INVALID;
  }
  // bf16 weights: fp32 checkpoints' matrices rounded by the caller; one GPU
  if (d.weights != KLLM_WEIGHTS_F32 && d.weights != KLLM_WEIGHTS_BF16) return KLLM_E_INVALID;
  const bool w16 = d.weights == KLLM_WEIGHTS_BF16;
  if (w16 && int8) return KLLM_E_INVALID;
  if (w16 && tp > 1) return KLLM_E_UNSUPPORTED;

  DecoderModel& m = *out;
  m.dim = d.dim, m.hidden_dim = d.hidden_dim, m.layer_num = d.layer_num, m.head_num = d.head_num;
  m.kv_head_num = d.kv_head_num, m.vocab_size = d.vocab_size, m.seq_len = d.seq_len;
  m.head_size = d.dim / (d.head_num * tp);
  m.kv_dim = d.kv_head_num * m.head_size;
  m.kv_mul = d.head_num / d.kv_head_num;
  m.q_rows = d.head_num * m.head_size;
  m.flavour = d.flavour;
  m.eps = flavour_eps(d.flavour);
  m.format = int8 ? WeightFormat::kInt8 : w16 ? WeightFormat::kBf16 : WeightFormat::kF32;
  m.group_size = d.group_size;
  m.group_shift = group_shift_of(d.group_size);
  m.tok_emb = d.tok_emb;
  m.final_norm = d.final_norm;
  m.cls = {d.wcls, nullptr, nullptr};
  if (int8) m.cls.scales = d.scls;
  m.layers.resize(d.layer_num);
  for (int l = 0; l < d.layer_num; ++l) {
    LayerWeights& lw = m.layers[l];
    lw = {d.attn_norm[l], d.ffn_norm[l], {d.wq[l]}, {d.wk[l]}, {d.wv[l]}, {d.wo[l]}, {d.w1[l]}, {d.w2[l]}, {d.w3[l]}};
    if (int8) {  // an fp32 or bf16 model's scale arrays are not read
      lw.q.scales = d.sq[l], lw.k.scales = d.sk[l], lw.v.scales = d.sv[l], lw.o.scales = d.so[l];
      lw.w1.scales = d.s1[l], lw.w2.scales = d.s2[l], lw.w3.scales = d.s3[l];
    }
    if (d.bq) lw.q.bias = d.bq[l];
    if (d.bk) lw.k.bias = d.bk[l];
    if (d.bv) lw.v.bias = d.bv[l];
  }
  return 0;
}

}  // namespace kllm

using namespace kllm;

struct kllm_decoder {
  kllm_decoder_desc d{};  // the caller's description (tp_size >= 1): its transport and cache settings
  DecoderModel m;         // the model it describes
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // device buffers
  float *x = nullptr, *q = nullptr, *k = nullptr, *v = nullptr, *attn = nullptr, *h = nullptr, *logits = nullptr;
  float *score = nullptr, *kcache = nullptr, *vcache = nullptr, *sin_t = nullptr, *cos_t = nullptr;
  float* tp_tmp = nullptr;
  // the fp8 KV cache's scales (KLLM_KV_FP8): [2][L][kv_head] s_k, s_v on the host (kllm_decoder_read_kv), and on the
  // device [4][L][kv_head] s_k, s_v, 1 / s_k, 1 / s_v
  std::vector<float> kv_scales;
  float* kv_scales_dev = nullptr;
  MegaEngine mega;
  bool use_mega = false;
  mega::State* st = nullptr;
  DrawSettings cfg{};                // the settings in force (put_settings)
  DrawSettings* d_cfg = nullptr;     // device: their copy, which both engines read
  int32_t* hist = nullptr;           // device [seq_len]: the id fed at each position, -1 for none
  float* penalized = nullptr;        // device [vocab]: the penalised logits of the last draw
  float* bias = nullptr;             // device [vocab]: the dense logit bias table (kllm_decoder_set_logit_bias)
  int32_t* marks = nullptr;          // device [vocab]: step 0's mark words, zero between tokens
  int32_t* out_tokens = nullptr;  // device [seq_len]
  int32_t* teacher = nullptr;     // device [seq_len]
  mega::State* st_host = nullptr;  // pinned: the state of an entry's first position (put_state), then its last
  sampling::LogprobRecord rec{};   // log-probabilities (kllm_decoder_set_logprobs), indexed by position
  int32_t* io_host = nullptr;     // pinned scratch
  cudaGraphExec_t exec = nullptr;  // the graph engine's captured step, in the mode of the uploaded state
  int launches_per_step = 0;
  // Mapped pinned host memory that kllm_decoder_generate_until streams the ids through: the count at
  // [0], the ids from [kStreamIds] (a line of their own, apart from the polled count).
  int32_t* stream_host = nullptr;
  int32_t* stream_dev = nullptr;  // the same memory as the device addresses it
  // batched wgmma prefill (kllm_decoder_prefill_tf32 / _w8): activations of one block of prompt positions
  float* pf_buf = nullptr;
  PrefillWorkspace pf_ws{};
  // kllm_decoder_verify (verify.cu): the per-position workspace, and the chain of each length captured on first use
  void* vf_buf = nullptr;
  VerifyWorkspace vf{};
  VerifyIo* vf_io_host = nullptr;  // pinned
  cudaGraphExec_t vf_exec[KLLM_MAX_VERIFY_TOKENS] = {};
  int vf_launches[KLLM_MAX_VERIFY_TOKENS] = {};
};

// A batch of decoders over one model (kllm_batch_create): member b is row b of one chain
struct kllm_batch {
  std::vector<kllm_decoder*> members;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  void* buf = nullptr;  // device: the chain's rows [n][.]
  ChainRows rows{};
  // device: the rows' ChainMember [n], then their BatchTarget [n].  Row r is member r, except inside
  // kllm_batch_generate_until, which puts the running members first and restores this order before it returns.
  void* tables = nullptr;
  ChainMember* chain = nullptr;
  BatchTarget* targets = nullptr;
  void* tables_host = nullptr;  // pinned: the staging of the tables' uploads
  int32_t* io_host = nullptr;  // pinned [n][seq_len]: the ids read back
  // exec[k - 1]: embedding, chain and draw of one step of rows [0, k).  The n-row step is captured at create, the
  // others on first use by kllm_batch_generate_until.
  cudaGraphExec_t exec[KLLM_MAX_BATCH] = {};
  int launches[KLLM_MAX_BATCH] = {};
  // kllm_batch_beam_search: beam_exec[0] the pass of one row, beam_exec[1] of n rows (embedding, chain,
  // candidates), captured on first use; the candidates reach the host through mapped memory
  cudaGraphExec_t beam_exec[2] = {};
  int beam_launches[2] = {};
  BeamCandidates* cand_host = nullptr;
  BeamCandidates* cand_dev = nullptr;
};

namespace {

// The settings `next` in force from the next entry on: no step may still be reading the old ones, and the next one
// reads the new.  The host's copy changes only once the device's has.
int put_settings(kllm_decoder* dc, DrawSettings next) {
  sampling::step0_finish(next.penalty);
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  KLLM_TRY(cudaMemcpyAsync(dc->d_cfg, &next, sizeof(next), cudaMemcpyHostToDevice, dc->stream));
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  dc->cfg = next;
  return 0;
}

// The log-probability record with no entries (ids -1), in stream order
int clear_record(kllm_decoder* dc) {
  const size_t S = dc->m.seq_len, T = S * sampling::kMaxTopLogprobs;
  KLLM_TRY(cudaMemsetAsync(dc->rec.id, 0xff, sizeof(int32_t) * S, dc->stream));
  KLLM_TRY(cudaMemsetAsync(dc->rec.lp, 0, sizeof(float) * S, dc->stream));
  KLLM_TRY(cudaMemsetAsync(dc->rec.top_ids, 0xff, sizeof(int32_t) * T, dc->stream));
  return static_cast<int>(cudaMemsetAsync(dc->rec.top_lp, 0, sizeof(float) * T, dc->stream));
}

// An entry's first position, queued for upload with the entry's mode (mega::State): `teacher` feeds the teacher's
// ids, `streamed` publishes every id to mapped host memory, the steps before `lp_from` are prompt positions, and
// `lp_target` is kllm_decoder_score's.  The upload goes on stream s, the decoder's own when s is null.  The pinned
// copy stays as written until the entry reads the state back.
int put_state(kllm_decoder* dc, int32_t token, int32_t pos, int teacher, int streamed, int lp_from, int lp_target,
              cudaStream_t s = nullptr) {
  *dc->st_host = mega::State{token, pos, 0, -1, teacher, streamed, lp_from, lp_target};
  return static_cast<int>(cudaMemcpyAsync(dc->st, dc->st_host, sizeof(mega::State), cudaMemcpyHostToDevice,
                                          s != nullptr ? s : dc->stream));
}

// Reads the state back after an entry's last position: *next is the id drawn there
int read_next(kllm_decoder* dc, int32_t* next) {
  KLLM_TRY(cudaMemcpyAsync(dc->st_host, dc->st, sizeof(mega::State), cudaMemcpyDeviceToHost, dc->stream));
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  *next = dc->st_host->next;
  return 0;
}

// Queues the upload of tokens[0 .. n) into the teacher through the pinned scratch
int put_teacher(kllm_decoder* dc, const int32_t* tokens, int n) {
  std::memcpy(dc->io_host, tokens, sizeof(int32_t) * n);
  return static_cast<int>(
      cudaMemcpyAsync(dc->teacher, dc->io_host, sizeof(int32_t) * n, cudaMemcpyHostToDevice, dc->stream));
}

// Captures what enqueue() queues on stream s into *exec, and the number of kernels it launched into *launches.
// Capturing does not execute: the launch accounting of the capture pass is undone.
template <typename Enqueue>
int capture_graph(cudaStream_t s, Enqueue&& enqueue, cudaGraphExec_t* exec, int* launches) {
  (void)cudaGetLastError();  // the chain checks its launches with cudaGetLastError: no earlier call's error is its own
  const uint64_t before = launch_counter().load();
  KLLM_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
  const int rc = enqueue();
  cudaGraph_t g = nullptr;
  const cudaError_t end = cudaStreamEndCapture(s, &g);
  const uint64_t n = launch_counter().load() - before;
  launch_counter().fetch_sub(n);
  if (rc != 0 || end != cudaSuccess) {
    if (g) cudaGraphDestroy(g);
    return rc != 0 ? rc : static_cast<int>(end);
  }
  const cudaError_t inst = cudaGraphInstantiate(exec, g, 0);
  cudaGraphDestroy(g);
  KLLM_TRY(inst);
  *launches = static_cast<int>(n);
  return 0;
}

// n launches of a captured graph on stream s, counted as `launches` kernels each
int replay(cudaGraphExec_t exec, int launches, int n, cudaStream_t s) {
  for (int i = 0; i < n; ++i) KLLM_TRY(cudaGraphLaunch(exec, s));
  count_launch(static_cast<uint64_t>(launches) * n);
  return 0;
}

// Waits for streamed id i: until the mapped count, which the draw publishes with release semantics, exceeds i.
// KLLM_E_STATE when stream s finished and the count did not get there, else the stream's own error.  A busy poll,
// since the wait is on the loop's critical path.
int wait_streamed(const int32_t* count, int i, cudaStream_t s) {
  while (__atomic_load_n(count, __ATOMIC_ACQUIRE) <= i) {
    const cudaError_t q = cudaStreamQuery(s);
    if (q == cudaSuccess && __atomic_load_n(count, __ATOMIC_ACQUIRE) <= i) return KLLM_E_STATE;
    if (q != cudaSuccess && q != cudaErrorNotReady) return static_cast<int>(q);
  }
  return 0;
}

// Whether id is one of the stop ids[0 .. n)
bool hits_stop(const int32_t* ids, int n, int32_t id) {
  for (int j = 0; j < n; ++j)
    if (ids[j] == id) return true;
  return false;
}

// A stop set of n ids: at most KLLM_MAX_STOP_IDS, given when n > 0, each in the vocabulary
int stop_args(const int32_t* ids, int32_t n, int vocab) {
  if (n < 0 || n > KLLM_MAX_STOP_IDS || (n > 0 && ids == nullptr)) return KLLM_E_INVALID;
  for (int32_t i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= vocab) return KLLM_E_INVALID;
  return 0;
}

// The arguments kllm_decoder_generate_until and kllm_decoder_generate_speculative share
int until_args(const kllm_decoder* dc, int32_t start_pos, int32_t max_steps, const int32_t* stop_ids, int32_t n_stop,
               const int32_t* out_tokens_host, const int32_t* n_out) {
  if (!dc || !out_tokens_host || !n_out || max_steps <= 0 || start_pos < 0) return KLLM_E_INVALID;
  if (static_cast<int64_t>(start_pos) + max_steps > dc->m.seq_len) return KLLM_E_INVALID;
  return stop_args(stop_ids, n_stop, dc->m.vocab_size);
}

// The next [n][per] floats of a workspace from `cursor`, which moves past them
float* take(float*& cursor, size_t n, size_t per) {
  float* r = cursor;
  cursor += n * per;
  return r;
}

// The chain's rows of n positions or members, in the one order the batch and the verify workspace carve them
ChainRows chain_rows(const DecoderModel& m, size_t n, float*& cursor) {
  ChainRows r;
  r.x = take(cursor, n, m.dim), r.q = take(cursor, n, m.q_rows), r.k = take(cursor, n, m.kv_dim);
  r.v = take(cursor, n, m.kv_dim), r.att = take(cursor, n, m.q_rows), r.h = take(cursor, n, m.hidden_dim);
  r.logits = take(cursor, n, m.vocab_size), r.score = take(cursor, n, static_cast<size_t>(m.head_num) * m.seq_len);
  return r;
}

// Runs n positions from the state put_state queued, in its mode, on the decoder's engine.  The persistent engine
// takes the mode in one launch's parameters: the teacher, its classifier skipped at the prompt positions before
// lp_from, and scoring's target mode, which records even with logprobs off.  The graph engine launches its
// captured step n times; argmax_advance_kernel reads the mode from the state.
int run_positions(kllm_decoder* dc, int n) {
  const mega::State& s = *dc->st_host;
  if (dc->use_mega) {
    DrawSettings cfg = dc->cfg;
    if (s.lp_target) cfg.lp_top_n = std::max(cfg.lp_top_n, 0);
    return dc->mega.run(cfg, n, s.teacher ? dc->teacher : nullptr, nullptr, -1, s.lp_from, s.lp_target);
  }
  return replay(dc->exec, dc->launches_per_step, n, dc->stream);
}

// The decoder's KV cache in its engine's layout -- the persistent engine's, or the graph engine's [seq][kv_dim] --
// and its RoPE tables
DecoderCache decoder_cache(const kllm_decoder* dc) {
  const DecoderModel& m = dc->m;
  const prefill::CacheLayout layout{dc->use_mega ? 1 : 0, m.seq_len, m.kv_dim, m.head_size,
                                    dc->use_mega ? dc->mega.attn_vsplit() : 1, dc->d.kv_cache};
  return {layout, dc->kcache, dc->vcache, dc->sin_t, dc->cos_t, dc->kv_scales_dev};
}

int enqueue_step(kllm_decoder* dc, cudaStream_t s) {
  const DecoderModel& m = dc->m;
  embed_token_kernel<<<4, 256, 0, s>>>(dc->st, m.tok_emb, dc->x, m.dim, m.vocab_size, dc->hist);
  count_launch();
  KLLM_TRY(cudaGetLastError());
  const ChainRows rows{dc->x, dc->q, dc->k, dc->v, dc->attn, dc->h, dc->score, dc->logits};
  const TpReduce tp{&dc->d, dc->tp_tmp};
  KLLM_TRY(enqueue_layers(m, decoder_cache(dc), rows, 1, ChainPos{PosArg{&dc->st->pos, 0}, nullptr},
                          dc->d.tp_size > 1 ? &tp : nullptr, s));
  // post_processing (llama3.cpp:733-745)
  argmax_advance_kernel<<<1, 1024, 0, s>>>(dc->logits, m.vocab_size, dc->d_cfg, dc->st, dc->out_tokens, dc->teacher,
                                           m.seq_len, dc->stream_dev + kStreamIds, dc->stream_dev, dc->hist,
                                           dc->penalized, dc->rec);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// The graph engine's step, captured once
int capture(kllm_decoder* dc) {
  return capture_graph(dc->stream, [dc] { return enqueue_step(dc, dc->stream); }, &dc->exec, &dc->launches_per_step);
}

// The batched prefill behind kllm_decoder_prefill_tf32 / _w8.  Each entry checks the arguments
// (prefill_args), then refuses what its GEMM cannot take, then calls run_prefill(): the workspace, the block loop,
// and the last position's classifier and argmax.
int prefill_args(const kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                 const int32_t* next_host) {
  if (!dc || !tokens_host || !next_host || n_tokens <= 0 || start_pos < 0) return KLLM_E_INVALID;
  if (start_pos + n_tokens > dc->m.seq_len) return KLLM_E_INVALID;
  // embed_rows_kernel has no embedding row for an id outside the vocabulary: refuse before any launch
  for (int32_t i = 0; i < n_tokens; ++i)
    if (tokens_host[i] < 0 || tokens_host[i] >= dc->m.vocab_size) return KLLM_E_INVALID;
  return 0;
}

int run_prefill(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                int32_t* next_host) {
  const DecoderModel& m = dc->m;
  constexpr int kBlock = 256;  // prompt positions per pass = the N of the wgmma
  const int q_rows = m.q_rows, kvd = m.kv_dim;
  if ((m.dim & 3) || (m.hidden_dim & 3) || (q_rows & 3)) return KLLM_E_UNSUPPORTED;
  if (dc->pf_buf == nullptr) {
    const size_t per_row = static_cast<size_t>(3 * m.dim + 2 * q_rows + 2 * kvd + 2 * m.hidden_dim);
    if (cudaMalloc(&dc->pf_buf, per_row * kBlock * sizeof(float)) != cudaSuccess)
      return static_cast<int>(cudaErrorMemoryAllocation);
    float* f = dc->pf_buf;
    PrefillWorkspace& w = dc->pf_ws;
    w.x = take(f, kBlock, m.dim), w.xn = take(f, kBlock, m.dim), w.tmp = take(f, kBlock, m.dim);
    w.q = take(f, kBlock, q_rows), w.att = take(f, kBlock, q_rows);
    w.k = take(f, kBlock, kvd), w.v = take(f, kBlock, kvd);
    w.h1 = take(f, kBlock, m.hidden_dim), w.h3 = take(f, kBlock, m.hidden_dim);
  }
  KLLM_TRY(prefill_attention_smem_opt_in(static_cast<size_t>(start_pos + n_tokens) * sizeof(float)));
  const DecoderCache pm = decoder_cache(dc);

  KLLM_TRY(put_teacher(dc, tokens_host, n_tokens));
  // the prompt rows' history (prefill_args refused ids outside the vocabulary), in stream order before the draw
  KLLM_TRY(cudaMemcpyAsync(dc->hist + start_pos, dc->teacher, sizeof(int32_t) * n_tokens, cudaMemcpyDeviceToDevice,
                           dc->stream));
  int last_rows = 0;
  for (int c0 = 0; c0 < n_tokens; c0 += kBlock) {
    const int T = std::min(kBlock, n_tokens - c0);
    KLLM_TRY(prefill_block(m, pm, dc->pf_ws, dc->teacher + c0, T, start_pos + c0, dc->stream));
    last_rows = T;
  }
  // last prompt position only: the classifier and the greedy id (post_processing, llama3.cpp:733-745) through the
  // decode path's fused GEMV and argmax
  KLLM_TRY(put_state(dc, tokens_host[n_tokens - 1], start_pos + n_tokens - 1, 0, 0, 0, 0));
  KLLM_TRY(enqueue_classifier(m, dc->pf_ws.x + static_cast<size_t>(last_rows - 1) * m.dim, dc->logits, 1,
                              dc->stream));
  argmax_advance_kernel<<<1, 1024, 0, dc->stream>>>(dc->logits, m.vocab_size, dc->d_cfg, dc->st, nullptr, nullptr,
                                                    m.seq_len, nullptr, nullptr, dc->hist, dc->penalized, dc->rec);
  count_launch();
  KLLM_TRY(cudaGetLastError());
  return read_next(dc, next_host);
}

// What the verify pass has no counterpart of: the fast numerics' fixed-point rows and flash attention (and with them
// the bf16 and fp8 caches), and tensor parallelism
int verify_supported(const kllm_decoder* dc) {
  if (dc->d.tp_size > 1 || dc->d.kv_cache != KLLM_KV_F32) return KLLM_E_UNSUPPORTED;
  if (dc->use_mega && dc->mega.fast()) return KLLM_E_UNSUPPORTED;
  return 0;
}

// One model: the same shape, flavour, group size, weight format and weight pointers, on the same engine with the same
// cache layout (so the same attention split).  Two such decoders run the same arithmetic on the same weights, so
// one chain serves both, and a cache prefix of one is a cache prefix of the other.
bool same_model(const kllm_decoder* a, const kllm_decoder* b) {
  const DecoderModel &x = a->m, &y = b->m;
  const int xs[] = {x.dim, x.hidden_dim, x.layer_num, x.head_num, x.kv_head_num, x.vocab_size, x.seq_len, x.head_size,
                    x.kv_dim, x.kv_mul, x.q_rows, x.flavour, x.group_size};
  const int ys[] = {y.dim, y.hidden_dim, y.layer_num, y.head_num, y.kv_head_num, y.vocab_size, y.seq_len, y.head_size,
                    y.kv_dim, y.kv_mul, y.q_rows, y.flavour, y.group_size};
  if (std::memcmp(xs, ys, sizeof(xs)) != 0 || x.format != y.format) return false;
  auto same = [](const Matrix& p, const Matrix& q) { return p.w == q.w && p.scales == q.scales && p.bias == q.bias; };
  if (x.tok_emb != y.tok_emb || x.final_norm != y.final_norm || !same(x.cls, y.cls)) return false;
  for (int l = 0; l < x.layer_num; ++l) {
    const LayerWeights &p = x.layers[l], &q = y.layers[l];
    if (p.attn_norm != q.attn_norm || p.ffn_norm != q.ffn_norm || !same(p.q, q.q) || !same(p.k, q.k) ||
        !same(p.v, q.v) || !same(p.o, q.o) || !same(p.w1, q.w1) || !same(p.w2, q.w2) || !same(p.w3, q.w3))
      return false;
  }
  const prefill::CacheLayout ca = decoder_cache(a).cache, cb = decoder_cache(b).cache;
  return a->use_mega == b->use_mega && ca.mega == cb.mega && ca.seq_len == cb.seq_len && ca.kv_dim == cb.kv_dim &&
         ca.head_size == cb.head_size && ca.split == cb.split && ca.elem == cb.elem;
}

// Embedding and chain of rows [0, k): each row's logits in the batch's rows
int enqueue_batch_chain(const kllm_batch* b, int k, cudaStream_t s) {
  const kllm_decoder* d0 = b->members[0];
  const DecoderModel& m = d0->m;
  batch_embed_kernel<<<dim3(4, k), 256, 0, s>>>(b->targets, m.tok_emb, b->rows.x, m.dim, m.vocab_size);
  count_launch();
  KLLM_TRY(cudaGetLastError());
  // the RoPE tables are member 0's: every member's hold the same values (kllm_sincos_init of the same shape)
  return enqueue_layers(m, decoder_cache(d0), b->rows, k, ChainPos{PosArg{nullptr, 0}, b->chain}, nullptr, s);
}

// Embedding, chain and draw of one step of rows [0, k): the graph engine's step (enqueue_step) at k rows
int enqueue_batch(const kllm_batch* b, int k, cudaStream_t s) {
  const DecoderModel& m = b->members[0]->m;
  KLLM_TRY(enqueue_batch_chain(b, k, s));
  batch_draw_kernel<<<k, 1024, 0, s>>>(b->rows.logits, m.vocab_size, b->targets, m.seq_len);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// The step of k rows, captured once
int batch_capture(kllm_batch* b, int k) {
  if (b->exec[k - 1] != nullptr) return 0;
  return capture_graph(b->stream, [b, k] { return enqueue_batch(b, k, b->stream); }, &b->exec[k - 1],
                       &b->launches[k - 1]);
}

size_t table_bytes(const kllm_batch* b) { return b->members.size() * (sizeof(ChainMember) + sizeof(BatchTarget)); }

// Queues the upload of the tables with rows[r] in row r, r < k, from the pinned staging: the caller does not write
// the staging again before this copy has run
int put_tables(kllm_batch* b, const int* rows, int k) {
  const size_t n = b->members.size();
  auto* chain = static_cast<ChainMember*>(b->tables_host);
  auto* targets = reinterpret_cast<BatchTarget*>(static_cast<char*>(b->tables_host) + n * sizeof(ChainMember));
  for (int r = 0; r < k; ++r) {
    kllm_decoder* dc = b->members[rows[r]];
    chain[r] = ChainMember{dc->kcache, dc->vcache, &dc->st->pos};
    targets[r] = BatchTarget{dc->st, dc->d_cfg, dc->hist, dc->penalized, dc->rec, dc->out_tokens, dc->teacher,
                             dc->logits, dc->stream_dev + kStreamIds, dc->stream_dev};
  }
  return static_cast<int>(
      cudaMemcpyAsync(b->tables, b->tables_host, table_bytes(b), cudaMemcpyHostToDevice, b->stream));
}

// put_tables with every member in its own row
int put_member_tables(kllm_batch* b) {
  const int n = static_cast<int>(b->members.size());
  int all[KLLM_MAX_BATCH];
  for (int i = 0; i < n; ++i) all[i] = i;
  return put_tables(b, all, n);
}

// The batch's workspace, member tables and captured step
int batch_prepare(kllm_batch* b) {
  const DecoderModel& m = b->members[0]->m;
  const int n = static_cast<int>(b->members.size());
  const size_t V = m.vocab_size;
  const size_t per_row = 2 * static_cast<size_t>(m.q_rows) + 2 * m.kv_dim + m.dim + m.hidden_dim + V +
                         static_cast<size_t>(m.head_num) * m.seq_len;
  if (cudaMalloc(&b->buf, per_row * n * sizeof(float)) != cudaSuccess) b->buf = nullptr;
  if (cudaMalloc(&b->tables, table_bytes(b)) != cudaSuccess) b->tables = nullptr;
  if (cudaMallocHost(&b->tables_host, table_bytes(b)) != cudaSuccess) b->tables_host = nullptr;
  if (cudaMallocHost(&b->io_host, sizeof(int32_t) * n * m.seq_len) != cudaSuccess) b->io_host = nullptr;
  if (cudaHostAlloc(&b->cand_host, sizeof(BeamCandidates), cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer(&b->cand_dev, b->cand_host, 0) != cudaSuccess)
    b->cand_dev = nullptr;
  if (!b->buf || !b->tables || !b->tables_host || !b->io_host || !b->cand_dev)
    return static_cast<int>(cudaErrorMemoryAllocation);
  float* f = static_cast<float*>(b->buf);
  b->rows = chain_rows(m, n, f);
  b->chain = static_cast<ChainMember*>(b->tables);
  b->targets = reinterpret_cast<BatchTarget*>(static_cast<char*>(b->tables) + n * sizeof(ChainMember));
  static_assert(sizeof(ChainMember) % alignof(BatchTarget) == 0, "the targets follow the chain table aligned");
  KLLM_TRY(put_member_tables(b));
  KLLM_TRY(cudaStreamSynchronize(b->stream));
  return batch_capture(b, n);
}

// n_steps steps of every member from tokens[b] at pos[b]; out [n][n_steps].  Every refusal comes before any launch.
int run_batch(kllm_batch* b, const int32_t* tokens, const int32_t* pos, int32_t n_steps, int32_t* out) {
  if (!b || !tokens || !pos || !out || n_steps <= 0) return KLLM_E_INVALID;
  const DecoderModel& m = b->members[0]->m;
  const size_t n = b->members.size();
  for (size_t i = 0; i < n; ++i) {
    if (tokens[i] < 0 || tokens[i] >= m.vocab_size || pos[i] < 0) return KLLM_E_INVALID;
    if (static_cast<int64_t>(pos[i]) + n_steps > m.seq_len) return KLLM_E_INVALID;
  }
  for (kllm_decoder* dc : b->members) KLLM_TRY(cudaStreamSynchronize(dc->stream));
  // each member's state as its own kllm_decoder_generate (no teacher) puts it; the pinned copies stay as written
  // until the synchronisation below
  for (size_t i = 0; i < n; ++i) KLLM_TRY(put_state(b->members[i], tokens[i], pos[i], 0, 0, 0, 0, b->stream));
  KLLM_TRY(replay(b->exec[n - 1], b->launches[n - 1], n_steps, b->stream));
  for (size_t i = 0; i < n; ++i)
    KLLM_TRY(cudaMemcpyAsync(b->io_host + i * n_steps, b->members[i]->out_tokens, sizeof(int32_t) * n_steps,
                             cudaMemcpyDeviceToHost, b->stream));
  KLLM_TRY(cudaStreamSynchronize(b->stream));
  std::memcpy(out, b->io_host, sizeof(int32_t) * n * n_steps);
  return 0;
}

// kllm_batch_generate_until's loop, after its refusals.  Pass p launches the step of the k members still running,
// which are rows [0, k) of the tables, waits for each one's id p through its mapped count and hands it over.  A member
// whose id p is one of its stop ids or its max_steps-th id is done: the tables are uploaded again with the members
// still running first, in member order, and the next pass launches the step of their number.  A finished member is
// in no later pass, so nothing of it is written after its end.
int run_batch_until(kllm_batch* b, const int32_t* tokens, const int32_t* pos, const int32_t* max_steps,
                    const int32_t* stop_ids, const int32_t* n_stop, kllm_batch_token_callback on_tokens, void* ctx,
                    int32_t* out, int32_t* n_out, kllm_batch_stats* stats) {
  const int n = static_cast<int>(b->members.size());
  int32_t M = 0;
  for (int i = 0; i < n; ++i) M = std::max(M, max_steps[i]);
  for (kllm_decoder* dc : b->members) KLLM_TRY(cudaStreamSynchronize(dc->stream));
  // each member's state as its own kllm_decoder_generate_until puts it, streamed through its own mapped area
  for (int i = 0; i < n; ++i) {
    kllm_decoder* dc = b->members[i];
    __atomic_store_n(dc->stream_host, 0, __ATOMIC_SEQ_CST);  // before the launch that writes it
    KLLM_TRY(put_state(dc, tokens[i], pos[i], 0, 1, 0, 0, b->stream));
  }
  int running[KLLM_MAX_BATCH];
  for (int i = 0; i < n; ++i) running[i] = i, n_out[i] = 0;
  int k = n, passes = 0, rows = 0;
  bool reordered = false;
  int rc = 0;
  for (int p = 0; k > 0 && rc == 0; ++p) {
    if (b->exec[k - 1] == nullptr) {  // first use of k rows: captured with nothing in flight
      if ((rc = static_cast<int>(cudaStreamSynchronize(b->stream))) != 0 || (rc = batch_capture(b, k)) != 0) break;
    }
    if ((rc = replay(b->exec[k - 1], b->launches[k - 1], 1, b->stream)) != 0) break;
    ++passes, rows += k;
    int still = 0;
    for (int r = 0; r < k; ++r) {
      const int i = running[r];
      if ((rc = wait_streamed(b->members[i]->stream_host, p, b->stream)) != 0) break;
      const int32_t id = b->members[i]->stream_host[kStreamIds + p];
      n_out[i] = p + 1;
      if (on_tokens != nullptr) on_tokens(ctx, i, &id, 1);
      const bool stop = p + 1 == max_steps[i] || hits_stop(stop_ids + i * KLLM_MAX_STOP_IDS, n_stop[i], id);
      if (!stop) running[still++] = i;
    }
    if (rc != 0) break;
    // the previous upload ran before this pass's step, so the staging is free
    if (still > 0 && still < k) rc = put_tables(b, running, still), reordered = true;
    k = still;
  }
  // the next call sees every member in its own row again
  cudaError_t s = cudaStreamSynchronize(b->stream);
  if (reordered && s == cudaSuccess) {
    s = static_cast<cudaError_t>(put_member_tables(b));
    if (s == cudaSuccess) s = cudaStreamSynchronize(b->stream);
  }
  if (rc == 0) rc = static_cast<int>(s);
  if (rc != 0) return rc;
  for (int i = 0; i < n; ++i)
    std::memcpy(out + static_cast<size_t>(i) * M, b->members[i]->stream_host + kStreamIds, sizeof(int32_t) * n_out[i]);
  if (stats != nullptr) *stats = kllm_batch_stats{passes, rows};
  return 0;
}

// A beam-search pass of rows [0, k): embedding, chain, and each row's candidates
int enqueue_beam_pass(const kllm_batch* b, int k, cudaStream_t s) {
  const DecoderModel& m = b->members[0]->m;
  KLLM_TRY(enqueue_batch_chain(b, k, s));
  const int top_n = static_cast<int>(b->members.size()) + KLLM_MAX_BEAM_EOS;
  beam_candidates_kernel<<<k, 1024, 0, s>>>(b->rows.logits, m.vocab_size, top_n, b->cand_dev);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// Queues the copy of rows [lo, hi) from member src[f] to member dst[f] for every f < n, in one launch
int fork_rows(kllm_batch* b, const int* src, const int* dst, int n, int lo, int hi) {
  if (n == 0 || hi <= lo) return 0;
  ForkTable t{};
  for (int f = 0; f < n; ++f) {
    const kllm_decoder *s = b->members[src[f]], *d = b->members[dst[f]];
    t.ks[f] = s->kcache, t.vs[f] = s->vcache, t.kd[f] = d->kcache, t.vd[f] = d->vcache;
  }
  const kllm_decoder* d0 = b->members[0];
  fork_rows_kernel<<<dim3(hi - lo, d0->m.layer_num, n), 256, 0, b->stream>>>(t, lo, decoder_cache(d0).cache);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// kllm_batch_beam_search's loop, after its refusals: the rule of kuiperllama_b200/beam.py, step for step.  Beam r of
// a pass is row r, carried by member rows[r].  Each pass puts every row's state (the beam's last id at the pass's
// position), launches the pass, reads the candidates, applies the rule, then queues the next pass's tables and the
// forks: a child whose parent's member is taken by an earlier child takes a dropped beam's member.
int run_batch_beam(kllm_batch* b, int32_t first_token, int32_t start_pos, int32_t max_new, const int32_t* eos,
                   int n_eos, float alpha, int early, int n_return, int32_t* out_ids, int32_t* out_len,
                   float* out_score, float* out_sum, kllm_beam_stats* stats) {
  const int B = static_cast<int>(b->members.size()), top = B + n_eos;
  struct Beam {
    std::vector<int32_t> ids;
    float sum;
    int member;
  };
  struct Cand {
    float s;
    int beam, k;
    int32_t id;
  };
  struct Hyp {
    float h, sum;
    std::vector<int32_t> ids;
  };
  for (kllm_decoder* dc : b->members) KLLM_TRY(cudaStreamSynchronize(dc->stream));
  for (int g = 0; g < (B > 1 ? 2 : 1); ++g) {  // first use: captured with nothing in flight
    if (b->beam_exec[g] != nullptr) continue;
    const int k = g == 0 ? 1 : B;
    KLLM_TRY(capture_graph(b->stream, [b, k] { return enqueue_beam_pass(b, k, b->stream); }, &b->beam_exec[g],
                           &b->beam_launches[g]));
  }
  std::vector<Beam> beams{Beam{{}, 0.f, 0}};
  std::vector<Hyp> slots;
  std::vector<Cand> cands;
  bool unsatisfied = true, reordered = false;
  kllm_beam_stats st{0, 0, 0};
  int rc = 0;
  for (int t = 1; t <= max_new && rc == 0; ++t) {
    const int k = static_cast<int>(beams.size()), g = k == 1 ? 0 : 1;
    const int pos = start_pos + t - 1;
    for (int r = 0; r < k && rc == 0; ++r)
      rc = put_state(b->members[beams[r].member], t == 1 ? first_token : beams[r].ids.back(), pos, 0, 0, 0, 0,
                     b->stream);
    if (rc != 0 || (rc = replay(b->beam_exec[g], b->beam_launches[g], 1, b->stream)) != 0) break;
    if ((rc = static_cast<int>(cudaStreamSynchronize(b->stream))) != 0) break;
    ++st.passes;
    // 2. candidates: s = fp32(S_b + lp), ordered by s descending, beam, the beam's own order
    const BeamCandidates& c = *b->cand_host;
    cands.clear();
    for (int r = 0; r < k; ++r)
      for (int j = 0; j < top; ++j) cands.push_back(Cand{beams[r].sum + c.lp[r][j], r, j, c.ids[r][j]});
    std::sort(cands.begin(), cands.end(), [](const Cand& x, const Cand& y) {
      if (x.s != y.s) return x.s > y.s;
      return x.beam != y.beam ? x.beam < y.beam : x.k < y.k;
    });
    // 3. finished hypotheses from the first B ranks, merged into the slots unless a gate is closed
    const bool last = t == max_new;
    auto is_eos = [&](int32_t id) { return hits_stop(eos, n_eos, id); };
    auto extend = [](const std::vector<int32_t>& ids, int32_t id) {
      std::vector<int32_t> r = ids;
      r.push_back(id);
      return r;
    };
    if (unsatisfied && !(static_cast<int>(slots.size()) == B && early == KLLM_BEAM_EARLY_ALL_DONE)) {
      const float div = static_cast<float>(std::pow(static_cast<double>(t), static_cast<double>(alpha)));
      for (int r = 0; r < B; ++r)
        if (last || is_eos(cands[r].id))
          slots.push_back(Hyp{cands[r].s / div, cands[r].s, extend(beams[cands[r].beam].ids, cands[r].id)});
      std::stable_sort(slots.begin(), slots.end(), [](const Hyp& x, const Hyp& y) { return x.h > y.h; });
      if (static_cast<int>(slots.size()) > B) slots.resize(B);
    }
    // 4. the next beams: the first B candidates that are not eos ids
    std::vector<Beam> next;
    std::vector<int> parent;
    for (const Cand& x : cands) {
      if (static_cast<int>(next.size()) == B) break;
      if (is_eos(x.id)) continue;
      next.push_back(Beam{extend(beams[x.beam].ids, x.id), x.s, -1});
      parent.push_back(x.beam);
    }
    // 5. the early-stop heuristic and the stop test
    const bool full = static_cast<int>(slots.size()) == B;
    if (unsatisfied) {
      const int L = early == KLLM_BEAM_EARLY_NEVER && alpha > 0.f ? max_new : t;
      const float best = next[0].sum / static_cast<float>(std::pow(static_cast<double>(L), static_cast<double>(alpha)));
      unsatisfied = !full || best > slots.back().h;
    }
    const bool stop = last || !unsatisfied || (full && early == KLLM_BEAM_EARLY_ALL_DONE);
    // forks: after pass 0 member 0's prompt rows to every other member, even when the search stops there
    int src[KLLM_MAX_BATCH], dst[KLLM_MAX_BATCH], nf = 0;
    if (t == 1) {
      for (int j = 0; j < B; ++j) next[j].member = j;
      for (int j = 1; j < B; ++j) src[nf] = 0, dst[nf] = j, ++nf;
      rc = fork_rows(b, src, dst, nf, 0, start_pos + 1);
      st.forks += nf, st.fork_rows += static_cast<int64_t>(nf) * (start_pos + 1);
    } else if (!stop) {
      bool kept[KLLM_MAX_BATCH] = {};  // old beam r's member went to its first child
      for (int j = 0; j < B; ++j)
        if (!kept[parent[j]]) kept[parent[j]] = true, next[j].member = beams[parent[j]].member;
      int free_members[KLLM_MAX_BATCH], n_free = 0;
      for (int r = 0; r < k; ++r)
        if (!kept[r]) free_members[n_free++] = beams[r].member;
      std::sort(free_members, free_members + n_free);
      for (int j = 0, f = 0; j < B; ++j)
        if (next[j].member < 0) {
          next[j].member = free_members[f++];
          src[nf] = beams[parent[j]].member, dst[nf] = next[j].member, ++nf;
        }
      rc = fork_rows(b, src, dst, nf, start_pos + 1, pos + 1);
      st.forks += nf, st.fork_rows += static_cast<int64_t>(nf) * (t - 1);
    }
    if (rc != 0 || stop) break;
    // the next pass's rows; the last upload ran before this pass, so the staging is free
    int rows[KLLM_MAX_BATCH];
    for (int j = 0; j < B; ++j) rows[j] = next[j].member;
    rc = put_tables(b, rows, B), reordered = true;
    beams = std::move(next);
  }
  // the next call sees every member in its own row again
  cudaError_t s = cudaStreamSynchronize(b->stream);
  if (reordered && s == cudaSuccess) {
    s = static_cast<cudaError_t>(put_member_tables(b));
    if (s == cudaSuccess) s = cudaStreamSynchronize(b->stream);
  }
  if (rc == 0) rc = static_cast<int>(s);
  if (rc != 0) return rc;
  for (int i = 0; i < n_return; ++i) {
    const Hyp& h = slots[i];
    std::memcpy(out_ids + static_cast<size_t>(i) * max_new, h.ids.data(), sizeof(int32_t) * h.ids.size());
    out_len[i] = static_cast<int32_t>(h.ids.size());
    out_score[i] = h.h, out_sum[i] = h.sum;
  }
  if (stats != nullptr) *stats = st;
  return 0;
}

// The verify workspace (once per decoder) and the captured chain of n positions (once per length)
int verify_prepare(kllm_decoder* dc, int n) {
  const DecoderModel& m = dc->m;
  constexpr int N = KLLM_MAX_VERIFY_TOKENS;
  if (dc->vf_buf == nullptr) {
    const size_t V = m.vocab_size, T = sampling::kMaxTopLogprobs;
    const size_t floats = N * (2 * static_cast<size_t>(m.dim) + 2 * m.q_rows + 2 * m.kv_dim + m.hidden_dim + 2 * V +
                               static_cast<size_t>(m.head_num) * m.seq_len);
    const size_t words = N * (V + 2 + 2 * T);  // marks, saved history, saved record
    const size_t bytes = (floats + words) * 4 + sizeof(VerifyIo);
    // both or neither: a later call allocates again
    if (cudaMalloc(&dc->vf_buf, bytes) != cudaSuccess) {
      dc->vf_buf = nullptr;
      return static_cast<int>(cudaErrorMemoryAllocation);
    }
    if (cudaMallocHost(&dc->vf_io_host, sizeof(VerifyIo)) != cudaSuccess) {
      cudaFree(dc->vf_buf);
      dc->vf_buf = nullptr, dc->vf_io_host = nullptr;
      return static_cast<int>(cudaErrorMemoryAllocation);
    }
    KLLM_TRY(cudaMemsetAsync(dc->vf_buf, 0, bytes, dc->stream));  // the marks start at zero
    float* f = static_cast<float*>(dc->vf_buf);
    VerifyWorkspace& w = dc->vf;
    w.rows = chain_rows(m, N, f);
    w.penalized = take(f, N, V);
    w.marks = reinterpret_cast<int32_t*>(take(f, N, V));
    w.saved_hist = reinterpret_cast<int32_t*>(take(f, N, 1));
    w.saved.id = reinterpret_cast<int32_t*>(take(f, N, 1));
    w.saved.lp = take(f, N, 1);
    w.saved.top_ids = reinterpret_cast<int32_t*>(take(f, N, T));
    w.saved.top_lp = take(f, N, T);
    w.io = reinterpret_cast<VerifyIo*>(f);
  }
  if (dc->vf_exec[n - 1] != nullptr) return 0;
  const VerifyTarget t{dc->d_cfg, dc->st, dc->hist, dc->rec, dc->logits};
  return capture_graph(dc->stream, [&] { return enqueue_verify(m, decoder_cache(dc), t, dc->vf, n, dc->stream); },
                       &dc->vf_exec[n - 1], &dc->vf_launches[n - 1]);
}

// One verify pass of tokens[0 .. n) at start_pos, acceptance ended at the first of the n_stop stop ids; the caller
// checked the arguments.  out_ids receives id_0 .. id_a.
int run_verify(kllm_decoder* dc, const int32_t* tokens, int n, int start_pos, const int32_t* stop_ids, int n_stop,
               int32_t* out_ids, int32_t* accepted) {
  KLLM_TRY(verify_prepare(dc, n));
  VerifyIo& io = *dc->vf_io_host;
  std::memcpy(io.tokens, tokens, sizeof(int32_t) * n);
  io.start_pos = start_pos;
  io.n_stop = n_stop;
  if (n_stop > 0) std::memcpy(io.stop, stop_ids, sizeof(int32_t) * n_stop);
  KLLM_TRY(cudaMemcpyAsync(dc->vf.io, &io, offsetof(VerifyIo, ids), cudaMemcpyHostToDevice, dc->stream));
  KLLM_TRY(replay(dc->vf_exec[n - 1], dc->vf_launches[n - 1], 1, dc->stream));
  KLLM_TRY(cudaMemcpyAsync(io.ids, dc->vf.io->ids, sizeof(int32_t) * (KLLM_MAX_VERIFY_TOKENS + 1),
                           cudaMemcpyDeviceToHost, dc->stream));
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  *accepted = io.accepted;
  std::memcpy(out_ids, io.ids, sizeof(int32_t) * (io.accepted + 1));
  return 0;
}

// The prompt-lookup draft (kllm_b200.h, kllm_decoder_generate_speculative) of c[0 .. L) into draft, at most m ids
int lookup_draft(const int32_t* c, int L, int ngram_max, int m, int32_t* draft) {
  if (m <= 0) return 0;
  for (int n = ngram_max; n >= 1; --n) {
    if (L < n) continue;
    const int32_t* suf = c + L - n;
    bool hole = false;
    for (int i = 0; i < n; ++i) hole |= suf[i] < 0;
    if (hole) continue;
    for (int s = L - 1 - n; s >= 0; --s) {
      if (std::memcmp(c + s, suf, sizeof(int32_t) * n) != 0) continue;
      int k = 0;
      for (int j = s + n; j < L && k < m && c[j] >= 0; ++j) draft[k++] = c[j];
      if (k > 0) return k;
      break;  // the largest match gives the draft for this n, empty or not
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int kllm_decoder_create(const kllm_decoder_desc* desc, void* stream, kllm_decoder** out) {
  if (!desc || !out) return KLLM_E_INVALID;
  const kllm_decoder_desc& d = *desc;
  DecoderModel model;
  KLLM_TRY(build_decoder_model(d, &model));
  const int tp = d.tp_size > 1 ? d.tp_size : 1;
  // bf16 and fp8 caches exist on the persistent engine's flash form only; the rest of the refusals come from its init
  const bool kv_lowp = d.kv_cache != KLLM_KV_F32;
  const char* want = getenv("KLLM_ENGINE");
  const bool force_graph = want != nullptr && strcmp(want, "graph") == 0;
  const bool force_mega = want != nullptr && strcmp(want, "persistent") == 0;
  if (kv_lowp && (tp > 1 || force_graph)) return KLLM_E_UNSUPPORTED;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return KLLM_E_NODEVICE;

  auto* dc = new kllm_decoder();
  dc->d = d;
  dc->d.tp_size = tp;
  dc->m = std::move(model);
  const DecoderModel& m = dc->m;

  if (stream != nullptr) {
    dc->stream = static_cast<cudaStream_t>(stream);
  } else {
    if (cudaStreamCreateWithFlags(&dc->stream, cudaStreamNonBlocking) != cudaSuccess) {
      delete dc;
      return KLLM_E_NODEVICE;
    }
    dc->own_stream = true;
    // A private non-blocking stream does not order against the legacy default stream: weights the
    // caller uploaded or produced there (or anywhere else) must have landed before the first launch.
    if (cudaDeviceSynchronize() != cudaSuccess) {
      cudaStreamDestroy(dc->stream);
      delete dc;
      return KLLM_E_NODEVICE;
    }
  }

  auto fail = [&](int rc) {
    kllm_decoder_destroy(dc);
    return rc;
  };
  auto dev_alloc = [&](float** p, size_t n) {
    if (cudaMalloc(p, n * sizeof(float)) != cudaSuccess) return 1;
    return static_cast<int>(cudaMemsetAsync(*p, 0, n * sizeof(float), dc->stream));
  };
  const size_t kv_elems = static_cast<size_t>(m.layer_num) * m.seq_len * m.kv_dim;
  // bf16 / fp8: a half / a quarter of the bytes behind the same pointers
  const size_t kv_floats = (kv_elems * prefill::kv_elem_bytes(d.kv_cache) + 3) / 4;
  if (dev_alloc(&dc->x, m.dim) || dev_alloc(&dc->q, m.q_rows) || dev_alloc(&dc->k, m.kv_dim) ||
      dev_alloc(&dc->v, m.kv_dim) || dev_alloc(&dc->attn, m.q_rows) ||
      dev_alloc(&dc->h, m.hidden_dim) || dev_alloc(&dc->logits, m.vocab_size) ||
      dev_alloc(&dc->score, static_cast<size_t>(m.head_num) * m.seq_len) ||
      dev_alloc(&dc->kcache, kv_floats) || dev_alloc(&dc->vcache, kv_floats) ||
      dev_alloc(&dc->sin_t, static_cast<size_t>(m.seq_len) * m.head_size) ||
      dev_alloc(&dc->cos_t, static_cast<size_t>(m.seq_len) * m.head_size) ||
      dev_alloc(&dc->tp_tmp, m.dim) || dev_alloc(&dc->penalized, m.vocab_size) ||
      dev_alloc(&dc->bias, m.vocab_size))
    return fail(static_cast<int>(cudaErrorMemoryAllocation));
  if (d.kv_cache == KLLM_KV_FP8) {
    const size_t n = static_cast<size_t>(m.layer_num) * m.kv_head_num;
    dc->kv_scales.assign(d.kv_scales, d.kv_scales + 2 * n);
    std::vector<float> dev(4 * n);
    for (size_t i = 0; i < 2 * n; ++i) dev[i] = dc->kv_scales[i], dev[2 * n + i] = 1.0f / dc->kv_scales[i];
    // a blocking copy into unset memory: no memset on dc->stream may land after it
    if (cudaMalloc(&dc->kv_scales_dev, 4 * n * sizeof(float)) != cudaSuccess ||
        cudaMemcpy(dc->kv_scales_dev, dev.data(), 4 * n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
      return fail(static_cast<int>(cudaErrorMemoryAllocation));
  }
  dc->d.kv_scales = nullptr;  // the caller's array is not read after create
  if (cudaMalloc(&dc->st, sizeof(mega::State)) != cudaSuccess ||
      cudaMalloc(&dc->d_cfg, sizeof(DrawSettings)) != cudaSuccess ||
      cudaMalloc(&dc->hist, sizeof(int32_t) * m.seq_len) != cudaSuccess ||
      cudaMalloc(&dc->marks, sizeof(int32_t) * m.vocab_size) != cudaSuccess ||
      cudaMalloc(&dc->out_tokens, sizeof(int32_t) * m.seq_len) != cudaSuccess ||
      cudaMalloc(&dc->teacher, sizeof(int32_t) * m.seq_len) != cudaSuccess ||
      cudaMallocHost(&dc->st_host, sizeof(mega::State)) != cudaSuccess ||
      cudaMalloc(&dc->rec.id, sizeof(int32_t) * m.seq_len) != cudaSuccess ||
      cudaMalloc(&dc->rec.lp, sizeof(float) * m.seq_len) != cudaSuccess ||
      cudaMalloc(&dc->rec.top_ids, sizeof(int32_t) * m.seq_len * sampling::kMaxTopLogprobs) != cudaSuccess ||
      cudaMalloc(&dc->rec.top_lp, sizeof(float) * m.seq_len * sampling::kMaxTopLogprobs) != cudaSuccess ||
      cudaMallocHost(&dc->io_host, sizeof(int32_t) * m.seq_len) != cudaSuccess ||
      cudaHostAlloc(&dc->stream_host, sizeof(int32_t) * (kStreamIds + m.seq_len), cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer(&dc->stream_dev, dc->stream_host, 0) != cudaSuccess)
    return fail(static_cast<int>(cudaErrorMemoryAllocation));
  std::memset(dc->stream_host, 0, sizeof(int32_t) * (kStreamIds + m.seq_len));
  DrawSettings off{};  // greedy, step 0 off until a setter turns a sub-step on, logprobs off
  off.penalty.marks = dc->marks;
  off.lp_top_n = -1;
  int rc = static_cast<int>(cudaMemsetAsync(dc->st, 0, sizeof(mega::State), dc->stream));
  if (rc == 0) rc = static_cast<int>(cudaMemsetAsync(dc->hist, 0xff, sizeof(int32_t) * m.seq_len, dc->stream));  // -1
  if (rc == 0) rc = static_cast<int>(cudaMemsetAsync(dc->marks, 0, sizeof(int32_t) * m.vocab_size, dc->stream));
  if (rc == 0) rc = clear_record(dc);
  if (rc == 0) rc = put_settings(dc, off);
  if (rc != 0) return fail(rc);

  rc = kllm_sincos_init(m.head_size, m.seq_len, m.flavour, dc->sin_t, dc->cos_t, dc->stream);
  if (rc != 0) return fail(rc);
  // Engine: the persistent megakernel (one cooperative launch per run) when the shape fits its
  // shared-memory ring, else the CUDA-graph chain of fused launches.  KLLM_ENGINE=graph|persistent
  // forces one (persistent fails loudly if unsupported).  Both are CUDA; neither is a fallback to
  // anything off-device.  A bf16 or fp8 cache never falls back to the graph engine.
  // tensor parallel: the persistent engine needs the peer-memory transport (its exchange IS
  // the all-reduce); with NCCL or a caller-supplied callback the graph engine is used
  unsigned long long* tp_areas[8] = {};
  int tp_world = 1, tp_rank = 0, tp_stride = 0;
  bool mega_ok = tp == 1;
  if (tp > 1 && d.comm != nullptr &&
      comm_tagged_areas(d.comm, tp_areas, &tp_world, &tp_rank, &tp_stride) == 0 && tp_world == tp &&
      tp_stride >= m.dim)
    mega_ok = true;
  if (!force_graph && mega_ok) {
    MegaModel mm{};
    mm.tp_world = tp, mm.tp_rank = tp_rank, mm.tp_stride = tp_stride;
    mm.numerics = d.numerics;
    mm.kv_cache = d.kv_cache;
    mm.kv_scales = dc->kv_scales_dev;
    for (int r = 0; r < 8; ++r) mm.tp_data[r] = tp_areas[r];
    mm.logits = dc->logits, mm.score = dc->score, mm.key_cache = dc->kcache, mm.value_cache = dc->vcache;
    mm.sin_cache = dc->sin_t, mm.cos_cache = dc->cos_t, mm.state = dc->st, mm.out_tokens = dc->out_tokens;
    mm.sampling = &dc->d_cfg->sample;
    mm.hist = dc->hist, mm.penalized = dc->penalized;
    mm.lp_rec = dc->rec;
    rc = dc->mega.init(m, mm, dc->stream);
    if (rc == 0) {
      dc->use_mega = true;
      dc->launches_per_step = 1;
    } else if (rc != KLLM_E_UNSUPPORTED || force_mega || kv_lowp) {
      return fail(rc);
    }
  } else if (force_mega || kv_lowp) {
    return fail(KLLM_E_UNSUPPORTED);
  }
  if (!dc->use_mega && (rc = capture(dc)) != 0) return fail(rc);
  if (const cudaError_t e = cudaStreamSynchronize(dc->stream)) return fail(static_cast<int>(e));
  *out = dc;
  return 0;
}

void kllm_decoder_destroy(kllm_decoder* dc) {
  if (!dc) return;
  if (dc->stream) cudaStreamSynchronize(dc->stream);
  dc->mega.destroy();
  if (dc->exec) cudaGraphExecDestroy(dc->exec);
  float* bufs[] = {dc->x, dc->q, dc->k, dc->v, dc->attn, dc->h, dc->logits, dc->score,
                   dc->kcache, dc->vcache, dc->sin_t, dc->cos_t, dc->tp_tmp, dc->penalized, dc->bias,
                   dc->kv_scales_dev};
  for (float* b : bufs)
    if (b) cudaFree(b);
  if (dc->st) cudaFree(dc->st);
  if (dc->d_cfg) cudaFree(dc->d_cfg);
  if (dc->hist) cudaFree(dc->hist);
  if (dc->marks) cudaFree(dc->marks);
  if (dc->out_tokens) cudaFree(dc->out_tokens);
  if (dc->teacher) cudaFree(dc->teacher);
  if (dc->pf_buf) cudaFree(dc->pf_buf);
  for (cudaGraphExec_t e : dc->vf_exec)
    if (e) cudaGraphExecDestroy(e);
  if (dc->vf_buf) cudaFree(dc->vf_buf);
  if (dc->vf_io_host) cudaFreeHost(dc->vf_io_host);
  if (dc->st_host) cudaFreeHost(dc->st_host);
  if (dc->rec.id) cudaFree(dc->rec.id);
  if (dc->rec.lp) cudaFree(dc->rec.lp);
  if (dc->rec.top_ids) cudaFree(dc->rec.top_ids);
  if (dc->rec.top_lp) cudaFree(dc->rec.top_lp);
  if (dc->io_host) cudaFreeHost(dc->io_host);
  if (dc->stream_host) cudaFreeHost(dc->stream_host);
  if (dc->own_stream && dc->stream) cudaStreamDestroy(dc->stream);
  delete dc;
}

int kllm_decoder_step(kllm_decoder* dc, int32_t token_host, int32_t pos, int is_prompt,
                      int32_t* next_host) {
  if (!dc || !next_host) return KLLM_E_INVALID;
  if (pos < 0 || pos >= dc->m.seq_len) return KLLM_E_INVALID;
  // a prompt position needs no logits (llama3.cpp:738-739 returns -1): no record entry, and the persistent engine
  // skips the classifier
  KLLM_TRY(put_state(dc, token_host, pos, 0, 0, is_prompt ? 1 : 0, 0));
  KLLM_TRY(run_positions(dc, 1));
  KLLM_TRY(read_next(dc, next_host));
  if (is_prompt) *next_host = -1;
  return 0;
}

int kllm_decoder_prompt(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                        int32_t* next_host) {
  if (!dc || !tokens_host || !next_host || n_tokens <= 0 || start_pos < 0) return KLLM_E_INVALID;
  if (start_pos + n_tokens > dc->m.seq_len) return KLLM_E_INVALID;
  KLLM_TRY(put_teacher(dc, tokens_host, n_tokens));
  // teacher forced; only the last position records an entry (and, on the persistent engine, runs the classifier:
  // ONE launch for the whole prompt)
  KLLM_TRY(put_state(dc, tokens_host[0], start_pos, 1, 0, n_tokens - 1, 0));
  KLLM_TRY(run_positions(dc, n_tokens));
  return read_next(dc, next_host);
}

int kllm_decoder_prefill_tf32(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                              int32_t* next_host) {
  KLLM_TRY(prefill_args(dc, tokens_host, n_tokens, start_pos, next_host));
  const DecoderModel& m = dc->m;
  if (m.group_size != 0 || dc->d.tp_size > 1) return KLLM_E_UNSUPPORTED;  // fp32 checkpoints, one GPU
  // what kllm_gemm_bf16_tf32 takes (in_dim % 8 == 0), for every projection's in_dim; checked before any launch, so
  // a refused call leaves the cache and the history as they were
  if (m.format == WeightFormat::kBf16 && ((m.dim & 7) || (m.hidden_dim & 7) || (m.q_rows & 7)))
    return KLLM_E_UNSUPPORTED;
  return run_prefill(dc, tokens_host, n_tokens, start_pos, next_host);
}

int kllm_decoder_prefill_w8(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                            int32_t* next_host) {
  KLLM_TRY(prefill_args(dc, tokens_host, n_tokens, start_pos, next_host));
  const DecoderModel& m = dc->m;
  const int g = m.group_size;
  if (m.format != WeightFormat::kInt8 || dc->d.tp_size > 1) return KLLM_E_UNSUPPORTED;  // int8 checkpoints, one GPU
  // what kllm_gemm_w8_tf32 takes, for the in_dim of every projection (dim, q_rows, hidden_dim); checked before
  // any launch, so a refused call leaves the cache as it was
  if (g % 32) return KLLM_E_UNSUPPORTED;
  for (int k : {m.dim, m.q_rows, m.hidden_dim})
    if (k % 16 || k % g) return KLLM_E_UNSUPPORTED;
  return run_prefill(dc, tokens_host, n_tokens, start_pos, next_host);
}

int kllm_decoder_generate(kllm_decoder* dc, int32_t first_token, int32_t start_pos,
                          int32_t n_steps, const int32_t* teacher_host,
                          int32_t* out_tokens_host) {
  if (!dc || n_steps <= 0 || start_pos < 0) return KLLM_E_INVALID;
  if (start_pos + n_steps > dc->m.seq_len) return KLLM_E_INVALID;
  if (teacher_host) KLLM_TRY(put_teacher(dc, teacher_host, n_steps));
  KLLM_TRY(put_state(dc, teacher_host ? teacher_host[0] : first_token, start_pos, teacher_host != nullptr, 0, 0, 0));
  KLLM_TRY(run_positions(dc, n_steps));
  if (out_tokens_host) {
    KLLM_TRY(cudaMemcpyAsync(dc->io_host, dc->out_tokens, sizeof(int32_t) * n_steps,
                             cudaMemcpyDeviceToHost, dc->stream));
  }
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  if (out_tokens_host) std::memcpy(out_tokens_host, dc->io_host, sizeof(int32_t) * n_steps);
  return 0;
}

int kllm_decoder_generate_until(kllm_decoder* dc, int32_t first_token, int32_t start_pos, int32_t max_steps,
                                const int32_t* stop_ids, int32_t n_stop, kllm_token_callback on_tokens, void* ctx,
                                int32_t* out_tokens_host, int32_t* n_out) {
  // every refusal comes before the first launch, so a refused call leaves the decoder as it was
  KLLM_TRY(until_args(dc, start_pos, max_steps, stop_ids, n_stop, out_tokens_host, n_out));
  *n_out = 0;
  int32_t* count = dc->stream_host;
  const int32_t* ids = dc->stream_host + kStreamIds;
  __atomic_store_n(count, 0, __ATOMIC_SEQ_CST);  // before the launch that writes it
  KLLM_TRY(put_state(dc, first_token, start_pos, 0, 1, 0, 0));
  int32_t n = 0;
  if (dc->use_mega) {
    // One launch that stops on the device; the host hands over whatever ids the count says have arrived
    // until the stream is done.
    KLLM_TRY(dc->mega.run_until(dc->cfg, max_steps, stop_ids, n_stop, dc->stream_dev + kStreamIds, dc->stream_dev));
    int32_t delivered = 0;
    cudaError_t q = cudaErrorNotReady;
    while (on_tokens != nullptr && q == cudaErrorNotReady) {
      q = cudaStreamQuery(dc->stream);  // before the count: after a success the count is final
      const int32_t c = __atomic_load_n(count, __ATOMIC_ACQUIRE);
      if (c > delivered) {
        on_tokens(ctx, ids + delivered, c - delivered);
        delivered = c;
      }
    }
    const cudaError_t e = cudaMemcpyAsync(dc->st_host, dc->st, sizeof(mega::State), cudaMemcpyDeviceToHost, dc->stream);
    const cudaError_t s = cudaStreamSynchronize(dc->stream);
    if (e != cudaSuccess || s != cudaSuccess) return static_cast<int>(e != cudaSuccess ? e : s);
    n = dc->st_host->step;
    dc->mega.account(n);  // the tags and barriers of the positions that ran, not of max_steps
    if (on_tokens != nullptr && n > delivered) on_tokens(ctx, ids + delivered, n - delivered);
  } else {
    // One captured step per launch, driven from the host: wait for the step's id through the mapped count,
    // then stop or launch the next step.  No step runs after the stop, on any tensor-parallel rank.
    for (int i = 0; i < max_steps;) {
      KLLM_TRY(replay(dc->exec, dc->launches_per_step, 1, dc->stream));
      KLLM_TRY(wait_streamed(count, i, dc->stream));
      const int32_t id = ids[i++];
      if (on_tokens != nullptr) on_tokens(ctx, &id, 1);
      n = i;
      if (hits_stop(stop_ids, n_stop, id)) break;
    }
    KLLM_TRY(cudaStreamSynchronize(dc->stream));
  }
  std::memcpy(out_tokens_host, ids, sizeof(int32_t) * n);
  *n_out = n;
  return 0;
}

int kllm_decoder_verify(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                        int32_t* out_ids_host, int32_t* n_accepted) {
  // every refusal comes before the first launch, so a refused call leaves the decoder as it was
  if (!dc || !tokens_host || !out_ids_host || !n_accepted) return KLLM_E_INVALID;
  KLLM_TRY(verify_supported(dc));
  if (n_tokens < 1 || n_tokens > KLLM_MAX_VERIFY_TOKENS || start_pos < 0) return KLLM_E_INVALID;
  if (static_cast<int64_t>(start_pos) + n_tokens > dc->m.seq_len) return KLLM_E_INVALID;
  for (int32_t i = 0; i < n_tokens; ++i)
    if (tokens_host[i] < 0 || tokens_host[i] >= dc->m.vocab_size) return KLLM_E_INVALID;
  return run_verify(dc, tokens_host, n_tokens, start_pos, nullptr, 0, out_ids_host, n_accepted);
}

int kllm_batch_create(kllm_decoder* const* members, int32_t n, void* stream, kllm_batch** out) {
  // every refusal comes before the first launch, so a refused call leaves every member as it was
  if (!members || !out || n < 1 || n > KLLM_MAX_BATCH) return KLLM_E_INVALID;
  for (int32_t i = 0; i < n; ++i) {
    if (members[i] == nullptr) return KLLM_E_INVALID;
    for (int32_t j = 0; j < i; ++j)
      if (members[j] == members[i]) return KLLM_E_INVALID;
  }
  for (int32_t i = 0; i < n; ++i) {
    KLLM_TRY(verify_supported(members[i]));
    if (!same_model(members[0], members[i])) return KLLM_E_UNSUPPORTED;
  }
  auto* b = new kllm_batch();
  b->members.assign(members, members + n);
  auto fail = [&](int rc) {
    kllm_batch_destroy(b);
    return rc;
  };
  if (stream != nullptr) {
    b->stream = static_cast<cudaStream_t>(stream);
  } else {
    if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(KLLM_E_NODEVICE);
    b->own_stream = true;
  }
  for (kllm_decoder* dc : b->members)
    if (const cudaError_t e = cudaStreamSynchronize(dc->stream)) return fail(static_cast<int>(e));
  if (const int rc = batch_prepare(b)) return fail(rc);
  *out = b;
  return 0;
}

void kllm_batch_destroy(kllm_batch* b) {
  if (!b) return;
  if (b->stream) cudaStreamSynchronize(b->stream);
  for (cudaGraphExec_t e : b->exec)
    if (e) cudaGraphExecDestroy(e);
  for (cudaGraphExec_t e : b->beam_exec)
    if (e) cudaGraphExecDestroy(e);
  if (b->cand_host) cudaFreeHost(b->cand_host);
  if (b->buf) cudaFree(b->buf);
  if (b->tables) cudaFree(b->tables);
  if (b->tables_host) cudaFreeHost(b->tables_host);
  if (b->io_host) cudaFreeHost(b->io_host);
  if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
  delete b;
}

int kllm_batch_step(kllm_batch* b, const int32_t* tokens_host, const int32_t* pos_host, int32_t* next_host) {
  return run_batch(b, tokens_host, pos_host, 1, next_host);
}

int kllm_batch_generate(kllm_batch* b, const int32_t* first_tokens_host, const int32_t* start_pos_host,
                        int32_t n_steps, int32_t* out_tokens_host) {
  return run_batch(b, first_tokens_host, start_pos_host, n_steps, out_tokens_host);
}

int kllm_batch_generate_until(kllm_batch* b, const int32_t* first_tokens_host, const int32_t* start_pos_host,
                              const int32_t* max_steps_host, const int32_t* stop_ids_host, const int32_t* n_stop_host,
                              kllm_batch_token_callback on_tokens, void* ctx, int32_t* out_tokens_host,
                              int32_t* n_out_host, kllm_batch_stats* stats) {
  // every refusal comes before the first launch, so a refused call leaves every member as it was
  if (!b || !first_tokens_host || !start_pos_host || !max_steps_host || !stop_ids_host || !n_stop_host ||
      !out_tokens_host || !n_out_host)
    return KLLM_E_INVALID;
  const DecoderModel& m = b->members[0]->m;
  for (size_t i = 0; i < b->members.size(); ++i) {
    const int32_t first = first_tokens_host[i], start = start_pos_host[i], steps = max_steps_host[i];
    if (first < 0 || first >= m.vocab_size || start < 0 || steps <= 0) return KLLM_E_INVALID;
    if (static_cast<int64_t>(start) + steps > m.seq_len) return KLLM_E_INVALID;
    KLLM_TRY(stop_args(stop_ids_host + i * KLLM_MAX_STOP_IDS, n_stop_host[i], m.vocab_size));
  }
  return run_batch_until(b, first_tokens_host, start_pos_host, max_steps_host, stop_ids_host, n_stop_host, on_tokens,
                         ctx, out_tokens_host, n_out_host, stats);
}

int kllm_batch_beam_search(kllm_batch* b, int32_t first_token, int32_t start_pos, int32_t max_new_tokens,
                           const int32_t* eos_ids, int32_t n_eos, float length_penalty, int32_t early_stopping,
                           int32_t n_return, int32_t* out_ids_host, int32_t* out_len_host, float* out_score_host,
                           float* out_sum_host, kllm_beam_stats* stats) {
  // every refusal comes before the first launch, so a refused call leaves every member as it was
  if (!b || !out_ids_host || !out_len_host || !out_score_host || !out_sum_host) return KLLM_E_INVALID;
  const DecoderModel& m = b->members[0]->m;
  const int B = static_cast<int>(b->members.size());
  if (first_token < 0 || first_token >= m.vocab_size || start_pos < 0 || max_new_tokens <= 0) return KLLM_E_INVALID;
  if (static_cast<int64_t>(start_pos) + max_new_tokens > m.seq_len) return KLLM_E_INVALID;
  if (n_eos < 0 || n_eos > KLLM_MAX_BEAM_EOS || (n_eos > 0 && eos_ids == nullptr)) return KLLM_E_INVALID;
  for (int32_t i = 0; i < n_eos; ++i)
    if (eos_ids[i] < 0 || eos_ids[i] >= m.vocab_size) return KLLM_E_INVALID;
  if (n_return < 1 || n_return > B || !std::isfinite(length_penalty)) return KLLM_E_INVALID;
  if (early_stopping < KLLM_BEAM_EARLY_HEURISTIC || early_stopping > KLLM_BEAM_EARLY_NEVER) return KLLM_E_INVALID;
  // the rule is over the raw logits: a member that would draw or adjust them is refused, not silently ignored
  for (const kllm_decoder* dc : b->members)
    if (dc->cfg.sample.temperature != 0.f || sampling::step0_active(dc->cfg.penalty)) return KLLM_E_UNSUPPORTED;
  if (static_cast<int64_t>(m.vocab_size) < static_cast<int64_t>(std::max(2, 1 + n_eos)) * B) return KLLM_E_UNSUPPORTED;
  return run_batch_beam(b, first_token, start_pos, max_new_tokens, eos_ids, n_eos, length_penalty, early_stopping,
                        n_return, out_ids_host, out_len_host, out_score_host, out_sum_host, stats);
}

int kllm_decoder_copy_prefix(kllm_decoder* dst, const kllm_decoder* src, int32_t n_pos) {
  // every refusal comes before the first launch, so a refused call copies nothing
  if (!dst || !src || dst == src || n_pos < 0) return KLLM_E_INVALID;
  if (dst->d.tp_size > 1 || src->d.tp_size > 1 || !same_model(dst, src) || dst->d.kv_cache != src->d.kv_cache ||
      dst->kv_scales != src->kv_scales)
    return KLLM_E_UNSUPPORTED;
  const DecoderModel& m = dst->m;
  if (n_pos > m.seq_len) return KLLM_E_INVALID;
  KLLM_TRY(cudaStreamSynchronize(src->stream));
  if (n_pos == 0) return 0;
  const prefill::CacheLayout c = decoder_cache(dst).cache;
  const dim3 grid(n_pos, m.layer_num);
  cudaStream_t s = dst->stream;
  if (c.elem == KLLM_KV_FP8) {
    copy_prefix_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src->kcache),
                                            reinterpret_cast<const uint8_t*>(src->vcache),
                                            reinterpret_cast<uint8_t*>(dst->kcache),
                                            reinterpret_cast<uint8_t*>(dst->vcache), c);
  } else if (c.elem == KLLM_KV_BF16) {
    copy_prefix_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint16_t*>(src->kcache),
                                            reinterpret_cast<const uint16_t*>(src->vcache),
                                            reinterpret_cast<uint16_t*>(dst->kcache),
                                            reinterpret_cast<uint16_t*>(dst->vcache), c);
  } else {
    copy_prefix_kernel<<<grid, 256, 0, s>>>(src->kcache, src->vcache, dst->kcache, dst->vcache, c);
  }
  count_launch();
  KLLM_TRY(cudaGetLastError());
  // the history and the record entries of the same positions
  const size_t P = n_pos, T = P * sampling::kMaxTopLogprobs;
  KLLM_TRY(cudaMemcpyAsync(dst->hist, src->hist, sizeof(int32_t) * P, cudaMemcpyDeviceToDevice, s));
  KLLM_TRY(cudaMemcpyAsync(dst->rec.id, src->rec.id, sizeof(int32_t) * P, cudaMemcpyDeviceToDevice, s));
  KLLM_TRY(cudaMemcpyAsync(dst->rec.lp, src->rec.lp, sizeof(float) * P, cudaMemcpyDeviceToDevice, s));
  KLLM_TRY(cudaMemcpyAsync(dst->rec.top_ids, src->rec.top_ids, sizeof(int32_t) * T, cudaMemcpyDeviceToDevice, s));
  KLLM_TRY(cudaMemcpyAsync(dst->rec.top_lp, src->rec.top_lp, sizeof(float) * T, cudaMemcpyDeviceToDevice, s));
  // src may change as soon as this returns
  return static_cast<int>(cudaStreamSynchronize(s));
}

int kllm_decoder_generate_speculative(kllm_decoder* dc, int32_t first_token, int32_t start_pos, int32_t max_steps,
                                      const int32_t* stop_ids, int32_t n_stop, int32_t draft_len, int32_t ngram_max,
                                      kllm_token_callback on_tokens, void* ctx, int32_t* out_tokens_host,
                                      int32_t* n_out, kllm_spec_stats* stats) {
  // every refusal comes before the first launch, so a refused call leaves the decoder as it was
  KLLM_TRY(until_args(dc, start_pos, max_steps, stop_ids, n_stop, out_tokens_host, n_out));
  if (draft_len < 1 || draft_len >= KLLM_MAX_VERIFY_TOKENS || ngram_max < 1 || ngram_max > 8) return KLLM_E_INVALID;
  if (first_token < 0 || first_token >= dc->m.vocab_size) return KLLM_E_INVALID;
  KLLM_TRY(verify_supported(dc));
  *n_out = 0;
  if (stats) *stats = kllm_spec_stats{0, 0, 0};
  // c: the history up to the next position, then the id fed there; the drafts are looked up in it
  std::vector<int32_t> c(static_cast<size_t>(start_pos) + max_steps + 1);
  if (start_pos > 0) {
    KLLM_TRY(cudaMemcpyAsync(dc->io_host, dc->hist, sizeof(int32_t) * start_pos, cudaMemcpyDeviceToHost, dc->stream));
    KLLM_TRY(cudaStreamSynchronize(dc->stream));
    std::memcpy(c.data(), dc->io_host, sizeof(int32_t) * start_pos);
  }
  c[start_pos] = first_token;
  int32_t produced = 0;
  int32_t tokens[KLLM_MAX_VERIFY_TOKENS], ids[KLLM_MAX_VERIFY_TOKENS];
  while (produced < max_steps) {
    const int p = start_pos + produced;
    const int m = std::min({draft_len, max_steps - produced - 1, dc->m.seq_len - p - 1});
    const int k = lookup_draft(c.data(), p + 1, ngram_max, m, tokens + 1);
    int32_t a = 0;
    if (k == 0) {  // no draft: one plain step on the decoder's engine
      KLLM_TRY(put_state(dc, c[p], p, 0, 0, 0, 0));
      KLLM_TRY(run_positions(dc, 1));
      KLLM_TRY(read_next(dc, &ids[0]));
    } else {
      tokens[0] = c[p];
      KLLM_TRY(run_verify(dc, tokens, k + 1, p, stop_ids, n_stop, ids, &a));
    }
    if (stats) stats->rounds += 1, stats->drafted += k, stats->accepted += a;
    if (on_tokens != nullptr) on_tokens(ctx, ids, a + 1);
    std::memcpy(out_tokens_host + produced, ids, sizeof(int32_t) * (a + 1));
    std::memcpy(c.data() + p + 1, ids, sizeof(int32_t) * (a + 1));
    produced += a + 1;
    if (hits_stop(stop_ids, n_stop, ids[a])) break;
  }
  *n_out = produced;
  return 0;
}

int kllm_decoder_set_sampling(kllm_decoder* dc, float temperature, int32_t top_k, uint64_t seed) {
  return kllm_decoder_set_sampling_top_p(dc, temperature, top_k, 1.f, seed);
}

int kllm_decoder_set_sampling_top_p(kllm_decoder* dc, float temperature, int32_t top_k, float top_p, uint64_t seed) {
  if (!dc || !std::isfinite(temperature) || temperature < 0.f || !(top_p > 0.f && top_p <= 1.f)) return KLLM_E_INVALID;
  DrawSettings next = dc->cfg;
  next.sample = SampleParams{temperature, top_k, seed, top_p};
  return put_settings(dc, next);
}

int kllm_decoder_set_repetition_penalty(kllm_decoder* dc, float penalty, int32_t last_n) {
  if (!dc || !std::isfinite(penalty) || !(penalty > 0.f) || last_n < 0) return KLLM_E_INVALID;
  DrawSettings next = dc->cfg;
  next.penalty.penalty = penalty, next.penalty.last_n = last_n;
  return put_settings(dc, next);
}

int kllm_decoder_set_frequency_presence(kllm_decoder* dc, float frequency, float presence, int32_t from_pos) {
  if (!dc || !std::isfinite(frequency) || !std::isfinite(presence) || from_pos < 0) return KLLM_E_INVALID;
  DrawSettings next = dc->cfg;
  next.penalty.frequency = frequency == 0.f ? 0.f : frequency;  // -0.0 is off, as 0
  next.penalty.presence = presence == 0.f ? 0.f : presence;
  next.penalty.from_pos = from_pos;
  return put_settings(dc, next);
}

int kllm_decoder_set_logit_bias(kllm_decoder* dc, const int32_t* ids_host, const float* bias_host, int32_t n) {
  if (!dc || n < 0 || (n > 0 && (!ids_host || !bias_host))) return KLLM_E_INVALID;
  const int V = dc->m.vocab_size;
  std::vector<float> table;
  if (n > 0) {
    std::vector<char> seen(V, 0);
    table.assign(V, 0.f);
    for (int32_t k = 0; k < n; ++k) {
      const int32_t id = ids_host[k];
      if (id < 0 || id >= V || seen[id] || !std::isfinite(bias_host[k])) return KLLM_E_INVALID;
      seen[id] = 1;
      table[id] = 0.f + bias_host[k];  // HF's table: 0 + b, so a -0.0 bias adds +0.0
    }
  }
  DrawSettings next = dc->cfg;
  next.penalty.bias = n > 0 ? dc->bias : nullptr;
  // no step may still be reading the old table
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  if (n > 0) KLLM_TRY(cudaMemcpy(dc->bias, table.data(), sizeof(float) * V, cudaMemcpyHostToDevice));
  return put_settings(dc, next);
}

int kllm_decoder_set_logprobs(kllm_decoder* dc, int32_t top_n) {
  if (!dc || top_n < -1 || top_n > KLLM_MAX_TOP_LOGPROBS) return KLLM_E_INVALID;
  static_assert(sampling::kMaxTopLogprobs == KLLM_MAX_TOP_LOGPROBS, "one top-N capacity");
  DrawSettings next = dc->cfg;
  next.lp_top_n = top_n;
  KLLM_TRY(clear_record(dc));  // in stream order, behind every step that may still write the record
  return put_settings(dc, next);
}

int kllm_decoder_read_logprobs(kllm_decoder* dc, int32_t start_pos, int32_t n, int32_t* ids_host, float* lp_host,
                               int32_t* top_ids_host, float* top_lp_host) {
  if (!dc || !ids_host || !lp_host || start_pos < 0 || n < 0) return KLLM_E_INVALID;
  if (static_cast<int64_t>(start_pos) + n > dc->m.seq_len) return KLLM_E_INVALID;
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  if (n == 0) return 0;
  KLLM_TRY(cudaMemcpy(ids_host, dc->rec.id + start_pos, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  KLLM_TRY(cudaMemcpy(lp_host, dc->rec.lp + start_pos, sizeof(float) * n, cudaMemcpyDeviceToHost));
  const int N = dc->cfg.lp_top_n;
  if (N <= 0 || (!top_ids_host && !top_lp_host)) return 0;
  constexpr int K = sampling::kMaxTopLogprobs;
  const size_t row0 = static_cast<size_t>(start_pos) * K, rows = static_cast<size_t>(n) * K;
  std::vector<int32_t> ti(rows);
  std::vector<float> tl(rows);
  KLLM_TRY(cudaMemcpy(ti.data(), dc->rec.top_ids + row0, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost));
  KLLM_TRY(cudaMemcpy(tl.data(), dc->rec.top_lp + row0, sizeof(float) * rows, cudaMemcpyDeviceToHost));
  for (int32_t i = 0; i < n; ++i)
    for (int r = 0; r < N; ++r) {
      if (top_ids_host) top_ids_host[static_cast<size_t>(i) * N + r] = ti[static_cast<size_t>(i) * K + r];
      if (top_lp_host) top_lp_host[static_cast<size_t>(i) * N + r] = tl[static_cast<size_t>(i) * K + r];
    }
  return 0;
}

int kllm_decoder_score(kllm_decoder* dc, const int32_t* tokens_host, int32_t n_tokens, int32_t start_pos,
                       float* lp_host) {
  // every refusal comes before the first launch
  if (!dc || !tokens_host || !lp_host || n_tokens < 2 || start_pos < 0) return KLLM_E_INVALID;
  if (static_cast<int64_t>(start_pos) + n_tokens > dc->m.seq_len) return KLLM_E_INVALID;
  for (int32_t i = 0; i < n_tokens; ++i)
    if (tokens_host[i] < 0 || tokens_host[i] >= dc->m.vocab_size) return KLLM_E_INVALID;
  const int steps = n_tokens - 1;
  // the targets: the teacher holds all n tokens, one more than the positions run, so step i's target is [i + 1]
  KLLM_TRY(put_teacher(dc, tokens_host, n_tokens));
  KLLM_TRY(put_state(dc, tokens_host[0], start_pos, 1, 0, 0, 1));
  KLLM_TRY(run_positions(dc, steps));
  KLLM_TRY(cudaMemcpyAsync(dc->io_host, dc->rec.lp + start_pos, sizeof(float) * steps, cudaMemcpyDeviceToHost,
                           dc->stream));
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  std::memcpy(lp_host, dc->io_host, sizeof(float) * steps);
  return 0;
}

int kllm_decoder_profile(kllm_decoder* dc, int32_t first_token, int32_t start_pos, int32_t n_steps,
                         int32_t profiled_step, uint64_t* stamps_host, int32_t capacity,
                         int32_t* grid_out, int32_t* phases_out) {
  if (!dc || !stamps_host || !grid_out || !phases_out || n_steps <= 0) return KLLM_E_INVALID;
  // no timeline kernel for the bf16 or fp8 cache or bf16 weights
  if (!dc->use_mega || dc->d.kv_cache != KLLM_KV_F32 || dc->m.format == WeightFormat::kBf16) return KLLM_E_UNSUPPORTED;
  if (start_pos < 0 || start_pos + n_steps > dc->m.seq_len) return KLLM_E_INVALID;
  const int grid = dc->mega.grid(), phases = dc->mega.phases();
  const size_t n = static_cast<size_t>(grid) * phases * mega::kProfStamps;
  *grid_out = grid;
  *phases_out = phases;
  if (static_cast<size_t>(capacity) < n) return KLLM_E_INVALID;
  KLLM_TRY(put_state(dc, first_token, start_pos, 0, 0, 0, 0));
  unsigned long long* d_prof = nullptr;
  KLLM_TRY(cudaMalloc(&d_prof, n * sizeof(unsigned long long)));
  int rc = static_cast<int>(cudaMemsetAsync(d_prof, 0, n * sizeof(unsigned long long), dc->stream));
  if (rc == 0) rc = dc->mega.run(dc->cfg, n_steps, nullptr, d_prof, profiled_step);
  if (rc == 0) rc = static_cast<int>(cudaStreamSynchronize(dc->stream));
  if (rc == 0)
    rc = static_cast<int>(cudaMemcpy(stamps_host, d_prof, n * sizeof(unsigned long long),
                                     cudaMemcpyDeviceToHost));
  cudaFree(d_prof);
  return rc;
}

int kllm_decoder_logits(kllm_decoder* dc, float* logits_host) {
  if (!dc || !logits_host) return KLLM_E_INVALID;
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  return static_cast<int>(cudaMemcpy(logits_host, dc->logits, sizeof(float) * dc->m.vocab_size,
                                     cudaMemcpyDeviceToHost));
}

const float* kllm_decoder_logits_device(const kllm_decoder* dc) { return dc ? dc->logits : nullptr; }

int kllm_decoder_read_kv(kllm_decoder* dc, float* key_host, float* value_host) {
  if (!dc || !key_host || !value_host) return KLLM_E_INVALID;
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  const DecoderModel& m = dc->m;
  const size_t S = m.seq_len, kvd = m.kv_dim, hs = m.head_size, layer = S * kvd, n = m.layer_num * layer;
  // each layer in the engine's layout -> reference [L][S][kv_dim], a bf16 element widened exactly, an fp8 one as
  // fp32(value(code) * s) at its layer's and kv head's scale s
  const prefill::CacheLayout c = decoder_cache(dc).cache;
  const size_t esz = prefill::kv_elem_bytes(c.elem);
  std::vector<unsigned char> kraw(n * esz), vraw(n * esz);
  KLLM_TRY(cudaMemcpy(kraw.data(), dc->kcache, n * esz, cudaMemcpyDeviceToHost));
  KLLM_TRY(cudaMemcpy(vraw.data(), dc->vcache, n * esz, cudaMemcpyDeviceToHost));
  auto at = [&](const std::vector<unsigned char>& raw, size_t i) {
    uint32_t u = 0;
    if (c.elem == KLLM_KV_FP8) return e4m3_value_host(raw[i]);
    if (c.elem == KLLM_KV_BF16) {
      uint16_t b;
      std::memcpy(&b, raw.data() + 2 * i, sizeof(b));
      u = static_cast<uint32_t>(b) << 16;
    } else {
      std::memcpy(&u, raw.data() + 4 * i, sizeof(u));
    }
    float f;
    std::memcpy(&f, &u, sizeof(f));
    return f;
  };
  const size_t nh = static_cast<size_t>(m.layer_num) * m.kv_head_num;
  for (size_t l = 0; l < static_cast<size_t>(m.layer_num); ++l)
    for (int t = 0; t < m.seq_len; ++t)
      for (int g = 0; g < m.kv_head_num; ++g) {
        float sk = 1.f, sv = 1.f;
        if (c.elem == KLLM_KV_FP8) sk = dc->kv_scales[l * m.kv_head_num + g], sv = dc->kv_scales[nh + l * m.kv_head_num + g];
        for (int i = 0; i < m.head_size; ++i) {
          const size_t dst = (l * S + t) * kvd + g * hs + i;
          const float k = at(kraw, l * layer + prefill::k_index(c, t, g, i));
          const float v = at(vraw, l * layer + prefill::v_index(c, t, g, i));
          key_host[dst] = c.elem == KLLM_KV_FP8 ? k * sk : k;
          value_host[dst] = c.elem == KLLM_KV_FP8 ? v * sv : v;
        }
      }
  return 0;
}

int kllm_decoder_read_history(kllm_decoder* dc, int32_t* ids_host) {
  if (!dc || !ids_host) return KLLM_E_INVALID;
  KLLM_TRY(cudaStreamSynchronize(dc->stream));
  return static_cast<int>(cudaMemcpy(ids_host, dc->hist, sizeof(int32_t) * dc->m.seq_len, cudaMemcpyDeviceToHost));
}

int kllm_decoder_launches_per_step(const kllm_decoder* dc) { return dc ? dc->launches_per_step : 0; }
int kllm_decoder_classifier_rows(const kllm_decoder* dc) {
  if (!dc) return 0;
  return dc->use_mega ? dc->mega.cls_rows() : dc->m.vocab_size;
}
const char* kllm_decoder_engine(const kllm_decoder* dc) {
  if (!dc) return "";
  return dc->use_mega ? "persistent" : "graph";
}
int kllm_decoder_attention_geometry(const kllm_decoder* dc, int* tile, int* split, int* tile_v, int* stage_bytes) {
  if (!dc || !tile || !split || !tile_v || !stage_bytes) return KLLM_E_INVALID;
  if (!dc->use_mega) return KLLM_E_UNSUPPORTED;
  *tile = dc->mega.attn_tile();
  *split = dc->mega.attn_split();
  *tile_v = dc->mega.attn_tile_v();
  *stage_bytes = dc->mega.stage_bytes();
  return 0;
}

}  // extern "C"
