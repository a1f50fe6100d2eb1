// Host/device shared declarations of the persistent decode megakernel (megakernel.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "decoder_model.h"
#include "sampling.cuh"

namespace kllm {
namespace mega {

enum {
  kPhaseGemv = 0,
  kPhaseAttention = 1 /* scores of the split attention */,
  kPhaseAttnPV = 2 /* softmax + P.V of the split attention */,
  kPhaseAttnFused = 3 /* whole attention of one head in one CTA (attn_split == 1) */,
  kPhaseAttnFlash = 4 /* toleranced: split by timestep, online softmax, partials merged by CTA 0 of the head */,
  kPhaseGather = 5 /* tensor parallel, classifier sharded by vocabulary: collect every rank's logits, argmax partials */
};
constexpr int kProfStamps = 16;  // uint64 stamps per (CTA, phase) of kllm_decoder_profile
constexpr int kMaxStopIds = 16;  // == KLLM_MAX_STOP_IDS

struct Seg {
  const void* w;        // fp32 or int8 [rows, in_dim]
  const float* scales;  // int8 only
  const float* bias;    // optional
  float* out;           // out[pos * pos_stride + row]
  long long pos_stride;
  int rows;
  int head_major;       // 1: out is the head-major value cache, index ((row/hs)*seq_len + pos)*hs + row%hs
  // optional local hand-off: row r is (also) published as a tagged 64-bit word at tag_out[r] for
  // the next phase to poll (out may then be null)
  unsigned long long* tag_out;
};

// One entry of the per-token schedule.  A GEMV phase's units (rows, or w1/w3 row pairs) are
// split evenly over the CTAs; each CTA streams its contiguous share through the stage ring.
struct Phase {
  int kind;
  int in_dim;
  int units;
  int n_seg;
  int swiglu;             // units are (w1 row, w3 row) pairs -> SiLU*gate epilogue
  int argmax;             // track (max, index) of the produced rows (classifier)
  int cls;                // classifier work: skipped for prompt positions (llama3.cpp:733-745 discards their logits)
  int group_size, group_shift;
  int rows_per_stage;     // whole rows per ring stage (chunks_per_row == 1)
  int chunks_per_row;     // > 1: a row spans this many stages (fp32 rows longer than a stage)
  int chunk_elems;
  int scale_off;          // byte offset of the scales region inside a stage (int8)
  int scale_row_bytes;
  int layer;              // attention: layer index
  float norm_eps;
  const float* norm_w;    // optional RMSNorm weight applied to the input vector
  // The input vector is the residual stream (tp_in), the previous phase's output (tag_in) or, when
  // neither is set (the QKV phase of layer 0), the embedding row of the current token.
  // Tagged exchange (replaces the grid barrier AND, under tensor parallelism, the all-reduce):
  //   tp_out: each produced row is published as {value, tag} -- one 64-bit store -- into every
  //           rank's exchange area instead of seg[0].out; no residual add, no barrier after.
  //   tp_in : the input vector is x_old + (p_0 + p_1 + ... + p_{world-1}), p_r = rank r's tagged
  //           partials of exchange `exch`, polled until their tag is current; x_old is the CTA's
  //           own shared-memory copy of the residual stream (it starts as the embedding row of the
  //           token and is updated by every exchange), so the stream never round-trips through
  //           global memory between CTAs.
  int tp_in, tp_out;
  int exch;      // index (within the token) of the exchange tp_in consumes
  int exch_out;  // ... of the exchange tp_out publishes (a phase may do both: the sharded classifier)
  // Local tagged hand-offs (same words, one rank): the phase's input vector is polled from tag_in
  // (GEMV) or tq/tk/tv (attention: this head's query, its kv head's raw key and value rows);
  // outputs go to seg[].tag_out (GEMV) or ta (attention).  hand_in / hand_out number the
  // hand-offs of a token for the tags.
  const unsigned long long* tag_in;
  const unsigned long long* tq;
  const unsigned long long* tk;
  const unsigned long long* tv;
  unsigned long long* ta;
  int hand_in, hand_out;
  int hand_aux;           // attention P.V phase: the q|k|v hand-off (value row of the current position)
  Seg seg[3];
};

// The device-resident step state of both engines: the loop state, then the mode of the entry that uploaded it.
// The persistent engine reads and writes the first four fields only; it takes the mode in its launch parameters.
struct State {
  int32_t token;  // input token of the current step
  int32_t pos;    // position of the current step
  int32_t step;   // steps done since the entry started
  int32_t next;   // id produced by the last step
  // the graph engine's per-entry switches (argmax_advance_kernel), written by the host only
  int32_t teacher;    // feed teacher[step + 1] instead of the id
  int32_t streamed;   // publish the id, then the count, to mapped host memory (kllm_decoder_generate_until)
  int32_t lp_from;    // the first step that writes a record entry: the steps before it are prompt positions
  int32_t lp_target;  // kllm_decoder_score: the entry's id is teacher[step + 1], recorded with top_n max(top_n, 0)
};

struct Params {
  const Phase* phases;
  int n_phases, n_tokens;
  int attn_vsplit;      // V cache layout [L][kv_head][attn_vsplit][seq_len][head_size / attn_vsplit]
  int int8_fast;       // int8 weights: 1 = fixed-point activations on dp4a (toleranced), 0 = the reference's per-element order
  int n_cls_phases;     // trailing phases that make up the classifier (1, or 2 with the vocabulary-sharded form)
  int skip_cls_tokens;  // the first skip_cls_tokens positions of this launch are prompt tokens: no classifier pass
  int num_stages, stage_bytes, xbuf_bytes;
  int xres_bytes;  // shared-memory copy of the residual stream behind the input vector
  int attn_tile;    // timesteps per K ring stage
  int attn_tile_v;  // timesteps per V ring stage (rows of head_size / attn_split floats)
  unsigned long long* scores;  // [head][seq_len] tagged scaled scores: scores phase -> P.V phase
  int attn_split;   // CTAs per query head: K tiles round-robin, P.V output dims split (bit-exact chains)
  int group_size;
  int dim, vocab_size, head_num, head_size, kv_dim, kv_mul, seq_len, flavour;
  const float* tok_emb;
  float* score;
  // [head][attn_split][seq_len]: the split P.V phase's probabilities when they do not fit shared memory, one row
  // per CTA (each CTA's softmax runs in place, so the SP CTAs of a head cannot share a row)
  float* probs;
  // KV cache in the persistent engine's own layout (see megakernel.cu "KV layout"):
  //   K [L][kv_head][head_size/4][seq_len][4]    V [L][kv_head][attn_split][seq_len][head_size/attn_split]
  // KLLM_KV_BF16 (flash form only): both caches hold bf16 elements behind these pointers,
  //   K [L][kv_head][head_size/8][seq_len][8]    V [L][kv_head][seq_len][head_size]
  // KLLM_KV_FP8 (flash form only): e4m3 codes, K [L][kv_head][head_size/16][seq_len][16], V as bf16's
  float* key_cache;
  const float* value_cache;
  const float* sin_cache;
  const float* cos_cache;
  State* state;
  int32_t* out_tokens;
  const int32_t* teacher;
  int max_steps;
  unsigned* barrier;
  // one grid barrier per token: token tok of this launch passes it when *barrier reaches barrier_base + (tok + 1) * grid
  unsigned barrier_base;
  // tagged exchange areas: tp_data[r] = rank r's area [2 slots][tp_world][tp_stride] of 64-bit
  // {tag:32 | fp32 bits:32}; tp_data[tp_rank] is local memory, the others NVLink peer mappings
  unsigned long long* tp_data[8];
  int tp_world, tp_rank, tp_stride, exch_per_token;
  unsigned tp_seq_base;
  unsigned hand_base;
  int hands_per_token;
  float* arg_val;
  int* arg_idx;
  const SampleParams* sampling;  // read when a token's id is drawn: changing it needs no new engine
  const float* logits;           // [vocab]: complete once the classifier's grid barrier is passed
  // Step 0 of the rule (sampling.cuh: logit bias, repetition, frequency and presence penalties): the settings of
  // this launch (a copy of the decoder's, which change only between launches, with its bias table and mark words),
  // hist[seq_len] the id fed at each position, penalized[vocab] the adjusted logits, complete behind the same
  // barrier as `logits` when step 0 is on.
  PenaltyParams penalty;
  int32_t* hist;
  float* penalized;
  // Stoppable run (kllm_decoder_generate_until): the run ends after the first token whose id is one of
  // stop_ids (unused entries are -1, so a run without stop ids compares against nothing), and each id is
  // also published to stream_ids[step] followed by stream_count = step + 1 (mapped host memory; null: off).
  int stop_ids[kMaxStopIds];
  int32_t* stream_ids;
  int32_t* stream_count;
  // optional phase timeline of one token: prof[(cta * n_phases + phase) * 4 + k], k = phase
  // entered / input staged / last stage consumed / grid barrier passed (globaltimer ns)
  unsigned long long* prof;
  int prof_token;
  // Log-probabilities (sampling.cuh, DESIGN.md 5.8).  lp_top_n -1 is off; else each CTA leaves its part's (m_c, S_c)
  // in lp_part and, for lp_top_n > 0, its top-N in lp_cand_v / lp_cand_i [grid][kMaxTopLogprobs]; CTA 0 folds them
  // behind the token's grid barrier into the record.  lp_target 1: the entry's id is teacher[step + 1].
  int lp_top_n, lp_target;
  float2* lp_part;
  float* lp_cand_v;
  int* lp_cand_i;
  sampling::LogprobRecord lp_rec;
  // the fp8 KV cache's scales (kv8_megakernel; null otherwise), each [L][kv_head]: s_k, s_v and their fp32 inverses
  const float* kv_scale_k;
  const float* kv_scale_v;
  const float* kv_inv_k;
  const float* kv_inv_v;
};

}  // namespace mega

// What the engine needs besides the model (DecoderModel): all pointers are device pointers, the buffers the decoder owns.
struct MegaModel {
  float* logits; float* score;
  float* key_cache; float* value_cache;
  const float* sin_cache; const float* cos_cache;
  mega::State* state;
  int32_t* out_tokens;
  const SampleParams* sampling;  // the sampling part of the decoder's device DrawSettings
  int32_t* hist;
  float* penalized;
  sampling::LogprobRecord lp_rec;
  // tensor parallel (tp_world > 1): exchange areas of every rank (kllm_comm, CUDA IPC)
  int tp_world, tp_rank;
  unsigned long long* tp_data[8];
  int tp_stride;
  int numerics;  // kllm_decoder_desc::numerics
  int kv_cache;  // kllm_decoder_desc::kv_cache: KLLM_KV_BF16 and KLLM_KV_FP8 need the fast numerics (flash attention)
  const float* kv_scales;  // KLLM_KV_FP8: device [4][L][kv_head], s_k, s_v, 1 / s_k, 1 / s_v
};

class MegaEngine {
 public:
  // Every refusal (KLLM_E_INVALID, KLLM_E_UNSUPPORTED, KLLM_E_NODEVICE) comes before the one allocation: an engine
  // that refuses holds nothing.  `dm` and `m` are read here only.
  int init(const DecoderModel& dm, const MegaModel& m, cudaStream_t stream);
  int destroy();  // the status of freeing the scratch block
  // Run n_tokens consecutive positions starting from the device-resident state, under the decoder's settings
  // `cfg` (its step 0 and logprob setting ride in the launch parameters; the sampling parameters are read through
  // MegaModel::sampling).  lp_target: kllm_decoder_score's run, whose record entries hold teacher[step + 1]
  // (cfg.lp_top_n >= 0, so that they are written even with logprobs off)
  int run(const DrawSettings& cfg, int n_tokens, const int32_t* teacher_dev, unsigned long long* prof_dev = nullptr,
          int prof_token = -1, int skip_cls_tokens = 0, int lp_target = 0);
  // Up to n_tokens positions, ending after the first id in stop_ids[0 .. n_stop); every id is streamed to
  // stream_ids / stream_count (device-visible pointers into mapped host memory).  The number of positions
  // that ran is known only once the launch has finished, so the tag and barrier bases are NOT advanced
  // here: the caller passes that number (state.step) to account() before the next launch.
  int run_until(const DrawSettings& cfg, int n_tokens, const int32_t* stop_ids, int n_stop, int32_t* stream_ids,
                int32_t* stream_count);
  void account(int n_tokens);
  int grid() const { return grid_; }
  int phases() const { return base_.n_phases; }
  int attn_vsplit() const { return base_.attn_vsplit; }  // slices of the V cache layout
  int fast() const { return fast_; }                     // numerics: 1 = toleranced (free summation order)
  int attn_tile() const { return base_.attn_tile; }      // timesteps per K (flash: K and V) ring stage
  int attn_split() const { return base_.attn_split; }    // CTAs per query head
  int attn_tile_v() const { return base_.attn_tile_v; }  // timesteps per V ring stage
  int stage_bytes() const { return base_.stage_bytes; }
  int cls_rows() const { return cls_rows_; }  // classifier rows this rank streams per token

 private:
  mega::Params params(const DrawSettings& cfg, int n_tokens) const;
  int launch(const mega::Params& P);
  mega::Params base_{};  // every launch parameter that stays the same from launch to launch
  // hand-off words, score words, exchange area (one GPU), phase table, barrier word, argmax and logprob partials
  void* scratch_ = nullptr;
  cudaStream_t stream_ = nullptr;
  unsigned barrier_base_ = 0, tp_seq_base_ = 0, hand_base_ = 0;
  int grid_ = 0;
  int fast_ = 0;  // numerics: 0 = bit-exact with the reference, 1 = toleranced (free summation order)
  int cls_rows_ = 0;
  // the instantiations of the weight format and KV cache (megakernel.cu, kernels_for)
  const void* kernel_ = nullptr;       // plain
  const void* kernel_prof_ = nullptr;  // records the phase timeline stamps; none with a bf16 or fp8 cache or bf16 weights
  const void* kernel_lp_ = nullptr;    // log-probabilities on
  size_t smem_bytes_ = 0;
  bool ready_ = false;
};

}  // namespace kllm
