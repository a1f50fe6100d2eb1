// model::LLama2Model -- the Llama-2 / Llama-3 / TinyLlama decoder behind the reference's class name
// and public API (reference kuiper/include/model/llama3.h); model::Qwen2Model (model/qwen2.h)
// derives from it.
//
// Two per-token paths share one set of uploaded weights:
//   predict() on an embedding row that came from embedding() / fill_input() -- the only way
//       demo/main.cpp drives a model -- recovers the token id and runs the fused, device-resident
//       decoder of libkllm_b200 (include/kllm_b200.h): one persistent sm_90a kernel per token;
//   forward() is the layer-by-layer orchestration over the op registry (same arithmetic, one
//       launch per op) for callers that hand in activations of their own; its named buffers and
//       KV cache are created on first use.
// A sequence must stay on one of the two paths (each has its own KV cache).
//
// Opt-in batched prompt prefill (set_batched_prefill / KUIPER_BATCHED_PREFILL=1): the first prompt row
// predict() gets runs every prompt position but the last through the decoder's batched tensor-core prefill
// (kllm_decoder_prefill_w8 / _tf32, TF32 tolerance), and the later prompt rows return at once.
#ifndef KLLM_KUIPER_MODEL_LLAMA3_H_
#define KLLM_KUIPER_MODEL_LLAMA3_H_
#include <base/cuda_config.h>

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "model.h"
#include "sampler/seeded_sampler.h"
#include "tensor_parallel.h"

struct kllm_decoder;  // include/kllm_b200.h
struct kllm_comm;

namespace model {
// Every operator instance of the model.  The *_layers_ vectors hold one entry per transformer
// layer; rmsnorm_layers_ holds [0, L) attention norms, [L, 2L) FFN norms, [2L] the final norm.
struct LLama2Layers {
  using LayerPtr = std::shared_ptr<op::Layer>;
  using LayerList = std::vector<LayerPtr>;

  LayerPtr embedding_layer_, cls_layer_;
  LayerList rmsnorm_layers_;
  LayerList wq_layers_, wk_layers_, wv_layers_, wo_layers_;  // attention projections
  LayerList w1_layers_, w2_layers_, w3_layers_;              // SwiGLU FFN: gate, down, up
  LayerPtr rope_layer_, mha_layer_, add_layer_, swiglu_layer_;  // weight-free, shared by all layers

  // bind the stream and upload every weight; matrices = false leaves the projection and classifier matrices on the
  // host (bf16 weights: LLama2Model uploads its own bf16 copies of them)
  void to_cuda(std::shared_ptr<kernel::CudaConfig> config, bool matrices = true);
};

class LLama2Model : public Model {
 public:
  LLama2Model(base::TokenizerType tokenizer_type, std::string token_path, std::string model_path,
              bool is_quant_model);
  ~LLama2Model() override;

  base::Status init(base::DeviceType device_type) override;  // kDeviceCUDA only
  base::Status predict(const tensor::Tensor& input, const tensor::Tensor& pos_tensor, bool is_prompt,
                       int& next) const override;
  base::Status forward(const tensor::Tensor& input, const tensor::Tensor& pos_tensor, int& next) const override;
  op::EmbeddingOutput embedding(const std::vector<int>& tokens) const override;
  // kForwardOutput mirrors the fused decoder's logits when the last step ran there
  tensor::Tensor& get_buffer(ModelBufferType buffer_idx) override;
  const tensor::Tensor& get_buffer(ModelBufferType buffer_idx) const override;

  // "persistent" / "graph": which engine the fused decoder picked (diagnostic)
  const char* decoder_engine() const;

  // Tensor parallelism (model/tensor_parallel.h): call before init(); without a call init() takes the
  // configuration from the KUIPER_TP_* environment (set by tools/kuiper_tp_launch), so the reference's
  // unchanged demo programs run sharded under the launcher.  One process per GPU; this process loads
  // only its shard of every layer matrix, and predict() is the only per-token path (forward() is the
  // single-GPU layer-by-layer path and refuses to run on a shard).
  void set_tensor_parallel(const TpConfig& config);
  const TpConfig& tensor_parallel() const { return tp_; }
  const TpShard& tensor_parallel_shard() const { return shard_; }

  // Batched prompt prefill under predict(): call before init(); without a call init() takes it from
  // KUIPER_BATCHED_PREFILL=1, so the reference's unchanged demos can opt in.  Off by default: every
  // prompt position is then one full single-token forward, bit-identical to the reference.  When on,
  // predict(row pos of the latest embedding() of n >= 3 tokens, pos, is_prompt = true), with the decoder
  // holding rows [0, pos) of the sequence, fills positions pos .. n - 2 in one batched prefill (the rows
  // whose logits a prompt throws away; int8 checkpoints through kllm_decoder_prefill_w8, fp32 through
  // kllm_decoder_prefill_tf32; KV rows within their stated TF32 tolerance, include/kllm_b200.h), and
  // the prompt calls for those positions then return next = -1 without running.  The last prompt row and
  // every later position step as before.  Single GPU: init() refuses it under tensor parallelism.
  void set_batched_prefill(bool on);
  bool batched_prefill() const { return batched_prefill_; }

  // bf16 KV cache in the fused decoder (kllm_decoder_desc::kv_cache = KLLM_KV_BF16): call before init();
  // without a call init() takes it from KUIPER_KV_CACHE=bf16.  Off by default.  Half the cache memory and
  // half the attention's cache reads, toleranced: it needs the fast numerics (KUIPER_NUMERICS=fast) on
  // one GPU, and init() fails rather than run without it.  The layer path (forward()) keeps fp32 rows;
  // the rows it takes over from the decoder are the widened bf16 values.
  void set_bf16_kv_cache(bool on);
  bool bf16_kv_cache() const { return bf16_kv_cache_; }

  // fp8 e4m3 KV cache in the fused decoder (kllm_decoder_desc::kv_cache = KLLM_KV_FP8): call before init(); without a
  // call init() takes it from KUIPER_KV_CACHE=fp8, with unit scales.  Off by default.  `scales` is empty (every scale
  // 1) or the [2][layer_num][kv_head_num] array of kllm_decoder_desc::kv_scales: the K scales, then the V scales.  A
  // quarter of the fp32 cache's memory and reads, toleranced: the fast numerics (KUIPER_NUMERICS=fast), one GPU and
  // head_size % 64 == 0, and init() fails rather than run without them.  The rows the layer path (forward()) takes
  // over from the decoder are the codes' values times their scales.
  void set_fp8_kv_cache(bool on, std::vector<float> scales = {});
  bool fp8_kv_cache() const { return fp8_kv_cache_; }

  // bf16 weights in the fused decoder (kllm_decoder_desc::weights = KLLM_WEIGHTS_BF16): call before init(); without
  // a call init() takes it from KUIPER_WEIGHTS=bf16|fp32 (fp32 by default).  The matrices wq wk wv wo w1 w2 w3 and the
  // classifier (a bf16 copy of the embedding when shared) are rounded to bf16, nearest even, while they are staged
  // for the upload: only the bf16 copies reach the device, half the upload and half their device memory.  Every
  // result equals the fp32 model's over the rounded weights.  fp32 checkpoints on one GPU only: init() fails for an
  // int8 checkpoint or under tensor parallelism; forward() (the layer path, which has no bf16 kernels) returns an
  // error in this mode.
  void set_bf16_weights(bool on);
  bool bf16_weights() const { return bf16_weights_; }

  // Speculative decoding in generate()'s step 3 (kllm_decoder_generate_speculative, DESIGN.md 5.13): prompt-lookup
  // drafts of up to draft_len ids (1..7) from the n-grams of up to ngram_max ids (1..8) of the sequence, each checked
  // by one verify pass over the weights.  The ids are generate()'s without it.  Call before init(); without a call
  // init() takes draft_len from KUIPER_SPECULATIVE=<draft_len> (0, the default, is off; ngram_max 3).  It needs the
  // exact numerics on one GPU: init() fails under KUIPER_NUMERICS=fast or tensor parallelism, or for a value outside
  // those ranges.
  void set_speculative(int32_t draft_len, int32_t ngram_max = 3);
  int32_t speculative() const { return spec_draft_len_; }

  // Seeded sampling instead of the greedy id (DESIGN.md "Sampling"): call before init(); without a call
  // init() takes it from KUIPER_TEMPERATURE, KUIPER_TOP_K and KUIPER_SEED, so the reference's unchanged
  // demos can sample.  Unset or temperature 0 is greedy.  predict() on the fused decoder and forward() +
  // post_processing on the layer path draw the same id: a pure function of the logits, the settings and
  // the position.  Under tensor parallelism every rank reads the same settings and draws the same id.
  void set_sampling(float temperature, int32_t top_k, uint64_t seed);
  // Nucleus sampling after top-k (kllm_decoder_set_sampling_top_p): call before init(); without a call init()
  // takes it from KUIPER_TOP_P.  Unset or 1 is off; init() refuses a value that is NaN, <= 0 or > 1.
  void set_top_p(float top_p);
  // HF's repetition penalty before every draw (kllm_decoder_set_repetition_penalty, DESIGN.md 5.7), over the ids fed
  // at the last `last_n` positions (0: the whole sequence): call before init(); without a call init() takes it from
  // KUIPER_REPETITION_PENALTY and KUIPER_REPEAT_LAST_N.  Unset or 1 is off; init() refuses a penalty that is not
  // finite or <= 0 and last_n < 0.  The fused paths take the ids from the decoder's history; predict() of a tensor
  // that is not a row of the last embedding() cannot know its id and is refused while the penalty is on.
  void set_repetition_penalty(float penalty, int32_t last_n = 0);
  // Frequency and presence penalties before every draw (kllm_decoder_set_frequency_presence, DESIGN.md 5.9): each id
  // fed c > 0 times at positions [from_pos, pos] loses frequency * c, then presence.  Call before init(); without a
  // call init() takes them from KUIPER_FREQUENCY_PENALTY and KUIPER_PRESENCE_PENALTY (from_pos 0).  Unset or 0 is
  // off; init() refuses a value that is not finite and from_pos < 0.  Like the repetition penalty, predict() of a
  // tensor that is not a row of the last embedding() is refused while they are on.
  void set_frequency_presence(float frequency, float presence, int32_t from_pos = 0);
  // Logit bias before every draw (kllm_decoder_set_logit_bias): id -> bias, added before the penalties.  Call before
  // init(), which refuses an id outside the vocabulary, a repeated id and a bias that is not finite.  Empty is off.
  void set_logit_bias(std::vector<std::pair<int32_t, float>> bias);
  // the draw settings in force (after init(): the environment's for each group no setter above was called for)
  const sampler::DrawConfig& draw_config() const { return draw_; }

  // A whole generation on the fused decoder, without a host round trip per token:
  //   1. the prompt from position 0 (the batched prefill for all but its last token when batched_prefill() is
  //      on, else kllm_decoder_prompt -- also under tensor parallelism);
  //   2. the id after the prompt; if it is a stop id, that one id is the result;
  //   3. kllm_decoder_generate_until for the rest, which stops on the device at the first stop id (with
  //      set_speculative: kllm_decoder_generate_speculative, the same ids).
  // `ids` receives at most max_new_tokens ids (fewer where the context ends), counting the stop id.  on_tokens,
  // if set, receives every id exactly once, in order, while the loop runs.  The stop set is the tokenizer's
  // generation-ending ids (what is_sentence_ending() accepts) plus set_stop_ids().  Afterwards predict() at
  // position prompt.size() + ids.size() - 1 with ids.back() continues the same sequence.
  base::Status generate(const std::vector<int32_t>& prompt, int32_t max_new_tokens, std::vector<int32_t>& ids,
                        const std::function<void(const int32_t*, int32_t)>& on_tokens = {}) const;
  // Log-probabilities of the returned ids (kllm_decoder_set_logprobs, DESIGN.md 5.8): call before init(), which
  // refuses a value outside [-1, KLLM_MAX_TOP_LOGPROBS].  -1 (the default) is off; 0 records each returned id's
  // log-probability over the raw logits, 1..20 also its top_n alternatives.  Entries are written by the fused
  // paths (predict() on the fused decoder, generate()), at every position whose classifier runs.
  void set_logprobs(int32_t top_n);
  int32_t logprobs_top_n() const { return draw_.logprobs_top_n; }
  // The record of positions [first_pos, first_pos + n) (kllm_decoder_read_logprobs): ids (-1: no entry), lp, and
  // top_ids / top_lp [n][logprobs_top_n()] (empty when it is <= 0).
  base::Status logprobs(int32_t first_pos, int32_t n, std::vector<int32_t>& ids, std::vector<float>& lp,
                        std::vector<int32_t>& top_ids, std::vector<float>& top_lp) const;
  // Teacher-forced scoring from position 0 (kllm_decoder_score): lp[i] = log p(tokens[i + 1] | tokens[0..i]),
  // tokens.size() - 1 values.  Afterwards the decoder holds positions 0 .. tokens.size() - 2.
  base::Status score(const std::vector<int32_t>& tokens, std::vector<float>& lp) const;
  // Extra stop ids for generate(), e.g. for tokenizers that stop on nothing.
  void set_stop_ids(std::vector<int32_t> ids) { extra_stop_ids_ = std::move(ids); }

 protected:
  // qkv_bias: the checkpoint carries a bias vector behind each layer's wq / wk / wv (Qwen2 files)
  LLama2Model(base::TokenizerType tokenizer_type, std::string token_path, std::string model_path,
              bool is_quant_model, bool qkv_bias);

 private:
  friend struct ModelInspector;
  // Model's loading hooks
  void init_mem() override;
  base::Status create_layers() override;
  void create_param_layers() override;
  void create_nonparam_layers() override;
  void create_param_quant_layers() override;
  int32_t post_processing(const tensor::Tensor& pos, bool is_prompt) const override;

  base::Status create_decoder();
  base::Status connect_ranks();
  void ensure_lazy_buffer(ModelBufferType buffer_idx) const;

  // the stages of forward(), one transformer layer at a time
  void attention_rms(int32_t layer_idx, const tensor::Tensor& input) const;
  void attention_qkv(int32_t layer_idx, const tensor::Tensor& pos_tensor) const;
  void attention_mha(int32_t layer_idx, const tensor::Tensor& pos_tensor) const;
  void feed_forward(int32_t layer_idx, const tensor::Tensor& input) const;
  void cls_logits(const tensor::Tensor& input) const;

  bool qkv_bias_ = false;
  std::shared_ptr<kernel::CudaConfig> cuda_config_;
  std::unique_ptr<LLama2Layers> llama_layers_;
  kllm_decoder* decoder_ = nullptr;
  // tokens of the most recent embedding() call: maps an input row back to its token id
  mutable std::vector<int32_t> last_tokens_;
  mutable const float* last_embeddings_ = nullptr;
  mutable bool logits_in_decoder_ = false;
  // leading positions of the current sequence present in the decoder's KV cache / in the layer
  // path's kKeyCache+kValueCache (the two are separate allocations with different layouts)
  mutable int32_t decoder_rows_ = 0;
  mutable int32_t layer_rows_ = 0;
  base::Status sync_layer_cache(int32_t pos) const;

  // batched prompt prefill: the switch, and which positions [prefilled_from_, prefilled_to_) of which
  // embedding() call (embedding_calls_ counts them) the decoder's cache holds from it
  bool batched_prefill_ = false;
  bool batched_prefill_explicit_ = false;
  bool bf16_kv_cache_ = false;
  bool bf16_kv_cache_explicit_ = false;
  bool fp8_kv_cache_ = false;
  bool fp8_kv_cache_explicit_ = false;
  std::vector<float> fp8_kv_scales_;
  std::vector<float> fp8_unit_scales_;  // the ones passed for an empty fp8_kv_scales_
  bool bf16_weights_ = false;
  bool bf16_weights_explicit_ = false;
  int32_t spec_draft_len_ = 0;  // 0: generate() runs kllm_decoder_generate_until
  int32_t spec_ngram_max_ = 3;
  bool spec_explicit_ = false;
  // bf16 weights: the device copies of the matrices, in create_decoder's order (wq.. per layer, then wcls)
  std::vector<std::shared_ptr<base::Buffer>> bf16_matrices_;
  base::Status upload_bf16_matrices();
  sampler::DrawConfig draw_;
  sampler::DrawGroups draw_set_;              // the groups a setter gave: init() keeps them over the environment
  sampler::SeededSampler* seeded_ = nullptr;  // sampler_ when sampling, else null
  std::vector<int32_t> extra_stop_ids_;       // set_stop_ids()
  mutable uint64_t embedding_calls_ = 0;
  mutable uint64_t prefilled_embedding_ = 0;
  mutable int32_t prefilled_from_ = 0, prefilled_to_ = 0;
  // predict() on row `pos` of the latest embedding(): true when the batched prefill has filled (or has just
  // filled) position pos, so there is nothing left to run
  base::Status prefill_prompt_rows(int32_t pos, bool* done) const;

  // tensor parallel state: who we are, what we own, the exchange and the start-up rendezvous; the host
  // staging buffers of the repacked column shards live until init_mem() has uploaded them
  TpConfig tp_;
  bool tp_explicit_ = false;
  TpShard shard_;
  kllm_comm* comm_ = nullptr;
  std::unique_ptr<TpRendezvous> rendezvous_;
  std::vector<std::shared_ptr<base::Buffer>> tp_staging_;
};
}  // namespace model
#endif  // KLLM_KUIPER_MODEL_LLAMA3_H_
