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
#ifndef KLLM_KUIPER_MODEL_LLAMA3_H_
#define KLLM_KUIPER_MODEL_LLAMA3_H_
#include <base/cuda_config.h>

#include <memory>
#include <string>
#include <vector>

#include "model.h"
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

  // bind the stream and upload every weight
  void to_cuda(std::shared_ptr<kernel::CudaConfig> config);
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
