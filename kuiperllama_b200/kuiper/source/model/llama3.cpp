// model::LLama2Model / Qwen2Model on the H100 backend (API of kuiper/include/model/llama3.h,
// behaviour of kuiper/source/model/llama3.cpp + qwen2.cpp in the reference).
//
// Loading: the checkpoint is mmap'd, every weight becomes an op layer that views the mapping
// and is then uploaded (LayerParam::to_cuda) -- as in the reference.  On top of the uploaded
// weights a fused, device-resident decoder (kllm_decoder, include/kllm_b200.h) is created; it
// shares the weight buffers and owns its activations and KV cache.
//
// Per token: predict() recognises the embedding row it is given (the only way demo/main.cpp
// feeds the model), recovers the token id and runs ONE persistent sm_90a kernel for the whole
// forward + greedy argmax.  forward() is the reference's layer-by-layer orchestration
// (llama3.cpp:147-167,600-745) over the op registry, for callers with their own activations;
// it keeps its own named buffers (allocated on first use) and its own KV cache, so a sequence
// must stay on one of the two paths.
#include "model/llama3.h"

#include <cuda_runtime_api.h>
#include <kllm_b200.h>
#include <op/decoder_layers.h>

#include <cstring>
#include <utility>

#include "../op/kernels/kernels_interface.h"

namespace model {
namespace {
std::shared_ptr<op::LayerParam> as_param(const std::shared_ptr<op::Layer>& l) {
  return std::static_pointer_cast<op::LayerParam>(l);
}
}  // namespace

void LLama2Layers::to_cuda(std::shared_ptr<kernel::CudaConfig> config) {
  auto move = [&](const std::shared_ptr<op::Layer>& l) {
    if (l) {
      l->set_cuda_config(config);
      l->to_cuda();
    }
  };
  move(add_layer_), move(rope_layer_), move(swiglu_layer_), move(mha_layer_);
  move(cls_layer_), move(embedding_layer_);
  for (auto* group : {&wq_layers_, &wk_layers_, &wv_layers_, &wo_layers_, &w1_layers_, &w2_layers_, &w3_layers_,
                      &rmsnorm_layers_})
    for (auto& l : *group) move(l);
}

LLama2Model::LLama2Model(base::TokenizerType tokenizer_type, std::string token_path, std::string model_path,
                         bool is_quant_model)
    : LLama2Model(tokenizer_type, std::move(token_path), std::move(model_path), is_quant_model, false) {}

LLama2Model::LLama2Model(base::TokenizerType tokenizer_type, std::string token_path, std::string model_path,
                         bool is_quant_model, bool qkv_bias)
    : Model(tokenizer_type, base::ModelType::kModelTypeLLama2, std::move(token_path), std::move(model_path),
            is_quant_model),
      qkv_bias_(qkv_bias) {}

LLama2Model::~LLama2Model() {
  if (comm_ != nullptr) {
    // nobody frees its exchange area while a peer's kernel may still push into it
    cudaDeviceSynchronize();
    if (rendezvous_ && rendezvous_->is_open()) rendezvous_->barrier();
  }
  if (decoder_ != nullptr) kllm_decoder_destroy(decoder_);
  if (comm_ != nullptr) kllm_comm_destroy(comm_);
}

void LLama2Model::set_tensor_parallel(const TpConfig& config) {
  tp_ = config;
  tp_explicit_ = true;
}

const char* LLama2Model::decoder_engine() const { return decoder_ ? kllm_decoder_engine(decoder_) : ""; }

base::Status LLama2Model::init(base::DeviceType device_type) {
  using namespace base;
  if (token_path_.empty()) return error::PathNotValid(token_path_);
  if (device_type != DeviceType::kDeviceCUDA)
    return error::InternalError(
        "This library is the H100 (sm_90a) backend: init(kDeviceCUDA) is the only supported device; it has "
        "no CPU path.");
  device_type_ = device_type;
  if (!tp_explicit_) tp_ = TpConfig::from_env();  // tools/kuiper_tp_launch: one process per GPU
  if (tp_.rank < 0 || tp_.rank >= tp_.world) return error::InvalidArgument("tensor parallel: rank outside the world");
  if (cudaSetDevice(tp_.cuda_device()) != cudaSuccess)
    return error::InternalError("No usable CUDA device " + std::to_string(tp_.cuda_device()) + ".");
  cuda_config_ = std::make_shared<kernel::CudaConfig>();
  if (cudaStreamCreate(&cuda_config_->stream) != cudaSuccess)
    return error::InternalError("The cuda handle create failed.");

  Status st = gen_model_from_file();
  if (!st) return st;
  init_mem();
  kernel::sin_cos_cache_calc_cu(config_->head_size_, config_->seq_len_, get_buffer(ModelBufferType::kSinCache),
                                get_buffer(ModelBufferType::kCosCache), cuda_config_->stream);
  sampler_ = std::make_unique<sampler::ArgmaxSampler>(device_type_);
  return create_decoder();
}

// ---- layers over the mmap'd checkpoint ------------------------------------------------------------
void LLama2Model::create_nonparam_layers() {
  CHECK(llama_layers_ != nullptr);
  llama_layers_->rope_layer_ =
      std::make_shared<op::RoPELayer>(device_type_, config_->dim_, config_->kv_dim_, config_->head_size_);
  llama_layers_->mha_layer_ = std::make_shared<op::MultiHeadAttention>(
      device_type_, 0, config_->kv_mul_, config_->kv_dim_, config_->seq_len_, config_->head_num_,
      config_->head_size_);
  llama_layers_->add_layer_ = std::make_shared<op::VecAddLayer>(device_type_);
  llama_layers_->swiglu_layer_ = std::make_shared<op::SwiGLULayer>(device_type_, config_->hidden_dim_);
}

// fp32 v0 (export.py:79-131): tok_emb, attn_norm[L], wq[L], wk[L], wv[L], wo[L], ffn_norm[L],
// w1[L], w2[L], w3[L], final_norm, freqs_cos, freqs_sin, [wcls].  Qwen2 (export_qwen2.py:103-110):
// a bias vector follows each layer's wq / wk / wv.
void LLama2Model::create_param_layers() {
  CHECK(!is_quant_model_);
  const auto cpu = base::DeviceType::kDeviceCPU;
  const int32_t dim = config_->dim_, kvd = config_->kv_dim_, hid = config_->hidden_dim_;
  const int32_t L = config_->layer_num_, V = config_->vocab_size_;
  const bool tp = tp_.on();
  size_t off = 0;  // in floats
  auto take = [&](size_t n) {
    const void* p = raw_model_data_->weight(off);
    off += n;
    return p;
  };
  // One [rows, cols] matrix per layer; under tensor parallelism only rows [r0, r1) (a contiguous span of
  // the file, viewed in place) or columns [c0, c1) (packed once into a host staging buffer) are kept.
  auto matmul_group = [&](std::vector<std::shared_ptr<op::Layer>>& dst, int32_t rows, int32_t cols, bool bias,
                          int32_t r0, int32_t r1, int32_t c0, int32_t c1) {
    const int32_t lr = r1 - r0, lc = c1 - c0;
    for (int32_t i = 0; i < L; ++i) {
      auto m = std::make_shared<op::MatmulLayer>(device_type_, lr, lc, false, bias);
      const float* full = static_cast<const float*>(take(static_cast<size_t>(rows) * cols));
      if (lc == cols) {
        m->set_weight(0, {lr, lc}, full + static_cast<size_t>(r0) * cols, cpu);
      } else {
        auto pack = std::make_shared<base::Buffer>(static_cast<size_t>(lr) * lc * sizeof(float),
                                                   base::CPUDeviceAllocatorFactory::get_instance());
        float* p = static_cast<float*>(pack->ptr());
        for (int32_t r = 0; r < lr; ++r)
          std::memcpy(p + static_cast<size_t>(r) * lc, full + static_cast<size_t>(r0 + r) * cols + c0,
                      static_cast<size_t>(lc) * sizeof(float));
        m->set_weight(0, {lr, lc}, p, cpu);
        tp_staging_.push_back(std::move(pack));
      }
      if (bias) {
        int32_t n = lr;
        m->set_bias(0, n, static_cast<const float*>(take(rows)) + r0, cpu);
      }
      dst.push_back(m);
    }
  };
  auto norm_group = [&](int32_t count) {
    for (int32_t i = 0; i < count; ++i) {
      auto n = std::make_shared<op::RmsNormLayer>(device_type_, dim);
      n->set_weight(0, {dim}, take(dim), cpu);
      llama_layers_->rmsnorm_layers_.push_back(n);
    }
  };
  const TpShard& sh = shard_;
  const int32_t q0 = tp ? sh.q0 : 0, q1 = tp ? sh.q1 : dim, k0 = tp ? sh.k0 : 0, k1 = tp ? sh.k1 : kvd;
  const int32_t f0 = tp ? sh.f0 : 0, f1 = tp ? sh.f1 : hid;

  auto emb = std::make_shared<op::EmbeddingLayer>(device_type_, dim, config_->seq_len_, V);
  const void* emb_ptr = take(static_cast<size_t>(V) * dim);
  emb->set_weight(0, {V, dim}, emb_ptr, cpu);
  llama_layers_->embedding_layer_ = emb;

  norm_group(L);  // attention norms -> rmsnorm_layers_[0, L)
  matmul_group(llama_layers_->wq_layers_, dim, dim, qkv_bias_, q0, q1, 0, dim);
  matmul_group(llama_layers_->wk_layers_, kvd, dim, qkv_bias_, k0, k1, 0, dim);
  matmul_group(llama_layers_->wv_layers_, kvd, dim, qkv_bias_, k0, k1, 0, dim);
  matmul_group(llama_layers_->wo_layers_, dim, dim, false, 0, dim, q0, q1);
  norm_group(L);  // ffn norms -> [L, 2L)
  matmul_group(llama_layers_->w1_layers_, hid, dim, false, f0, f1, 0, dim);
  matmul_group(llama_layers_->w2_layers_, dim, hid, false, 0, dim, f0, f1);
  matmul_group(llama_layers_->w3_layers_, hid, dim, false, f0, f1, 0, dim);
  norm_group(1);  // final norm -> [2L]
  take(static_cast<size_t>(config_->seq_len_) * config_->head_size_);  // freqs_cos + freqs_sin: unused

  auto cls = std::make_shared<op::MatmulLayer>(device_type_, V, dim);
  cls->set_weight(0, {V, dim}, config_->is_shared_weight_ ? emb_ptr : take(static_cast<size_t>(V) * dim), cpu);
  llama_layers_->cls_layer_ = cls;
}

// int8 v3 (export.py:134-210): for wq wk wv wo w1 w2 w3, per layer: int8 block then fp32 group
// scales; [wcls]; then fp32 tok_emb, attn_norm[L], ffn_norm[L], final_norm.
void LLama2Model::create_param_quant_layers() {
  CHECK(is_quant_model_);
  const auto cpu = base::DeviceType::kDeviceCPU;
  const int32_t dim = config_->dim_, kvd = config_->kv_dim_, hid = config_->hidden_dim_;
  const int32_t L = config_->layer_num_, V = config_->vocab_size_;
  const int32_t g = group_size_;
  const bool tp = tp_.on();
  size_t off = 0;  // in bytes
  // One tensor of the file: int8 [rows, cols] followed by its fp32 scales [rows * cols / g].  Under tensor
  // parallelism rows [r0, r1) keep viewing the file (the weight slice and the scale slice are two
  // contiguous spans); columns [c0, c1) -- c0, c1 multiples of g -- are packed into host staging buffers.
  auto quant_matmul = [&](int32_t rows, int32_t cols, int32_t r0, int32_t r1, int32_t c0, int32_t c1) {
    const int32_t lr = r1 - r0, lc = c1 - c0;
    auto m = std::make_shared<op::MatmulLayer>(device_type_, lr, lc, true);
    m->set_group_size(g);
    const int8_t* full = static_cast<const int8_t*>(raw_model_data_->weight(off));
    const size_t numel = static_cast<size_t>(rows) * cols;
    const float* full_scales = reinterpret_cast<const float*>(full + numel);
    off += numel + numel / g * sizeof(float);
    if (lr == rows && lc == cols) {
      m->set_weight(0, {rows, cols}, full, cpu);  // scales: right behind the block
      return m;
    }
    CHECK(cols % g == 0 && c0 % g == 0 && lc % g == 0) << "quantisation groups straddle the shard";
    const size_t n_scales = static_cast<size_t>(lr) * lc / g;
    const int8_t* w_ptr;
    const float* s_ptr;
    if (lc == cols) {
      w_ptr = full + static_cast<size_t>(r0) * cols;
      s_ptr = full_scales + static_cast<size_t>(r0) * cols / g;
    } else {
      auto pack = std::make_shared<base::Buffer>(static_cast<size_t>(lr) * lc + n_scales * sizeof(float),
                                                 base::CPUDeviceAllocatorFactory::get_instance());
      int8_t* pw = static_cast<int8_t*>(pack->ptr());
      float* ps = reinterpret_cast<float*>(pw + static_cast<size_t>(lr) * lc);  // lr * lc % 4 == 0
      for (int32_t r = 0; r < lr; ++r) {
        std::memcpy(pw + static_cast<size_t>(r) * lc, full + static_cast<size_t>(r0 + r) * cols + c0, lc);
        std::memcpy(ps + static_cast<size_t>(r) * (lc / g), full_scales + (static_cast<size_t>(r0 + r) * cols + c0) / g,
                    static_cast<size_t>(lc / g) * sizeof(float));
      }
      w_ptr = pw, s_ptr = ps;
      tp_staging_.push_back(std::move(pack));
    }
    m->set_weight(0, {lr, lc}, w_ptr, cpu);
    tensor::Tensor scales(base::DataType::kDataTypeFp32, static_cast<int32_t>(n_scales), false, nullptr,
                          const_cast<float*>(s_ptr));
    scales.set_device_type(cpu);
    m->set_scales(scales);
    return m;
  };
  auto group = [&](std::vector<std::shared_ptr<op::Layer>>& dst, int32_t rows, int32_t cols, int32_t r0, int32_t r1,
                   int32_t c0, int32_t c1) {
    for (int32_t i = 0; i < L; ++i) dst.push_back(quant_matmul(rows, cols, r0, r1, c0, c1));
  };
  const TpShard& sh = shard_;
  const int32_t q0 = tp ? sh.q0 : 0, q1 = tp ? sh.q1 : dim, k0 = tp ? sh.k0 : 0, k1 = tp ? sh.k1 : kvd;
  const int32_t f0 = tp ? sh.f0 : 0, f1 = tp ? sh.f1 : hid;
  group(llama_layers_->wq_layers_, dim, dim, q0, q1, 0, dim);
  group(llama_layers_->wk_layers_, kvd, dim, k0, k1, 0, dim);
  group(llama_layers_->wv_layers_, kvd, dim, k0, k1, 0, dim);
  group(llama_layers_->wo_layers_, dim, dim, 0, dim, q0, q1);
  group(llama_layers_->w1_layers_, hid, dim, f0, f1, 0, dim);
  group(llama_layers_->w2_layers_, dim, hid, 0, dim, f0, f1);
  group(llama_layers_->w3_layers_, hid, dim, f0, f1, 0, dim);
  // A shared classifier cannot be expressed in this format: the exporter writes no int8 copy of
  // the embedding and the reference then reads the fp32 table as int8 (llama3.cpp:259-277).
  CHECK(!config_->is_shared_weight_)
      << "int8 checkpoints with a shared classifier are not loadable (reference defect, see DESIGN.md)";
  llama_layers_->cls_layer_ = quant_matmul(V, dim, 0, V, 0, dim);

  const float* f = static_cast<const float*>(raw_model_data_->weight(off));
  auto emb = std::make_shared<op::EmbeddingLayer>(device_type_, dim, config_->seq_len_, V);
  emb->set_weight(0, {V, dim}, f, cpu);
  llama_layers_->embedding_layer_ = emb;
  f += static_cast<size_t>(V) * dim;
  for (int32_t i = 0; i < 2 * L + 1; ++i) {
    auto n = std::make_shared<op::RmsNormLayer>(device_type_, dim);
    n->set_weight(0, {dim}, f, cpu);
    llama_layers_->rmsnorm_layers_.push_back(n);
    f += dim;
  }
}

base::Status LLama2Model::create_layers() {
  using namespace base;
  if (!llama_layers_) llama_layers_ = std::make_unique<LLama2Layers>();
  if (tp_.on()) {
    if (Status st = tp_shard(*config_, is_quant_model_ ? group_size_ : 0, tp_.world, tp_.rank, &shard_); !st) return st;
    LOG(INFO) << "tensor parallel rank " << tp_.rank << " of " << tp_.world << ": heads [" << shard_.q0 / config_->head_size_
              << ", " << shard_.q1 / config_->head_size_ << "), kv rows [" << shard_.k0 << ", " << shard_.k1
              << "), FFN rows [" << shard_.f0 << ", " << shard_.f1 << ")";
  }
  // the file must hold exactly what the header promises before any view is taken
  {
    const size_t dim = config_->dim_, kvd = config_->kv_dim_, hid = config_->hidden_dim_, L = config_->layer_num_,
                 V = config_->vocab_size_;
    const size_t mats = L * (2 * dim * dim + 2 * kvd * dim + 3 * hid * dim);
    size_t need;
    if (!is_quant_model_) {
      need = 28 + 4 * (V * dim + (2 * L + 1) * dim + mats + static_cast<size_t>(config_->seq_len_) * config_->head_size_ +
                       (config_->is_shared_weight_ ? 0 : V * dim) + (qkv_bias_ ? L * (dim + 2 * kvd) : 0));
    } else {
      if (group_size_ <= 0) return error::ModelParseError("The int8 checkpoint has no valid group size.");
      const size_t q = mats + (config_->is_shared_weight_ ? 0 : V * dim);
      need = 32 + q + q / group_size_ * 4 + 4 * (V * dim + (2 * L + 1) * dim);
    }
    if (raw_model_data_->file_size < need)
      return error::ModelParseError("The checkpoint is smaller than its header implies (" +
                                    std::to_string(raw_model_data_->file_size) + " < " + std::to_string(need) +
                                    " bytes): wrong quant flag or flavour?");
  }
  if (is_quant_model_) {
    create_param_quant_layers();
  } else {
    create_param_layers();
  }
  create_nonparam_layers();
  const size_t L = config_->layer_num_;
  const LLama2Layers& ly = *llama_layers_;
  if (!ly.embedding_layer_ || !ly.cls_layer_ || ly.rmsnorm_layers_.size() != 2 * L + 1 || ly.wq_layers_.size() != L ||
      ly.wk_layers_.size() != L || ly.wv_layers_.size() != L || ly.wo_layers_.size() != L ||
      ly.w1_layers_.size() != L || ly.w2_layers_.size() != L || ly.w3_layers_.size() != L || !ly.rope_layer_ ||
      !ly.add_layer_ || !ly.mha_layer_ || !ly.swiglu_layer_)
    return error::InternalError("Create the layers for the llama model failed!");
  return error::Success();
}

// ---- buffers -----------------------------------------------------------------------------------------
void LLama2Model::init_mem() {
  CHECK(device_type_ == base::DeviceType::kDeviceCUDA);
  CHECK_NE(cuda_config_, nullptr);
  llama_layers_->to_cuda(cuda_config_);  // weights: mmap (or the packed column shards) -> device
  cudaStreamSynchronize(cuda_config_->stream);
  tp_staging_.clear();
  // the host mapping is no longer needed for the weights that now live on the device
  auto cpu = base::CPUDeviceAllocatorFactory::get_instance();
  auto gpu = base::CUDADeviceAllocatorFactory::get_instance();
  const auto f32 = base::DataType::kDataTypeFp32;
  const int32_t dim = config_->dim_;

  CHECK(insert_buffer(ModelBufferType::kInputTokens, tensor::Tensor(base::DataType::kDataTypeInt32, 1, true, cpu)));
  CHECK(insert_buffer(ModelBufferType::kInputEmbeddings, tensor::Tensor(f32, 1, dim, true, gpu)));
  CHECK(insert_buffer(ModelBufferType::kInputPos, tensor::Tensor(base::DataType::kDataTypeInt32, 1, true, cpu)));
  const int32_t table = config_->head_size_ * config_->seq_len_;
  CHECK(insert_buffer(ModelBufferType::kSinCache, tensor::Tensor(f32, table, true, gpu)));
  CHECK(insert_buffer(ModelBufferType::kCosCache, tensor::Tensor(f32, table, true, gpu)));
  // Everything else (activations of the layer-by-layer path, its KV cache, the logits mirror) is
  // created on first use by ensure_lazy_buffer(): the fused decoder keeps its own.
}

void LLama2Model::ensure_lazy_buffer(ModelBufferType idx) const {
  if (buffers_.count(idx) > 0) return;
  auto gpu = base::CUDADeviceAllocatorFactory::get_instance();
  auto cpu = base::CPUDeviceAllocatorFactory::get_instance();
  const auto f32 = base::DataType::kDataTypeFp32;
  const TransformerConfig& c = *config_;
  auto put = [&](ModelBufferType k, const tensor::Tensor& t) { buffers_.insert({k, t}); };
  switch (idx) {
    // one dim-sized scratch serves four roles, as in the reference (llama3.cpp:456-460)
    case ModelBufferType::kOutputRMSNorm:
    case ModelBufferType::kOutputMHA:
    case ModelBufferType::kW2Output:
    case ModelBufferType::kFFNRMSNorm: {
      tensor::Tensor t(f32, c.dim_, true, gpu);
      put(ModelBufferType::kOutputRMSNorm, t), put(ModelBufferType::kOutputMHA, t);
      put(ModelBufferType::kW2Output, t), put(ModelBufferType::kFFNRMSNorm, t);
      break;
    }
    case ModelBufferType::kQuery:
    case ModelBufferType::kAttnOutput: {  // aliased too (llama3.cpp:478-489)
      tensor::Tensor t(f32, c.dim_, true, gpu);
      put(ModelBufferType::kQuery, t), put(ModelBufferType::kAttnOutput, t);
      break;
    }
    case ModelBufferType::kW1Output: put(idx, tensor::Tensor(f32, c.hidden_dim_, true, gpu)); break;
    case ModelBufferType::kW3Output: put(idx, tensor::Tensor(f32, c.hidden_dim_, true, gpu)); break;
    case ModelBufferType::kKeyCache:
    case ModelBufferType::kValueCache: {
      tensor::Tensor t(f32, c.layer_num_, c.seq_len_, c.kv_dim_, true, gpu);
      gpu->memset_zero(t.ptr<float>(), t.byte_size(), cuda_config_->stream);
      put(idx, t);
      break;
    }
    case ModelBufferType::kScoreStorage: put(idx, tensor::Tensor(f32, c.head_num_, c.seq_len_, true, gpu)); break;
    case ModelBufferType::kForwardOutput: put(idx, tensor::Tensor(f32, c.vocab_size_, true, gpu)); break;
    case ModelBufferType::kForwardOutputCPU: put(idx, tensor::Tensor(f32, c.vocab_size_, true, cpu)); break;
    default: break;
  }
}

tensor::Tensor& LLama2Model::get_buffer(ModelBufferType idx) {
  return const_cast<tensor::Tensor&>(static_cast<const LLama2Model*>(this)->get_buffer(idx));
}

const tensor::Tensor& LLama2Model::get_buffer(ModelBufferType idx) const {
  ensure_lazy_buffer(idx);
  if (idx == ModelBufferType::kForwardOutput && logits_in_decoder_) {
    // the last step ran in the fused decoder: mirror its logits into the named buffer
    const tensor::Tensor& out = Model::get_buffer(idx);
    cudaMemcpyAsync(const_cast<float*>(out.ptr<float>()), kllm_decoder_logits_device(decoder_), out.byte_size(),
                    cudaMemcpyDeviceToDevice, cuda_config_->stream);
    cudaStreamSynchronize(cuda_config_->stream);
    logits_in_decoder_ = false;
    return out;
  }
  return Model::get_buffer(idx);
}

// ---- the fused decoder over the uploaded weights -------------------------------------------------
base::Status LLama2Model::create_decoder() {
  const TransformerConfig& c = *config_;
  const int32_t L = c.layer_num_;
  auto weight_ptrs = [&](const std::vector<std::shared_ptr<op::Layer>>& v) {
    std::vector<const void*> p;
    for (auto& l : v) p.push_back(as_param(l)->get_weight(0).ptr<int8_t>());
    return p;
  };
  auto scale_ptrs = [&](const std::vector<std::shared_ptr<op::Layer>>& v) {
    std::vector<const float*> p;
    for (auto& l : v) p.push_back(as_param(l)->get_scales().ptr<float>());
    return p;
  };
  auto bias_ptrs = [&](const std::vector<std::shared_ptr<op::Layer>>& v) {
    std::vector<const float*> p;
    for (auto& l : v) p.push_back(std::static_pointer_cast<op::MatmulLayer>(l)->get_bias(0).ptr<float>());
    return p;
  };
  std::vector<const float*> attn_norm, ffn_norm;
  for (int32_t l = 0; l < L; ++l) {
    attn_norm.push_back(as_param(llama_layers_->rmsnorm_layers_[l])->get_weight(0).ptr<float>());
    ffn_norm.push_back(as_param(llama_layers_->rmsnorm_layers_[l + L])->get_weight(0).ptr<float>());
  }
  const auto wq = weight_ptrs(llama_layers_->wq_layers_), wk = weight_ptrs(llama_layers_->wk_layers_),
             wv = weight_ptrs(llama_layers_->wv_layers_), wo = weight_ptrs(llama_layers_->wo_layers_),
             w1 = weight_ptrs(llama_layers_->w1_layers_), w2 = weight_ptrs(llama_layers_->w2_layers_),
             w3 = weight_ptrs(llama_layers_->w3_layers_);
  std::vector<const float*> sq, sk, sv, so, s1, s2, s3, bq, bk, bv;

  kllm_decoder_desc d{};
  d.dim = c.dim_, d.hidden_dim = c.hidden_dim_, d.layer_num = L, d.head_num = c.head_num_;
  d.kv_head_num = c.kv_head_num_, d.vocab_size = c.vocab_size_, d.seq_len = c.seq_len_;
  d.flavour = kernel::build_flavour();
  d.group_size = is_quant_model_ ? group_size_ : 0;
  d.tok_emb = as_param(llama_layers_->embedding_layer_)->get_weight(0).ptr<float>();
  d.attn_norm = attn_norm.data(), d.ffn_norm = ffn_norm.data();
  d.final_norm = as_param(llama_layers_->rmsnorm_layers_[2 * L])->get_weight(0).ptr<float>();
  d.wq = wq.data(), d.wk = wk.data(), d.wv = wv.data(), d.wo = wo.data();
  d.w1 = w1.data(), d.w2 = w2.data(), d.w3 = w3.data();
  d.wcls = as_param(llama_layers_->cls_layer_)->get_weight(0).ptr<int8_t>();
  if (is_quant_model_) {
    sq = scale_ptrs(llama_layers_->wq_layers_), sk = scale_ptrs(llama_layers_->wk_layers_);
    sv = scale_ptrs(llama_layers_->wv_layers_), so = scale_ptrs(llama_layers_->wo_layers_);
    s1 = scale_ptrs(llama_layers_->w1_layers_), s2 = scale_ptrs(llama_layers_->w2_layers_);
    s3 = scale_ptrs(llama_layers_->w3_layers_);
    d.sq = sq.data(), d.sk = sk.data(), d.sv = sv.data(), d.so = so.data();
    d.s1 = s1.data(), d.s2 = s2.data(), d.s3 = s3.data();
    d.scls = as_param(llama_layers_->cls_layer_)->get_scales().ptr<float>();
  }
  if (qkv_bias_) {
    bq = bias_ptrs(llama_layers_->wq_layers_), bk = bias_ptrs(llama_layers_->wk_layers_);
    bv = bias_ptrs(llama_layers_->wv_layers_);
    d.bq = bq.data(), d.bk = bk.data(), d.bv = bv.data();
  }
  d.tp_size = 1;
  if (tp_.on()) {
    // this rank's shard: LOCAL head / kv-head / FFN counts, full model dim (include/kllm_b200.h)
    if (base::Status st = connect_ranks(); !st) return st;
    d.head_num = shard_.head_num, d.kv_head_num = shard_.kv_head_num, d.hidden_dim = shard_.hidden_dim;
    d.tp_size = tp_.world, d.tp_rank = tp_.rank;
    d.comm = comm_;
  }
  if (const char* mode = std::getenv("KUIPER_NUMERICS"); mode && std::string(mode) == "fast") d.numerics = KLLM_NUMERICS_FAST;
  const int rc = kllm_decoder_create(&d, cuda_config_->stream, &decoder_);
  if (rc != 0)
    return base::error::InternalError(std::string("kllm_decoder_create failed: ") + kllm_error_string(rc));
  LOG(INFO) << "fused decoder engine: " << kllm_decoder_engine(decoder_) << ", "
            << kllm_decoder_launches_per_step(decoder_) << " launch(es) per token";
  if (tp_.on()) {
    // every rank has built its engine (and zeroed its exchange area) before anybody's first token
    cudaDeviceSynchronize();
    if (base::Status st = rendezvous_->barrier(); !st) return st;
  }
  return base::error::Success();
}

// The exchange between the ranks: create this rank's kllm_comm (peer-memory transport), swap the 64-byte
// CUDA-IPC handles of the exchange areas over the rendezvous, map every peer.  What tensor_parallel.Comm
// does through torch.distributed on the Python side.
base::Status LLama2Model::connect_ranks() {
  using base::error::InternalError;
  if (comm_ != nullptr) return base::error::Success();
  rendezvous_ = std::make_unique<TpRendezvous>();
  if (base::Status st = rendezvous_->open(tp_); !st) return st;
  int rc = kllm_comm_create(tp_.world, tp_.rank, KLLM_COMM_PEER, tp_comm_words(*config_, tp_.world), nullptr, &comm_);
  if (rc != 0) return InternalError(std::string("kllm_comm_create: ") + kllm_error_string(rc));
  unsigned char mine[64] = {0};
  rc = kllm_comm_ipc_handle(comm_, mine);
  if (rc != 0) return InternalError(std::string("kllm_comm_ipc_handle: ") + kllm_error_string(rc));
  std::vector<unsigned char> all(static_cast<size_t>(64) * tp_.world);
  if (base::Status st = rendezvous_->all_gather(mine, sizeof(mine), all.data()); !st) return st;
  rc = kllm_comm_connect(comm_, all.data());
  if (rc != 0) return InternalError(std::string("kllm_comm_connect: ") + kllm_error_string(rc));
  cudaDeviceSynchronize();
  return rendezvous_->barrier();  // every rank has mapped every peer before the first exchange
}

// ---- embedding / predict -----------------------------------------------------------------------------
op::EmbeddingOutput LLama2Model::embedding(const std::vector<int>& tokens) const {
  auto input_tokens = get_buffer(ModelBufferType::kInputTokens);
  auto input_embeddings = get_buffer(ModelBufferType::kInputEmbeddings);
  const int32_t n = static_cast<int32_t>(tokens.size());
  if (input_tokens.size() != tokens.size()) {
    input_tokens.reshape({n});
    input_embeddings.reshape({n, config_->dim_});
  }
  for (int32_t i = 0; i < n; ++i) input_tokens.index<int32_t>(i) = tokens[i];
  tensor::Tensor input_token_num(base::DataType::kDataTypeInt32, n);
  LOG_IF(FATAL, !llama_layers_->embedding_layer_) << "The embedding layer in the llama2 model is null pointer.";
  STATUS_CHECK(llama_layers_->embedding_layer_->forward(input_tokens, input_token_num, input_embeddings));
  last_tokens_.assign(tokens.begin(), tokens.end());
  last_embeddings_ = input_embeddings.ptr<float>();
  return op::EmbeddingOutput(input_tokens, input_embeddings, input_token_num);
}

base::Status LLama2Model::predict(const tensor::Tensor& input, const tensor::Tensor& pos_tensor, bool is_prompt,
                                  int& next) const {
  if (input.is_empty()) return base::error::InvalidArgument("The input tensor is empty.");
  const int32_t pos = pos_tensor.index<int32_t>(0);
  // Is `input` a row of the last embedding() result?  Then its token id is known and the whole
  // step runs in the fused decoder.  The decoder and the layer-by-layer path keep separate KV
  // caches; decoder_rows_ / layer_rows_ count the leading positions each one holds, and a step is
  // only routed to a path whose cache has every row below `pos` (sync_layer_cache() copies the
  // decoder's rows over when the layer path has to continue a sequence the decoder started).
  const float* p = input.ptr<float>();
  if (decoder_ != nullptr && last_embeddings_ != nullptr && p >= last_embeddings_) {
    const ptrdiff_t delta = p - last_embeddings_;
    const ptrdiff_t row = delta / config_->dim_;
    const bool rows_present = pos <= decoder_rows_ || pos > layer_rows_;  // else only the layer path has them
    if (delta % config_->dim_ == 0 && row < static_cast<ptrdiff_t>(last_tokens_.size()) && rows_present) {
      int32_t nxt = -1;
      const int rc = kllm_decoder_step(decoder_, last_tokens_[row], pos, is_prompt ? 1 : 0, &nxt);
      if (rc != 0) return base::error::InternalError(std::string("kllm_decoder_step: ") + kllm_error_string(rc));
      next = nxt;
      logits_in_decoder_ = true;
      if (pos <= decoder_rows_) decoder_rows_ = pos + 1;  // rows above pos belong to an older sequence
      return base::error::Success();
    }
  }
  if (tp_.on())
    return base::error::InvalidArgument(
        "tensor parallel: predict() needs a row of the last embedding() call (the fused decoder is the only "
        "sharded path)");
  base::Status st = forward(input, pos_tensor, next);
  if (!st) return st;
  next = post_processing(pos_tensor, is_prompt);
  return base::error::Success();
}

// Rows [0, pos) of the sequence live in the fused decoder's cache but not (all) in the layer path's:
// copy them over (reference layout [layer][seq_len][kv_dim], llama3.cpp:469-475) so that forward()
// attends over the same history.  Rare path (a caller that hands predict()/forward() a tensor that
// is not an embedding() row in the middle of a sequence): a blocking round trip through the host.
base::Status LLama2Model::sync_layer_cache(int32_t pos) const {
  if (decoder_ == nullptr || pos <= layer_rows_ || decoder_rows_ < pos) return base::error::Success();
  const tensor::Tensor& kc = get_buffer(ModelBufferType::kKeyCache);
  const tensor::Tensor& vc = get_buffer(ModelBufferType::kValueCache);
  std::vector<float> kh(kc.size()), vh(vc.size());
  const int rc = kllm_decoder_read_kv(decoder_, kh.data(), vh.data());
  if (rc != 0) return base::error::InternalError(std::string("kllm_decoder_read_kv: ") + kllm_error_string(rc));
  cudaStreamSynchronize(cuda_config_->stream);
  if (cudaMemcpy(const_cast<float*>(kc.ptr<float>()), kh.data(), kc.byte_size(), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(const_cast<float*>(vc.ptr<float>()), vh.data(), vc.byte_size(), cudaMemcpyHostToDevice) != cudaSuccess)
    return base::error::InternalError("copying the decoder's KV rows to the layer path's cache failed");
  layer_rows_ = decoder_rows_;
  return base::error::Success();
}

// ---- the layer-by-layer path (reference orchestration, llama3.cpp:147-167, 600-745) -------------------
base::Status LLama2Model::forward(const tensor::Tensor& input, const tensor::Tensor& pos_tensor, int& next) const {
  UNUSED(next);
  if (input.is_empty()) return base::error::InvalidArgument("The input tensor is empty.");
  if (tp_.on())
    return base::error::FunctionNotImplement("forward() is the single-GPU layer-by-layer path; a tensor-parallel "
                                             "model steps through predict()");
  const int32_t pos = pos_tensor.index<int32_t>(0);
  if (base::Status st = sync_layer_cache(pos); !st) return st;
  for (int32_t l = 0; l < config_->layer_num_; ++l) {
    attention_rms(l, input);
    attention_qkv(l, pos_tensor);
    attention_mha(l, pos_tensor);
    feed_forward(l, input);
  }
  cls_logits(input);
  logits_in_decoder_ = false;
  if (pos <= layer_rows_) layer_rows_ = pos + 1;
  return base::error::Success();
}

void LLama2Model::attention_rms(int32_t layer_idx, const tensor::Tensor& input) const {
  tensor::Tensor out = get_buffer(ModelBufferType::kOutputRMSNorm);
  STATUS_CHECK(llama_layers_->rmsnorm_layers_.at(layer_idx)->forward(input, out));
}

void LLama2Model::attention_qkv(int32_t layer_idx, const tensor::Tensor& pos_tensor) const {
  tensor::Tensor query = get_buffer(ModelBufferType::kQuery);
  const int32_t pos = pos_tensor.index<int32_t>(0);
  get_buffer(ModelBufferType::kKeyCache), get_buffer(ModelBufferType::kValueCache);  // materialise
  const auto& [key, val] = slice_kv_cache(layer_idx, pos);  // k, v land in the cache row directly
  tensor::Tensor normed = get_buffer(ModelBufferType::kOutputRMSNorm);
  STATUS_CHECK(llama_layers_->wq_layers_.at(layer_idx)->forward(normed, query));
  STATUS_CHECK(llama_layers_->wk_layers_.at(layer_idx)->forward(normed, key));
  STATUS_CHECK(llama_layers_->wv_layers_.at(layer_idx)->forward(normed, val));
  STATUS_CHECK(llama_layers_->rope_layer_->forward(query, key, pos_tensor, get_buffer(ModelBufferType::kSinCache),
                                                   get_buffer(ModelBufferType::kCosCache), tensor::Tensor{}));
}

void LLama2Model::attention_mha(int32_t layer_idx, const tensor::Tensor& pos_tensor) const {
  tensor::Tensor key_cache = get_buffer(ModelBufferType::kKeyCache);
  tensor::Tensor val_cache = get_buffer(ModelBufferType::kValueCache);
  tensor::Tensor mha_output = get_buffer(ModelBufferType::kOutputMHA);
  tensor::Tensor score = get_buffer(ModelBufferType::kScoreStorage);
  tensor::Tensor query = get_buffer(ModelBufferType::kQuery);
  auto mha = std::static_pointer_cast<op::MultiHeadAttention>(llama_layers_->mha_layer_);
  mha->set_pos(pos_tensor.index<int32_t>(0));
  mha->set_layer_idx(layer_idx);
  STATUS_CHECK(llama_layers_->mha_layer_->forward(query, score, key_cache, val_cache, mha_output));
  tensor::Tensor attn_output = get_buffer(ModelBufferType::kAttnOutput);
  STATUS_CHECK(llama_layers_->wo_layers_.at(layer_idx)->forward(mha_output, attn_output));
}

void LLama2Model::feed_forward(int32_t layer_idx, const tensor::Tensor& input) const {
  STATUS_CHECK(llama_layers_->add_layer_->forward(input, get_buffer(ModelBufferType::kAttnOutput), input));
  tensor::Tensor ffn_norm = get_buffer(ModelBufferType::kFFNRMSNorm);
  STATUS_CHECK(llama_layers_->rmsnorm_layers_.at(layer_idx + config_->layer_num_)->forward(input, ffn_norm));
  tensor::Tensor w1_out = get_buffer(ModelBufferType::kW1Output);
  tensor::Tensor w3_out = get_buffer(ModelBufferType::kW3Output);
  STATUS_CHECK(llama_layers_->w1_layers_.at(layer_idx)->forward(ffn_norm, w1_out));
  STATUS_CHECK(llama_layers_->w3_layers_.at(layer_idx)->forward(ffn_norm, w3_out));
  STATUS_CHECK(llama_layers_->swiglu_layer_->forward(w1_out, w3_out, w1_out));
  tensor::Tensor w2_out = get_buffer(ModelBufferType::kW2Output);
  STATUS_CHECK(llama_layers_->w2_layers_.at(layer_idx)->forward(w1_out, w2_out));
  STATUS_CHECK(llama_layers_->add_layer_->forward(input, w2_out, input));
}

void LLama2Model::cls_logits(const tensor::Tensor& input) const {
  STATUS_CHECK(llama_layers_->rmsnorm_layers_.at(2 * config_->layer_num_)->forward(input, input));
  tensor::Tensor logits = get_buffer(ModelBufferType::kForwardOutput);
  STATUS_CHECK(llama_layers_->cls_layer_->forward(input, logits));
}

int32_t LLama2Model::post_processing(const tensor::Tensor& pos, bool is_prompt) const {
  UNUSED(pos);
  if (is_prompt) return -1;
  const tensor::Tensor& logits = Model::get_buffer(ModelBufferType::kForwardOutput);
  return static_cast<int32_t>(sampler_->sample(logits.ptr<float>(), logits.size(), cuda_config_->stream));
}
}  // namespace model
