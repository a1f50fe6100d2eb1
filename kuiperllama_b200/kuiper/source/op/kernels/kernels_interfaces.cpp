// Registry getters + the Tensor -> C-ABI adapters (see kernels_interface.h).
#include "kernels_interface.h"

#include <kllm_b200.h>

#include "sampler/argmax_sampler.h"
#include "sampler/seeded_sampler.h"

namespace kernel {
namespace {
#if defined(QWEN2_SUPPORT)
constexpr int kFlavour = KLLM_FLAVOUR_QWEN2;
constexpr float kEps = 1e-6f;
#elif defined(LLAMA3_SUPPORT)
constexpr int kFlavour = KLLM_FLAVOUR_LLAMA3;
constexpr float kEps = 1e-5f;
#else
constexpr int kFlavour = KLLM_FLAVOUR_LLAMA2;
constexpr float kEps = 1e-5f;
#endif

constexpr auto kCUDA = base::DeviceType::kDeviceCUDA;

inline void ok(int rc, const char* what) {
  CHECK(rc == 0) << what << " failed: " << rc << " (" << kllm_error_string(rc) << ")";
}
template <typename T>
inline T* mut(const tensor::Tensor& t) {
  return const_cast<T*>(t.ptr<T>());  // registry convention: outputs arrive const
}

template <typename Fn>
Fn no_cpu_backend(const char* op) {
  LOG(FATAL) << "kernel registry: " << op
             << " requested for a non-CUDA device.  This library is the H100 (sm_90a) backend "
                "only; it has no CPU kernels and never falls back to the host.";
  return nullptr;
}

// ---- adapters ------------------------------------------------------------------------------------
void add_kernel_cu(const tensor::Tensor& in1, const tensor::Tensor& in2, const tensor::Tensor& out,
                   void* stream) {
  CHECK(!in1.is_empty() && !in2.is_empty() && !out.is_empty());
  CHECK_EQ(in1.size(), in2.size());
  CHECK_EQ(in1.size(), out.size());
  ok(kllm_add_f32(in1.ptr<float>(), in2.ptr<float>(), mut<float>(out), static_cast<int>(in1.size()), stream),
     "kllm_add_f32");
}

void matmul_kernel_cu(const tensor::Tensor& input, const tensor::Tensor& weight,
                      const tensor::Tensor& output, float scale, const CudaConfig* config) {
  UNUSED(scale);  // ignored on CUDA in the reference as well (matmul_kernel.cu:89-109)
  CHECK(!input.is_empty() && input.dims_size() <= 2 && input.device_type() == kCUDA);
  CHECK(!weight.is_empty() && weight.dims_size() == 2 && weight.device_type() == kCUDA);
  const int K = weight.get_dim(0), M = weight.get_dim(1);
  CHECK_EQ(M, input.get_dim(0));
  ok(kllm_gemv_f32(input.ptr<float>(), weight.ptr<float>(), mut<float>(output), M, K,
                   config ? config->stream : nullptr),
     "kllm_gemv_f32");
}

void matmul_kernel_cu_qint8(const tensor::Tensor& input, const tensor::Tensor& weight,
                            const tensor::Tensor& output, int32_t group_size,
                            const tensor::Tensor& scale, const CudaConfig* config) {
  CHECK(config != nullptr);
  CHECK(!input.is_empty() && input.dims_size() <= 2 && input.device_type() == kCUDA);
  CHECK(!weight.is_empty() && weight.dims_size() == 2 && weight.device_type() == kCUDA);
  const int K = weight.get_dim(0), M = weight.get_dim(1);
  CHECK_EQ(M % 4, 0);
  CHECK_EQ(M, input.get_dim(0));
  ok(kllm_gemv_w8(input.ptr<float>(), weight.ptr<int8_t>(), scale.ptr<float>(), mut<float>(output), M, K,
                  group_size, config->stream),
     "kllm_gemv_w8");
}

void emb_kernel_cu(const tensor::Tensor& input, const tensor::Tensor& weight, const tensor::Tensor& output,
                   int32_t vocab_size, void* stream) {
  CHECK(weight.device_type() == output.device_type());
  CHECK(output.device_type() == kCUDA);
  const int n = static_cast<int>(input.size());
  const int dim = weight.get_dim(1);
  // the ids may live on the host (the reference requires that); stage them without the
  // reference's blocking pool allocation per call
  const int32_t* ids = input.ptr<int32_t>();
  tensor::Tensor staged;
  if (input.device_type() != kCUDA) {
    staged = tensor::Tensor(base::DataType::kDataTypeInt32, n, true, base::CUDADeviceAllocatorFactory::get_instance());
    CHECK(cudaMemcpyAsync(staged.ptr<int32_t>(), ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice,
                          static_cast<cudaStream_t>(stream)) == cudaSuccess);
    ids = staged.ptr<int32_t>();
  }
  ok(kllm_embedding_f32(ids, n, weight.ptr<float>(), mut<float>(output), dim, vocab_size, stream),
     "kllm_embedding_f32");
  if (input.device_type() != kCUDA) cudaStreamSynchronize(static_cast<cudaStream_t>(stream));  // staged dies here
}

void swiglu_kernel_cu(const tensor::Tensor& in1, const tensor::Tensor& in2, const tensor::Tensor& out,
                      void* stream) {
  CHECK(!in1.is_empty() && in1.device_type() == kCUDA);
  CHECK(!in2.is_empty() && in2.device_type() == kCUDA);
  CHECK(!out.is_empty() && out.device_type() == kCUDA);
  ok(kllm_swiglu_f32(in1.ptr<float>(), in2.ptr<float>(), mut<float>(out), static_cast<int>(in1.size()), stream),
     "kllm_swiglu_f32");
}

void mha_kernel_cu(int32_t pos, int32_t head_num, int32_t layer_index, int32_t seq_len, int32_t kv_dim,
                   int32_t kv_mul, int32_t head_size, const tensor::Tensor& mha_out,
                   const tensor::Tensor& query, const tensor::Tensor& score, const tensor::Tensor& key_cache,
                   const tensor::Tensor& value_cache, base::DeviceType device_type, CudaConfig* config) {
  UNUSED(device_type);
  ok(kllm_mha_decode_f32(pos, head_num, layer_index, seq_len, kv_dim, kv_mul, head_size, mut<float>(mha_out),
                         query.ptr<float>(), mut<float>(score), key_cache.ptr<float>(),
                         value_cache.ptr<float>(), config ? config->stream : nullptr),
     "kllm_mha_decode_f32");
}

void rmsnorm_kernel_cu(const tensor::Tensor& input, const tensor::Tensor& weight, const tensor::Tensor& output,
                       void* stream) {
  CHECK(!input.is_empty() && !weight.is_empty() && !output.is_empty());
  CHECK(input.device_type() == kCUDA && weight.device_type() == kCUDA && output.device_type() == kCUDA);
  ok(kllm_rmsnorm_f32(input.ptr<float>(), weight.ptr<float>(), mut<float>(output),
                      static_cast<int>(input.size()), kEps, stream),
     "kllm_rmsnorm_f32");
}

void rope_kernel_cu(int32_t dim, int32_t kv_dim, int32_t head_size, const tensor::Tensor& q,
                    const tensor::Tensor& k, const tensor::Tensor& pos_tensor, const tensor::Tensor& sin_cache,
                    const tensor::Tensor& cos_cache, void* stream) {
  const int32_t pos = *pos_tensor.ptr<int32_t>(0);  // host tensor, as in rope_kernel.cu:157
  ok(kllm_rope_f32(kFlavour, dim, kv_dim, head_size, mut<float>(q), mut<float>(k), pos, sin_cache.ptr<float>(),
                   cos_cache.ptr<float>(), stream),
     "kllm_rope_f32");
}
}  // namespace

int build_flavour() { return kFlavour; }

void sin_cos_cache_calc_cu(int head_size, int max_seq_len, const tensor::Tensor& sin_cache,
                           const tensor::Tensor& cos_cache, cudaStream_t stream) {
  CHECK(!sin_cache.is_empty() && !cos_cache.is_empty());
  ok(kllm_sincos_init(head_size, max_seq_len, kFlavour, mut<float>(sin_cache), mut<float>(cos_cache), stream),
     "kllm_sincos_init");
}

size_t argmax_kernel_cu(const float* input_ptr, size_t size, void* stream) {
  const int64_t idx = kllm_argmax_f32_sync(input_ptr, static_cast<int64_t>(size), stream);
  CHECK_GE(idx, 0) << "kllm_argmax_f32_sync failed";
  return static_cast<size_t>(idx);
}

#define KLLM_GETTER(Type, name, cuda_fn)                                  \
  Type name(base::DeviceType device_type) {                               \
    if (device_type == base::DeviceType::kDeviceCUDA) return cuda_fn;     \
    return no_cpu_backend<Type>(#name);                                   \
  }

KLLM_GETTER(AddKernel, get_add_kernel, add_kernel_cu)
KLLM_GETTER(EmbeddingKernel, get_emb_kernel, emb_kernel_cu)
KLLM_GETTER(MatmulKernel, get_matmul_kernel, matmul_kernel_cu)
KLLM_GETTER(MatmulKernelQuant, get_matmul_kernel_quant8, matmul_kernel_cu_qint8)
KLLM_GETTER(MHAKernel, get_mha_kernel, mha_kernel_cu)
KLLM_GETTER(RMSNormKernel, get_rmsnorm_kernel, rmsnorm_kernel_cu)
KLLM_GETTER(RoPEKernel, get_rope_kernel, rope_kernel_cu)
#undef KLLM_GETTER

SwigluKernel get_swiglu_kernel(base::DeviceType device_type, void* stream) {
  UNUSED(stream);
  if (device_type == base::DeviceType::kDeviceCUDA) return swiglu_kernel_cu;
  return no_cpu_backend<SwigluKernel>("get_swiglu_kernel");
}

// scale / softmax / scale_sum exist only as CPU kernels in the reference
// (kernels_interfaces.cpp:85-101,125-132); no device version is registered there either.
ScaleKernel get_scale_kernel(base::DeviceType) { return no_cpu_backend<ScaleKernel>("get_scale_kernel"); }
SoftmaxInplaceKernel get_softmax_kernel(base::DeviceType) {
  return no_cpu_backend<SoftmaxInplaceKernel>("get_softmax_kernel");
}
ScaleSumKernel get_scale_sum_kernel(base::DeviceType) {
  return no_cpu_backend<ScaleSumKernel>("get_scale_sum_kernel");
}
}  // namespace kernel

// sampler::ArgmaxSampler (sampler/argmax_sampler.h): greedy sampling runs where the logits are; this
// library has no host path
size_t sampler::ArgmaxSampler::sample(const float* logits, size_t size, void* stream) {
  CHECK(device_type_ == base::DeviceType::kDeviceCUDA) << "ArgmaxSampler: CUDA logits only (no CPU backend)";
  return kernel::argmax_kernel_cu(logits, size, stream);
}

size_t sampler::SeededSampler::sample(const float* logits, size_t size, void* stream) {
  CHECK(device_type_ == base::DeviceType::kDeviceCUDA) << "SeededSampler: CUDA logits only (no CPU backend)";
  static thread_local int64_t* d_idx = nullptr;
  if (d_idx == nullptr) CHECK(cudaMalloc(reinterpret_cast<void**>(&d_idx), sizeof(int64_t)) == cudaSuccess) << "SeededSampler: cudaMalloc";
  if (cfg_.step0()) {  // step 0 on a copy of the logits, then the draw from that copy
    static thread_local float* d_pen = nullptr;
    static thread_local size_t pen_cap = 0;
    static thread_local int32_t* d_ids = nullptr;
    static thread_local size_t ids_cap = 0;
    if (pen_cap < size) {
      if (d_pen != nullptr) cudaFree(d_pen);
      CHECK(cudaMalloc(reinterpret_cast<void**>(&d_pen), size * sizeof(float)) == cudaSuccess) << "SeededSampler: cudaMalloc";
      pen_cap = size;
    }
    if (ids_cap < fed_.size()) {
      if (d_ids != nullptr) cudaFree(d_ids);
      CHECK(cudaMalloc(reinterpret_cast<void**>(&d_ids), fed_.size() * sizeof(int32_t)) == cudaSuccess)
          << "SeededSampler: cudaMalloc";
      ids_cap = fed_.size();
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (!fed_.empty())
      CHECK(cudaMemcpyAsync(d_ids, fed_.data(), fed_.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s) ==
            cudaSuccess) << "SeededSampler: copy of the fed ids";
    // the windows of sampling.cuh (window_lo, step0_history): H(pos) = fed[rep_lo, pos], C(pos) = fed[cnt_lo, pos]
    const int32_t n_fed = static_cast<int32_t>(fed_.size());
    const int32_t rep_lo = std::min(n_fed, cfg_.last_n == 0 ? 0 : std::max(0, pos_ - cfg_.last_n + 1));
    const int32_t cnt_lo = std::min(n_fed, cfg_.from_pos);
    if (cfg_.step0_extras()) {
      std::vector<int32_t> bias_ids;
      std::vector<float> bias;
      for (const auto& [id, b] : cfg_.logit_bias) bias_ids.push_back(id), bias.push_back(b);
      const int prc = kllm_logit_penalties_f32(
          logits, d_pen, static_cast<int64_t>(size), bias_ids.data(), bias.data(), static_cast<int32_t>(bias.size()),
          cfg_.penalty, d_ids + rep_lo, n_fed - rep_lo, cfg_.frequency, cfg_.presence, d_ids + cnt_lo, n_fed - cnt_lo,
          stream);
      CHECK(prc == 0) << "kllm_logit_penalties_f32: " << kllm_error_string(prc);
    } else {
      const int prc = kllm_repetition_penalty_f32(logits, d_pen, static_cast<int64_t>(size), d_ids + rep_lo,
                                                  n_fed - rep_lo, cfg_.penalty, stream);
      CHECK(prc == 0) << "kllm_repetition_penalty_f32: " << kllm_error_string(prc);
    }
    logits = d_pen;
  }
  const int rc = kllm_sample_top_p_f32(logits, static_cast<int64_t>(size), cfg_.temperature, cfg_.top_k, cfg_.top_p,
                                       cfg_.seed, pos_, d_idx, stream);
  CHECK(rc == 0) << "kllm_sample_top_p_f32: " << kllm_error_string(rc);
  int64_t h = -1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CHECK(cudaMemcpyAsync(&h, d_idx, sizeof(h), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
        cudaStreamSynchronize(s) == cudaSuccess)
      << "SeededSampler: copy of the id";
  return static_cast<size_t>(h);
}
