// GPU oracle: C-ABI wrappers around the UNMODIFIED reference sources, compiled where they
// lie in the reference checkout by oracle/Makefile into oracle/_ref/libkuiper_ref.so.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under kuiperllama_b200/ links, loads or calls this
// library; only tests/, __graft_entry__.smoke() and bench.py's reference leg do, and only
// as the checker / the reference timing arm.  No reference source is copied into the repo:
// this file is our own glue that calls the reference's public entry points
//   kernel::get_*_kernel(DeviceType)            kuiper/source/op/kernels/kernels_interface.h:6-68
//   kernel::sin_cos_cache_calc_cu               kuiper/source/op/kernels/cuda/rope_kernel.cu:138-151
//   kernel::argmax_kernel_cu                    kuiper/source/op/kernels/cuda/argmax_kernel.cu:73-87
//   model::LLama2Model::{init,embedding,fill_input,predict,get_buffer}   kuiper/include/model/model.h:15-56
// with tensors that wrap caller-owned device pointers.
#include <cuda_runtime_api.h>

#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "base/base.h"
#include "base/cuda_config.h"
#ifndef KREF_KERNELS_ONLY
#include "model/llama3.h"
#endif
#include "tensor/tensor.h"
// The registry header lives next to the sources, exactly as the reference's own tests
// include it (test/test_op/test_cu_matmul.cpp:5).
#include "../source/op/kernels/kernels_interface.h"
// The registry getters (kernels_interfaces.cpp:21-132) return exactly these functions for
// kDeviceCUDA; calling them directly lets the kernels-only (Qwen2 flavour) build skip the
// registry translation unit, which also references the CPU kernels.
#include "../source/op/kernels/cuda/add_kernel.cuh"
#include "../source/op/kernels/cuda/argmax_kernel.cuh"
#include "../source/op/kernels/cuda/emb_kernel.cuh"
#include "../source/op/kernels/cuda/matmul_kernel.cuh"
#include "../source/op/kernels/cuda/mha_kernel.cuh"
#include "../source/op/kernels/cuda/rmsnorm_kernel.cuh"
#include "../source/op/kernels/cuda/rope_kernel.cuh"
#include "../source/op/kernels/cuda/swiglu_kernel.cuh"

namespace {
using base::DataType;
using base::DeviceType;
using tensor::Tensor;

Tensor wrap1(DataType dt, int32_t n, const void* p) {
  Tensor t(dt, n, false, nullptr, const_cast<void*>(p));
  t.set_device_type(DeviceType::kDeviceCUDA);
  return t;
}

Tensor wrap2(DataType dt, int32_t d0, int32_t d1, const void* p) {
  Tensor t(dt, d0, d1, false, nullptr, const_cast<void*>(p));
  t.set_device_type(DeviceType::kDeviceCUDA);
  return t;
}

Tensor wrap3(DataType dt, int32_t d0, int32_t d1, int32_t d2, const void* p) {
  Tensor t(dt, d0, d1, d2, false, nullptr, const_cast<void*>(p));
  t.set_device_type(DeviceType::kDeviceCUDA);
  return t;
}

// CudaConfig's destructor destroys its stream; the caller owns ours, so detach first.
struct BorrowedConfig {
  kernel::CudaConfig cfg;
  explicit BorrowedConfig(void* stream) { cfg.stream = static_cast<cudaStream_t>(stream); }
  ~BorrowedConfig() { cfg.stream = nullptr; }
};

constexpr auto kCUDA = DeviceType::kDeviceCUDA;
}  // namespace

extern "C" {

const char* kref_flavour() {
#if defined(QWEN2_SUPPORT)
  return "qwen2";
#elif defined(LLAMA3_SUPPORT)
  return "llama3";
#else
  return "llama2";
#endif
}

// out[K] = W[K,M] . x[M]            (matmul_kernel.cu:89-109)
void kref_matmul_f32(const float* x, const float* w, float* out, int M, int K, void* stream) {
  BorrowedConfig bc(stream);
  kernel::matmul_kernel_cu(wrap1(DataType::kDataTypeFp32, M, x),
                                   wrap2(DataType::kDataTypeFp32, K, M, w),
                                   wrap1(DataType::kDataTypeFp32, K, out), 1.f, &bc.cfg);
}

// int8 group-dequant GEMV              (matmul_kernel.cu:111-134)
void kref_matmul_w8(const float* x, const int8_t* w, const float* scales, float* out, int M, int K,
                    int group_size, void* stream) {
  BorrowedConfig bc(stream);
  const int32_t nscale = static_cast<int32_t>((int64_t(M) * K) / group_size);
  kernel::matmul_kernel_cu_qint8(
      wrap1(DataType::kDataTypeFp32, M, x), wrap2(DataType::kDataTypeInt8, K, M, w),
      wrap1(DataType::kDataTypeFp32, K, out), group_size,
      wrap1(DataType::kDataTypeFp32, nscale, scales), &bc.cfg);
}

void kref_rmsnorm(const float* x, const float* w, float* out, int n, void* stream) {
  kernel::rmsnorm_kernel_cu(wrap1(DataType::kDataTypeFp32, n, x),
                                    wrap1(DataType::kDataTypeFp32, n, w),
                                    wrap1(DataType::kDataTypeFp32, n, out), stream);
}

void kref_add(const float* a, const float* b, float* out, int n, void* stream) {
  kernel::add_kernel_cu(wrap1(DataType::kDataTypeFp32, n, a),
                                wrap1(DataType::kDataTypeFp32, n, b),
                                wrap1(DataType::kDataTypeFp32, n, out), stream);
}

void kref_swiglu(const float* a, const float* b, float* out, int n, void* stream) {
  kernel::swiglu_kernel_cu(wrap1(DataType::kDataTypeFp32, n, a),
                                   wrap1(DataType::kDataTypeFp32, n, b),
                                   wrap1(DataType::kDataTypeFp32, n, out), stream);
}

void kref_sincos(int head_size, int seq_len, float* sin_cache, float* cos_cache, void* stream) {
  kernel::sin_cos_cache_calc_cu(head_size, seq_len,
                                wrap1(DataType::kDataTypeFp32, head_size * seq_len, sin_cache),
                                wrap1(DataType::kDataTypeFp32, head_size * seq_len, cos_cache),
                                static_cast<cudaStream_t>(stream));
}

// q[dim], k[kv_dim] rotated in place; pos is passed by value (the reference reads it from a
// host int32 tensor, rope_kernel.cu:157).
void kref_rope(int dim, int kv_dim, int head_size, float* q, float* k, int pos,
               const float* sin_cache, const float* cos_cache, int seq_len, void* stream) {
  int32_t pos_host = pos;
  Tensor pos_t(DataType::kDataTypeInt32, 1, false, nullptr, &pos_host);
  pos_t.set_device_type(DeviceType::kDeviceCPU);
  kernel::rope_kernel_cu(dim, kv_dim, head_size, wrap1(DataType::kDataTypeFp32, dim, q),
                                 wrap1(DataType::kDataTypeFp32, kv_dim, k), pos_t,
                                 wrap1(DataType::kDataTypeFp32, head_size * seq_len, sin_cache),
                                 wrap1(DataType::kDataTypeFp32, head_size * seq_len, cos_cache),
                                 stream);
}

void kref_mha(int pos, int head_num, int layer_index, int seq_len, int kv_dim, int kv_mul,
              int head_size, float* out, const float* q, float* score, const float* key_cache,
              const float* value_cache, int layer_num, void* stream) {
  BorrowedConfig bc(stream);
  kernel::mha_kernel_cu(
      pos, head_num, layer_index, seq_len, kv_dim, kv_mul, head_size,
      wrap1(DataType::kDataTypeFp32, head_num * head_size, out),
      wrap1(DataType::kDataTypeFp32, head_num * head_size, q),
      wrap2(DataType::kDataTypeFp32, head_num, seq_len, score),
      wrap3(DataType::kDataTypeFp32, layer_num, seq_len, kv_dim, key_cache),
      wrap3(DataType::kDataTypeFp32, layer_num, seq_len, kv_dim, value_cache), kCUDA, &bc.cfg);
}

// tokens are HOST int32 (embedding.cpp:24-25); table/out are device pointers.
void kref_embedding(const int32_t* tokens_host, int n_tokens, const float* table, float* out,
                    int dim, int vocab, void* stream) {
  Tensor tok(DataType::kDataTypeInt32, n_tokens, false, nullptr,
             const_cast<int32_t*>(tokens_host));
  tok.set_device_type(DeviceType::kDeviceCPU);
  // emb_kernel_cu clones + to_cuda()s the token tensor, which needs an allocator on the
  // source buffer; give it one by cloning into an owned CPU tensor first.
  Tensor tok_owned(DataType::kDataTypeInt32, n_tokens, true,
                   base::CPUDeviceAllocatorFactory::get_instance());
  std::memcpy(tok_owned.ptr<int32_t>(), tokens_host, sizeof(int32_t) * n_tokens);
  kernel::emb_kernel_cu(tok_owned, wrap2(DataType::kDataTypeFp32, vocab, dim, table),
                                wrap2(DataType::kDataTypeFp32, n_tokens, dim, out), vocab, stream);
}

int64_t kref_argmax(const float* logits, int64_t n, void* stream) {
  size_t idx = kernel::argmax_kernel_cu(logits, static_cast<size_t>(n), stream);
  cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  return static_cast<int64_t>(idx);
}

#ifndef KREF_KERNELS_ONLY
// ---------------------------------------------------------------------------------------
// Whole-model runner: the reference's own LLama2Model on its stock CUDA path.
// ---------------------------------------------------------------------------------------
struct KrefModel {
  std::unique_ptr<model::LLama2Model> m;
};

void* kref_model_create(const char* checkpoint_path, int is_quant) {
  auto h = std::make_unique<KrefModel>();
  h->m = std::make_unique<model::LLama2Model>(base::TokenizerType::kEncodeSpe, "stub-tokenizer",
                                              checkpoint_path, is_quant != 0);
  auto st = h->m->init(DeviceType::kDeviceCUDA);
  if (!st) {
    fprintf(stderr, "kref_model_create: %s\n", st.get_err_msg().c_str());
    return nullptr;
  }
  return h.release();
}

void kref_model_destroy(void* handle) { delete static_cast<KrefModel*>(handle); }

// One decode position, exactly the way demo/main.cpp:18-29 drives the model.
// Returns the greedy next id; if logits_host != nullptr copies the fp32 logits out.
int kref_model_step(void* handle, int token, int pos, float* logits_host, int vocab) {
  auto* h = static_cast<KrefModel*>(handle);
  const model::LLama2Model& m = *h->m;
  tensor::Tensor pos_tensor = m.get_buffer(model::ModelBufferType::kInputPos);
  pos_tensor.index<int32_t>(0) = pos;
  std::vector<int32_t> tokens{token};
  const auto& emb = m.embedding(tokens);
  tensor::Tensor input = m.fill_input(pos_tensor, emb, false);
  int next = -1;
  m.predict(input, pos_tensor, false, next);
  if (logits_host) {
    const tensor::Tensor& logits = m.get_buffer(model::ModelBufferType::kForwardOutput);
    cudaDeviceSynchronize();
    cudaMemcpy(logits_host, logits.ptr<float>(), sizeof(float) * vocab, cudaMemcpyDeviceToHost);
  }
  return next;
}
#endif  // KREF_KERNELS_ONLY

}  // extern "C"
