// The kernel registry: the plug point of the kuiper:: operator API.  A layer asks
// `kernel::get_<op>_kernel(device_type)` for a plain function pointer and calls it with tensors;
// type names, getter names and argument order/meaning are those of the reference's
// kuiper/source/op/kernels/kernels_interface.h, so its layers and tests bind unchanged (outputs are
// passed as `const Tensor&` and written through, as there).
//
// Here every getter answers kDeviceCUDA with an adapter (kernels_interfaces.cpp) that unwraps the
// tensors and calls the sm_90a C-ABI of include/kllm_b200.h.  There is NO CPU backend: asking for
// kDeviceCPU is a fatal error saying so (the CPU restatement of the reference lives under oracle/
// and is test infrastructure only).  The scale / softmax / scale-sum entries exist because the
// reference's CPU attention is assembled from them; on CUDA attention is one kernel.
#ifndef KLLM_KUIPER_KERNELS_INTERFACE_H_
#define KLLM_KUIPER_KERNELS_INTERFACE_H_
#include <base/cuda_config.h>

#include "tensor/tensor.h"

namespace kernel {
using Ref = const tensor::Tensor&;  // every tensor argument, inputs and outputs alike

// element-wise
using AddKernel = void (*)(Ref a, Ref b, Ref out, void* stream);                      // out = a + b
using SwigluKernel = void (*)(Ref gate, Ref up, Ref out, void* stream);               // out = silu(gate) * up
using ScaleKernel = void (*)(float scale, Ref inout, void* stream);               // inout *= scale
using SoftmaxInplaceKernel = void (*)(Ref inout, void* stream);
using ScaleSumKernel = void (*)(Ref value, Ref scale, Ref out, int t, int size, int stride, void* stream);
// row-wise
using RMSNormKernel = void (*)(Ref x, Ref weight, Ref out, void* stream);             // out = x * rsqrt(mean x^2 + eps) * weight
using EmbeddingKernel = void (*)(Ref token_ids, Ref table, Ref out, int32_t vocab_size, void* stream);
// out[K] = weight[K, M] . x[M]; `scale` is ignored on CUDA; int8: fp32 scale per group_size weights
using MatmulKernel = void (*)(Ref x, Ref weight, Ref out, float scale, const CudaConfig* config);
using MatmulKernelQuant = void (*)(Ref x, Ref weight, Ref out, int32_t group_size, Ref scales, const CudaConfig* config);
// rotates q[dim] and k[kv_dim] in place by the angles of position *pos (a CPU int32 tensor)
using RoPEKernel = void (*)(int32_t dim, int32_t kv_dim, int32_t head_size, Ref q, Ref k, Ref pos, Ref sin_cache,
                            Ref cos_cache, void* stream);
// one position of grouped-query attention over cache rows [0, pos] of layer `layer_index`
using MHAKernel = void (*)(int32_t pos, int32_t head_num, int32_t layer_index, int32_t seq_len, int32_t kv_dim,
                           int32_t kv_mul, int32_t head_size, Ref mha_out, Ref query, Ref score, Ref key_cache,
                           Ref value_cache, base::DeviceType device_type, CudaConfig* config);

AddKernel get_add_kernel(base::DeviceType device_type);
SwigluKernel get_swiglu_kernel(base::DeviceType device_type, void* stream = nullptr);
ScaleKernel get_scale_kernel(base::DeviceType device_type);
SoftmaxInplaceKernel get_softmax_kernel(base::DeviceType device_type);
ScaleSumKernel get_scale_sum_kernel(base::DeviceType device_type);
RMSNormKernel get_rmsnorm_kernel(base::DeviceType device_type);
EmbeddingKernel get_emb_kernel(base::DeviceType device_type);
MatmulKernel get_matmul_kernel(base::DeviceType device_type);
MatmulKernelQuant get_matmul_kernel_quant8(base::DeviceType device_type);
RoPEKernel get_rope_kernel(base::DeviceType device_type);
MHAKernel get_mha_kernel(base::DeviceType device_type);

// Entry points model code calls directly: the RoPE sin / cos tables [max_seq_len, head_size] and
// the blocking greedy argmax (index of the maximum, lowest index on ties).
void sin_cos_cache_calc_cu(int head_size, int max_seq_len, Ref sin_cache, Ref cos_cache, cudaStream_t stream);
size_t argmax_kernel_cu(const float* input_ptr, size_t size, void* stream);

// RoPE pairing / constants this library was built for: KLLM_FLAVOUR_* of kllm_b200.h, chosen by
// the same compile definitions as the reference (LLAMA3_SUPPORT / QWEN2_SUPPORT / none).
int build_flavour();
}  // namespace kernel
#endif  // KLLM_KUIPER_KERNELS_INTERFACE_H_
