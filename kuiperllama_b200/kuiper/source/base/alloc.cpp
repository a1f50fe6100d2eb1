// Allocators + memcpy/memset helpers (reference alloc.cpp:4-60, alloc_cpu.cpp:13-31,
// alloc_cu.cpp:7-112 for the behaviour; the pooling strategy is ours, see base/memory.h).
#include "base/memory.h"

#include <cuda_runtime_api.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

namespace base {
namespace {
cudaMemcpyKind to_cuda_kind(MemcpyKind k) {
  switch (k) {
    case MemcpyKind::kMemcpyCPU2CUDA: return cudaMemcpyHostToDevice;
    case MemcpyKind::kMemcpyCUDA2CPU: return cudaMemcpyDeviceToHost;
    case MemcpyKind::kMemcpyCUDA2CUDA: return cudaMemcpyDeviceToDevice;
    default: return cudaMemcpyHostToHost;
  }
}
// pooled sizes: round up so that similar requests share a bucket
size_t bucket_size(size_t n) {
  if (n <= 256) return 256;
  if (n <= (1u << 20)) {  // next power of two up to 1 MiB
    size_t p = 512;
    while (p < n) p <<= 1;
    return p;
  }
  const size_t mib = size_t(1) << 20;  // then 1 MiB granularity
  return (n + mib - 1) / mib * mib;
}
}  // namespace

void DeviceAllocator::memcpy(const void* src_ptr, void* dest_ptr, size_t byte_size,
                             MemcpyKind memcpy_kind, void* stream, bool need_sync) const {
  CHECK_NE(src_ptr, nullptr);
  CHECK_NE(dest_ptr, nullptr);
  if (byte_size == 0) return;
  if (memcpy_kind == MemcpyKind::kMemcpyCPU2CPU) {
    std::memcpy(dest_ptr, src_ptr, byte_size);
  } else if (memcpy_kind == MemcpyKind::kMemcpyCPU2CUDA && stream != nullptr && byte_size >= PinnedUploader::kMinBytes &&
             PinnedUploader::instance().upload(dest_ptr, src_ptr, byte_size, stream)) {
    // checkpoint-sized host -> device copy: pinned, double-buffered (see PinnedUploader)
  } else {
    cudaError_t e;
    if (stream != nullptr) {
      e = cudaMemcpyAsync(dest_ptr, src_ptr, byte_size, to_cuda_kind(memcpy_kind),
                          static_cast<cudaStream_t>(stream));
    } else {
      e = cudaMemcpy(dest_ptr, src_ptr, byte_size, to_cuda_kind(memcpy_kind));
    }
    CHECK(e == cudaSuccess) << "memcpy failed: " << cudaGetErrorString(e);
  }
  if (need_sync) cudaDeviceSynchronize();
}

// ---- PinnedUploader ------------------------------------------------------------------------------------
PinnedUploader& PinnedUploader::instance() {
  static PinnedUploader u;
  return u;
}
bool PinnedUploader::ensure() {
  if (failed_) return false;
  if (pinned_[0] != nullptr) return true;
  for (int i = 0; i < 2; ++i) {
    cudaEvent_t ev = nullptr;
    if (cudaMallocHost(&pinned_[i], kChunkBytes) != cudaSuccess ||
        cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
      failed_ = true;
      cudaGetLastError();
      return false;
    }
    done_[i] = ev;
  }
  return true;
}
bool PinnedUploader::upload(void* dst_device, const void* src_host, size_t bytes, void* stream) {
  std::lock_guard<std::mutex> lock(mu_);
  if (!ensure()) return false;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* src = static_cast<const char*>(src_host);
  char* dst = static_cast<char*>(dst_device);
  for (size_t off = 0; off < bytes; off += kChunkBytes) {
    const size_t n = std::min(kChunkBytes, bytes - off);
    const int b = next_;
    next_ ^= 1;
    if (busy_[b]) cudaEventSynchronize(static_cast<cudaEvent_t>(done_[b]));  // its previous DMA has drained
    std::memcpy(pinned_[b], src + off, n);  // page faults + host copy overlap the other buffer's DMA
    if (cudaMemcpyAsync(dst + off, pinned_[b], n, cudaMemcpyHostToDevice, s) != cudaSuccess) return false;
    cudaEventRecord(static_cast<cudaEvent_t>(done_[b]), s);
    busy_[b] = true;
  }
  uploaded_ += bytes;
  return true;
}
bool PinnedUploader::upload_bf16(void* dst_device, const float* src_host, size_t n, void* stream) {
  std::lock_guard<std::mutex> lock(mu_);
  if (!ensure()) return false;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* dst = static_cast<char*>(dst_device);
  const size_t per_chunk = kChunkBytes / sizeof(uint16_t);
  for (size_t off = 0; off < n; off += per_chunk) {
    const size_t k = std::min(per_chunk, n - off);
    const int b = next_;
    next_ ^= 1;
    if (busy_[b]) cudaEventSynchronize(static_cast<cudaEvent_t>(done_[b]));
    uint16_t* staged = static_cast<uint16_t*>(pinned_[b]);
    for (size_t i = 0; i < k; ++i) staged[i] = fp32_to_bf16_rne(src_host[off + i]);
    if (cudaMemcpyAsync(dst + off * sizeof(uint16_t), staged, k * sizeof(uint16_t), cudaMemcpyHostToDevice, s) !=
        cudaSuccess)
      return false;
    cudaEventRecord(static_cast<cudaEvent_t>(done_[b]), s);
    busy_[b] = true;
  }
  uploaded_ += n * sizeof(uint16_t);
  return true;
}
PinnedUploader::~PinnedUploader() {
  for (int i = 0; i < 2; ++i) {
    if (done_[i]) cudaEventDestroy(static_cast<cudaEvent_t>(done_[i]));
    if (pinned_[i]) cudaFreeHost(pinned_[i]);
  }
}

void DeviceAllocator::memset_zero(void* ptr, size_t byte_size, void* stream, bool need_sync) {
  CHECK(device_type_ != DeviceType::kDeviceUnknown);
  if (device_type_ == DeviceType::kDeviceCPU) {
    std::memset(ptr, 0, byte_size);
    return;
  }
  if (stream != nullptr) {
    cudaMemsetAsync(ptr, 0, byte_size, static_cast<cudaStream_t>(stream));
  } else {
    cudaMemset(ptr, 0, byte_size);
  }
  if (need_sync) cudaDeviceSynchronize();
}

// ---- CPU -------------------------------------------------------------------------------------

void* CPUDeviceAllocator::allocate(size_t byte_size) const {
  if (byte_size == 0) return nullptr;
  void* p = nullptr;
  // 64-byte alignment: cache line, and enough for any vector load the host side does
  if (posix_memalign(&p, 64, byte_size) != 0) return nullptr;
  return p;
}

void CPUDeviceAllocator::release(void* ptr) const {
  if (ptr != nullptr) std::free(ptr);
}

// ---- CUDA ------------------------------------------------------------------------------------

CUDADeviceAllocator::~CUDADeviceAllocator() {
  // process teardown: the driver may already be gone, so errors are ignored on purpose
  for (auto& kv : free_)
    for (void* p : kv.second) cudaFree(p);
}

void* CUDADeviceAllocator::allocate(size_t byte_size) const {
  if (byte_size == 0) return nullptr;
  int dev = -1;
  CHECK(cudaGetDevice(&dev) == cudaSuccess) << "no CUDA device";
  const size_t want = bucket_size(byte_size);
  std::lock_guard<std::mutex> lock(mu_);
  auto it = free_.find({dev, want});
  if (it != free_.end() && !it->second.empty()) {
    void* p = it->second.back();
    it->second.pop_back();
    cached_ -= want;
    live_[p] = Block{dev, want};
    return p;
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, want);
  if (e != cudaSuccess) {
    // give cached blocks back to the driver once, then retry
    for (auto& kv : free_) {
      for (void* q : kv.second) cudaFree(q);
      kv.second.clear();
    }
    cached_ = 0;
    cudaGetLastError();
    e = cudaMalloc(&p, want);
  }
  if (e != cudaSuccess) {
    LOG(ERROR) << "CUDA error when allocating " << (want >> 20) << " MB: " << cudaGetErrorString(e);
    return nullptr;
  }
  live_[p] = Block{dev, want};
  return p;
}

void CUDADeviceAllocator::release(void* ptr) const {
  if (ptr == nullptr) return;
  std::lock_guard<std::mutex> lock(mu_);
  auto it = live_.find(ptr);
  if (it == live_.end()) {
    // not ours (or already released): hand it to the driver like the reference's fallback
    cudaFree(ptr);
    return;
  }
  const Block b = it->second;
  live_.erase(it);
  // keep at most 1 GiB parked (the reference trims its small-buffer list at the same mark)
  if (cached_ + b.bytes > (size_t(1) << 30)) {
    cudaFree(ptr);
    return;
  }
  free_[{b.device, b.bytes}].push_back(ptr);
  cached_ += b.bytes;
}

size_t CUDADeviceAllocator::cached_bytes() const {
  std::lock_guard<std::mutex> lock(mu_);
  return cached_;
}

}  // namespace base
