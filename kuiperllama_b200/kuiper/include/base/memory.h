// Memory of the kuiper:: API surface: device allocators and base::Buffer (the reference splits
// these over base/alloc.h and base/buffer.h; both forward here).
//
//   DeviceAllocator       allocate / release / memcpy / memset_zero for one kind of device
//   CPUDeviceAllocator    aligned host memory
//   CUDADeviceAllocator   pooled cudaMalloc: released blocks go to size-keyed free lists per device
//                         and are handed out again (the reference scans two vectors linearly per
//                         call; nothing on the per-token path allocates here at all)
//   *AllocatorFactory     process-wide instances, `get_instance()`
//   Buffer                a byte range + who frees it: owns memory from an allocator, or wraps a
//                         pointer the caller keeps alive (use_external) -- checkpoint views
#ifndef KLLM_KUIPER_BASE_MEMORY_H_
#define KLLM_KUIPER_BASE_MEMORY_H_
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <utility>
#include <vector>

#include "base.h"

namespace base {
enum class MemcpyKind { kMemcpyCPU2CPU = 0, kMemcpyCPU2CUDA = 1, kMemcpyCUDA2CPU = 2, kMemcpyCUDA2CUDA = 3 };

class DeviceAllocator {
 public:
  explicit DeviceAllocator(DeviceType device_type) : device_type_(device_type) {}
  virtual ~DeviceAllocator() = default;
  virtual DeviceType device_type() const { return device_type_; }

  virtual void* allocate(size_t byte_size) const = 0;
  virtual void release(void* ptr) const = 0;
  // copies on `stream` when one is given (async unless need_sync), else blocking
  virtual void memcpy(const void* src_ptr, void* dest_ptr, size_t byte_size,
                      MemcpyKind memcpy_kind = MemcpyKind::kMemcpyCPU2CPU, void* stream = nullptr,
                      bool need_sync = false) const;
  virtual void memset_zero(void* ptr, size_t byte_size, void* stream, bool need_sync = false);

 private:
  DeviceType device_type_ = DeviceType::kDeviceUnknown;
};

// Host -> device staging for checkpoint uploads.  The reference copies every weight straight out of
// the pageable mmap with a blocking cudaMemcpy (tensor.cpp:104-119 via alloc.cpp:14-38), which the
// driver serialises through its own bounce buffer: page faults, the host copy and the DMA take turns.
// Here large copies go through two pinned buffers: while the copy engine drains one, the host fills
// the other from the mapping (page-cache reads overlap the DMA).  One instance per process; copies of
// less than kMinBytes, and everything after a failed pinned allocation, take the plain path.
// fp32 -> bf16 bits, round to nearest even (torch.Tensor.to(torch.bfloat16)): finite values past the largest bf16
// become inf, NaN stays a quiet NaN of the same sign.
inline uint16_t fp32_to_bf16_rne(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40u);
  return static_cast<uint16_t>((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

class PinnedUploader {
 public:
  static constexpr size_t kChunkBytes = size_t(32) << 20;
  static constexpr size_t kMinBytes = size_t(1) << 20;
  static PinnedUploader& instance();
  ~PinnedUploader();
  // enqueue host -> device on `stream`; returns false if the pinned path is unavailable
  bool upload(void* dst_device, const void* src_host, size_t bytes, void* stream);
  // the same for n fp32 values that land on the device as bf16 (fp32_to_bf16_rne), rounded chunk by chunk while
  // they are staged: only the 2-byte values cross the bus
  bool upload_bf16(void* dst_device, const float* src_host, size_t n, void* stream);
  size_t bytes_uploaded() const { return uploaded_; }

 private:
  PinnedUploader() = default;
  bool ensure();
  void* pinned_[2] = {nullptr, nullptr};
  void* done_[2] = {nullptr, nullptr};  // cudaEvent_t: the DMA out of pinned_[i] has finished
  bool busy_[2] = {false, false};
  int next_ = 0;
  bool failed_ = false;
  size_t uploaded_ = 0;
  std::mutex mu_;
};

class CPUDeviceAllocator final : public DeviceAllocator {
 public:
  CPUDeviceAllocator() : DeviceAllocator(DeviceType::kDeviceCPU) {}
  void* allocate(size_t byte_size) const override;
  void release(void* ptr) const override;
};

class CUDADeviceAllocator final : public DeviceAllocator {
 public:
  CUDADeviceAllocator() : DeviceAllocator(DeviceType::kDeviceCUDA) {}
  ~CUDADeviceAllocator() override;
  void* allocate(size_t byte_size) const override;
  void release(void* ptr) const override;
  size_t cached_bytes() const;  // parked in the free lists, all devices

 private:
  struct Block {
    int device;
    size_t bytes;
  };
  mutable std::mutex mu_;
  mutable std::unordered_map<void*, Block> live_;                      // handed out
  mutable std::map<std::pair<int, size_t>, std::vector<void*>> free_;  // (device, size) -> blocks
  mutable size_t cached_ = 0;
};

template <typename Allocator>
struct AllocatorFactory {
  static std::shared_ptr<Allocator> get_instance() {
    static const std::shared_ptr<Allocator> instance = std::make_shared<Allocator>();
    return instance;
  }
};
using CPUDeviceAllocatorFactory = AllocatorFactory<CPUDeviceAllocator>;
using CUDADeviceAllocatorFactory = AllocatorFactory<CUDADeviceAllocator>;

class Buffer : public NoCopyable, public std::enable_shared_from_this<Buffer> {
 public:
  Buffer() = default;
  // no ptr + an allocator: allocate now and own the memory;
  // ptr: wrap it -- with use_external the buffer never frees it
  explicit Buffer(size_t byte_size, std::shared_ptr<DeviceAllocator> allocator = nullptr, void* ptr = nullptr,
                  bool use_external = false);
  virtual ~Buffer();

  bool allocate();  // (re)allocate byte_size() bytes from the allocator; false without one
  // copies min(byte sizes) bytes, direction from the two device types
  void copy_from(const Buffer& buffer) const;
  void copy_from(const Buffer* buffer) const;

  void* ptr() { return ptr_; }
  const void* ptr() const { return ptr_; }
  size_t byte_size() const { return byte_size_; }
  bool is_external() const { return use_external_; }
  std::shared_ptr<DeviceAllocator> allocator() const { return allocator_; }
  DeviceType device_type() const { return device_type_; }
  void set_device_type(DeviceType device_type) { device_type_ = device_type; }
  std::shared_ptr<Buffer> get_shared_from_this() { return shared_from_this(); }

 private:
  size_t byte_size_ = 0;
  void* ptr_ = nullptr;
  bool use_external_ = false;
  DeviceType device_type_ = DeviceType::kDeviceUnknown;
  std::shared_ptr<DeviceAllocator> allocator_;
};
}  // namespace base
#endif  // KLLM_KUIPER_BASE_MEMORY_H_
