// dietgpu_b200_compat.hpp -- the reference's C++ API surface, header-only, on top of the C ABI.
//
// A caller of facebookresearch/dietgpu's C++ API (dietgpu/ans/GpuANSCodec.h:65-341,
// dietgpu/float/GpuFloatCodec.h:31-292, dietgpu/utils/StackDeviceMemory.h) can include this
// header instead, link libdietgpu_b200.so, and keep its call sites: same namespace, same
// function names, same argument order and meaning, same status types.  Every function forwards
// to one dgb_* entry point of include/dietgpu_b200.h.
//
// Error behaviour mirrors the reference: API misuse / CUDA failure aborts the process with a
// message (the reference's glog CHECK, utils/DeviceUtils.h:33-39); a checksum mismatch is
// returned in the status struct (ans/GpuANSDecode.cuh:581-590).
//
// Written for this repository from the API's documented contract; it shares no source text with
// the reference headers.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

#include "dietgpu_b200.h"

namespace dietgpu {

constexpr int kANSRequiredAlignment = DGB_ANS_REQUIRED_ALIGNMENT;  // ans/GpuANSCodec.h:16
constexpr int kANSDefaultProbBits = DGB_ANS_DEFAULT_PROB_BITS;     // ans/GpuANSCodec.h:20

namespace detail {
[[noreturn]] inline void fail(const char* what, int code) {
  std::fprintf(stderr, "dietgpu_b200: %s failed: %s (code %d, cudaError %d)\n", what,
               dgb_error_string(code), code, dgb_last_cuda_error());
  std::abort();
}
inline void check(const char* what, int code) {
  if (code != DGB_OK && code != DGB_ERR_CHECKSUM) fail(what, code);
}
}  // namespace detail

// ---- utils/StackDeviceMemory.h:17-299 ----------------------------------------------------------
// The scratch arena every API call takes as its first argument: a LIFO bump allocator over one
// device region (owned or caller-provided), 256 B granularity, with the reference's overflow
// behaviour -- a Temporary request that does not fit, and every Permanent request, is served by
// cudaMalloc (Temporary overflows warn on stderr) and freed on release
// (utils/StackDeviceMemory.cpp:105-184).  Temporary reservations must be released in reverse
// order (:181); GpuMemoryReservation<T> does that on destruction.
constexpr size_t kDefaultStackSize = 256 * 1024 * 1024;  // utils/StackDeviceMemory.h:19
constexpr size_t kSDMAlignment = 256;                    // utils/StackDeviceMemory.h:24

enum class AllocType { Temporary, Permanent };

class StackDeviceMemory;

template <typename T>
struct GpuMemoryReservation {
  GpuMemoryReservation() = default;
  GpuMemoryReservation(StackDeviceMemory* r, int dev, cudaStream_t str, void* p, size_t n, size_t szAlloc)
      : res(r), device(dev), stream(str), ptr(p), num(n), sizeAllocated(szAlloc) {}
  GpuMemoryReservation(const GpuMemoryReservation&) = delete;
  GpuMemoryReservation& operator=(const GpuMemoryReservation&) = delete;
  GpuMemoryReservation(GpuMemoryReservation&& m) noexcept { take(m); }
  GpuMemoryReservation& operator=(GpuMemoryReservation&& m) {
    if (this != &m) {
      release();
      take(m);
    }
    return *this;
  }
  ~GpuMemoryReservation() { release(); }

  T* data() { return static_cast<T*>(ptr); }
  const T* data() const { return static_cast<const T*>(ptr); }

  // device -> host std::vector<T>, ordered after `onStream` (pageable destination: the copy has
  // completed when this returns, which is what the reference's tests rely on)
  std::vector<T> copyToHost(cudaStream_t onStream) const {
    std::vector<T> out(num);
    if (num && cudaMemcpyAsync(out.data(), ptr, num * sizeof(T), cudaMemcpyDeviceToHost, onStream) != cudaSuccess)
      detail::fail("GpuMemoryReservation::copyToHost", DGB_ERR_CUDA);
    return out;
  }

  inline void release();

  StackDeviceMemory* res = nullptr;
  int device = 0;
  cudaStream_t stream = nullptr;
  void* ptr = nullptr;
  size_t num = 0;            // valid elements of T
  size_t sizeAllocated = 0;  // bytes taken from the arena

 private:
  void take(GpuMemoryReservation& m) {
    res = m.res; device = m.device; stream = m.stream; ptr = m.ptr; num = m.num; sizeAllocated = m.sizeAllocated;
    m.res = nullptr; m.ptr = nullptr; m.num = 0; m.sizeAllocated = 0;
  }
};

class StackDeviceMemory {
 public:
  StackDeviceMemory(int device, size_t allocPerDevice) : device_(device) {
    if (allocPerDevice) {
      int prev = 0;
      cudaGetDevice(&prev);
      cudaSetDevice(device);
      const size_t bytes = (allocPerDevice + kSDMAlignment - 1) / kSDMAlignment * kSDMAlignment;
      if (cudaMalloc(&owned_, bytes) != cudaSuccess) detail::fail("StackDeviceMemory cudaMalloc", DGB_ERR_CUDA);
      cudaSetDevice(prev);
      setRegion(owned_, bytes);
    }
  }
  StackDeviceMemory(int device, void* p, size_t size) : device_(device) { setRegion(p, p ? size : 0); }
  StackDeviceMemory(const StackDeviceMemory&) = delete;
  StackDeviceMemory& operator=(const StackDeviceMemory&) = delete;
  // movable only while no reservation is outstanding (reservations point back at the arena)
  StackDeviceMemory(StackDeviceMemory&& o) noexcept { swap(o); }
  StackDeviceMemory& operator=(StackDeviceMemory&& o) noexcept {
    swap(o);
    return *this;
  }
  ~StackDeviceMemory() {
    for (auto& ov : overflow_) cudaFree(ov.first);
    if (owned_) cudaFree(owned_);
  }

  int getDevice() const { return device_; }

  template <typename T>
  GpuMemoryReservation<T> alloc(cudaStream_t stream, size_t num, AllocType type = AllocType::Temporary) {
    size_t bytes = (num * sizeof(T) + kSDMAlignment - 1) / kSDMAlignment * kSDMAlignment;
    bytes = std::max(bytes, kSDMAlignment);
    return GpuMemoryReservation<T>(this, device_, stream, allocPointer(stream, bytes, type), num, bytes);
  }
  // host (or device) array -> new reservation, copy ordered on `stream`
  template <typename T>
  GpuMemoryReservation<T> copyAlloc(cudaStream_t stream, const T* src, size_t num, AllocType type = AllocType::Temporary) {
    auto mem = alloc<T>(stream, num, type);
    if (num && cudaMemcpyAsync(mem.data(), src, num * sizeof(T), cudaMemcpyDefault, stream) != cudaSuccess)
      detail::fail("StackDeviceMemory::copyAlloc", DGB_ERR_CUDA);
    return mem;
  }
  template <typename T>
  GpuMemoryReservation<T> copyAlloc(cudaStream_t stream, const std::vector<T>& v, AllocType type = AllocType::Temporary) {
    return copyAlloc<T>(stream, v.data(), v.size(), type);
  }

  // size: a multiple of kSDMAlignment
  void* allocPointer(cudaStream_t, size_t size, AllocType type) {
    if (size == 0 || size % kSDMAlignment) detail::fail("StackDeviceMemory::allocPointer (size not 256 B granular)", DGB_ERR_INVALID_ARG);
    void* out = nullptr;
    const size_t used = (size_t)(head_ - start_);
    if (type == AllocType::Permanent || size > getSizeAvailable()) {
      if (type == AllocType::Temporary) {
        std::fprintf(stderr,
                     "dietgpu_b200 WARNING: StackDeviceMemory: %zu bytes requested with %zu available; calling "
                     "cudaMalloc. Size the temporary memory to >= %zu bytes to avoid this.\n",
                     size, getSizeAvailable(), std::max(maxSeen_, used + overflowBytes_ + size));
      }
      int prev = 0;
      cudaGetDevice(&prev);
      if (prev != device_) cudaSetDevice(device_);
      if (cudaMalloc(&out, size) != cudaSuccess) detail::fail("StackDeviceMemory overflow cudaMalloc", DGB_ERR_CUDA);
      if (prev != device_) cudaSetDevice(prev);
      overflow_.emplace_back(out, size);
      overflowBytes_ += size;
    } else {
      out = head_;
      head_ += size;
    }
    maxSeen_ = std::max(maxSeen_, (size_t)(head_ - start_) + overflowBytes_);
    return out;
  }
  void deallocPointer(int device, cudaStream_t stream, size_t size, void* p) {
    if (!p || device != device_) detail::fail("StackDeviceMemory::deallocPointer", DGB_ERR_INVALID_ARG);
    for (size_t i = 0; i < overflow_.size(); ++i) {
      if (overflow_[i].first == p) {
        // kernels that use the region may still be queued on the stream it was handed out for
        cudaStreamSynchronize(stream);
        cudaFree(p);
        overflowBytes_ -= overflow_[i].second;
        overflow_.erase(overflow_.begin() + (long)i);
        return;
      }
    }
    char* pc = static_cast<char*>(p);
    // Temporary reservations are returned in reverse order (utils/StackDeviceMemory.cpp:181)
    if (pc < start_ || pc + size != head_) detail::fail("StackDeviceMemory: reservations released out of order", DGB_ERR_INVALID_ARG);
    head_ = pc;
  }

  size_t getSizeAvailable() const { return (size_t)(end_ - head_); }
  size_t getSizeTotal() const { return (size_t)(end_ - start_); }
  size_t getMaxMemoryUsage() const { return maxSeen_; }
  void resetMaxMemoryUsage() { maxSeen_ = 0; }
  std::string toString() const {
    return "SDM device " + std::to_string(device_) + ": total " + std::to_string(getSizeTotal()) + " B, available " +
           std::to_string(getSizeAvailable()) + " B, maximum seen usage " + std::to_string(maxSeen_) + " B\n";
  }

  // One scratch region for the duration of a codec call (the C ABI takes a plain pointer + size).
  struct Lease {
    GpuMemoryReservation<uint8_t> mem;
    void* ptr = nullptr;
    size_t bytes = 0;
  };
  Lease lease(size_t need, cudaStream_t stream) {
    Lease l;
    l.mem = alloc<uint8_t>(stream, std::max<size_t>(need, 1));
    l.ptr = l.mem.data();
    l.bytes = need;
    return l;
  }

 private:
  void setRegion(void* p, size_t size) {
    // allocations are handed out on 256 B boundaries whatever the caller's pointer is
    const uintptr_t a = (reinterpret_cast<uintptr_t>(p) + kSDMAlignment - 1) & ~uintptr_t(kSDMAlignment - 1);
    const size_t pad = (size_t)(a - reinterpret_cast<uintptr_t>(p));
    start_ = head_ = reinterpret_cast<char*>(a);
    end_ = start_ + (size > pad ? (size - pad) / kSDMAlignment * kSDMAlignment : 0);
  }
  void swap(StackDeviceMemory& o) {
    std::swap(device_, o.device_); std::swap(owned_, o.owned_); std::swap(start_, o.start_);
    std::swap(end_, o.end_); std::swap(head_, o.head_); std::swap(overflow_, o.overflow_);
    std::swap(overflowBytes_, o.overflowBytes_); std::swap(maxSeen_, o.maxSeen_);
  }
  int device_ = 0;
  void* owned_ = nullptr;
  char* start_ = nullptr;
  char* end_ = nullptr;
  char* head_ = nullptr;
  std::vector<std::pair<void*, size_t>> overflow_;
  size_t overflowBytes_ = 0;
  size_t maxSeen_ = 0;
};

template <typename T>
inline void GpuMemoryReservation<T>::release() {
  if (ptr && res) res->deallocPointer(device, stream, sizeAllocated, ptr);
  res = nullptr;
  ptr = nullptr;
  num = 0;
  sizeAllocated = 0;
}

// utils/StackDeviceMemory.h:297-299 / .cpp:248-250
inline StackDeviceMemory makeStackMemory(size_t bytes = kDefaultStackSize) {
  int dev = 0;
  cudaGetDevice(&dev);
  return StackDeviceMemory(dev, bytes);
}

// ---- ans/GpuANSCodec.h:22-59 ----
inline uint32_t getMaxCompressedSize(uint32_t uncompressedBytes) { return dgb_ans_max_compressed_size(uncompressedBytes); }

struct ANSCodecConfig {
  ANSCodecConfig() : probBits(kANSDefaultProbBits), useChecksum(false) {}
  explicit ANSCodecConfig(int pb, bool checksum = false) : probBits(pb), useChecksum(checksum) {}
  int probBits;
  bool useChecksum;
};

enum class ANSDecodeError : uint32_t { None = 0, ChecksumMismatch = 1 };

struct ANSDecodeStatus {
  ANSDecodeStatus() : error(ANSDecodeError::None) {}
  ANSDecodeError error;
  std::vector<std::pair<int, std::string>> errorInfo;
};

// ---- float/GpuFloatCodec.h:18-97 ----
// kFloat64, kFloat16Sparse, kBFloat16Sparse, kFloat32Sparse: this library's extensions (archives of float types
// 4, 5, 6 and 8, which the reference cannot read)
enum class FloatType : uint32_t {
  kUndefined = 0,
  kFloat16 = 1,
  kBFloat16 = 2,
  kFloat32 = 3,
  kFloat64 = 4,
  kFloat16Sparse = 5,
  kBFloat16Sparse = 6,
  kFloat32Sparse = 8
};

inline uint32_t getMaxFloatCompressedSize(FloatType ft, uint32_t size) {
  return dgb_float_max_compressed_size((int)ft, size);
}

struct FloatCodecConfig {
  FloatCodecConfig() : floatType(FloatType::kFloat16), useChecksum(false), is16ByteAligned(false) {}
  FloatCodecConfig(FloatType ft, const ANSCodecConfig& ansConf, bool align, bool checksum = false)
      : floatType(ft), useChecksum(checksum), ansConfig(ansConf), is16ByteAligned(align) {}
  FloatType floatType;
  bool useChecksum;
  ANSCodecConfig ansConfig;
  bool is16ByteAligned;  // accepted for compatibility; the fused decode needs no alignment hint
};
using FloatCompressConfig = FloatCodecConfig;
using FloatDecompressConfig = FloatCodecConfig;

enum class FloatDecompressError : uint32_t { None = 0, ChecksumMismatch = 1 };

struct FloatDecompressStatus {
  FloatDecompressStatus() : error(FloatDecompressError::None) {}
  FloatDecompressError error;
  std::vector<std::pair<int, std::string>> errorInfo;
};

namespace detail {
template <typename Status, typename Err>
Status makeStatus(int rc, const std::vector<uint8_t>& mismatch, Err mismatchErr) {
  Status st;
  if (rc == DGB_ERR_CHECKSUM) {
    st.error = mismatchErr;
    for (size_t i = 0; i < mismatch.size(); ++i)
      if (mismatch[i]) st.errorInfo.emplace_back((int)i, "Checksum mismatch in batch member " + std::to_string(i) + "\n");
  }
  return st;
}
inline uint32_t maxOf(const uint32_t* v, uint32_t n) {
  uint32_t m = 0;
  for (uint32_t i = 0; i < n; ++i) m = std::max(m, v[i]);
  return m;
}
}  // namespace detail

// ---- encode (ans/GpuANSCodec.h:65-164) ----
inline void ansEncodeBatchStride(StackDeviceMemory& res, const ANSCodecConfig& config, uint32_t numInBatch,
                                 const void* in_dev, uint32_t inPerBatchSize, uint32_t inPerBatchStride,
                                 const uint32_t* histogram_dev, void* out_dev, uint32_t outPerBatchStride,
                                 uint32_t* outBatchSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_encode_temp_bytes(numInBatch, inPerBatchSize), stream);
  detail::check("ansEncodeBatchStride",
                dgb_ans_encode_stride(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in_dev,
                                      inPerBatchSize, inPerBatchStride, histogram_dev, out_dev, outPerBatchStride,
                                      outBatchSize_dev, stream));
}

inline void ansEncodeBatchPointer(StackDeviceMemory& res, const ANSCodecConfig& config, uint32_t numInBatch,
                                  const void** in, const uint32_t* inSize, const uint32_t* histogram_dev,
                                  void** out, uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_encode_temp_bytes(numInBatch, detail::maxOf(inSize, numInBatch)), stream);
  detail::check("ansEncodeBatchPointer",
                dgb_ans_encode_pointer(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in, inSize,
                                       histogram_dev, out, outSize_dev, stream));
}

inline void ansEncodeBatchSplitSize(StackDeviceMemory& res, const ANSCodecConfig& config, uint32_t numInBatch,
                                    const void* in_dev, const uint32_t* inSplitSizes, const uint32_t* histogram_dev,
                                    void* out_dev, uint32_t outStride, uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_encode_temp_bytes(numInBatch, detail::maxOf(inSplitSizes, numInBatch)), stream);
  detail::check("ansEncodeBatchSplitSize",
                dgb_ans_encode_split_size(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in_dev,
                                          inSplitSizes, histogram_dev, out_dev, outStride, outSize_dev, stream));
}

// ---- decode (ans/GpuANSCodec.h:170-303) ----
inline ANSDecodeStatus ansDecodeBatchStride(StackDeviceMemory& res, const ANSCodecConfig& config, uint32_t numInBatch,
                                            const void* in_dev, uint32_t inPerBatchStride, void* out_dev,
                                            uint32_t outPerBatchStride, uint32_t outPerBatchCapacity,
                                            uint8_t* outSuccess_dev, uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_decode_temp_bytes(numInBatch), stream);
  std::vector<uint8_t> mm(numInBatch);
  int rc = dgb_ans_decode_stride(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in_dev,
                                 inPerBatchStride, out_dev, outPerBatchStride, outPerBatchCapacity, outSuccess_dev,
                                 outSize_dev, mm.data(), stream);
  detail::check("ansDecodeBatchStride", rc);
  return detail::makeStatus<ANSDecodeStatus>(rc, mm, ANSDecodeError::ChecksumMismatch);
}

inline ANSDecodeStatus ansDecodeBatchPointer(StackDeviceMemory& res, const ANSCodecConfig& config, uint32_t numInBatch,
                                             const void** in, void** out, const uint32_t* outCapacity,
                                             uint8_t* outSuccess_dev, uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_decode_temp_bytes(numInBatch), stream);
  std::vector<uint8_t> mm(numInBatch);
  int rc = dgb_ans_decode_pointer(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in, out,
                                  outCapacity, outSuccess_dev, outSize_dev, mm.data(), stream);
  detail::check("ansDecodeBatchPointer", rc);
  return detail::makeStatus<ANSDecodeStatus>(rc, mm, ANSDecodeError::ChecksumMismatch);
}

inline ANSDecodeStatus ansDecodeBatchSplitSize(StackDeviceMemory& res, const ANSCodecConfig& config,
                                               uint32_t numInBatch, const void** in, void* out_dev,
                                               const uint32_t* outSplitSizes, uint8_t* outSuccess_dev,
                                               uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_ans_decode_temp_bytes(numInBatch), stream);
  std::vector<uint8_t> mm(numInBatch);
  int rc = dgb_ans_decode_split_size(l.ptr, l.bytes, config.probBits, config.useChecksum, numInBatch, in, out_dev,
                                     outSplitSizes, outSuccess_dev, outSize_dev, mm.data(), stream);
  detail::check("ansDecodeBatchSplitSize", rc);
  return detail::makeStatus<ANSDecodeStatus>(rc, mm, ANSDecodeError::ChecksumMismatch);
}

// ---- information (ans/GpuANSCodec.h:309-341) ----
inline void ansGetCompressedInfo(StackDeviceMemory& res, const void** in, uint32_t numInBatch,
                                 uint32_t* outSizes_dev, uint32_t* outChecksum_dev, cudaStream_t stream) {
  auto l = res.lease(sizeof(void*) * (size_t)numInBatch + 256, stream);
  detail::check("ansGetCompressedInfo",
                dgb_ans_get_compressed_info(l.ptr, l.bytes, in, 0, numInBatch, outSizes_dev, outChecksum_dev, stream));
}
inline void ansGetCompressedInfoDevice(StackDeviceMemory&, const void** in_dev, uint32_t numInBatch,
                                       uint32_t* outSizes_dev, uint32_t* outChecksum_dev, cudaStream_t stream) {
  detail::check("ansGetCompressedInfoDevice",
                dgb_ans_get_compressed_info(nullptr, 0, in_dev, 1, numInBatch, outSizes_dev, outChecksum_dev, stream));
}

// ---- float codec (float/GpuFloatCodec.h:103-292) ----
inline void floatCompress(StackDeviceMemory& res, const FloatCompressConfig& config, uint32_t numInBatch,
                          const void** in, const uint32_t* inSize, void** out, uint32_t* outSize_dev,
                          cudaStream_t stream) {
  auto l = res.lease(dgb_float_compress_temp_bytes((int)config.floatType, numInBatch, detail::maxOf(inSize, numInBatch)), stream);
  detail::check("floatCompress",
                dgb_float_compress_pointer(l.ptr, l.bytes, (int)config.floatType, config.ansConfig.probBits,
                                           config.useChecksum, numInBatch, in, inSize, out, outSize_dev, stream));
}

inline void floatCompressSplitSize(StackDeviceMemory& res, const FloatCompressConfig& config, uint32_t numInBatch,
                                   const void* in_dev, const uint32_t* inSplitSizes, void* out_dev,
                                   uint32_t outStride, uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_float_compress_temp_bytes((int)config.floatType, numInBatch, detail::maxOf(inSplitSizes, numInBatch)), stream);
  detail::check("floatCompressSplitSize",
                dgb_float_compress_split_size(l.ptr, l.bytes, (int)config.floatType, config.ansConfig.probBits,
                                              config.useChecksum, numInBatch, in_dev, inSplitSizes, out_dev, outStride,
                                              outSize_dev, stream));
}

inline FloatDecompressStatus floatDecompress(StackDeviceMemory& res, const FloatDecompressConfig& config,
                                             uint32_t numInBatch, const void** in, void** out,
                                             const uint32_t* outCapacity, uint8_t* outSuccess_dev,
                                             uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_float_decompress_temp_bytes((int)config.floatType, numInBatch, 0), stream);
  std::vector<uint8_t> mm(numInBatch);
  int rc = dgb_float_decompress_pointer(l.ptr, l.bytes, (int)config.floatType, config.ansConfig.probBits,
                                        config.useChecksum, numInBatch, in, out, outCapacity, outSuccess_dev,
                                        outSize_dev, mm.data(), stream);
  detail::check("floatDecompress", rc);
  return detail::makeStatus<FloatDecompressStatus>(rc, mm, FloatDecompressError::ChecksumMismatch);
}

inline FloatDecompressStatus floatDecompressSplitSize(StackDeviceMemory& res, const FloatDecompressConfig& config,
                                                      uint32_t numInBatch, const void** in, void* out_dev,
                                                      const uint32_t* outSplitSizes, uint8_t* outSuccess_dev,
                                                      uint32_t* outSize_dev, cudaStream_t stream) {
  auto l = res.lease(dgb_float_decompress_temp_bytes((int)config.floatType, numInBatch, 0), stream);
  std::vector<uint8_t> mm(numInBatch);
  int rc = dgb_float_decompress_split_size(l.ptr, l.bytes, (int)config.floatType, config.ansConfig.probBits,
                                           config.useChecksum, numInBatch, in, out_dev, outSplitSizes,
                                           outSuccess_dev, outSize_dev, mm.data(), stream);
  detail::check("floatDecompressSplitSize", rc);
  return detail::makeStatus<FloatDecompressStatus>(rc, mm, FloatDecompressError::ChecksumMismatch);
}

inline void floatGetCompressedInfo(StackDeviceMemory& res, const void** in, uint32_t numInBatch,
                                   uint32_t* outSizes_dev, uint32_t* outTypes_dev, uint32_t* outChecksum_dev,
                                   cudaStream_t stream) {
  auto l = res.lease(sizeof(void*) * (size_t)numInBatch + 256, stream);
  detail::check("floatGetCompressedInfo",
                dgb_float_get_compressed_info(l.ptr, l.bytes, in, 0, numInBatch, outSizes_dev, outTypes_dev,
                                              outChecksum_dev, stream));
}
inline void floatGetCompressedInfoDevice(StackDeviceMemory&, const void** in_dev, uint32_t numInBatch,
                                         uint32_t* outSizes_dev, uint32_t* outTypes_dev,
                                         uint32_t* outChecksum_dev, cudaStream_t stream) {
  detail::check("floatGetCompressedInfoDevice",
                dgb_float_get_compressed_info(nullptr, 0, in_dev, 1, numInBatch, outSizes_dev, outTypes_dev,
                                              outChecksum_dev, stream));
}

}  // namespace dietgpu
