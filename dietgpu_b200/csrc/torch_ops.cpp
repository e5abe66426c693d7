// torch_ops.cpp -- torch.ops.dietgpu.* backed by libdietgpu_b200.so.
//
// Registers the reference's ten operators with the reference's exact schema strings
// (/root/reference/dietgpu/DietGpu.cpp:915-937) so that code written against
// `torch.ops.load_library(<dietgpu>)` works by loading this library instead.  Argument validation,
// return values and error behaviour follow DietGpu.cpp:149-911; tensors are only handles to device
// memory -- all compute is in the CUDA library (include/dietgpu_b200.h).
//
// Every codec call goes to a dgb_* entry point and every return code becomes a TORCH_CHECK, so input the C ABI
// refuses raises RuntimeError instead of aborting the process (the compat header keeps the reference's abort for
// C++ callers; here only its StackDeviceMemory leases the scratch).  Where the reference would write or read
// memory the caller did not hand over, these operators differ on purpose, as dietgpu_b200/ops.py does: byte
// batches of mixed dtypes get rows sized by their largest member in bytes, split sizes must fit the tensor they
// index, float outputs must share one dtype, and archives and output rows must be 16 B aligned.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/types.h>

#include <limits>
#include <optional>
#include <tuple>
#include <vector>

#include "../../include/dietgpu_b200_compat.hpp"

namespace dgt {
using namespace dietgpu;
using torch::Tensor;

constexpr int kPrecision = 10;  // DietGpu.cpp:114

FloatType floatTypeOf(const Tensor& t) {
  switch (t.scalar_type()) {
    case at::ScalarType::Half: return FloatType::kFloat16;
    case at::ScalarType::BFloat16: return FloatType::kBFloat16;
    case at::ScalarType::Float: return FloatType::kFloat32;
    case at::ScalarType::Double: return FloatType::kFloat64;
    default: TORCH_CHECK(false, "dietgpu: unsupported float dtype ", t.scalar_type());
  }
  return FloatType::kUndefined;
}
at::ScalarType dtypeOf(FloatType ft) {
  switch (ft) {
    case FloatType::kFloat16: return at::ScalarType::Half;
    case FloatType::kBFloat16: return at::ScalarType::BFloat16;
    case FloatType::kFloat32: return at::ScalarType::Float;
    case FloatType::kFloat64: return at::ScalarType::Double;
    default: TORCH_CHECK(false, "dietgpu: invalid float type in archive");
  }
  return at::ScalarType::Half;
}

// largest member in elements and, separately, in bytes (a byte batch may mix dtypes)
std::tuple<int64_t, int64_t> maxNumelAndBytes(const std::vector<Tensor>& ts) {
  int64_t mx = 0, mxBytes = 0;
  for (auto& t : ts) {
    TORCH_CHECK((uint64_t)t.numel() * t.element_size() <= std::numeric_limits<uint32_t>::max());
    mx = std::max<int64_t>(mx, t.numel());
    mxBytes = std::max<int64_t>(mxBytes, t.numel() * t.element_size());
  }
  return {mx, mxBytes};
}

void checkRc(int rc, const char* what) {
  TORCH_CHECK(rc == DGB_OK, "dietgpu: ", what, " failed: ", dgb_error_string(rc), " (code ", rc,
              rc == DGB_ERR_CUDA ? ", cudaError " + std::to_string(dgb_last_cuda_error()) : std::string(), ")");
}
void checkDecodeRc(int rc, bool asFloat, const char* what) {
  TORCH_CHECK(rc != DGB_ERR_CHECKSUM, asFloat ? "floatDecompress" : "ANSDecode",
              ": checksum mismatch seen on decoded data; archive cannot be unpacked");
  checkRc(rc, what);
}
void checkArchiveAligned(const Tensor& t) {
  TORCH_CHECK(uintptr_t(t.data_ptr()) % 16 == 0, "dietgpu: compressed input is not 16 B aligned");
}
void checkSplitTotal(const std::vector<uint32_t>& split, int64_t capacity, const char* what) {
  int64_t total = 0;
  for (auto s : split) total += s;
  TORCH_CHECK(total <= capacity, "dietgpu: split sizes sum to ", total, ", more than ", what, " holds (", capacity,
              ")");
}

StackDeviceMemory makeRes(const std::optional<Tensor>& temp, const Tensor& like) {
  if (temp) {
    TORCH_CHECK(temp->is_cuda() && temp->is_contiguous());
    TORCH_CHECK(temp->get_device() == like.get_device());
    return StackDeviceMemory(like.get_device(), temp->data_ptr(), temp->numel() * temp->element_size());
  }
  return StackDeviceMemory(like.get_device(), nullptr, 0);
}

// The scratch of one codec call: `need` bytes leased from temp_mem when it holds them at a 256 B boundary.
// The reference falls back to cudaMalloc inside StackDeviceMemory when scratch is missing; here the op
// uses a stream-ordered torch allocation instead, so the common "no temp_mem" call stays asynchronous
// and the lease never takes StackDeviceMemory's cudaMalloc path.
struct Scratch {
  Tensor owned;
  StackDeviceMemory res;
  StackDeviceMemory::Lease lease;  // declared last: released before `res` goes away
  Scratch(const std::optional<Tensor>& temp, const Tensor& like, size_t need, cudaStream_t stream)
      : res(makeRes(temp, like)) {
    const size_t granular = (std::max<size_t>(need, 1) + kSDMAlignment - 1) / kSDMAlignment * kSDMAlignment;
    if (res.getSizeAvailable() < granular) {
      owned = torch::empty({(int64_t)granular + 256}, at::TensorOptions().device(like.device()).dtype(torch::kByte));
      res = StackDeviceMemory(like.get_device(), owned.data_ptr(), granular + 256);
    }
    lease = res.lease(need, stream);
  }
  void* ptr() const { return lease.ptr; }
  size_t bytes() const { return lease.bytes; }
  int64_t used() const { return (int64_t)res.getMaxMemoryUsage(); }
};

// ---- sizes ----------------------------------------------------------------
// The C ABI reports "worst-case archive exceeds the format's 32-bit sizes" as 0 (the reference
// CHECK-aborts, ans/GpuANSEncode.cu:22); never size an output tensor from that.
int64_t bound(uint32_t v) {
  TORCH_CHECK(v != 0, "dietgpu: input too large for one archive (32-bit format limit)");
  return (int64_t)v;
}
std::tuple<int64_t, int64_t> max_float_compressed_output_size(const std::vector<Tensor>& ts) {
  TORCH_CHECK(!ts.empty());
  auto s = maxNumelAndBytes(ts);
  return {(int64_t)ts.size(), bound(getMaxFloatCompressedSize(floatTypeOf(ts[0]), std::get<0>(s)))};
}
int64_t max_float_compressed_size(const Tensor& dtype, int64_t size) {
  return bound(getMaxFloatCompressedSize(floatTypeOf(dtype), size));
}
std::tuple<int64_t, int64_t> max_any_compressed_output_size(const std::vector<Tensor>& ts) {
  TORCH_CHECK(!ts.empty());
  // rows sized by the largest member in bytes; the reference multiplies the largest element count by the
  // first member's element size (DietGpu.cpp:134), too small for a batch of mixed dtypes
  auto s = maxNumelAndBytes(ts);
  return {(int64_t)ts.size(), bound(getMaxCompressedSize(std::get<1>(s)))};
}
int64_t max_any_compressed_size(int64_t bytes) { return bound(getMaxCompressedSize(bytes)); }

// ---- compress ---------------------------------------------------------------
void validateOut(const std::optional<Tensor>& outCompressed, const std::optional<Tensor>& outSizes, int64_t n,
                 int64_t cols, const Tensor& like, Tensor& comp, Tensor& sizes) {
  if (outCompressed) {
    TORCH_CHECK(outCompressed->dtype() == torch::kByte && outCompressed->is_cuda() && outCompressed->is_contiguous());
    TORCH_CHECK(outCompressed->dim() == 2 && outCompressed->size(0) >= n && outCompressed->size(1) >= cols);
    TORCH_CHECK(outCompressed->get_device() == like.get_device());
    TORCH_CHECK(uintptr_t(outCompressed->data_ptr()) % 16 == 0 && (n <= 1 || outCompressed->size(1) % 16 == 0),
                "dietgpu: out_compressed rows are not 16 B aligned");
    comp = *outCompressed;
  } else {
    comp = torch::empty({n, cols}, at::TensorOptions().device(like.device()).dtype(torch::kByte));
  }
  if (outSizes) {
    TORCH_CHECK(outSizes->dtype() == torch::kInt && outSizes->is_cuda() && outSizes->dim() == 1);
    TORCH_CHECK(outSizes->is_contiguous() && outSizes->size(0) >= n && outSizes->get_device() == like.get_device());
    sizes = *outSizes;
  } else {
    sizes = torch::empty({n}, at::TensorOptions().device(like.device()).dtype(torch::kInt));
  }
}

std::tuple<Tensor, Tensor, int64_t> compress_data(bool asFloat, const std::vector<Tensor>& tIns, bool checksum,
                                                   const std::optional<Tensor>& tempMem,
                                                   const std::optional<Tensor>& outCompressed,
                                                   const std::optional<Tensor>& outSizes) {
  TORCH_CHECK(!tIns.empty());
  c10::cuda::CUDAGuard guard(tIns.front().device());
  for (auto& t : tIns) {
    TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.get_device() == tIns[0].get_device());
    if (asFloat) {
      TORCH_CHECK(t.dtype() == tIns[0].dtype());
      floatTypeOf(t);
    }
  }
  const int64_t n = tIns.size();
  auto mo = asFloat ? max_float_compressed_output_size(tIns) : max_any_compressed_output_size(tIns);
  Tensor comp, sizes;
  validateOut(outCompressed, outSizes, n, std::get<1>(mo), tIns[0], comp, sizes);
  std::vector<const void*> in(n);
  std::vector<uint32_t> inSize(n);
  std::vector<void*> out(n);
  uint32_t maxSize = 0;
  for (int64_t i = 0; i < n; ++i) {
    in[i] = tIns[i].data_ptr();
    inSize[i] = asFloat ? tIns[i].numel() : tIns[i].numel() * tIns[i].element_size();
    out[i] = (uint8_t*)comp.data_ptr() + i * comp.size(1);
    maxSize = std::max(maxSize, inSize[i]);
  }
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (asFloat) {
    const int ft = (int)floatTypeOf(tIns[0]);
    Scratch sc(tempMem, tIns[0], dgb_float_compress_temp_bytes(ft, n, maxSize), stream);
    checkRc(dgb_float_compress_pointer(sc.ptr(), sc.bytes(), ft, kPrecision, checksum, n, in.data(), inSize.data(),
                                       out.data(), (uint32_t*)sizes.data_ptr(), stream),
            "compress_data");
    return {comp, sizes, sc.used()};
  }
  Scratch sc(tempMem, tIns[0], dgb_ans_encode_temp_bytes(n, maxSize), stream);
  checkRc(dgb_ans_encode_pointer(sc.ptr(), sc.bytes(), kPrecision, checksum, n, in.data(), inSize.data(), nullptr,
                                 out.data(), (uint32_t*)sizes.data_ptr(), stream),
          "compress_data");
  return {comp, sizes, sc.used()};
}

std::vector<Tensor> matrixToTensors(int64_t n, Tensor& matrix, Tensor& sizes) {
  auto host = sizes.narrow(0, 0, n).to(torch::kCPU);  // synchronises, DietGpu.cpp:75-103
  auto flat = matrix.view({matrix.numel()});
  auto cols = matrix.size(1);
  std::vector<Tensor> out(n);
  for (int64_t i = 0; i < n; ++i) out[i] = flat.narrow(0, i * cols, host.data_ptr<int32_t>()[i]);
  return out;
}

std::tuple<std::vector<Tensor>, Tensor, int64_t> compress_data_split_size(
    bool asFloat, const Tensor& tIn, const Tensor& tSplit, bool checksum, const std::optional<Tensor>& tempMem,
    const std::optional<Tensor>& outCompressed, const std::optional<Tensor>& outSizes) {
  c10::cuda::CUDAGuard guard(tIn.device());
  TORCH_CHECK(tIn.is_cuda() && tIn.is_contiguous());
  auto ft = asFloat ? floatTypeOf(tIn) : FloatType::kUndefined;
  if (!asFloat) TORCH_CHECK(uintptr_t(tIn.data_ptr()) % kANSRequiredAlignment == 0, "start pointer is not aligned");
  TORCH_CHECK(tSplit.is_contiguous() && tSplit.device().type() == at::kCPU && tSplit.dtype() == torch::kInt);
  const int64_t n = tSplit.numel();
  std::vector<uint32_t> split(n);
  uint32_t maxSize = 0;
  for (int64_t i = 0; i < n; ++i) {
    auto size = tSplit.data_ptr<int32_t>()[i];
    TORCH_CHECK(size > 0);
    split[i] = size;
    maxSize = std::max<uint32_t>(maxSize, size);
    if (!asFloat && i != n - 1)
      TORCH_CHECK(size % kANSRequiredAlignment == 0, "the size of an interior split is not a multiple of 4 bytes");
  }
  // splits count words of tIn's dtype for floats, bytes otherwise
  checkSplitTotal(split, asFloat ? tIn.numel() : tIn.numel() * tIn.element_size(), "t_in");
  const int64_t cols = bound(asFloat ? getMaxFloatCompressedSize(ft, maxSize) : getMaxCompressedSize(maxSize));
  Tensor comp, sizes;
  validateOut(outCompressed, outSizes, n, cols, tIn, comp, sizes);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  int64_t used = 0;
  if (asFloat) {
    Scratch sc(tempMem, tIn, dgb_float_compress_temp_bytes((int)ft, n, maxSize), stream);
    checkRc(dgb_float_compress_split_size(sc.ptr(), sc.bytes(), (int)ft, kPrecision, checksum, n, tIn.data_ptr(),
                                          split.data(), comp.data_ptr(), comp.size(1), (uint32_t*)sizes.data_ptr(),
                                          stream),
            "compress_data_split_size");
    used = sc.used();
  } else {
    Scratch sc(tempMem, tIn, dgb_ans_encode_temp_bytes(n, maxSize), stream);
    checkRc(dgb_ans_encode_split_size(sc.ptr(), sc.bytes(), kPrecision, checksum, n, tIn.data_ptr(), split.data(),
                                      nullptr, comp.data_ptr(), comp.size(1), (uint32_t*)sizes.data_ptr(), stream),
            "compress_data_split_size");
    used = sc.used();
  }
  return {matrixToTensors(n, comp, sizes), sizes, used};
}

std::vector<Tensor> compress_data_simple(bool asFloat, const std::vector<Tensor>& tIns, bool checksum,
                                         const std::optional<int64_t>& tempMem) {
  TORCH_CHECK(!tIns.empty());
  std::optional<Tensor> scratch;
  if (tempMem && *tempMem > 0)
    scratch = torch::empty({*tempMem}, at::TensorOptions().device(tIns[0].device()).dtype(torch::kByte));
  auto r = compress_data(asFloat, tIns, checksum, scratch, std::nullopt, std::nullopt);
  auto& comp = std::get<0>(r);
  auto host = std::get<1>(r).to(torch::kCPU);
  std::vector<Tensor> out;
  for (size_t i = 0; i < tIns.size(); ++i)
    out.push_back(comp[i].narrow(0, 0, host.data_ptr<int32_t>()[i]).clone());
  return out;
}

// ---- decompress -------------------------------------------------------------
void validateStatus(const std::optional<Tensor>& outStatus, const std::optional<Tensor>& outSizes, int64_t n,
                    const Tensor& like) {
  if (outStatus)
    TORCH_CHECK(outStatus->is_contiguous() && outStatus->is_cuda() && outStatus->dtype() == torch::kByte &&
                outStatus->numel() == n && outStatus->get_device() == like.get_device());
  if (outSizes)
    TORCH_CHECK(outSizes->is_contiguous() && outSizes->is_cuda() && outSizes->dtype() == torch::kInt32 &&
                outSizes->numel() == n && outSizes->get_device() == like.get_device());
}

int64_t decompressImpl(bool asFloat, const std::vector<Tensor>& tIns, const std::vector<Tensor>& tOuts, bool checksum,
                       const std::optional<Tensor>& tempMem, const std::optional<Tensor>& outStatus,
                       const std::optional<Tensor>& outSizes) {
  TORCH_CHECK(!tIns.empty() && tIns.size() == tOuts.size());
  c10::cuda::CUDAGuard guard(tIns.front().device());
  const int64_t n = tIns.size();
  std::vector<const void*> in(n);
  std::vector<void*> out(n);
  std::vector<uint32_t> cap(n);
  for (int64_t i = 0; i < n; ++i) {
    auto& ti = tIns[i];
    auto& to = tOuts[i];
    TORCH_CHECK(ti.is_cuda() && ti.is_contiguous() && ti.dtype() == torch::kByte);
    TORCH_CHECK(ti.get_device() == tIns[0].get_device());
    checkArchiveAligned(ti);
    TORCH_CHECK(to.is_cuda() && to.is_contiguous() && to.get_device() == ti.get_device());
    if (asFloat) {
      floatTypeOf(to);
      // capacities are counted in words of one float type
      TORCH_CHECK(to.dtype() == tOuts[0].dtype(), "dietgpu: float outputs must all have the same dtype");
    }
    in[i] = ti.data_ptr();
    out[i] = to.data_ptr();
    auto c = asFloat ? to.numel() : to.numel() * to.element_size();
    TORCH_CHECK((uint64_t)c <= std::numeric_limits<uint32_t>::max());
    cap[i] = c;
  }
  validateStatus(outStatus, outSizes, n, tIns[0]);
  auto st = (uint8_t*)(outStatus ? outStatus->data_ptr() : nullptr);
  auto sz = (uint32_t*)(outSizes ? outSizes->data_ptr() : nullptr);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (asFloat) {
    const int ft = (int)floatTypeOf(tOuts[0]);
    Scratch sc(tempMem, tIns[0], dgb_float_decompress_temp_bytes(ft, n, 0), stream);
    checkDecodeRc(dgb_float_decompress_pointer(sc.ptr(), sc.bytes(), ft, kPrecision, checksum, n, in.data(),
                                               out.data(), cap.data(), st, sz, nullptr, stream),
                  true, "decompress_data");
    return sc.used();
  }
  Scratch sc(tempMem, tIns[0], dgb_ans_decode_temp_bytes(n), stream);
  checkDecodeRc(dgb_ans_decode_pointer(sc.ptr(), sc.bytes(), kPrecision, checksum, n, in.data(), out.data(),
                                       cap.data(), st, sz, nullptr, stream),
                false, "decompress_data");
  return sc.used();
}

int64_t decompress_data(bool asFloat, const std::vector<Tensor>& tIns, const std::vector<Tensor>& tOuts, bool checksum,
                        const std::optional<Tensor>& tempMem, const std::optional<Tensor>& outStatus,
                        const std::optional<Tensor>& outSizes) {
  return decompressImpl(asFloat, tIns, tOuts, checksum, tempMem, outStatus, outSizes);
}

int64_t decompress_data_split_size(bool asFloat, const std::vector<Tensor>& tIns, Tensor& tOut, const Tensor& tSplit,
                                   bool checksum, const std::optional<Tensor>& tempMem,
                                   const std::optional<Tensor>& outStatus, const std::optional<Tensor>& outSizes) {
  TORCH_CHECK(!tIns.empty());
  c10::cuda::CUDAGuard guard(tIns.front().device());
  const int64_t n = tSplit.numel();
  TORCH_CHECK(tSplit.device().type() == at::kCPU && tSplit.dtype() == torch::kInt && tSplit.is_contiguous());
  TORCH_CHECK(n == (int64_t)tIns.size());
  std::vector<const void*> in(n);
  std::vector<uint32_t> split(n);
  for (int64_t i = 0; i < n; ++i) {
    TORCH_CHECK(tIns[i].is_cuda() && tIns[i].is_contiguous() && tIns[i].dtype() == torch::kByte);
    TORCH_CHECK(tIns[i].get_device() == tIns[0].get_device());
    checkArchiveAligned(tIns[i]);
    in[i] = tIns[i].data_ptr();
    auto s = tSplit.data_ptr<int32_t>()[i];
    TORCH_CHECK(s > 0);
    split[i] = s;
  }
  TORCH_CHECK(tOut.is_cuda() && tOut.is_contiguous());
  TORCH_CHECK(tOut.get_device() == tIns[0].get_device(), "dietgpu: t_out is not on the device of the compressed inputs");
  const int ft = asFloat ? (int)floatTypeOf(tOut) : 0;
  checkSplitTotal(split, asFloat ? tOut.numel() : tOut.numel() * tOut.element_size(), "t_out");
  validateStatus(outStatus, outSizes, n, tIns[0]);
  auto st = (uint8_t*)(outStatus ? outStatus->data_ptr() : nullptr);
  auto sz = (uint32_t*)(outSizes ? outSizes->data_ptr() : nullptr);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (asFloat) {
    Scratch sc(tempMem, tIns[0], dgb_float_decompress_temp_bytes(ft, n, 0), stream);
    checkDecodeRc(dgb_float_decompress_split_size(sc.ptr(), sc.bytes(), ft, kPrecision, checksum, n, in.data(),
                                                  tOut.data_ptr(), split.data(), st, sz, nullptr, stream),
                  true, "decompress_data_split_size");
    return sc.used();
  }
  Scratch sc(tempMem, tIns[0], dgb_ans_decode_temp_bytes(n), stream);
  checkDecodeRc(dgb_ans_decode_split_size(sc.ptr(), sc.bytes(), kPrecision, checksum, n, in.data(), tOut.data_ptr(),
                                          split.data(), st, sz, nullptr, stream),
                false, "decompress_data_split_size");
  return sc.used();
}

std::vector<Tensor> decompress_data_simple(bool asFloat, const std::vector<Tensor>& tIns, bool checksum,
                                           const std::optional<int64_t>& tempMem) {
  TORCH_CHECK(!tIns.empty());
  c10::cuda::CUDAGuard guard(tIns.front().device());
  const int64_t n = tIns.size();
  auto opts = at::TensorOptions().device(tIns[0].device());
  auto sizes = torch::empty({n}, opts.dtype(torch::kInt));
  auto types = torch::zeros({n}, opts.dtype(torch::kInt));
  std::vector<const void*> in(n);
  for (int64_t i = 0; i < n; ++i) {
    TORCH_CHECK(tIns[i].is_cuda() && tIns[i].get_device() == tIns[0].get_device());
    checkArchiveAligned(tIns[i]);
    in[i] = tIns[i].data_ptr();
  }
  {
    cudaStream_t stream = at::cuda::getCurrentCUDAStream();
    Scratch sc(std::nullopt, tIns[0], sizeof(void*) * n + 256, stream);
    checkRc(asFloat ? dgb_float_get_compressed_info(sc.ptr(), sc.bytes(), in.data(), 0, n, (uint32_t*)sizes.data_ptr(),
                                                    (uint32_t*)types.data_ptr(), nullptr, stream)
                    : dgb_ans_get_compressed_info(sc.ptr(), sc.bytes(), in.data(), 0, n, (uint32_t*)sizes.data_ptr(),
                                                  nullptr, stream),
            "get_compressed_info");
  }
  auto hs = sizes.to(torch::kCPU), ht = types.to(torch::kCPU);
  std::vector<Tensor> outs;
  for (int64_t i = 0; i < n; ++i) {
    auto size = hs.data_ptr<int32_t>()[i];
    if (asFloat) {
      TORCH_CHECK(ht.data_ptr<int32_t>()[i] == ht.data_ptr<int32_t>()[0],
                  "dietgpu: inconsistent / invalid float type in archives");
      outs.push_back(torch::empty({size}, opts.dtype(dtypeOf((FloatType)ht.data_ptr<int32_t>()[i]))));
    } else {
      outs.push_back(torch::empty({size}, opts.dtype(torch::kByte)));
    }
  }
  std::optional<Tensor> scratch;
  if (tempMem && *tempMem >= 256) scratch = torch::empty({*tempMem}, opts.dtype(torch::kByte));
  decompressImpl(asFloat, tIns, outs, checksum, scratch, std::nullopt, std::nullopt);
  return outs;
}

}  // namespace dgt

// Schema strings: DietGpu.cpp:915-937, verbatim (they are the interface).
TORCH_LIBRARY_FRAGMENT(dietgpu, m) {
  m.def("max_float_compressed_output_size(Tensor[] ts) -> (int, int)");
  m.def("max_float_compressed_size(Tensor dtype, int size) -> int");
  m.def("max_any_compressed_output_size(Tensor[] ts) -> (int, int)");
  m.def("max_any_compressed_size(int bytes) -> int");
  m.def("compress_data(bool compress_as_float, Tensor[] ts_in, bool checksum=False, Tensor? temp_mem=None, Tensor? out_compressed=None, Tensor? out_compressed_bytes=None) -> (Tensor, Tensor, int)");
  m.def("compress_data_split_size(bool compress_as_float, Tensor t_in, Tensor t_in_split_sizes, bool checksum=False, Tensor? temp_mem=None, Tensor? out_compressed=None, Tensor? out_compressed_bytes=None) -> (Tensor[], Tensor, int)");
  m.def("compress_data_simple(bool compress_as_float, Tensor[] ts_in, bool checksum=False, int? temp_mem=67108864) -> Tensor[]");
  m.def("decompress_data(bool compress_as_float, Tensor[] ts_in, Tensor[] ts_out, bool checksum=False, Tensor? temp_mem=None, Tensor? out_status=None, Tensor? out_decompressed_words=None) -> (int)");
  m.def("decompress_data_split_size(bool compress_as_float, Tensor[] ts_in, Tensor t_out, Tensor t_out_split_sizes, bool checksum=False, Tensor? temp_mem=None, Tensor? out_status=None, Tensor? out_decompressed_words=None) -> (int)");
  m.def("decompress_data_simple(bool compress_as_float, Tensor[] ts_in, bool checksum=False, int? temp_mem=67108864) -> Tensor[]");
}

TORCH_LIBRARY(dietgpu, m) {
  m.impl("max_float_compressed_output_size", TORCH_FN(dgt::max_float_compressed_output_size));
  m.impl("max_float_compressed_size", TORCH_FN(dgt::max_float_compressed_size));
  m.impl("max_any_compressed_output_size", TORCH_FN(dgt::max_any_compressed_output_size));
  m.impl("max_any_compressed_size", TORCH_FN(dgt::max_any_compressed_size));
  m.impl("compress_data", TORCH_FN(dgt::compress_data));
  m.impl("compress_data_split_size", TORCH_FN(dgt::compress_data_split_size));
  m.impl("compress_data_simple", TORCH_FN(dgt::compress_data_simple));
  m.impl("decompress_data", TORCH_FN(dgt::decompress_data));
  m.impl("decompress_data_split_size", TORCH_FN(dgt::decompress_data_split_size));
  m.impl("decompress_data_simple", TORCH_FN(dgt::decompress_data_simple));
}
