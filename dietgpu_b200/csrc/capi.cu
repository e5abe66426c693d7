// capi.cu -- the extern "C" boundary declared in include/dietgpu_b200.h.
// Maps the reference's three batch-addressing forms (pointer / stride / split
// size; ans/BatchProvider.cuh) onto one internal member list, so every kernel
// sees a single descriptor table.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace dgb {

// Tuning options: one process-wide set (dgb_set_option) and an optional per-thread copy that overrides it
// (dgb_set_thread_option), so threads that drive different streams can run different variants without racing;
// every codec call snapshots the effective set at entry.
static Options gOptions;
static thread_local Options tlsOptions;
static thread_local bool tlsHasOptions = false;
Options& options() { return tlsHasOptions ? tlsOptions : gOptions; }

static thread_local cudaError_t tlsLastCuda = cudaSuccess;
void setLastCudaError(cudaError_t e) { tlsLastCuda = e; }

// ---- per-kernel timing -------------------------------------------------------
namespace {
struct TimedLaunch { int slot; cudaEvent_t a, b; };
std::vector<TimedLaunch>& timedLaunches() { static std::vector<TimedLaunch> v; return v; }
std::vector<cudaEvent_t>& eventPool() { static std::vector<cudaEvent_t> v; return v; }
std::mutex& timerMutex() { static std::mutex m; return m; }  // guards the two vectors above (calls may come from several host threads)
cudaEvent_t takeEvent() {
  {
    std::lock_guard<std::mutex> lock(timerMutex());
    auto& pool = eventPool();
    if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
  }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
thread_local TimedLaunch tlsOpen[kNumSlots];
}  // namespace

HostStage& hostStage() {
  static thread_local HostStage h;
  return h;
}

namespace {
// uploadTable while capturing: up to kTableWords 8-byte words per launch, in the kernel parameters (32 KiB are allowed
// since CUDA 12.1); most tables fit the small form, which keeps the parameter block of a launch at 4 KiB
template <uint32_t WORDS>
struct TableChunk {
  unsigned long long* dst;
  uint32_t words;
  uint32_t pad;
  unsigned long long w[WORDS];
};
constexpr uint32_t kTableWordsSmall = 500, kTableWords = 4080;
static_assert(sizeof(TableChunk<kTableWordsSmall>) <= 4096 && sizeof(TableChunk<kTableWords>) <= 32764, "");

template <uint32_t WORDS>
__global__ void __launch_bounds__(256) tableKernel(const __grid_constant__ TableChunk<WORDS> c) {
  for (uint32_t i = threadIdx.x; i < c.words; i += blockDim.x) c.dst[i] = c.w[i];
}

template <uint32_t WORDS>
int launchTable(unsigned long long* dst, const unsigned long long* src, uint32_t words, cudaStream_t stream) {
  static thread_local TableChunk<WORDS> c;
  c.dst = dst;
  c.words = words;
  std::memcpy(c.w, src, (size_t)words * 8u);
  tableKernel<WORDS><<<1, 256, 0, stream>>>(c);
  DGB_CUDA_TRY(cudaGetLastError());
  return DGB_OK;
}
}  // namespace

int uploadTable(void* dst, const void* src, size_t bytes, cudaStream_t stream) {
  if ((bytes | reinterpret_cast<uintptr_t>(dst)) & 7u) return DGB_ERR_INVALID_ARG;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  DGB_CUDA_TRY(cudaStreamIsCapturing(stream, &st));
  if (st == cudaStreamCaptureStatusNone) {
    // an ordinary call: a copy from pageable memory has staged `src` when it returns, and it costs the device
    // less than a copy kernel whose parameter block holds the table (256 members, c4 in tools/walltime.py on an
    // H100 at 400 W: encode and decode each 2-5 us faster).  A captured copy would read `src` at every replay.
    DGB_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    return DGB_OK;
  }
  auto* d = static_cast<unsigned long long*>(dst);
  const auto* s = static_cast<const unsigned long long*>(src);
  for (size_t w = 0, words = bytes / 8u; w < words; w += kTableWords) {
    const uint32_t k = (uint32_t)std::min<size_t>(kTableWords, words - w);
    const int rc = k <= kTableWordsSmall ? launchTable<kTableWordsSmall>(d + w, s + w, k, stream)
                                         : launchTable<kTableWords>(d + w, s + w, k, stream);
    if (rc != DGB_OK) return rc;
  }
  return DGB_OK;
}

int checkNotCapturing(cudaStream_t stream) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  DGB_CUDA_TRY(cudaStreamIsCapturing(stream, &st));
  return st == cudaStreamCaptureStatusNone ? DGB_OK : DGB_ERR_CAPTURING;
}

int smCount() {
  // per device (a process may drive several); racing first calls write the same value
  static int cached[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!cached[dev]) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = v > 0 ? v : 132;
  }
  return cached[dev];
}

int residentCtasPerSm(const void* kernel, int threads, size_t smemBytes, int maxDynamicSmem, int* out) {
  // function attributes are per device; a thread that drives several devices keeps an entry per device.
  // A full cache overwrites its oldest entry, which costs one recomputation later.
  struct Entry {
    const void* kernel;
    int dev, threads;
    size_t smem;
    int perSm;  // 0: only the shared-memory limit is set
  };
  constexpr int kEntries = 64;
  static thread_local Entry cache[kEntries];
  static thread_local int nextEntry = 0;
  int dev = 0;
  DGB_CUDA_TRY(cudaGetDevice(&dev));
  bool limitSet = false;
  for (const Entry& e : cache) {
    if (e.kernel != kernel || e.dev != dev) continue;
    limitSet = true;
    if (!out) return DGB_OK;
    if (e.perSm && e.threads == threads && e.smem == smemBytes) {
      *out = e.perSm;
      return DGB_OK;
    }
  }
  if (!limitSet) DGB_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, maxDynamicSmem));
  int perSm = 0;
  if (out) {
    DGB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kernel, threads, smemBytes));
    perSm = std::max(perSm, 1);
    *out = perSm;
  }
  cache[nextEntry] = Entry{kernel, dev, threads, smemBytes, perSm};
  nextEntry = (nextEntry + 1) % kEntries;
  return DGB_OK;
}

// ---- sub-batches -------------------------------------------------------------
struct StreamPool {
  cudaStream_t s[kMaxParts];
  cudaEvent_t start, done[kMaxParts];
};

namespace {
// One pool per (host thread, device): the fork/join events of a call must not be shared with a call
// that another thread, or the same thread on another device, makes at the same time.  Lazily created.
int streamPool(StreamPool** out) {
  constexpr int kMaxDevices = 64;
  struct Slot {
    StreamPool pool;
    bool ready = false;
  };
  static thread_local Slot slots[kMaxDevices];
  int dev = 0;
  DGB_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) return DGB_ERR_INVALID_ARG;
  Slot& sl = slots[dev];
  if (!sl.ready) {
    // all or nothing: a partly created pool is torn down again, so a later call can retry cleanly
    StreamPool p{};
    bool ok = cudaEventCreateWithFlags(&p.start, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < kMaxParts; ++i) {
      ok = cudaStreamCreateWithFlags(&p.s[i], cudaStreamNonBlocking) == cudaSuccess &&
           cudaEventCreateWithFlags(&p.done[i], cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) {
      setLastCudaError(cudaGetLastError());
      if (p.start) cudaEventDestroy(p.start);
      for (int i = 0; i < kMaxParts; ++i) {
        if (p.s[i]) cudaStreamDestroy(p.s[i]);
        if (p.done[i]) cudaEventDestroy(p.done[i]);
      }
      return DGB_ERR_CUDA;
    }
    sl.pool = p;
    sl.ready = true;
  }
  *out = &sl.pool;
  return DGB_OK;
}

// cuts members [0,n) into `parts` contiguous ranges of roughly equal bytes; bounds has parts+1 entries
void splitParts(const MemberDesc* members, uint32_t n, uint32_t wordBytes, int parts, const Options& opt,
                uint32_t* bounds) {
  auto weight = [&](uint32_t i) { return (uint64_t)members[i].size * wordBytes; };
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; ++i) total += weight(i);
  bounds[0] = 0;
  uint64_t acc = 0;
  uint32_t idx = 0;
  // options first_part_pct / last_part_pct: size of the first / last sub-batch in percent of an equal share
  // (100 = equal); the middle sub-batches share the rest equally
  const int fp = parts > 2 ? std::max(10, std::min(200, opt.first_part_pct)) : 100;
  const int lp = parts > 2 ? std::max(10, std::min(200, opt.last_part_pct)) : 100;
  const uint64_t eq = total / (uint64_t)parts;
  const uint64_t first = eq * (uint64_t)fp / 100u, last = eq * (uint64_t)lp / 100u;
  const uint64_t mid = parts > 2 && total > first + last ? (total - first - last) / (uint64_t)(parts - 2) : eq;
  for (int p = 1; p < parts; ++p) {
    const uint64_t target = (parts > 2 && (fp != 100 || lp != 100)) ? first + mid * (uint64_t)(p - 1) : eq * (uint64_t)p;
    const uint32_t mustLeave = (uint32_t)(parts - p);  // one member for every later part
    while (idx + mustLeave < n && (idx < bounds[p - 1] + 1 || acc + weight(idx) / 2 <= target)) acc += weight(idx++);
    bounds[p] = idx;
  }
  bounds[parts] = n;
}

int autoParts(int kind, uint32_t n, uint64_t totalBytes, const Options& o) {
  if (o.timing) return 1;  // per-kernel timing wants un-overlapped launches
  int p = o.parts;
  // float encode of large batches runs in sub-batches so that the bandwidth-bound statistics kernel of
  // one sub-batch runs beside the issue-bound coder of the previous one; on H100 (400 W, tools/walltime.py,
  // 256 MiB batches) c3 encode takes 293 / 282 / 286 us with 1 / 2 / 4 sub-batches and c4 304 / 292 / 299,
  // 2 and 4 within the run-to-run spread; byte inputs gain nothing (c2: 426 / 429 us with 1 / 2)
  if (p <= 0) {
    const bool big = kind != kKindBytes && totalBytes >= (64ull << 20);
    p = !big ? 1 : (n >= 16 ? 4 : (n >= 8 ? 2 : 1));
  }
  p = std::min(p, kMaxParts);
  return (int)std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)p, n));
}
}  // namespace

SubBatches::SubBatches(int kind, const MemberDesc* members, uint32_t n, const Options& opt, bool split,
                       cudaStream_t stream)
    : stream_(stream) {
  const uint32_t wb = wordBytes(kind);
  uint64_t totalBytes = 0;
  for (uint32_t i = 0; i < n; ++i) totalBytes += (uint64_t)members[i].size * wb;
  parts_ = split ? autoParts(kind, n, totalBytes, opt) : 1;
  splitParts(members, n, wb, parts_, opt, bounds_);
}

int SubBatches::fork() {
  if (parts_ == 1) return DGB_OK;
  const int rc = streamPool(&pool_);
  if (rc != DGB_OK) return rc;
  DGB_CUDA_TRY(cudaEventRecord(pool_->start, stream_));
  return DGB_OK;
}

int SubBatches::stream(int k, cudaStream_t* out) {
  *out = stream_;
  if (parts_ == 1) return DGB_OK;
  DGB_CUDA_TRY(cudaStreamWaitEvent(pool_->s[k], pool_->start, 0));
  forked_[k] = true;
  *out = pool_->s[k];
  return DGB_OK;
}

SubBatches::~SubBatches() {
  if (!pool_) return;
  for (int k = 0; k < kMaxParts; ++k)
    if (forked_[k] && cudaEventRecord(pool_->done[k], pool_->s[k]) == cudaSuccess)
      cudaStreamWaitEvent(stream_, pool_->done[k], 0);
}

// kernels launched by this library since load (every codec launch site calls timerBegin first)
static std::atomic<int> gLaunches{0};

void timerBegin(const Options& opt, int slot, cudaStream_t stream) {
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  if (!opt.timing) return;
  TimedLaunch t{slot, takeEvent(), takeEvent()};
  cudaEventRecord(t.a, stream);
  tlsOpen[slot] = t;
}
void timerEnd(const Options& opt, int slot, cudaStream_t stream) {
  if (!opt.timing) return;
  cudaEventRecord(tlsOpen[slot].b, stream);
  std::lock_guard<std::mutex> lock(timerMutex());
  timedLaunches().push_back(tlsOpen[slot]);
}

namespace {

bool validFloatType(int ft) {
  return ft == DGB_FLOAT16 || ft == DGB_BFLOAT16 || ft == DGB_FLOAT32 || ft == DGB_FLOAT64 || isSparseKind(ft);
}

// the calling thread's member list, sized for n members
HostMember* stageMembers(uint32_t n) {
  std::vector<HostMember>& v = hostStage().members;
  v.resize(n);
  return v.data();
}

// pointer form
int buildPointer(uint32_t n, const void* const* in, const uint32_t* size, void* const* out, HostMember** members) {
  if (n && (!in || !size || !out)) return DGB_ERR_INVALID_ARG;
  HostMember* v = *members = stageMembers(n);
  for (uint32_t i = 0; i < n; ++i) v[i] = HostMember{in[i], out[i], size[i]};
  return DGB_OK;
}

}  // namespace
}  // namespace dgb

using namespace dgb;

extern "C" {

int dgb_version(void) { return 1; }

const char* dgb_error_string(int code) {
  switch (code) {
    case DGB_OK: return "ok";
    case DGB_ERR_INVALID_ARG: return "invalid argument";
    case DGB_ERR_TEMP_TOO_SMALL: return "temporary device memory too small";
    case DGB_ERR_CUDA: return "CUDA runtime error";
    case DGB_ERR_CHECKSUM: return "checksum mismatch";
    case DGB_ERR_TOO_LARGE: return "size exceeds format limits";
    case DGB_ERR_CAPTURING: return "checksum verification synchronises the stream and cannot be captured into a CUDA graph";
    default: return "unknown error";
  }
}

int dgb_last_cuda_error(void) { return (int)tlsLastCuda; }

uint32_t dgb_ans_max_compressed_size(uint32_t bytes) {
  // ans/GpuANSEncode.cu:13-25 (the header overhead is charged for a constant 4096 blocks)
  // The reference CHECKs rawSize <= INT32_MAX (process abort); this ABI returns 0 = "too large"
  // instead of a wrapped value a caller would size its output buffer from.
  uint64_t raw = ansOverhead(kBlockBytes);
  raw += (uint64_t)roundUp(kBlockBytes + kBlockBytes / 4u, 16u) * (((uint64_t)bytes + kBlockBytes - 1) / kBlockBytes);
  raw = roundUp64(raw, 16);
  return raw <= 0x7fffffffull ? (uint32_t)raw : 0u;
}

uint32_t dgb_float_max_compressed_size(int ft, uint32_t n) {
  if (!validFloatType(ft)) return 0;
  const uint32_t ans = dgb_ans_max_compressed_size(n);
  if (ans == 0u) return 0u;  // too large (see above)
  const uint64_t total = isSparseKind(ft) ? sparseExtraBytes<uint64_t>(ft, n, n) + ans
                                          : (uint64_t)kFloatHeaderBytes + ans + floatPlanesBytes<uint64_t>(ft, n);
  return total <= 0xffffffffull ? (uint32_t)total : 0u;
}

size_t dgb_ans_encode_temp_bytes(uint32_t n, uint32_t maxBytes) {
  return encodeTempBytes(kKindBytes, n, maxBytes);
}
size_t dgb_ans_decode_temp_bytes(uint32_t n) { return decodeTempBytes(kKindBytes, n); }
size_t dgb_float_compress_temp_bytes(int ft, uint32_t n, uint32_t maxFloats) {
  return validFloatType(ft) ? encodeTempBytes(ft, n, maxFloats) : 0;
}
size_t dgb_float_decompress_temp_bytes(int ft, uint32_t n, uint32_t /*maxFloats*/) {
  // the fp8 types: the scratch of their decode-and-sum
  return validFloatType(ft) || isFp8Kind(ft) ? decodeTempBytes(ft, n) : 0;
}

// ---- encode ----------------------------------------------------------------

int dgb_ans_encode_pointer(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                           const void* const* in, const uint32_t* inSize,
                           const uint32_t* histogram_dev, void* const* out, uint32_t* outSize_dev,
                           void* stream) {
  HostMember* v = nullptr;
  int rc = buildPointer(n, in, inSize, out, &v);
  if (rc) return rc;
  return encodeBatch(kKindBytes, temp, tempBytes, pb, useChecksum != 0, n, v, histogram_dev,
                     outSize_dev, (cudaStream_t)stream);
}

int dgb_ans_encode_stride(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                          const void* in_dev, uint32_t inSize, uint32_t inStride,
                          const uint32_t* histogram_dev, void* out_dev, uint32_t outStride,
                          uint32_t* outSize_dev, void* stream) {
  if (n && (!out_dev || (inSize && !in_dev))) return DGB_ERR_INVALID_ARG;
  HostMember* v = stageMembers(n);
  for (uint32_t i = 0; i < n; ++i)
    v[i] = HostMember{static_cast<const uint8_t*>(in_dev) + (size_t)i * inStride,
                      static_cast<uint8_t*>(out_dev) + (size_t)i * outStride, inSize};
  return encodeBatch(kKindBytes, temp, tempBytes, pb, useChecksum != 0, n, v, histogram_dev,
                     outSize_dev, (cudaStream_t)stream);
}

int dgb_ans_encode_split_size(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                              const void* in_dev, const uint32_t* splitSizes,
                              const uint32_t* histogram_dev, void* out_dev, uint32_t outStride,
                              uint32_t* outSize_dev, void* stream) {
  if (n && (!splitSizes || !out_dev)) return DGB_ERR_INVALID_ARG;
  HostMember* v = stageMembers(n);
  size_t off = 0;
  for (uint32_t i = 0; i < n; ++i) {
    // ans/GpuANSEncode.cu:132-140: interior splits must keep 4 B alignment
    if (i + 1 != n && (splitSizes[i] % DGB_ANS_REQUIRED_ALIGNMENT)) return DGB_ERR_INVALID_ARG;
    v[i] = HostMember{static_cast<const uint8_t*>(in_dev) + off,
                      static_cast<uint8_t*>(out_dev) + (size_t)i * outStride, splitSizes[i]};
    off += splitSizes[i];
  }
  return encodeBatch(kKindBytes, temp, tempBytes, pb, useChecksum != 0, n, v, histogram_dev,
                     outSize_dev, (cudaStream_t)stream);
}

int dgb_float_compress_pointer(void* temp, size_t tempBytes, int ft, int pb, int useChecksum,
                               uint32_t n, const void* const* in, const uint32_t* inSize,
                               void* const* out, uint32_t* outSize_dev, void* stream) {
  if (!validFloatType(ft)) return DGB_ERR_INVALID_ARG;
  HostMember* v = nullptr;
  int rc = buildPointer(n, in, inSize, out, &v);
  if (rc) return rc;
  return encodeBatch(ft, temp, tempBytes, pb, useChecksum != 0, n, v, nullptr, outSize_dev,
                     (cudaStream_t)stream);
}

int dgb_float_compress_to(void* temp, size_t tempBytes, int inFt, int ft, int pb, int useChecksum, uint32_t n,
                          const void* const* in, const uint32_t* inSize, void* const* out, uint32_t* outSize_dev,
                          void* stream) {
  int kind;
  if (inFt == ft && (ft == DGB_FLOAT16 || ft == DGB_BFLOAT16 || ft == DGB_FLOAT32))
    kind = ft;  // dgb_float_compress_pointer
  else if (inFt == DGB_FLOAT32 && ft == DGB_FLOAT16)
    kind = kKindF32toF16;
  else if (inFt == DGB_FLOAT32 && ft == DGB_BFLOAT16)
    kind = kKindF32toBF16;
  else
    return DGB_ERR_INVALID_ARG;
  HostMember* v = nullptr;
  int rc = buildPointer(n, in, inSize, out, &v);
  if (rc) return rc;
  return encodeBatch(kind, temp, tempBytes, pb, useChecksum != 0, n, v, nullptr, outSize_dev, (cudaStream_t)stream);
}

int dgb_float_compress_to_ef(void* temp, size_t tempBytes, int inFt, int ft, int pb, int useChecksum, uint32_t n,
                             const void* const* in, const uint32_t* inSize, float* const* err, void* const* out,
                             uint32_t* outSize_dev, void* stream) {
  int kind;
  if (inFt == DGB_FLOAT32 && ft == DGB_FLOAT16)
    kind = kKindF32toF16EF;
  else if (inFt == DGB_FLOAT32 && ft == DGB_BFLOAT16)
    kind = kKindF32toBF16EF;
  else
    return DGB_ERR_INVALID_ARG;
  if (!err) return DGB_ERR_INVALID_ARG;
  HostMember* v = nullptr;
  int rc = buildPointer(n, in, inSize, out, &v);
  if (rc) return rc;
  for (uint32_t i = 0; i < n; ++i) {
    if (v[i].size == 0) continue;  // an empty member reads no residual (nor input)
    if (!err[i] || ((reinterpret_cast<uintptr_t>(err[i]) ^ reinterpret_cast<uintptr_t>(v[i].in)) & 15u))
      return DGB_ERR_INVALID_ARG;
  }
  return encodeBatch(kind, temp, tempBytes, pb, useChecksum != 0, n, v, nullptr, outSize_dev, (cudaStream_t)stream, err);
}

int dgb_float_cast_fp8(int inFt, int fp8Ft, uint32_t n, const void* const* in, const uint32_t* inSize,
                       const float* scale_dev, void* const* out, uint32_t* histogram_dev, void* stream) {
  if ((inFt != DGB_FLOAT32 && inFt != DGB_BFLOAT16) || !isFp8Kind(fp8Ft)) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(scale_dev) & 3u) return DGB_ERR_INVALID_ARG;
  return castFp8(inFt, fp8Ft, n, in, inSize, scale_dev, out, histogram_dev, (cudaStream_t)stream);
}

int dgb_float_compress_split_size(void* temp, size_t tempBytes, int ft, int pb, int useChecksum,
                                  uint32_t n, const void* in_dev, const uint32_t* splitSizes,
                                  void* out_dev, uint32_t outStride, uint32_t* outSize_dev,
                                  void* stream) {
  if (!validFloatType(ft)) return DGB_ERR_INVALID_ARG;
  if (n && (!splitSizes || !out_dev)) return DGB_ERR_INVALID_ARG;
  HostMember* v = stageMembers(n);
  size_t off = 0;
  for (uint32_t i = 0; i < n; ++i) {
    v[i] = HostMember{static_cast<const uint8_t*>(in_dev) + off * wordBytes(ft),
                      static_cast<uint8_t*>(out_dev) + (size_t)i * outStride, splitSizes[i]};
    off += splitSizes[i];
  }
  return encodeBatch(ft, temp, tempBytes, pb, useChecksum != 0, n, v, nullptr, outSize_dev,
                     (cudaStream_t)stream);
}

// ---- decode ----------------------------------------------------------------

static int decodePointerCommon(int kind, void* temp, size_t tempBytes, int pb, int useChecksum,
                               uint32_t n, const void* const* in, void* const* out,
                               const uint32_t* cap, uint8_t* outSuccess_dev, uint32_t* outSize_dev,
                               uint8_t* mismatchHost, void* stream) {
  HostMember* v = nullptr;
  int rc = buildPointer(n, in, cap, out, &v);
  if (rc) return rc;
  return decodeBatch(kind, temp, tempBytes, pb, useChecksum != 0, n, v, outSuccess_dev,
                     outSize_dev, mismatchHost, (cudaStream_t)stream);
}

static int decodeSplitCommon(int kind, void* temp, size_t tempBytes, int pb, int useChecksum,
                             uint32_t n, const void* const* in, void* out_dev,
                             const uint32_t* splitSizes, uint8_t* outSuccess_dev,
                             uint32_t* outSize_dev, uint8_t* mismatchHost, void* stream) {
  if (n && (!in || !splitSizes)) return DGB_ERR_INVALID_ARG;
  HostMember* v = stageMembers(n);
  size_t off = 0;
  for (uint32_t i = 0; i < n; ++i) {
    v[i] = HostMember{in[i], static_cast<uint8_t*>(out_dev) + off * wordBytes(kind), splitSizes[i]};
    off += splitSizes[i];
  }
  return decodeBatch(kind, temp, tempBytes, pb, useChecksum != 0, n, v, outSuccess_dev,
                     outSize_dev, mismatchHost, (cudaStream_t)stream);
}

int dgb_ans_decode_pointer(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                           const void* const* in, void* const* out, const uint32_t* cap,
                           uint8_t* outSuccess_dev, uint32_t* outSize_dev, uint8_t* mismatchHost,
                           void* stream) {
  return decodePointerCommon(kKindBytes, temp, tempBytes, pb, useChecksum, n, in, out, cap,
                             outSuccess_dev, outSize_dev, mismatchHost, stream);
}

int dgb_ans_decode_stride(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                          const void* in_dev, uint32_t inStride, void* out_dev, uint32_t outStride,
                          uint32_t outCapacity, uint8_t* outSuccess_dev, uint32_t* outSize_dev,
                          uint8_t* mismatchHost, void* stream) {
  if (n && !in_dev) return DGB_ERR_INVALID_ARG;
  HostMember* v = stageMembers(n);
  for (uint32_t i = 0; i < n; ++i)
    v[i] = HostMember{static_cast<const uint8_t*>(in_dev) + (size_t)i * inStride,
                      static_cast<uint8_t*>(out_dev) + (size_t)i * outStride, outCapacity};
  return decodeBatch(kKindBytes, temp, tempBytes, pb, useChecksum != 0, n, v, outSuccess_dev,
                     outSize_dev, mismatchHost, (cudaStream_t)stream);
}

int dgb_ans_decode_split_size(void* temp, size_t tempBytes, int pb, int useChecksum, uint32_t n,
                              const void* const* in, void* out_dev, const uint32_t* splitSizes,
                              uint8_t* outSuccess_dev, uint32_t* outSize_dev, uint8_t* mismatchHost,
                              void* stream) {
  return decodeSplitCommon(kKindBytes, temp, tempBytes, pb, useChecksum, n, in, out_dev, splitSizes,
                           outSuccess_dev, outSize_dev, mismatchHost, stream);
}

int dgb_float_decompress_pointer(void* temp, size_t tempBytes, int ft, int pb, int useChecksum,
                                 uint32_t n, const void* const* in, void* const* out,
                                 const uint32_t* cap, uint8_t* outSuccess_dev,
                                 uint32_t* outSize_dev, uint8_t* mismatchHost, void* stream) {
  if (!validFloatType(ft)) return DGB_ERR_INVALID_ARG;
  return decodePointerCommon(ft, temp, tempBytes, pb, useChecksum, n, in, out, cap, outSuccess_dev,
                             outSize_dev, mismatchHost, stream);
}

int dgb_float_decompress_split_size(void* temp, size_t tempBytes, int ft, int pb, int useChecksum,
                                    uint32_t n, const void* const* in, void* out_dev,
                                    const uint32_t* splitSizes, uint8_t* outSuccess_dev,
                                    uint32_t* outSize_dev, uint8_t* mismatchHost, void* stream) {
  if (!validFloatType(ft)) return DGB_ERR_INVALID_ARG;
  return decodeSplitCommon(ft, temp, tempBytes, pb, useChecksum, n, in, out_dev, splitSizes,
                           outSuccess_dev, outSize_dev, mismatchHost, stream);
}

int dgb_float_decompress_reduce(void* temp, size_t tempBytes, int ft, int pb, uint32_t numGroups,
                                uint32_t archivesPerGroup, const void* const* in, void* const* out,
                                const uint32_t* outSize, int accumulate, uint8_t* outSuccess_dev, void* stream) {
  return decodeReduce(ft, ft, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, false, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int dgb_float_decompress_reduce_to(void* temp, size_t tempBytes, int ft, int outFt, int pb, uint32_t numGroups,
                                   uint32_t archivesPerGroup, const void* const* in, void* const* out,
                                   const uint32_t* outSize, int accumulate, uint8_t* outSuccess_dev, void* stream) {
  return decodeReduce(ft, outFt, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, false, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int dgb_float_decompress_reduce_sparse(void* temp, size_t tempBytes, int ft, int outFt, int pb, uint32_t numGroups,
                                       uint32_t archivesPerGroup, const void* const* in, void* const* out,
                                       const uint32_t* outSize, int accumulate, uint8_t* outSuccess_dev, void* stream) {
  return decodeReduce(ft, outFt, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, true, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int dgb_float_decompress_reduce_scaled(void* temp, size_t tempBytes, int ft, int outFt, int pb, uint32_t numGroups,
                                       uint32_t archivesPerGroup, const void* const* in, void* const* out,
                                       const uint32_t* outSize, int accumulate, float scale, uint8_t* outSuccess_dev,
                                       void* stream) {
  // the dense pairs of dgb_float_decompress_reduce_to and the sparse pairs of dgb_float_decompress_reduce_sparse
  return decodeReduce(ft, outFt, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, isSparseKind(ft), &scale, nullptr, nullptr, (cudaStream_t)stream);
}

int dgb_float_decompress_reduce_scaled_dev(void* temp, size_t tempBytes, int ft, int outFt, int pb,
                                           uint32_t numGroups, uint32_t archivesPerGroup, const void* const* in,
                                           void* const* out, const uint32_t* outSize, int accumulate,
                                           const float* scale_dev, float* foundInf_dev, uint8_t* outSuccess_dev,
                                           void* stream) {
  // the pairs of dgb_float_decompress_reduce_scaled; the scale is read by the kernels, never on the host
  if (!scale_dev || (reinterpret_cast<uintptr_t>(scale_dev) & 3u)) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(foundInf_dev) & 3u) return DGB_ERR_INVALID_ARG;
  return decodeReduce(ft, outFt, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, isSparseKind(ft), nullptr, scale_dev, foundInf_dev, (cudaStream_t)stream);
}

int dgb_float_decompress_reduce_narrow(void* temp, size_t tempBytes, int ft, int pb, uint32_t numGroups,
                                       uint32_t archivesPerGroup, const void* const* in, float* const* acc,
                                       void* const* out, const uint32_t* outSize, int accumulate, const float* scale,
                                       const float* scale_dev, float* foundInf_dev, uint8_t* outSuccess_dev,
                                       void* stream) {
  // fp16 / bf16 archives, dense or sparse, summed in fp32 from the fp32 accumulators acc[g] into outputs of the
  // archives' 16-bit type; unscaled, host-scaled (scale) or device-scale (scale_dev, with the optional flag)
  if (ft != kKindF16 && ft != kKindBF16 && ft != kKindF16S && ft != kKindBF16S) return DGB_ERR_INVALID_ARG;
  if (scale && scale_dev) return DGB_ERR_INVALID_ARG;
  if (foundInf_dev && !scale_dev) return DGB_ERR_INVALID_ARG;
  if (scale_dev && (reinterpret_cast<uintptr_t>(scale_dev) & 3u)) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(foundInf_dev) & 3u) return DGB_ERR_INVALID_ARG;
  if (numGroups && !out) return DGB_ERR_INVALID_ARG;
  return decodeReduce(ft, kKindF32, temp, tempBytes, pb, numGroups, archivesPerGroup, in,
                      reinterpret_cast<void* const*>(acc), outSize, accumulate != 0, outSuccess_dev, isSparseKind(ft),
                      scale, scale_dev, foundInf_dev, (cudaStream_t)stream, out);
}

int dgb_float_decompress_reduce_scaled_dev_norm(void* temp, size_t tempBytes, int ft, int outFt, int pb,
                                                uint32_t numGroups, uint32_t archivesPerGroup, const void* const* in,
                                                void* const* out, const uint32_t* outSize, int accumulate,
                                                const float* scale_dev, float* foundInf_dev, double* sqNorm_dev,
                                                uint8_t* outSuccess_dev, void* stream) {
  // dgb_float_decompress_reduce_scaled_dev, and the squared norm of each group's stored words into sqNorm_dev[g]
  if (!scale_dev || (reinterpret_cast<uintptr_t>(scale_dev) & 3u)) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(foundInf_dev) & 3u) return DGB_ERR_INVALID_ARG;
  if (!sqNorm_dev || (reinterpret_cast<uintptr_t>(sqNorm_dev) & 7u)) return DGB_ERR_INVALID_ARG;
  return decodeReduce(ft, outFt, temp, tempBytes, pb, numGroups, archivesPerGroup, in, out, outSize, accumulate != 0,
                      outSuccess_dev, isSparseKind(ft), nullptr, scale_dev, foundInf_dev, (cudaStream_t)stream,
                      nullptr, sqNorm_dev);
}

int dgb_float_decompress_reduce_narrow_norm(void* temp, size_t tempBytes, int ft, int pb, uint32_t numGroups,
                                            uint32_t archivesPerGroup, const void* const* in, float* const* acc,
                                            void* const* out, const uint32_t* outSize, int accumulate,
                                            const float* scale_dev, float* foundInf_dev, double* sqNorm_dev,
                                            uint8_t* outSuccess_dev, void* stream) {
  // dgb_float_decompress_reduce_narrow with the device scale, and the squared norm of each group's 16-bit results
  if (ft != kKindF16 && ft != kKindBF16 && ft != kKindF16S && ft != kKindBF16S) return DGB_ERR_INVALID_ARG;
  if (!scale_dev || (reinterpret_cast<uintptr_t>(scale_dev) & 3u)) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(foundInf_dev) & 3u) return DGB_ERR_INVALID_ARG;
  if (!sqNorm_dev || (reinterpret_cast<uintptr_t>(sqNorm_dev) & 7u)) return DGB_ERR_INVALID_ARG;
  if (numGroups && !out) return DGB_ERR_INVALID_ARG;
  return decodeReduce(ft, kKindF32, temp, tempBytes, pb, numGroups, archivesPerGroup, in,
                      reinterpret_cast<void* const*>(acc), outSize, accumulate != 0, outSuccess_dev, isSparseKind(ft),
                      nullptr, scale_dev, foundInf_dev, (cudaStream_t)stream, out, sqNorm_dev);
}

size_t dgb_float_decompress_reduce_norm_temp_bytes(int ft, uint32_t numGroups, uint32_t archivesPerGroup,
                                                   const uint32_t* outSize) {
  const uint64_t n = (uint64_t)numGroups * archivesPerGroup;
  if (!(validFloatType(ft) || isFp8Kind(ft)) || n > 0xffffffffull || (numGroups && !outSize)) return 0;
  return decodeTempBytes(ft, (uint32_t)n) + sqNormScratchBytes(numGroups, sqNormBlocks(numGroups, outSize));
}

size_t dgb_float_sq_norm_temp_bytes(uint32_t numGroups, const uint32_t* size) {
  if (numGroups && !size) return 0;
  return floatSqNormTempBytes(numGroups, size);
}

int dgb_float_sq_norm(void* temp, size_t tempBytes, int ft, uint32_t numGroups, const void* const* in,
                      const uint32_t* size, double* sqNorm_dev, void* stream) {
  if (ft != kKindF16 && ft != kKindBF16 && ft != kKindF32) return DGB_ERR_INVALID_ARG;
  if (!sqNorm_dev || (reinterpret_cast<uintptr_t>(sqNorm_dev) & 7u)) return DGB_ERR_INVALID_ARG;
  return floatSqNorm(ft, temp, tempBytes, numGroups, in, size, sqNorm_dev, (cudaStream_t)stream);
}

// ---- info ------------------------------------------------------------------

int dgb_ans_get_compressed_info(void* temp, size_t tempBytes, const void* const* in,
                                int inIsDevice, uint32_t n, uint32_t* outSizes_dev,
                                uint32_t* outChecksum_dev, void* stream) {
  return getInfo(kKindBytes, temp, tempBytes, in, inIsDevice != 0, n, outSizes_dev, nullptr,
                 outChecksum_dev, (cudaStream_t)stream);
}

int dgb_float_get_compressed_info(void* temp, size_t tempBytes, const void* const* in,
                                  int inIsDevice, uint32_t n, uint32_t* outSizes_dev,
                                  uint32_t* outTypes_dev, uint32_t* outChecksum_dev, void* stream) {
  return getInfo(kKindF16, temp, tempBytes, in, inIsDevice != 0, n, outSizes_dev, outTypes_dev,
                 outChecksum_dev, (cudaStream_t)stream);
}

// ---- host front end helpers ---------------------------------------------------
int dgb_copy_async(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes == 0) return DGB_OK;
  if (!dst || !src) return DGB_ERR_INVALID_ARG;
  DGB_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
  return DGB_OK;
}

int dgb_copy_rows_async(void* dst, size_t dst_pitch, const void* src, size_t src_pitch,
                        size_t width_bytes, size_t rows, void* stream) {
  if (width_bytes == 0 || rows == 0) return DGB_OK;
  if (!dst || !src || width_bytes > dst_pitch || width_bytes > src_pitch) return DGB_ERR_INVALID_ARG;
  DGB_CUDA_TRY(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width_bytes, rows, cudaMemcpyDefault,
                                 (cudaStream_t)stream));
  return DGB_OK;
}

int dgb_archives_pull(int float_type, uint32_t num_in_batch, const void* const* src, void* const* dst,
                      const uint32_t* dst_capacity, uint32_t* out_bytes_dev, void* stream) {
  if (float_type != 0 && !validFloatType(float_type)) return DGB_ERR_INVALID_ARG;
  return dgb::pullArchives(float_type, num_in_batch, src, dst, dst_capacity, out_bytes_dev, (cudaStream_t)stream);
}

// ---- options ---------------------------------------------------------------

static int* optionSlot(Options& o, const char* name) {
  if (!name) return nullptr;
  if (!std::strcmp(name, "decode_fused")) return &o.decode_fused;
  if (!std::strcmp(name, "decode_warps")) return &o.decode_warps;
  if (!std::strcmp(name, "decode_slot_words")) return &o.decode_slot_words;
  if (!std::strcmp(name, "encode_warps")) return &o.encode_warps;
  if (!std::strcmp(name, "encode_canonical")) return &o.encode_canonical;
  if (!std::strcmp(name, "encode_fused")) return &o.encode_fused;
  if (!std::strcmp(name, "fused_stats_every")) return &o.fused_stats_every;
  if (!std::strcmp(name, "fused_stage")) return &o.fused_stage;
  if (!std::strcmp(name, "fused_chunk_blocks")) return &o.fused_chunk_blocks;
  if (!std::strcmp(name, "encode_wide_table")) return &o.encode_wide_table;
  if (!std::strcmp(name, "encode_slot_words")) return &o.encode_slot_words;
  if (!std::strcmp(name, "stats_stage")) return &o.stats_stage;
  if (!std::strcmp(name, "stats_stage_kb")) return &o.stats_stage_kb;
  if (!std::strcmp(name, "encode_k2_ctas")) return &o.encode_k2_ctas;
  if (!std::strcmp(name, "hist_slab_kb")) return &o.hist_slab_kb;
  if (!std::strcmp(name, "hist_ctas_per_sm")) return &o.hist_ctas_per_sm;
  if (!std::strcmp(name, "inline_members")) return &o.inline_members;
  if (!std::strcmp(name, "pull_ctas")) return &o.pull_ctas;
  if (!std::strcmp(name, "first_part_pct")) return &o.first_part_pct;
  if (!std::strcmp(name, "last_part_pct")) return &o.last_part_pct;
  if (!std::strcmp(name, "timing")) return &o.timing;
  if (!std::strcmp(name, "parts")) return &o.parts;
  return nullptr;
}

int dgb_set_option(const char* name, int value) {
  int* s = optionSlot(dgb::gOptions, name);
  if (!s) return DGB_ERR_INVALID_ARG;
  *s = value;
  return DGB_OK;
}

int dgb_set_thread_option(const char* name, int value) {
  dgb::Options probe;
  if (!optionSlot(probe, name)) return DGB_ERR_INVALID_ARG;
  if (!dgb::tlsHasOptions) {
    dgb::tlsOptions = dgb::gOptions;
    dgb::tlsHasOptions = true;
  }
  *optionSlot(dgb::tlsOptions, name) = value;
  return DGB_OK;
}

int dgb_clear_thread_options(void) {
  dgb::tlsHasOptions = false;
  return DGB_OK;
}

// Sum of the event-timed durations (ms) and launch counts per kernel slot since the last
// call; synchronises the device.  Slots: 0 stats(K1) 1 encode(K2) 2 plan 3 decode 4 checksum.
int dgb_kernel_times(float* ms, int* counts, int nslots) {
  if (cudaDeviceSynchronize() != cudaSuccess) return DGB_ERR_CUDA;
  std::lock_guard<std::mutex> lock(timerMutex());
  for (int i = 0; i < nslots; ++i) { if (ms) ms[i] = 0.f; if (counts) counts[i] = 0; }
  for (auto& t : timedLaunches()) {
    float e = 0.f;
    cudaEventElapsedTime(&e, t.a, t.b);
    if (t.slot < nslots) { if (ms) ms[t.slot] += e; if (counts) counts[t.slot] += 1; }
    eventPool().push_back(t.a);
    eventPool().push_back(t.b);
  }
  timedLaunches().clear();
  return DGB_OK;
}

int dgb_get_option(const char* name, int* value) {
  // read-only counter: hot-path kernels launched so far (stats, encode, plan, decode)
  if (name && value && !std::strcmp(name, "launches")) {
    *value = dgb::gLaunches.load(std::memory_order_relaxed);
    return DGB_OK;
  }
  int* s = optionSlot(dgb::options(), name);
  if (!s || !value) return DGB_ERR_INVALID_ARG;
  *value = *s;
  return DGB_OK;
}

}  // extern "C"
