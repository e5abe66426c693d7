// decode_norm.cu -- the squared-norm kernels and their launchers, in a module of their own: the device-scale
// decode-and-sum kernels | kSqNorm (decode.cu, compiled once more with DGB_DECODE_NORM_TU), the squared norm of dense
// fp16 / bf16 / fp32 words (floatSqNormKernel) and the fold of the block partials into one fp64 value per group
// (sqNormFoldKernel).  Apart from decode.o and decode_narrow.o, so that the kernels there keep their code.
#define DGB_DECODE_NORM_TU
#include "decode.cu"

namespace dgb {

namespace {

constexpr int kFoldThreads = 256;
constexpr int kNormWarps = 8;

// Step 3 of the definition (include/dietgpu_b200.h): thread t of group g's CTA sums q[t], q[t + 256], ... from +0 in
// increasing block order, each warp folds its 32 sums with the xor butterfly, and thread 0 adds the 8 warp sums in
// warp order.  groupOk (the decode-and-sum's verdicts; null: every group is valid): a group marked 0 is not written.
__global__ void __launch_bounds__(kFoldThreads)
sqNormFoldKernel(const double* __restrict__ part, const uint32_t* __restrict__ off,
                 const uint32_t* __restrict__ groupOk, double* __restrict__ sqNorm) {
  __shared__ double sWarp[kFoldThreads / 32];
  const uint32_t g = blockIdx.x, t = threadIdx.x;
  if (groupOk && groupOk[g] == 0u) return;
  const uint32_t b0 = off[g], nb = off[g + 1] - b0;
  double s = 0.0;
  for (uint32_t k = t; k < nb; k += kFoldThreads) s += part[b0 + k];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((t & 31u) == 0) sWarp[t >> 5] = s;
  __syncthreads();
  if (t == 0) {
    double r = sWarp[0];
    for (int w = 1; w < kFoldThreads / 32; ++w) r += sWarp[w];
    sqNorm[g] = r;
  }
}

// Steps 1 and 2 over words already in memory: one warp per 4096-word block of the flat block space [0, off[G]).  Lane
// l adds the squares of its words of the block's partial row first, then of its full rows from the top down (the
// decoder's order), and the butterfly of decodeReduceBlock gives the block's partial.  Rows are loaded 16 at a time
// ahead of their adds, so each lane has 16 loads in flight.
template <int KIND>
__global__ void __launch_bounds__(kNormWarps * 32)
floatSqNormKernel(const void* const* __restrict__ in, const uint32_t* __restrict__ off,
                  const uint32_t* __restrict__ size, uint32_t groups, double* __restrict__ part) {
  typedef typename std::conditional<KIND == kKindF32, uint32_t, uint16_t>::type T;
  constexpr int U = 16;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t total = off[groups];
  for (uint32_t b = blockIdx.x * kNormWarps + (threadIdx.x >> 5); b < total; b += gridDim.x * kNormWarps) {
    // the group of block b: off[lo] <= b < off[lo + 1] (an empty group shares its offset with the next one)
    uint32_t lo = 0, hi = groups;
    while (hi - lo > 1u) {
      const uint32_t mid = (lo + hi) >> 1;
      if (off[mid] <= b) lo = mid;
      else hi = mid;
    }
    const uint32_t k = b - off[lo];
    const uint32_t n = min((uint32_t)kBlockBytes, size[lo] - k * kBlockBytes);
    const T* p = static_cast<const T*>(in[lo]) + (size_t)k * kBlockBytes + lane;
    uint32_t row = n >> 5;
    double s = 0.0;
    if (lane < (n & 31u)) {
      const double v = wordF64<KIND>(__ldg(p + row * 32u));
      s = fma(v, v, s);
    }
    while (row >= (uint32_t)U) {
      row -= U;
      uint32_t w[U];
#pragma unroll
      for (int j = 0; j < U; ++j) w[j] = __ldg(p + (row + j) * 32u);
#pragma unroll
      for (int j = U - 1; j >= 0; --j) {
        const double v = wordF64<KIND>(w[j]);
        s = fma(v, v, s);
      }
    }
    while (row > 0) {
      --row;
      const double v = wordF64<KIND>(__ldg(p + row * 32u));
      s = fma(v, v, s);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) part[b] = s;
  }
}

int launchSqNormFold(const Options& opt, const SqNormScratch& ns, uint32_t groups, bool checked, double* sqNorm,
                     cudaStream_t stream) {
  timerBegin(opt, kSlotDecode, stream);
  sqNormFoldKernel<<<groups, kFoldThreads, 0, stream>>>(ns.part, ns.off, checked ? ns.ok : nullptr, sqNorm);
  DGB_CUDA_TRY(cudaGetLastError());
  timerEnd(opt, kSlotDecode, stream);
  return DGB_OK;
}

}  // namespace

int sqNormFoldValid(const Options& opt, const SqNormScratch& norm, uint32_t groups, double* sqNorm,
                    cudaStream_t stream) {
  return launchSqNormFold(opt, norm, groups, true, sqNorm, stream);
}

int sqNormPrepare(uint8_t* base, uint32_t groups, const uint32_t* size, SqNormScratch* out, cudaStream_t stream) {
  const uint64_t blocks = sqNormBlocks(groups, size);
  if (blocks > 0xffffffffull) return DGB_ERR_TOO_LARGE;
  // G + 1 offsets, then the G sizes, padded to whole 8 B words for the upload
  std::vector<uint32_t>& off = hostStage().sqNormOff;
  off.assign(2 * (size_t)groups + 2, 0u);
  uint32_t b = 0;
  for (uint32_t g = 0; g < groups; ++g) {
    off[g] = b;
    b += divUp(size[g], kBlockBytes);
    off[groups + 1 + g] = size[g];
  }
  off[groups] = b;
  out->off = reinterpret_cast<uint32_t*>(base);
  out->size = out->off + groups + 1;
  out->ok = reinterpret_cast<uint32_t*>(base + alignUp256(8 * (size_t)groups + 8));
  out->part = reinterpret_cast<double*>(base + alignUp256(8 * (size_t)groups + 8) + alignUp256(4 * (size_t)groups));
  return uploadTable(out->off, off.data(), 4 * off.size(), stream);
}

int launchDecodeReduceNorm(int kind, int pb, bool widen, const Options& opt, MemberDesc* members, uint32_t* next,
                           const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                           bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                           float* foundInf, void* const* narrowTable, const SqNormScratch& norm, double* sqNorm) {
  DecodeScratch sc{};
  sc.members = members;
  sc.next = next;
  sc.seen = next + (size_t)groups * width;
  const int rc = withKind(kind, [&](auto K) { return withPb(pb, [&](auto P) {
    constexpr int KIND = decltype(K)::value, PB = decltype(P)::value;
    constexpr int DK = denseKind(KIND);
    auto launch = [&](auto WK) {
      return launchDecodeReduce<decltype(WK)::value | kScaled | kDevScale | kSqNorm, PB>(
          opt, sc, im, groups, width, totalChunks, accumulate, outSuccess, stream, scaleDev, foundInf, narrowTable,
          &norm);
    };
    if constexpr (DK == kKindF16 || DK == kKindBF16) {
      if (narrowTable) return launch(IntC<KIND | kWidenF32 | kNarrowOut>());
      if (widen) return launch(IntC<KIND | kWidenF32>());
      return launch(IntC<KIND>());
    } else if constexpr (DK == kKindF32) {
      return launch(IntC<KIND>());
    } else {
      return (int)DGB_ERR_INVALID_ARG;  // not reached (decodeReduce checks the kind)
    }
  }); });
  if (rc != DGB_OK) return rc;
  return launchSqNormFold(opt, norm, groups, true, sqNorm, stream);
}

size_t floatSqNormTempBytes(uint32_t groups, const uint32_t* size) {
  return alignUp256(8 * (size_t)groups) + sqNormScratchBytes(groups, sqNormBlocks(groups, size));
}

int floatSqNorm(int kind, void* temp, size_t tempBytes, uint32_t groups, const void* const* in, const uint32_t* size,
                double* sqNorm, cudaStream_t stream) {
  // kind (fp16, bf16 or fp32) and sqNorm are checked by the entry point
  if (groups == 0) return DGB_OK;
  if (!in || !size) return DGB_ERR_INVALID_ARG;
  const uint32_t wb = wordBytes(kind);
  for (uint32_t g = 0; g < groups; ++g)
    if (size[g] && (!in[g] || (reinterpret_cast<uintptr_t>(in[g]) & (wb - 1u)))) return DGB_ERR_INVALID_ARG;
  if (!temp || tempBytes < floatSqNormTempBytes(groups, size)) return DGB_ERR_TEMP_TOO_SMALL;
  if (reinterpret_cast<uintptr_t>(temp) & 255u) return DGB_ERR_INVALID_ARG;
  const Options opt = options();
  uint8_t* base = static_cast<uint8_t*>(temp);
  SqNormScratch ns;
  int rc = sqNormPrepare(base + alignUp256(8 * (size_t)groups), groups, size, &ns, stream);
  if (rc != DGB_OK) return rc;
  rc = uploadTable(base, in, 8 * (size_t)groups, stream);
  if (rc != DGB_OK) return rc;
  const uint32_t blocks = hostStage().sqNormOff[groups];
  if (blocks) {
    const uint32_t grid = std::min<uint32_t>(divUp(blocks, (uint32_t)kNormWarps), (uint32_t)smCount() * 8u);
    timerBegin(opt, kSlotDecode, stream);
    withKind(kind, [&](auto K) {
      constexpr int KIND = decltype(K)::value;
      if constexpr (KIND == kKindF16 || KIND == kKindBF16 || KIND == kKindF32)
        floatSqNormKernel<KIND><<<grid, kNormWarps * 32, 0, stream>>>(
            static_cast<const void* const*>(temp), ns.off, ns.size, groups, ns.part);
      return (int)DGB_OK;
    });
    DGB_CUDA_TRY(cudaGetLastError());
    timerEnd(opt, kSlotDecode, stream);
  }
  return launchSqNormFold(opt, ns, groups, false, sqNorm, stream);
}

}  // namespace dgb
