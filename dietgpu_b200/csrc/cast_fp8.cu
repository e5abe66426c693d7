// cast_fp8.cu -- dgb_float_cast_fp8: the scaled fp8 cast of fp32 / bf16 words, q = cvt.rn.satfinite.fp8(fp32(x) * s),
// with the byte histogram of q taken in the same pass, so that the byte encoder given that histogram
// (dgb_ans_encode_pointer(histogram_dev=)) skips its statistics pass and an fp8 compress reads its input once.
// The histogram is the byte statistics pass's scheme (encode.cu statsBytesItem): one 256-bin shared-memory histogram
// per warp counted with shared atomics, summed over the warps and added to the member's global bins once per CTA.
#include <algorithm>

#include "common.cuh"

namespace dgb {

namespace {

constexpr int kCastThreads = 256;
constexpr int kCastWarps = kCastThreads / 32;
constexpr int kCastUnroll = 4;               // 16 B loads in flight per thread
constexpr uint32_t kCastSlabVecs = 4096;     // 16 B input vectors per CTA iteration (64 KiB)
constexpr uint32_t kCastBatch = 64;          // members per launch (their table travels in the kernel parameters)
constexpr uint32_t kCastMaxSlabCtas = 1024;  // CTAs per member and launch; more slabs are walked by grid stride

struct CastMembers {
  const void* in[kCastBatch];
  uint8_t* out[kCastBatch];
  uint32_t size[kCastBatch];
};

// two products to two fp8 bytes, lo in bits 0..7 and hi in bits 8..15: cvt.rn.satfinite (round to nearest even,
// out-of-range and infinite values to +-max), the one fp8 conversion sm_90 has (ptxas refuses it without .satfinite)
template <int FP8>
__device__ __forceinline__ uint32_t fp8Pair(float lo, float hi) {
  unsigned short r;
  if constexpr (FP8 == kKindE4M3)
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// the fp32 value of an input word (bf16: the high half of the fp32 word, exact)
template <int IN>
__device__ __forceinline__ float inValue(uint32_t w) {
  return __uint_as_float(IN == kKindF32 ? w : w << 16);
}

template <bool HIST>
__device__ __forceinline__ void count(uint32_t* wh, uint32_t q) {
  if constexpr (HIST) atomicAdd(&wh[q], 1u);
}

// Member blockIdx.y of the launch, slabs blockIdx.x, blockIdx.x + gridDim.x, ... of its 16 B input vectors; CTA 0
// also takes the head (the words before the first 16 B boundary) and the tail.  Every product is one __fmul_rn, which
// nvcc never contracts.  hist: the launch's first member's 256 bins (zeroed by the host), or unused.
template <int IN, int FP8, bool HIST>
__global__ void __launch_bounds__(kCastThreads)
castFp8Kernel(const __grid_constant__ CastMembers cm, const float* __restrict__ scaleDev, uint32_t* __restrict__ hist) {
  __shared__ uint32_t sHist[kCastWarps][kNumSymbols];
  constexpr uint32_t WB = IN == kKindF32 ? 4u : 2u, E = 16u / WB;  // word bytes, words per vector
  const uint32_t m = blockIdx.y, t = threadIdx.x;
  // shuffle => the histogram base is provably warp-uniform
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  const uint32_t size = cm.size[m];
  const uint8_t* in = static_cast<const uint8_t*>(cm.in[m]);
  uint8_t* out = cm.out[m];
  const uint32_t head = min(size, ((16u - (uint32_t)(reinterpret_cast<uintptr_t>(in) & 15u)) & 15u) / WB);
  const uint32_t nVec = (size - head) / E;
  const uint32_t tail = size - head - nVec * E;
  const uint32_t nSlabs = max(1u, divUp(nVec, kCastSlabVecs));
  if (size == 0 || blockIdx.x >= nSlabs) return;  // the whole CTA, before any barrier
  const float s = scaleDev ? __ldg(scaleDev) : 1.0f;
  uint32_t* wh = sHist[warp];
  if constexpr (HIST) {
#pragma unroll
    for (int w = 0; w < kCastWarps; ++w) sHist[w][t] = 0;
    __syncthreads();
  }
  if (blockIdx.x == 0) {
    const uint32_t i = t < head ? t : head + nVec * E + (t - head);
    if (t < head + tail) {  // head < E and tail < E words
      const uint32_t w = IN == kKindF32 ? reinterpret_cast<const uint32_t*>(in)[i] : reinterpret_cast<const uint16_t*>(in)[i];
      const uint32_t q = fp8Pair<FP8>(__fmul_rn(inValue<IN>(w), s), 0.0f) & 0xffu;
      out[i] = (uint8_t)q;
      count<HIST>(wh, q);
    }
  }
  const uint4* vec = reinterpret_cast<const uint4*>(in + head * WB);
  uint8_t* ov = out + head;
  const bool aligned = (reinterpret_cast<uintptr_t>(ov) & (E - 1u)) == 0;  // one E-byte store per vector
  for (uint32_t slab = blockIdx.x; slab < nSlabs; slab += gridDim.x) {
    const uint32_t v0 = slab * kCastSlabVecs, v1 = min(nVec, v0 + kCastSlabVecs);
    for (uint32_t i0 = v0 + t; i0 < v1; i0 += kCastUnroll * kCastThreads) {
      uint4 vv[kCastUnroll];
#pragma unroll
      for (int k = 0; k < kCastUnroll; ++k) {
        const uint32_t i = i0 + k * kCastThreads;
        vv[k] = i < v1 ? __ldcs(vec + i) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int k = 0; k < kCastUnroll; ++k) {
        const uint32_t i = i0 + k * kCastThreads;
        if (i >= v1) break;
        const uint32_t w4[4] = {vv[k].x, vv[k].y, vv[k].z, vv[k].w};
        uint32_t q[2] = {0u, 0u};  // the vector's E bytes, little-endian
        if constexpr (IN == kKindF32) {
          q[0] = fp8Pair<FP8>(__fmul_rn(inValue<IN>(w4[0]), s), __fmul_rn(inValue<IN>(w4[1]), s)) |
                 fp8Pair<FP8>(__fmul_rn(inValue<IN>(w4[2]), s), __fmul_rn(inValue<IN>(w4[3]), s)) << 16;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t p = fp8Pair<FP8>(__fmul_rn(__uint_as_float(w4[j] << 16), s),
                                             __fmul_rn(__uint_as_float(w4[j] & 0xffff0000u), s));
            q[j >> 1] |= p << (16 * (j & 1));
          }
        }
        uint8_t* o = ov + (size_t)i * E;
        if (aligned) {
          if constexpr (E == 4) *reinterpret_cast<uint32_t*>(o) = q[0];
          else *reinterpret_cast<uint2*>(o) = make_uint2(q[0], q[1]);
        } else {
#pragma unroll
          for (uint32_t b = 0; b < E; ++b) o[b] = (uint8_t)(q[b >> 2] >> (8 * (b & 3)));
        }
#pragma unroll
        for (uint32_t b = 0; b < E; ++b) count<HIST>(wh, (q[b >> 2] >> (8 * (b & 3))) & 0xffu);
      }
    }
  }
  if constexpr (HIST) {
    __syncthreads();
    uint32_t c = 0;
#pragma unroll
    for (int w = 0; w < kCastWarps; ++w) c += sHist[w][t];
    if (c) atomicAdd(hist + (size_t)m * kNumSymbols + t, c);
  }
}

}  // namespace

int castFp8(int inKind, int fp8Kind, uint32_t n, const void* const* in, const uint32_t* size, const float* scaleDev,
            void* const* out, uint32_t* histogram, cudaStream_t stream) {
  if (n == 0) return DGB_OK;
  if (!in || !size || !out) return DGB_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(histogram) & 3u) return DGB_ERR_INVALID_ARG;
  const uint32_t wb = wordBytes(inKind);
  for (uint32_t i = 0; i < n; ++i)
    if (size[i] && (!in[i] || !out[i] || (reinterpret_cast<uintptr_t>(in[i]) & (wb - 1u)))) return DGB_ERR_INVALID_ARG;
  if (histogram) DGB_CUDA_TRY(cudaMemsetAsync(histogram, 0, 4 * (size_t)kNumSymbols * n, stream));
  const uint32_t e = 16u / wb;
  for (uint32_t m0 = 0; m0 < n; m0 += kCastBatch) {
    const uint32_t k = std::min(kCastBatch, n - m0);
    CastMembers cm{};
    uint32_t slabs = 1;
    for (uint32_t j = 0; j < k; ++j) {
      cm.in[j] = in[m0 + j];
      cm.out[j] = static_cast<uint8_t*>(out[m0 + j]);
      cm.size[j] = size[m0 + j];
      slabs = std::max(slabs, divUp(size[m0 + j] / e, kCastSlabVecs));
    }
    const dim3 grid(std::min(slabs, kCastMaxSlabCtas), k);
    uint32_t* h = histogram ? histogram + (size_t)m0 * kNumSymbols : nullptr;
    auto launch = [&](auto IN, auto FP8) {
      constexpr int I = decltype(IN)::value, F = decltype(FP8)::value;
      if (h) castFp8Kernel<I, F, true><<<grid, kCastThreads, 0, stream>>>(cm, scaleDev, h);
      else castFp8Kernel<I, F, false><<<grid, kCastThreads, 0, stream>>>(cm, scaleDev, h);
    };
    if (inKind == kKindF32) {
      if (fp8Kind == kKindE4M3) launch(IntC<kKindF32>(), IntC<kKindE4M3>());
      else launch(IntC<kKindF32>(), IntC<kKindE5M2>());
    } else {
      if (fp8Kind == kKindE4M3) launch(IntC<kKindBF16>(), IntC<kKindE4M3>());
      else launch(IntC<kKindBF16>(), IntC<kKindE5M2>());
    }
    DGB_CUDA_TRY(cudaGetLastError());
  }
  return DGB_OK;
}

}  // namespace dgb
