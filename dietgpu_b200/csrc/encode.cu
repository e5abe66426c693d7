// encode.cu -- batched rANS encode (bytes) and float compress (fp16/bf16/fp32/fp64, sparse fp16/bf16/fp32, and
// float32 inputs narrowed to fp16/bf16 archives, with or without error feedback)
// for sm_90a (H100).  Two launches per call, whatever the batch size:
//
//   K1  stats*Kernel     a pure read of the raw input: 256-bin histogram of the coded byte, taken out of
//                        the raw bytes / float words with one shift and one mask per element (+ XOR
//                        checksum); float kinds also write the 16 B float header and zero the
//                        padding of the stored plane(s).  The LAST CTA of each member (atomic
//                        ticket) normalises the histogram, bit-identical to the reference
//                        (ans/GpuANSStatistics.cuh:178-367), writes the pdf into the archive and
//                        the encoder table to scratch.
//   K2  encodeKernelFast one resident wave of CTAs, each owning a contiguous range of 4 KiB
//                        blocks (one shared table load per member); each warp runs the
//                        32-lane interleaved rANS state machine of its block
//                        (ans/GpuANSEncode.cuh:49-211) over the member's RAW words (cp.async ring; float
//                        kinds write the stored plane(s) of the archive from the same ring slot, which
//                        replaces the reference's split pass, float/GpuFloatCompress.cuh:280-365)
//                        into a shared-memory staging slot and takes its place in the archive's data section with one 64-bit
//                        atomic, so the words go from shared memory straight to their final
//                        place (the reference's uncoalesced scratch, prefix-sum kernels and
//                        coalesce kernel -- ans/GpuANSEncode.cuh:515-672,
//                        ans/BatchPrefixSum.cuh -- do not exist here).  Streams land in
//                        completion order, which the format allows (the decoder follows
//                        blockWords[k].y).  Option encode_canonical selects encodeKernel:
//                        ordered per-warp tickets + a decoupled look-back, block order,
//                        byte-identical to the reference, slower.
//   Large batches are cut by member into sub-batches on internal streams (capi.cu autoParts).
//
// The archive produced is field-for-field the reference's (A.4 of SURVEY.md);
// bits the reference leaves undefined are zero.
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "../../include/dietgpu_b200_device.cuh"

namespace dgb {

namespace {

constexpr int kStatsThreads = 256;  // == kNumSymbols: thread <-> symbol in the epilogue
constexpr int kStatsWarps = kStatsThreads / 32;
#ifndef DGB_STATS_UNROLL
#define DGB_STATS_UNROLL 4
#endif
constexpr int kStatsUnroll = DGB_STATS_UNROLL;     // independent 16 B loads in flight per thread

__device__ __forceinline__ uint4 ldStream16(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

// TMA landing buffer of a statistics item (fused launch): the item's whole slab arrives in shared
// memory by one bulk copy (cp.async.bulk + mbarrier), so its HBM latency is covered by bytes in
// flight, not by resident warps -- the item runs at full speed next to encoder CTAs.  The two-kernel
// path (STAGED = false) keeps the register-pipelined global loads.
struct StatsStage {
  uint4* buf = nullptr;     // shared memory, 16 B aligned, >= slabVecs vectors
  uint32_t bar = 0;         // shared address of the mbarrier
  uint32_t* phase = nullptr;
};

struct EncodeScratch {
  MemberDesc* members;            // [n]
  uint32_t* hist;                 // [n][256]      (zeroed per call)
  uint32_t* histDone;             // [n]           (zeroed)
  uint32_t* checksum;             // [n]           (zeroed)
  uint32_t* ticket;               // [4]           (zeroed)
  unsigned long long* lookback;   // [totalTickets](zeroed)   canonical (ordered) layout only
  unsigned long long* allocDone;  // [n]           (zeroed)   low: words handed out, high: blocks placed
  uint8_t* spill;                 // [resident warps][maxBlockWords] u16: overflow of small staging slots
  uint4* table;                   // [n][tableSlots(kind)] slots of 16 B (packed entries use the first half)
  bool wideTable;                 // entry format: EncEntryWide (16 B) or EncEntry (8 B)
  uint32_t blockZerosOff;         // sparse kinds: see blockZeros() (in the padding after wideTable: the kernel
                                  // parameters of the other kinds keep their layout)
  // fused single-launch encoder only
  const uint2* workIdx;           // [n + 1] {first stats item, first encode chunk} of member i
  uint32_t* ready;                // [n]  (zeroed) 1 once the member's table is published
};
static_assert(sizeof(EncodeScratch) == 96, "");

// The sparse kinds never run the fused launch, so they keep their counters in its (zeroed) `ready` array:
// +0 and -0 words of member m, and the +-0 words of the 4 KiB block with ticket work0 + k.
__device__ __forceinline__ uint32_t* zeroCounts(const EncodeScratch& sc, uint32_t m) { return sc.ready + 2u * m; }
__device__ __forceinline__ uint32_t* blockZeros(const EncodeScratch& sc, uint32_t work0) {
  return sc.ready + sc.blockZerosOff + work0;
}

// ---------------------------------------------------------------------------
// Normalisation epilogue: 256 threads, thread t owns symbol t.
// Restates ans/GpuANSStatistics.cuh:178-367 (see SURVEY.md A.1); the sort is a
// rank-by-counting over the 256 unique keys (q << 16 | sym), descending.
// ---------------------------------------------------------------------------
__device__ void normalizeAndPublish(const uint32_t* __restrict__ histGlobal, uint32_t total,
                                    int pb, bool wideTable, uint4* __restrict__ tableOut,
                                    uint8_t* __restrict__ ansArchive) {
  const uint32_t t = threadIdx.x;
  const uint32_t K = 1u << pb;
  // the normalisation itself is the device-level API's routine (include/dietgpu_b200_device.cuh): one
  // implementation of the reference's quirks for the library and for user kernels
  uint32_t cdf;
  const uint32_t pdf = dietgpu_b200::device::blockNormalizedPdf(__ldcg(histGlobal + t), total, pb, &cdf);

  // Division constants.  The reference (:343-358) uses the round-up magic that needs
  // hi32(x * magic) + x; the coder state is always < 2^31 here, so the plain round-up
  // reciprocal M = ceil(2^(32+s) / pdf), s = ceil(log2 pdf) - 1, already gives the exact
  // quotient as hi32(x * M) >> s (x * (M * pdf - 2^(32+s)) < 2^31 * pdf <= 2^(32+s)), one add
  // and one register pair cheaper per symbol.  pdf == 1 has no such M below 2^32: it uses
  // M = 2^32 - 1 (quotient x - 1) and folds the missing (K - 1) into the cdf term.
  uint32_t shift = 0, magic = 0, cdfTerm = cdf;
  if (pdf > 1) {
    shift = 31u - (uint32_t)__clz((int)(pdf - 1));
    magic = (uint32_t)(((1ull << (32 + shift)) + pdf - 1) / pdf);
  } else if (pdf == 1) {
    magic = 0xffffffffu;
    cdfTerm = cdf + (K - 1u);
  }
  if (wideTable) {
    EncEntryWide e;
    e.thr = pdf << (31 - pb);
    e.magic = magic;
    e.kmp = K - pdf;
    e.cdfShift = shift | (cdfTerm << 5);
    reinterpret_cast<EncEntryWide*>(tableOut)[t] = e;
  } else {
    EncEntry e;
    e.magic = magic;
    e.pack = shift | ((K - pdf) << kEncKmpShift) | (cdfTerm << kEncCdfShift);
    reinterpret_cast<EncEntry*>(tableOut)[t] = e;
  }
  // archive: u16 pdf[256] right after the 32 B header (ans/GpuANSEncode.cuh:572-577)
  reinterpret_cast<uint16_t*>(ansArchive + kAnsHeaderBytes)[t] = (uint16_t)pdf;
}

// Header + empty pdf for a zero-sized member (ans/ANSTest.cu:243-246 ZeroSized).
__device__ void publishEmptyMember(uint8_t* ansArchive, int pb, bool useChecksum,
                                   uint32_t* outSize, uint32_t m, uint32_t extraBytes) {
  const uint32_t t = threadIdx.x;
  reinterpret_cast<uint16_t*>(ansArchive + kAnsHeaderBytes)[t] = 0;
  if (t == 0) {
    uint4* h = reinterpret_cast<uint4*>(ansArchive);
    h[0] = make_uint4(kAnsMagicVersion, 0u, 0u, 0u);
    h[1] = make_uint4((uint32_t)pb | ((useChecksum ? 1u : 0u) << 4), 0u, 0u, 0u);
    if (outSize) outSize[m] = ansOverhead(0) + extraBytes;
  }
}

// Encoder table of a member: 16 B slots in scratch, entries in shared memory.  The sparse kinds have two more
// entries: 256 for +0 and 257 for -0 words (copies of the entries of E+ and E-, or of the natural symbols when
// nothing is elided), so the coder turns a word into its table entry without any per-member escape state.
__host__ __device__ constexpr uint32_t tableSlots(int kind) { return isSparseKind(kind) ? 260u : kNumSymbols; }
__host__ __device__ constexpr uint32_t encTabVecs(bool wide, int kind) {
  return isSparseKind(kind) ? (wide ? 258u : 130u) : (wide ? kNumSymbols : kNumSymbols / 2);
}
__host__ __device__ constexpr uint32_t encTabBytes(int kind) { return isSparseKind(kind) ? 2080u : kNumSymbols * 8u; }

__device__ __forceinline__ uint32_t foldXor(uint32_t v) {
  return (v ^ (v >> 8) ^ (v >> 16) ^ (v >> 24)) & 0xffu;
}

// Adds this CTA's per-warp histograms to the global one, takes the member's
// completion ticket and tells whether this CTA is the last one.
__device__ bool flushAndTicket(uint32_t (*sHist)[kNumSymbols], uint32_t* histGlobal,
                               uint32_t* histDone, uint32_t expected, bool doHist,
                               uint32_t xorAcc, uint32_t* checksumGlobal, bool doChecksum) {
  __shared__ uint32_t sLast;
  __syncthreads();
  const uint32_t t = threadIdx.x;
  if (doHist) {
    uint32_t s = 0;
#pragma unroll
    for (int w = 0; w < kStatsWarps; ++w) s += sHist[w][t];
    if (s) atomicAdd(histGlobal + t, s);
  }
  if (doChecksum) {
    uint32_t x = foldXor(xorAcc);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, d);
    if ((t & 31) == 0 && x) atomicXor(checksumGlobal, x);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) sLast = (atomicAdd(histDone, 1u) == expected - 1u);
  __syncthreads();
  const bool last = sLast != 0;
  if (last) __threadfence();
  return last;
}

// ---------------------------------------------------------------------------
// K1 (bytes): histogram + checksum + normalisation epilogue.
// grid = (n, Y): CTA (m, y) walks slabs y, y+Y, ... of member m.
// ---------------------------------------------------------------------------
// Slab accounting shared by host (work-item counts of the fused launch) and device.
__host__ __device__ inline uint32_t bytesHeadLen(const void* in, uint32_t size) {
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(in) & 15u);
  const uint32_t head = (16u - mis) & 15u;
  return size < head ? size : head;
}
__host__ __device__ inline uint32_t bytesSlabs(const void* in, uint32_t size, uint32_t slabVecs, bool doPass) {
  if (!doPass) return 0u;
  const uint32_t nVec = (size - bytesHeadLen(in, size)) / 16u;
  const uint32_t s = divUp(nVec, slabVecs);
  return s > 0u ? s : (size > 0u ? 1u : 0u);
}

// Work of CTA y of Y on member m (Y = gridDim.y of the two-kernel path, the member's item count in
// the fused kernel).  Returns true in the CTA that finished the member (its table is published).
template <bool STAGED>
__device__ __forceinline__ bool statsBytesItem(const EncodeScratch& sc, uint32_t (*sHist)[kNumSymbols],
                                               const uint32_t* __restrict__ histogramGiven, int pb,
                                               bool useChecksum, uint32_t slabVecs, const MemberDesc& md,
                                               uint32_t m, uint32_t y,
                                               uint32_t Y, uint32_t* __restrict__ outSize,
                                               const StatsStage& stage = StatsStage()) {
  // shuffle => the histogram base is provably warp-uniform (ATOMS [R + UR], no per-symbol add)
  const uint32_t t = threadIdx.x, warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  const uint8_t* in = static_cast<const uint8_t*>(md.in);
  const uint32_t size = md.size;
  uint8_t* archive = static_cast<uint8_t*>(md.out);
  const bool doHist = histogramGiven == nullptr;
  const bool doPass = doHist || useChecksum;

  // member = [head bytes | 16 B vectors | tail bytes]
  const uint32_t head = bytesHeadLen(in, size);
  const uint32_t nVec = (size - head) / 16u;
  const uint32_t tail = size - head - nVec * 16u;
  const uint32_t nSlabs = bytesSlabs(in, size, slabVecs, doPass);
  const uint32_t participants = min(nSlabs, Y);

  if (participants == 0) {
    if (y != 0) return false;
  } else {
    if (y >= participants) return false;
    const uint4* vec = reinterpret_cast<const uint4*>(in + head);
    if (STAGED && t == 0) {
      const uint32_t v0 = y * slabVecs, v1 = min(nVec, v0 + slabVecs);
      if (v1 > v0) {
        fenceProxyAsync();  // the region was last touched through the generic proxy (coder staging)
        mbarExpectTx(stage.bar, (v1 - v0) * 16u);
        bulkLoad(smemAddr(stage.buf), vec + v0, (v1 - v0) * 16u, stage.bar);
      }
    }
#pragma unroll
    for (int w = 0; w < kStatsWarps; ++w) sHist[w][t] = 0;
    __syncthreads();
    uint32_t* wh = sHist[warp];
    uint32_t xorAcc = 0;
    if (y == 0) {
      if (t < head) { uint32_t b = in[t]; atomicAdd(&wh[b], 1u); xorAcc ^= b; }
      if (t < tail) { uint32_t b = in[head + nVec * 16u + t]; atomicAdd(&wh[b], 1u); xorAcc ^= b; }
    }
    for (uint32_t slab = y; slab < nSlabs; slab += Y) {
      const uint32_t v0 = slab * slabVecs, v1 = min(nVec, v0 + slabVecs);
      if (STAGED && v1 > v0) {  // one slab per item (Y == nSlabs): the copy was issued above
        mbarWait(stage.bar, *stage.phase);
        *stage.phase ^= 1u;
      }
      for (uint32_t i0 = v0 + t; i0 < v1; i0 += kStatsUnroll * kStatsThreads) {
        uint4 vv[kStatsUnroll];
#pragma unroll
        for (int k = 0; k < kStatsUnroll; ++k) {
          const uint32_t i = i0 + k * kStatsThreads;
          vv[k] = i < v1 ? (STAGED ? stage.buf[i - v0] : ldStream16(vec + i)) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int k = 0; k < kStatsUnroll; ++k) {
          if (i0 + k * kStatsThreads >= v1) break;
          const uint4 v = vv[k];
          xorAcc ^= v.x ^ v.y ^ v.z ^ v.w;
          if (doHist) {
            const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              atomicAdd(&wh[w4[q] & 0xffu], 1u);
              atomicAdd(&wh[(w4[q] >> 8) & 0xffu], 1u);
              atomicAdd(&wh[(w4[q] >> 16) & 0xffu], 1u);
              atomicAdd(&wh[w4[q] >> 24], 1u);
            }
          }
        }
      }
    }
    if (!flushAndTicket(sHist, sc.hist + m * kNumSymbols, sc.histDone + m, participants, doHist,
                        xorAcc, sc.checksum + m, useChecksum))
      return false;
  }

  // ---- last CTA of the member ----
  if (size == 0) {
    publishEmptyMember(archive, pb, useChecksum, outSize, m, 0);
    return true;
  }
  const uint32_t* h = doHist ? sc.hist + m * kNumSymbols : histogramGiven + m * kNumSymbols;
  normalizeAndPublish(h, size, pb, sc.wideTable, sc.table + m * kNumSymbols, archive);
  return true;
}

__global__ void __launch_bounds__(kStatsThreads)
statsBytesKernel(EncodeScratch sc, const __grid_constant__ InlineMembers im, const uint32_t* __restrict__ histogramGiven, int pb,
                 bool useChecksum, uint32_t slabVecs, uint32_t memberBase, uint32_t* __restrict__ outSize) {
  __shared__ uint32_t sHist[kStatsWarps][kNumSymbols];
  const uint32_t m = blockIdx.x + memberBase;
  statsBytesItem<false>(sc, sHist, histogramGiven, pb, useChecksum, slabVecs, memberAt(im, sc.members, m), m, blockIdx.y,
                        gridDim.y, outSize);
}

// ---------------------------------------------------------------------------
// K1 (floats): split + histogram of the comp byte + header + epilogue.
// float/GpuFloatCompress.cuh:280-365 (splitFloat), float/GpuFloatUtils.cuh:
// 100-204 (split rules), restated with packed-word bit tricks:
//   fp16 : comp = w >> 8,            non = w & 0xff
//   bf16 : w' = rotl16(w, 1); comp = w' >> 8, non = w' & 0xff
//   fp32 : w' = rotl32(w, 1); comp = w' >> 24, non = w' & 0xffffff
//          stored as a u16 plane (low 16 bits) then a u8 plane (bits 16..23)
//   fp64 : v = rotl64(w, 1); comp = v >> 56 (exponent bits 10..3), non = the low 56 bits, stored as a u32,
//          a u16 and a u8 plane; comp is fp32's coded byte taken from the word's high 32-bit half
// ---------------------------------------------------------------------------
template <int FT>
__device__ __forceinline__ uint32_t rot16x2(uint32_t w) {
  if (FT == DGB_BFLOAT16) {
    // rotate both 16-bit halves left by one: bitwise select between w << 1 and w >> 15 under one
    // mask, a single LOP3 (written as two AND/ORs, ptxas emits two LOP3s for the two constants)
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(r) : "r"(w << 1), "r"(w >> 15), "r"(0xfffefffeu));
    return r;
  }
  return w;
}

// member = [head elements up to the first 16 B boundary | 16 B vectors | tail elements]
__host__ __device__ inline uint32_t floatHeadLen(const void* in, uint32_t size, uint32_t wordBytes) {
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(in) & 15u);
  const uint32_t head = ((16u - mis) & 15u) / wordBytes;
  return size < head ? size : head;
}
__host__ __device__ inline uint32_t floatSlabs(const void* in, uint32_t size, uint32_t wordBytes, uint32_t slabVecs) {
  if (size == 0) return 0u;
  const uint32_t nVec = (size - floatHeadLen(in, size, wordBytes)) / (16u / wordBytes);
  const uint32_t s = divUp(nVec, slabVecs);
  return s > 0u ? s : 1u;
}

// Histogram index (x4, the byte offset into a 256-bin u32 histogram) of the coded byte of the
// element in bits [LO, LO + 16) of a packed 16-bit pair, or of a 32-bit word: one shift, one mask.
//   fp16 coded = w >> 8, bf16 coded = (w >> 7) & 0xff, fp32 coded = (w >> 23) & 0xff
template <int FT>
__device__ __forceinline__ uint32_t histOffLo(uint32_t w) {  // low half (or the whole fp32 word, or fp64's high half)
  return FT == DGB_FLOAT32 || FT == DGB_FLOAT64 ? (w >> 21) & 0x3fcu : (w >> (FT == DGB_BFLOAT16 ? 5 : 6)) & 0x3fcu;
}
template <int FT>
__device__ __forceinline__ uint32_t histOffHi(uint32_t w) {  // high half of a 16-bit pair
  return (w >> (FT == DGB_BFLOAT16 ? 21 : 22)) & 0x3fcu;
}
__device__ __forceinline__ void histAdd(uint32_t* wh, uint32_t byteOff) {
  atomicAdd(reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(wh) + byteOff), 1u);
}
// Narrowing kinds: two float32 words rounded to the archive type's 16-bit words at once (lo -> bits 0..15,
// hi -> bits 16..31), round to nearest even: the packed form of the instruction torch's CUDA cast uses
// (__float2half: cvt.rn.f16.f32, __float2bfloat16: cvt.rn.bf16.f32), with the same result for every float32
// bit pattern, NaNs included (tests/test_gpu_narrow.py checks all 2^32).
template <int KIND>
__device__ __forceinline__ uint32_t narrowPair(uint32_t lo, uint32_t hi) {
  uint32_t r;
  if (archiveKind(KIND) == DGB_FLOAT16)
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(__uint_as_float(hi)), "f"(__uint_as_float(lo)));
  else
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(__uint_as_float(hi)), "f"(__uint_as_float(lo)));
  return r;
}
// One word, in bits 0..15 (the high half rounds +0 to 0).  Not the scalar cvt.rn.f16.f32: ptxas lowers a byte
// store of that instruction's 16-bit result as a float-to-integer conversion (F2I.U8.F16), not as its low byte.
template <int KIND>
__device__ __forceinline__ uint32_t narrowWord(uint32_t w) {
  return narrowPair<KIND>(w, 0u);
}

// ---- error feedback (the EF kinds) ----
// y = x + e: one round-to-nearest fp32 add, subnormals kept (torch's CUDA add); __fadd_rn never joins a multiply
__device__ __forceinline__ uint32_t efSum(uint32_t x, uint32_t e) {
  return __float_as_uint(__fadd_rn(__uint_as_float(x), __uint_as_float(e)));
}
// The residual of y whose rounded 16-bit word is h (bits 0..15): y - float(h), exact for a finite h, and +0 when h
// is inf or NaN, so that one overflow or one non-finite gradient does not poison every later step.
template <int KIND>
__device__ __forceinline__ uint32_t efResidual(uint32_t y, uint32_t h) {
  float wf;
  bool finite;
  if constexpr (archiveKind(KIND) == DGB_FLOAT16) {
    asm("cvt.f32.f16 %0, %1;" : "=f"(wf) : "h"((unsigned short)h));
    finite = (h & 0x7c00u) != 0x7c00u;
  } else {
    wf = __uint_as_float(h << 16);
    finite = (h & 0x7f80u) != 0x7f80u;
  }
  return finite ? __float_as_uint(__fsub_rn(__uint_as_float(y), wf)) : 0u;
}

template <int FT>
__device__ __forceinline__ uint32_t codedScalar(const uint8_t* in, uint32_t e) {
  if constexpr (isNarrowKind(FT)) {
    const uint32_t w = narrowWord<FT>(reinterpret_cast<const uint32_t*>(in)[e]);
    return archiveKind(FT) == DGB_BFLOAT16 ? (w >> 7) & 0xffu : w >> 8;
  }
  if (FT == DGB_FLOAT64) return (reinterpret_cast<const uint32_t*>(in)[2u * (size_t)e + 1u] >> 23) & 0xffu;
  if (FT == DGB_FLOAT32) return (reinterpret_cast<const uint32_t*>(in)[e] >> 23) & 0xffu;
  const uint32_t w = reinterpret_cast<const uint16_t*>(in)[e];
  return FT == DGB_BFLOAT16 ? (w >> 7) & 0xffu : w >> 8;
}
// EF kinds: the rounded word of y = x + e (statistics pass: e is read, never written)
template <int FT>
__device__ __forceinline__ uint32_t efWordScalar(const uint8_t* in, const float* err, uint32_t e) {
  return narrowWord<FT>(efSum(reinterpret_cast<const uint32_t*>(in)[e], __float_as_uint(err[e])));
}
template <int FT>
__device__ __forceinline__ uint32_t codedScalarEf(const uint8_t* in, const float* err, uint32_t e) {
  const uint32_t w = efWordScalar<FT>(in, err, e);
  return archiveKind(FT) == DGB_BFLOAT16 ? (w >> 7) & 0xffu : w >> 8;
}

// The vector body of a float statistics slab: vectors [v0, v1) of the member, 16 B each: a pure
// read (the coder takes the coded byte out of the raw words itself and writes the stored planes).
// EF kinds: `evec` is the member's residual words, vector for vector beside `vec` (same address mod 16), and the
// words counted are round(x + e).
template <int FT, bool STAGED>
__device__ __forceinline__ void histVectors(const uint4* __restrict__ vec, const StatsStage& stage, uint32_t v0,
                                            uint32_t v1, uint32_t t, uint32_t* wh,
                                            const uint4* __restrict__ evec = nullptr) {
  for (uint32_t i0 = v0 + t; i0 < v1; i0 += kStatsUnroll * kStatsThreads) {
    uint4 vv[kStatsUnroll];
    [[maybe_unused]] uint4 ev[kStatsUnroll];
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t i = i0 + k * kStatsThreads;
      vv[k] = i < v1 ? (STAGED ? stage.buf[i - v0] : ldStream16(vec + i)) : make_uint4(0, 0, 0, 0);
      if constexpr (isEfKind(FT)) ev[k] = i < v1 ? ldStream16(evec + i) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t i = i0 + k * kStatsThreads;
      if (i >= v1) break;
      if constexpr (isEfKind(FT)) {
        vv[k] = make_uint4(efSum(vv[k].x, ev[k].x), efSum(vv[k].y, ev[k].y), efSum(vv[k].z, ev[k].z),
                           efSum(vv[k].w, ev[k].w));
      }
      if constexpr (isNarrowKind(FT)) {  // four float32 words -> two packed pairs of the archive type
        constexpr int AT = archiveKind(FT);
        const uint32_t p0 = narrowPair<FT>(vv[k].x, vv[k].y), p1 = narrowPair<FT>(vv[k].z, vv[k].w);
        histAdd(wh, histOffLo<AT>(p0));
        histAdd(wh, histOffHi<AT>(p0));
        histAdd(wh, histOffLo<AT>(p1));
        histAdd(wh, histOffHi<AT>(p1));
        continue;
      }
      if (FT == DGB_FLOAT64) {  // two words per vector: the coded byte is in each odd 32-bit half
        histAdd(wh, histOffLo<FT>(vv[k].y));
        histAdd(wh, histOffLo<FT>(vv[k].w));
        continue;
      }
      const uint32_t w4[4] = {vv[k].x, vv[k].y, vv[k].z, vv[k].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        histAdd(wh, histOffLo<FT>(w4[q]));
        if (FT != DGB_FLOAT32) histAdd(wh, histOffHi<FT>(w4[q]));
      }
    }
  }
}

// ---- sparse kinds: the +0 / -0 counts of the statistics pass ----------------------------------------------
// Bit j = element j of a 16 B vector of 16-bit words is +0 or -0; pz / nz count the +0 / -0 words.
__device__ __forceinline__ uint32_t zeroMask8(const uint4& v, uint32_t& pz, uint32_t& nz) {
  const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
  uint32_t m = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t lo = w4[q] & 0xffffu, hi = w4[q] >> 16;
    m |= (uint32_t)((lo & 0x7fffu) == 0u) << (2 * q);
    m |= (uint32_t)((hi & 0x7fffu) == 0u) << (2 * q + 1);
    pz += (uint32_t)(lo == 0u) + (uint32_t)(hi == 0u);
    nz += (uint32_t)(lo == 0x8000u) + (uint32_t)(hi == 0x8000u);
  }
  return m;
}

// The vector body for the sparse kinds: the natural symbols' histogram as for the dense type BT, plus the +-0
// words per member (registers) and per 4 KiB block (`bz`, global).  The 32 vectors a warp reads at once
// are 256 consecutive elements, so they touch at most two blocks: one warp reduction per block, one atomic each.
// `head` = elements before the first vector; when it is not 0 every block boundary falls inside a vector.
template <int BT>
__device__ __forceinline__ void histZeroVectors(const uint4* __restrict__ vec, uint32_t v0, uint32_t v1, uint32_t t,
                                                uint32_t* wh, uint32_t head, uint32_t* __restrict__ bz,
                                                uint32_t& pz, uint32_t& nz) {
  const uint32_t lane = t & 31u;
  for (uint32_t w0 = v0 + (t & ~31u); w0 < v1; w0 += kStatsUnroll * kStatsThreads) {  // warp-uniform
    uint4 vv[kStatsUnroll];
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t i = w0 + lane + k * kStatsThreads;
      vv[k] = i < v1 ? ldStream16(vec + i) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t wi = w0 + k * kStatsThreads;  // the warp's first vector
      if (wi >= v1) break;
      const uint32_t i = wi + lane;
      const uint32_t wb = (head + 8u * wi) >> 12;  // block of the warp's first element
      uint32_t c0 = 0, c1 = 0;                     // +-0 words in blocks wb and wb + 1
      if (i < v1) {
        const uint32_t w4[4] = {vv[k].x, vv[k].y, vv[k].z, vv[k].w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          histAdd(wh, histOffLo<BT>(w4[q]));
          histAdd(wh, histOffHi<BT>(w4[q]));
        }
        const uint32_t zm = zeroMask8(vv[k], pz, nz);
        const uint32_t e0 = head + 8u * i, bA = e0 >> 12;
        uint32_t cA = __popc(zm), cB = 0;
        if (((e0 + 7u) >> 12) != bA) {  // straddles a boundary: elements j < 8 - head are in block bA
          const uint32_t j = 8u - head;
          cA = __popc(zm & ((1u << j) - 1u));
          cB = __popc(zm >> j);
        }
        c0 = bA == wb ? cA : 0u;
        c1 = bA == wb ? cB : cA;
      }
      const uint32_t s0 = __reduce_add_sync(0xffffffffu, c0), s1 = __reduce_add_sync(0xffffffffu, c1);
      if (lane == 0) {
        if (s0) atomicAdd(bz + wb, s0);
        if (s1) atomicAdd(bz + wb + 1, s1);
      }
    }
  }
}

// Sparse fp32: the same counts over 16 B vectors of four 32-bit words (a warp's 32 vectors are 128 consecutive
// elements, so they too touch at most two blocks).  `head` = elements before the first vector (0..3).
__device__ __forceinline__ uint32_t zeroMask4(const uint4& v, uint32_t& pz, uint32_t& nz) {
  const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
  uint32_t m = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    m |= (uint32_t)((w4[q] & 0x7fffffffu) == 0u) << q;
    pz += (uint32_t)(w4[q] == 0u);
    nz += (uint32_t)(w4[q] == 0x80000000u);
  }
  return m;
}
__device__ __forceinline__ void histZeroVectors32(const uint4* __restrict__ vec, uint32_t v0, uint32_t v1, uint32_t t,
                                                  uint32_t* wh, uint32_t head, uint32_t* __restrict__ bz,
                                                  uint32_t& pz, uint32_t& nz) {
  const uint32_t lane = t & 31u;
  for (uint32_t w0 = v0 + (t & ~31u); w0 < v1; w0 += kStatsUnroll * kStatsThreads) {  // warp-uniform
    uint4 vv[kStatsUnroll];
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t i = w0 + lane + k * kStatsThreads;
      vv[k] = i < v1 ? ldStream16(vec + i) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int k = 0; k < kStatsUnroll; ++k) {
      const uint32_t wi = w0 + k * kStatsThreads;  // the warp's first vector
      if (wi >= v1) break;
      const uint32_t i = wi + lane;
      const uint32_t wb = (head + 4u * wi) >> 12;  // block of the warp's first element
      uint32_t c0 = 0, c1 = 0;                     // +-0 words in blocks wb and wb + 1
      if (i < v1) {
        histAdd(wh, histOffLo<DGB_FLOAT32>(vv[k].x));
        histAdd(wh, histOffLo<DGB_FLOAT32>(vv[k].y));
        histAdd(wh, histOffLo<DGB_FLOAT32>(vv[k].z));
        histAdd(wh, histOffLo<DGB_FLOAT32>(vv[k].w));
        const uint32_t zm = zeroMask4(vv[k], pz, nz);
        const uint32_t e0 = head + 4u * i, bA = e0 >> 12;
        uint32_t cA = __popc(zm), cB = 0;
        if (((e0 + 3u) >> 12) != bA) {  // straddles a boundary: elements j < 4 - head are in block bA
          const uint32_t j = 4u - head;
          cA = __popc(zm & ((1u << j) - 1u));
          cB = __popc(zm >> j);
        }
        c0 = bA == wb ? cA : 0u;
        c1 = bA == wb ? cB : cA;
      }
      const uint32_t s0 = __reduce_add_sync(0xffffffffu, c0), s1 = __reduce_add_sync(0xffffffffu, c1);
      if (lane == 0) {
        if (s0) atomicAdd(bz + wb, s0);
        if (s1) atomicAdd(bz + wb + 1, s1);
      }
    }
  }
}

// Last CTA of a sparse member (256 threads, thread t = symbol t): picks E+ and E-, moves the +0 / -0 counts from
// their natural symbols (+0: 0; -0: 0x80 for fp16, 0 for bf16 and fp32) to them, normalises, and writes the block
// table, the 32 B header, the zero padding of the table and the stored plane(s), the pdf and the encoder table.
template <int FT>
__device__ void finishSparseMember(const EncodeScratch& sc, int pb, bool useChecksum, const MemberDesc& md, uint32_t m,
                                   uint32_t* __restrict__ outSize) {
  constexpr uint32_t kNegSym = FT == kKindF16S ? 0x80u : 0u;
  __shared__ uint32_t sFree[kStatsWarps];
  __shared__ uint32_t sScan[kStatsWarps];
  const uint32_t t = threadIdx.x;
  const uint32_t size = md.size;
  uint8_t* archive = static_cast<uint8_t*>(md.out);
  const uint32_t pz = __ldcg(zeroCounts(sc, m)), nz = __ldcg(zeroCounts(sc, m) + 1);
  uint32_t* hist = sc.hist + m * kNumSymbols;
  const uint32_t other = __ldcg(hist + t) - (t == 0u ? pz : 0u) - (t == kNegSym ? nz : 0u);  // words neither +0 nor -0
  const uint32_t freeMask = __ballot_sync(0xffffffffu, other == 0u);
  if ((t & 31u) == 0u) sFree[t >> 5] = freeMask;
  __syncthreads();
  // E+ / E-: the two smallest symbols no other word uses (both or neither, see DESIGN.md section 0)
  uint32_t ep = 0, em = 0, found = 0;
  for (uint32_t w = 0; w < (uint32_t)kStatsWarps && found < 2u; ++w) {
    for (uint32_t f = sFree[w]; f != 0u && found < 2u; f &= f - 1u, ++found) {
      const uint32_t s = 32u * w + (uint32_t)__ffs((int)f) - 1u;
      if (found == 0u) ep = s; else em = s;
    }
  }
  const bool elide = found == 2u;
  const uint32_t esc = elide ? (ep | (em << 8) | (1u << 16)) : 0u;
  if (elide) hist[t] = other + (t == ep ? pz : 0u) + (t == em ? nz : 0u);  // read back by this thread below

  // block table: exclusive prefix of the stored bytes per block; each thread takes a contiguous run of blocks
  const uint32_t nb = divUp(size, kBlockBytes);
  uint32_t* table = reinterpret_cast<uint32_t*>(archive + kSparseHeaderBytes);
  const uint32_t* bz = blockZeros(sc, md.work0);
  const uint32_t per = divUp(nb, (uint32_t)kStatsThreads);
  const uint32_t b0 = min(nb, t * per), b1 = min(nb, b0 + per);
  auto kept = [&](uint32_t b) { return min(kBlockBytes, size - b * kBlockBytes) - (elide ? __ldcg(bz + b) : 0u); };
  uint32_t sum = 0;
  for (uint32_t b = b0; b < b1; ++b) sum += kept(b);
  uint32_t S;
  uint32_t run = blockExclusiveScan<kStatsThreads>(sum, sScan, &S);
  for (uint32_t b = b0; b < b1; ++b) {
    table[b] = run;
    run += kept(b);
  }
  for (uint32_t b = nb + t; b < roundUp(nb, 4u); b += kStatsThreads) table[b] = 0;
  uint8_t* plane = archive + kSparseHeaderBytes + sparseTableBytes<uint32_t>(size);
  if constexpr (FT == kKindF32S) {  // u16 plane, then u8 plane
    const uint32_t p8 = 2u * roundUp(S, 8u);
    for (uint32_t i = 2u * S + t; i < p8; i += kStatsThreads) plane[i] = 0;
    for (uint32_t i = S + t; i < roundUp(S, 16u); i += kStatsThreads) plane[p8 + i] = 0;
  } else {
    for (uint32_t i = S + t; i < roundUp(S, 16u); i += kStatsThreads) plane[i] = 0;
  }
  if (t == 0) {
    uint4* h = reinterpret_cast<uint4*>(archive);
    h[0] = make_uint4(kFloatMagicVersion, size, (uint32_t)FT | ((useChecksum ? 1u : 0u) << 4),
                      useChecksum ? __ldcg(sc.checksum + m) : 0u);
    h[1] = make_uint4(S, esc, 0u, 0u);
  }
  uint8_t* ansArchive;
  if constexpr (FT == kKindF32S)
    ansArchive = archive + sparseExtraBytes<uint32_t>(FT, size, S);
  else
    ansArchive = archive + sparseExtraBytes<uint32_t>(size, S);
  if (size == 0) {
    publishEmptyMember(ansArchive, pb, false, outSize, m, kSparseHeaderBytes);
    return;
  }
  uint4* tab = sc.table + (size_t)m * tableSlots(FT);
  normalizeAndPublish(hist, size, pb, sc.wideTable, tab, ansArchive);
  // entries 256 (+0) and 257 (-0); thread t reads back the entry it has just written
  const uint32_t srcP = elide ? ep : 0u, srcN = elide ? em : kNegSym;
  if (t == srcP || t == srcN) {
    if (sc.wideTable) {
      const uint4 e = tab[t];
      if (t == srcP) tab[256] = e;
      if (t == srcN) tab[257] = e;
    } else {
      uint2* p = reinterpret_cast<uint2*>(tab);
      const uint2 e = p[t];
      if (t == srcP) p[256] = e;
      if (t == srcN) p[257] = e;
    }
  }
}

// Work of CTA y of Y on member m; returns true in the CTA that finished the member.
template <int FT, bool STAGED>
__device__ __forceinline__ bool statsFloatItem(const EncodeScratch& sc, uint32_t (*sHist)[kNumSymbols], int pb,
                                               bool useChecksum, uint32_t slabVecs, const MemberDesc& md,
                                               uint32_t m, uint32_t y,
                                               uint32_t Y, uint32_t* __restrict__ outSize,
                                               const StatsStage& stage = StatsStage(),
                                               const float* __restrict__ err = nullptr) {  // EF kinds: residuals
  constexpr bool SPARSE = isSparseKind(FT);
  constexpr int BT = denseKind(FT);  // the dense type whose natural symbols the histogram counts
  constexpr bool NARROW = isNarrowKind(FT);  // float32 input words, archives of type AT
  constexpr int AT = archiveKind(FT);
  constexpr uint32_t EPV = (BT == DGB_FLOAT64) ? 2u : (BT == DGB_FLOAT32 || NARROW) ? 4u : 8u;  // input elements per 16 B vector
  constexpr uint32_t WB = 16u / EPV;                                                           // input word bytes
  // shuffle => the histogram base is provably warp-uniform (ATOMS [R + UR], no per-symbol add)
  const uint32_t t = threadIdx.x, warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  const uint8_t* in = static_cast<const uint8_t*>(md.in);
  const uint32_t size = md.size;  // float words
  uint8_t* archive = static_cast<uint8_t*>(md.out);
  uint8_t* non = archive + kFloatHeaderBytes;
  const uint32_t nonBytes = floatNonCompBytes(AT, size);
  uint8_t* ansArchive = non + nonBytes;

  const uint32_t head = floatHeadLen(in, size, WB);
  const uint32_t nVec = (size - head) / EPV;
  const uint32_t nSlabs = floatSlabs(in, size, WB, slabVecs);
  const uint32_t participants = min(nSlabs, Y);

  if (participants == 0) {
    if (y != 0) return false;
  } else {
    if (y >= participants) return false;
    const uint4* vec = reinterpret_cast<const uint4*>(in + (size_t)head * WB);
    if (STAGED && t == 0) {
      const uint32_t v0 = y * slabVecs, v1 = min(nVec, v0 + slabVecs);
      if (v1 > v0) {
        fenceProxyAsync();  // the region was last touched through the generic proxy (coder staging)
        mbarExpectTx(stage.bar, (v1 - v0) * 16u);
        bulkLoad(smemAddr(stage.buf), vec + v0, (v1 - v0) * 16u, stage.bar);
      }
    }
#pragma unroll
    for (int w = 0; w < kStatsWarps; ++w) sHist[w][t] = 0;
    __syncthreads();
    uint32_t* wh = sHist[warp];
    uint32_t xorAcc = 0;
    uint32_t pz = 0, nz = 0;  // sparse kinds: +0 / -0 words seen by this thread

    // ---- vector body ----
    for (uint32_t slab = y; slab < nSlabs; slab += Y) {
      const uint32_t v0 = slab * slabVecs, v1 = min(nVec, v0 + slabVecs);
      if (STAGED && v1 > v0) {  // one slab per item (Y == nSlabs): the copy was issued above
        mbarWait(stage.bar, *stage.phase);
        *stage.phase ^= 1u;
      }
      // four independent 16 B loads per thread are issued before any of them is consumed: the
      // kernel is a pure stream and was latency-bound with one load in flight
      if constexpr (FT == kKindF32S)
        histZeroVectors32(vec, v0, v1, t, wh, head, blockZeros(sc, md.work0), pz, nz);
      else if constexpr (SPARSE)
        histZeroVectors<BT>(vec, v0, v1, t, wh, head, blockZeros(sc, md.work0), pz, nz);
      else if constexpr (isEfKind(FT))  // err has in's address mod 16, so its vectors start at the same element
        histVectors<FT, STAGED>(vec, stage, v0, v1, t, wh, reinterpret_cast<const uint4*>(err + head));
      else
        histVectors<FT, STAGED>(vec, stage, v0, v1, t, wh);
    }
    if constexpr (SPARSE) {
      if (y == 0) {
        // scalar head and tail; the 32 B header, the table and the padding are written by the last CTA
        const uint32_t tailStart = head + nVec * EPV;
        uint32_t* bz = blockZeros(sc, md.work0);
        if constexpr (FT == kKindF32S) {
          const uint32_t* in32 = reinterpret_cast<const uint32_t*>(in);
          auto scalar = [&](uint32_t e) {
            const uint32_t w = in32[e];
            atomicAdd(&wh[(w >> 23) & 0xffu], 1u);
            if ((w & 0x7fffffffu) == 0u) {
              pz += w == 0u;
              nz += w != 0u;
              atomicAdd(bz + (e >> 12), 1u);
            }
          };
          if (t < head) scalar(t);
          if (t < size - tailStart) scalar(tailStart + t);
        } else {
          const uint16_t* in16 = reinterpret_cast<const uint16_t*>(in);
          auto scalar = [&](uint32_t e) {
            const uint32_t w = in16[e];
            atomicAdd(&wh[BT == DGB_BFLOAT16 ? (w >> 7) & 0xffu : w >> 8], 1u);
            if ((w & 0x7fffu) == 0u) {
              pz += w == 0u;
              nz += w != 0u;
              atomicAdd(bz + (e >> 12), 1u);
            }
          };
          if (t < head) scalar(t);
          if (t < size - tailStart) scalar(tailStart + t);
        }
      }
      const uint32_t p = __reduce_add_sync(0xffffffffu, pz), q = __reduce_add_sync(0xffffffffu, nz);
      if ((t & 31u) == 0u) {
        if (p) atomicAdd(zeroCounts(sc, m), p);
        if (q) atomicAdd(zeroCounts(sc, m) + 1, q);
      }
    } else if (y == 0) {
      // ---- scalar head and tail (fewer than one vector each) ----
      const uint32_t tailStart = head + nVec * EPV;
      if constexpr (isEfKind(FT)) {
        if (t < head) atomicAdd(&wh[codedScalarEf<FT>(in, err, t)], 1u);
        if (t < size - tailStart) atomicAdd(&wh[codedScalarEf<FT>(in, err, tailStart + t)], 1u);
      } else {
        if (t < head) atomicAdd(&wh[codedScalar<FT>(in, t)], 1u);
        if (t < size - tailStart) atomicAdd(&wh[codedScalar<FT>(in, tailStart + t)], 1u);
      }
      // float header (float/GpuFloatCompress.cuh:324-337) and zero padding of the planes
      if (t == 0) {
        // float-level checksum is patched in by the epilogue CTA
        *reinterpret_cast<uint4*>(archive) =
            make_uint4(kFloatMagicVersion, size, (uint32_t)AT | ((useChecksum ? 1u : 0u) << 4), 0u);
      }
      if (FT == DGB_FLOAT64) {
        const uint32_t p16 = floatU16PlaneOffset<uint32_t>(FT, size), p8 = floatU8PlaneOffset<uint32_t>(FT, size);
        for (uint32_t i = 4u * size + t; i < p16; i += kStatsThreads) non[i] = 0;
        for (uint32_t i = p16 + 2u * size + t; i < p8; i += kStatsThreads) non[i] = 0;
        for (uint32_t i = p8 + size + t; i < nonBytes; i += kStatsThreads) non[i] = 0;
      } else if (FT == DGB_FLOAT32) {
        const uint32_t p16 = 2u * roundUp(size, 8u);
        for (uint32_t i = 2u * size + t; i < p16; i += kStatsThreads) non[i] = 0;
        for (uint32_t i = p16 + size + t; i < nonBytes; i += kStatsThreads) non[i] = 0;
      } else {
        for (uint32_t i = size + t; i < nonBytes; i += kStatsThreads) non[i] = 0;
      }
    }
    if (isEfKind(FT) && useChecksum) {  // the rounded words of y = x + e
      for (uint32_t j = y * kStatsThreads + t; j < (size >> 1); j += participants * kStatsThreads)
        xorAcc ^= efWordScalar<FT>(in, err, j);
      if ((size & 1u) && y == 0 && t == 0) xorAcc ^= efWordScalar<FT>(in, err, size >> 1) & 0xffu;
    } else if (NARROW && useChecksum) {
      // the same rule over the ROUNDED data: its first size / 2 16-bit words, then the low byte of the next
      // one when size is odd (foldXor folds both bytes of a word into the byte checksum)
      const uint32_t* in32 = reinterpret_cast<const uint32_t*>(in);
      for (uint32_t j = y * kStatsThreads + t; j < (size >> 1); j += participants * kStatsThreads)
        xorAcc ^= narrowWord<FT>(in32[j]);
      if ((size & 1u) && y == 0 && t == 0) xorAcc ^= narrowWord<FT>(in32[size >> 1]) & 0xffu;
    } else if (useChecksum) {
      // SURVEY A.6 / B6: the float checksum covers the first `size` BYTES only (fp64: the first size / 8 words)
      const uint32_t cbytes = size;  // bytes, not words
      for (uint32_t i = y * kStatsThreads + t; i < cbytes; i += participants * kStatsThreads)
        xorAcc ^= in[i];
    }
    if (!flushAndTicket(sHist, sc.hist + m * kNumSymbols, sc.histDone + m, participants, true,
                        xorAcc, sc.checksum + m, useChecksum))
      return false;
  }

  // ---- last CTA of the member ----
  if constexpr (SPARSE) {
    finishSparseMember<FT>(sc, pb, useChecksum, md, m, outSize);
    return true;
  }
  if (size == 0) {
    if (t == 0) {
      *reinterpret_cast<uint4*>(archive) =
          make_uint4(kFloatMagicVersion, 0u, (uint32_t)AT | ((useChecksum ? 1u : 0u) << 4), 0u);
    }
    publishEmptyMember(ansArchive, pb, false, outSize, m, kFloatHeaderBytes + nonBytes);
    return true;
  }
  if (useChecksum && t == 0) {
    reinterpret_cast<uint32_t*>(archive)[3] = __ldcg(sc.checksum + m);
  }
  normalizeAndPublish(sc.hist + m * kNumSymbols, size, pb, sc.wideTable, sc.table + m * kNumSymbols, ansArchive);
  return true;
}

template <int FT>
__global__ void __launch_bounds__(kStatsThreads)
statsFloatKernel(EncodeScratch sc, const __grid_constant__ InlineMembers im, int pb, bool useChecksum, uint32_t slabVecs,
                 uint32_t memberBase, uint32_t* __restrict__ outSize) {
  __shared__ uint32_t sHist[kStatsWarps][kNumSymbols];
  const uint32_t m = blockIdx.x + memberBase;
  statsFloatItem<FT, false>(sc, sHist, pb, useChecksum, slabVecs, memberAt(im, sc.members, m), m, blockIdx.y, gridDim.y,
                            outSize);
}

// K1 of the EF kinds: statsFloatKernel plus the residual table (read only: the coder overwrites the residuals)
template <int FT>
__global__ void __launch_bounds__(kStatsThreads)
statsFloatEfKernel(EncodeScratch sc, const __grid_constant__ InlineMembers im, const __grid_constant__ EfMembers ef,
                   int pb, bool useChecksum, uint32_t slabVecs, uint32_t memberBase, uint32_t* __restrict__ outSize) {
  __shared__ uint32_t sHist[kStatsWarps][kNumSymbols];
  const uint32_t m = blockIdx.x + memberBase;
  statsFloatItem<FT, false>(sc, sHist, pb, useChecksum, slabVecs, memberAt(im, sc.members, m), m, blockIdx.y, gridDim.y,
                            outSize, StatsStage(), efAt(ef, m));
}

// K1 with the slab landed in shared memory by one TMA bulk copy per CTA (option stats_stage): the
// bytes in flight per SM no longer depend on the number of resident statistics warps, so the kernel
// keeps its bandwidth when it only gets the SM resources the coder of the previous sub-batch leaves
// free.  gridDim.y must equal the slab count (one slab per CTA); dynamic shared memory = slab bytes.
template <int FT>
__global__ void __launch_bounds__(kStatsThreads)
statsFloatStagedKernel(EncodeScratch sc, int pb, bool useChecksum, uint32_t slabVecs, uint32_t memberBase,
                       uint32_t* __restrict__ outSize) {
  extern __shared__ __align__(16) uint8_t stageSmem[];
  __shared__ uint32_t sHist[kStatsWarps][kNumSymbols];
  __shared__ __align__(8) unsigned long long sBar;
  uint32_t phase = 0;
  StatsStage stage;
  stage.buf = reinterpret_cast<uint4*>(stageSmem);
  stage.bar = smemAddr(&sBar);
  stage.phase = &phase;
  if (threadIdx.x == 0) mbarInit(stage.bar, 1);
  fenceBarrierInit();
  __syncthreads();
  const uint32_t m = blockIdx.x + memberBase;
  statsFloatItem<FT, true>(sc, sHist, pb, useChecksum, slabVecs, sc.members[m], m, blockIdx.y, gridDim.y, outSize, stage);
}

// ---------------------------------------------------------------------------
// K2: the rANS state machine + single-pass packing.
//
// Every WARP is an independent worker: it draws ORDERED tickets (one 4 KiB block
// each) from a global counter, keeps its own copy of the member's encoder table
// and its own staging slot in shared memory, streams the block's input bytes
// through a small cp.async ring, and resolves the packed offset of its block
// with a warp-wide decoupled look-back over the tickets of the same member.
// There is no CTA-wide barrier anywhere in the loop (a per-ticket
// __syncthreads would make every warp wait for the slowest block of the CTA).
// ---------------------------------------------------------------------------
#ifndef DGB_ENC_GROUP_ROWS
#define DGB_ENC_GROUP_ROWS 16
#endif
constexpr int kEncGroupRows = DGB_ENC_GROUP_ROWS;  // rows per cp.async group

// ---------------------------------------------------------------------------
// Input side of the coder, per data kind.  The coder reads the member's RAW words (bytes, or the
// fp16 / bf16 / fp32 words themselves): for float kinds it takes the coded byte out of each word on
// the way to the table lookup and writes the stored plane(s) of the float archive from the same
// shared-memory copy of the input.  The reference (and round 1 here) splits in a separate pass that
// writes the coded bytes to scratch for the coder to read back (float/GpuFloatCompress.cuh:280-365):
// one byte per element written and one read, which is a quarter of the statistics pass's traffic;
// here the statistics pass is a pure read.
//   fp16 : coded = w >> 8,        stored = w & 0xff                     (float/GpuFloatUtils.cuh:111-119)
//   bf16 : coded = (w >> 7) & ff, stored = (w & 7f) << 1 | w >> 15      (:141-159)
//   fp32 : coded = (w >> 23) & ff, stored = low 24 bits of rotl(w, 1): u16 plane then u8 plane (:181-203)
//   fp64 : coded = (hi >> 23) & ff, stored = low 56 bits of rotl64(w, 1): u32, u16 then u8 plane
// ---------------------------------------------------------------------------
struct StoredPlanes {
  uint8_t* non;   // fp16 / bf16: the stored byte plane; fp32: the u16 plane; fp64: the u32 plane
  uint8_t* non1;  // fp32: the u8 plane; fp64: the u16 plane
  uint8_t* non2;  // fp64: the u8 plane
  // sparse kinds: `non` holds the kept words' bytes, block k's from table[k] on
  const uint32_t* table;
  uint32_t keepAll;  // 1: nothing is elided (esc == 0), every word stores its byte
  float* err;        // EF kinds: the member's residual words (indexed like the member's elements)
};

template <int KIND>
struct EncIn;

template <>
struct EncIn<kKindBytes> {
  static constexpr uint32_t kWordBytes = 1, kRingSlots = 4;
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    return STRIDE * ldsU8<J * 32>(ringLane);
  }
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(uint32_t w) { return STRIDE * w; }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) { return in[e]; }
  static __device__ __forceinline__ void storeScalar(const StoredPlanes&, uint32_t, uint32_t) {}
  static __device__ __forceinline__ void storeGroup(uint32_t, const StoredPlanes&, uint32_t, uint32_t) {}
};

#ifndef DGB_ENC_RING16
#define DGB_ENC_RING16 3  // 3 slots = 3 KiB per warp: 4 CTAs per SM (4 slots: 3)
#endif
template <int KIND>
struct EncIn16 {
  static constexpr uint32_t kWordBytes = 2, kRingSlots = DGB_ENC_RING16;
  static constexpr uint32_t kCodedBit = KIND == kKindBF16 ? 7u : 8u;
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(uint32_t w) {
    // STRIDE * ((w >> kCodedBit) & 0xff) in one shift and one mask (STRIDE is 8 or 16)
    constexpr uint32_t lg = STRIDE == 16 ? 4u : 3u;
    return (w >> (kCodedBit - lg)) & (0xffu << lg);
  }
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    uint32_t w;
    if (KIND == kKindF16) {
      // the coded byte of fp16 IS the word's high byte: read it alone, no shift / mask
      asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 64 + 1));
      return STRIDE * w;
    }
    asm volatile("ld.shared.u16 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 64));
    return tabOffsetOf<STRIDE>(w);
  }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) {
    return __ldg(reinterpret_cast<const uint16_t*>(in) + e);
  }
  static __device__ __forceinline__ uint32_t storedOf(uint32_t w) {
    return KIND == kKindBF16 ? (((w << 1) | (w >> 15)) & 0xffu) : (w & 0xffu);
  }
  static __device__ __forceinline__ void storeScalar(const StoredPlanes& pl, uint32_t e, uint32_t w) {
    pl.non[e] = (uint8_t)storedOf(w);
  }
  // stored bytes of one group of 16 rows (512 elements, 1 KiB in the ring slot at `slot`): lane l
  // handles the 16 B vectors l and l + 32 -> 8 stored bytes each, one 8 B store
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t elem0,
                                                    uint32_t lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t v = lane + 32u * h;
      uint4 x;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(slot + v * 16u));
      const uint32_t r0 = rot16x2<KIND>(x.x), r1 = rot16x2<KIND>(x.y), r2 = rot16x2<KIND>(x.z), r3 = rot16x2<KIND>(x.w);
      uint2 nn;
      nn.x = __byte_perm(r0, r1, 0x6420);
      nn.y = __byte_perm(r2, r3, 0x6420);
      *reinterpret_cast<uint2*>(pl.non + elem0 + v * 8u) = nn;
    }
  }
};
template <> struct EncIn<kKindF16> : EncIn16<kKindF16> {};
template <> struct EncIn<kKindBF16> : EncIn16<kKindBF16> {};

// Sparse fp16 / bf16: a +0 / -0 word looks up table entry 256 / 257 (see tableSlots), every other word its
// natural symbol's.  The stored bytes of the kept words are compacted in element order: per group by a warp scan
// of the lanes' kept counts, per scalar row by a ballot; `cur` is the plane offset of the next kept byte.
template <int KIND>
struct EncInSparse {
  static constexpr int BT = denseKind(KIND);
  static constexpr uint32_t kWordBytes = 2, kRingSlots = DGB_ENC_RING16;
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(uint32_t w) {
    const uint32_t nat = BT == kKindBF16 ? (w >> 7) & 0xffu : w >> 8;
    return STRIDE * ((w & 0x7fffu) == 0u ? 256u + (w >> 15) : nat);
  }
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    uint32_t w;
    asm volatile("ld.shared.u16 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 64));
    return tabOffsetOf<STRIDE>(w);
  }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) {
    return __ldg(reinterpret_cast<const uint16_t*>(in) + e);
  }
  // one row of words, whole warp (lanes without a word pass valid = false)
  static __device__ __forceinline__ void storeRow(const StoredPlanes& pl, uint32_t& cur, uint32_t w, bool valid,
                                                  uint32_t ltMask) {
    const bool keep = valid && (pl.keepAll != 0u || (w & 0x7fffu) != 0u);
    const uint32_t b = __ballot_sync(0xffffffffu, keep);
    if (keep) pl.non[cur + __popc(b & ltMask)] = (uint8_t)EncIn16<BT>::storedOf(w);
    cur += __popc(b);
  }
  // one group of 16 rows (512 elements in the ring slot): lane l takes vectors l and l + 32, 8 elements each
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t& cur,
                                                    uint32_t lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t v = lane + 32u * h;
      uint4 x;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(slot + v * 16u));
      const uint32_t w4[4] = {x.x, x.y, x.z, x.w};
      uint32_t keep = 0xffu;
      if (!pl.keepAll) {
        keep = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          keep |= (uint32_t)((w4[q] & 0x7fffu) != 0u) << (2 * q);
          keep |= (uint32_t)((w4[q] & 0x7fff0000u) != 0u) << (2 * q + 1);
        }
      }
      const uint32_t lo = __byte_perm(rot16x2<BT>(x.x), rot16x2<BT>(x.y), 0x6420);
      const uint32_t hi = __byte_perm(rot16x2<BT>(x.z), rot16x2<BT>(x.w), 0x6420);
      const uint32_t c = __popc(keep);
      uint32_t incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t s = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (uint32_t)d) incl += s;
      }
      uint8_t* p = pl.non + cur + (incl - c);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if ((keep >> j) & 1u) *p++ = (uint8_t)((j < 4 ? lo : hi) >> (8 * (j & 3)));
      }
      cur += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
};
template <> struct EncIn<kKindF16S> : EncInSparse<kKindF16S> {};
template <> struct EncIn<kKindBF16S> : EncInSparse<kKindBF16S> {};

template <>
struct EncIn<kKindF32> {
  static constexpr uint32_t kWordBytes = 4, kRingSlots = 3;
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(uint32_t w) {
    constexpr uint32_t lg = STRIDE == 16 ? 4u : 3u;
    return (w >> (23u - lg)) & (0xffu << lg);
  }
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    uint32_t w;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 128));
    return tabOffsetOf<STRIDE>(w);
  }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) {
    return __ldg(reinterpret_cast<const uint32_t*>(in) + e);
  }
  static __device__ __forceinline__ void storeScalar(const StoredPlanes& pl, uint32_t e, uint32_t w) {
    const uint32_t r = __funnelshift_l(w, w, 1);
    reinterpret_cast<uint16_t*>(pl.non)[e] = (uint16_t)r;
    pl.non1[e] = (uint8_t)(r >> 16);
  }
  // one group of 16 rows = 512 words = 2 KiB in the ring slot: lane l handles vectors l + 32 h
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t elem0,
                                                    uint32_t lane) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const uint32_t v = lane + 32u * h;
      uint4 x;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(slot + v * 16u));
      const uint32_t r0 = __funnelshift_l(x.x, x.x, 1), r1 = __funnelshift_l(x.y, x.y, 1);
      const uint32_t r2 = __funnelshift_l(x.z, x.z, 1), r3 = __funnelshift_l(x.w, x.w, 1);
      uint2 lo;
      lo.x = __byte_perm(r0, r1, 0x5410);
      lo.y = __byte_perm(r2, r3, 0x5410);
      *reinterpret_cast<uint2*>(pl.non + 2u * (size_t)(elem0 + v * 4u)) = lo;
      const uint32_t hi = __byte_perm(__byte_perm(r0, r1, 0x0062), __byte_perm(r2, r3, 0x0062), 0x5410);
      *reinterpret_cast<uint32_t*>(pl.non1 + elem0 + v * 4u) = hi;
    }
  }
};

// Narrowing kinds: float32 words in the ring (fp32's geometry, 2 KiB per group of 16 rows), each rounded to the
// archive type's 16-bit word before the archive type's own coded-byte and stored-byte rules apply.  loadWord
// returns the rounded word, so the scalar paths use the 16-bit kind's tabOffsetOf and storeScalar unchanged.
template <int KIND>
struct EncInNarrow : EncIn16<archiveKind(KIND)> {
  static constexpr int AT = archiveKind(KIND);
  static constexpr uint32_t kWordBytes = 4, kRingSlots = 3;
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    uint32_t w;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 128));
    return EncIn16<AT>::template tabOffsetOf<STRIDE>(narrowWord<KIND>(w));
  }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) {
    return narrowWord<KIND>(__ldg(reinterpret_cast<const uint32_t*>(in) + e));
  }
  // one group of 16 rows = 512 words = 2 KiB in the ring slot: lane l handles vectors l + 32 h, as fp32 does, so
  // every shared load is conflict-free; a vector's four words round to two pairs whose stored bytes are one
  // 4 B store, and the warp's 32 stores of a step cover 128 contiguous bytes of the plane
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t elem0,
                                                    uint32_t lane) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const uint32_t v = lane + 32u * h;
      uint4 x;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(slot + v * 16u));
      const uint32_t r0 = rot16x2<AT>(narrowPair<KIND>(x.x, x.y)), r1 = rot16x2<AT>(narrowPair<KIND>(x.z, x.w));
      *reinterpret_cast<uint32_t*>(pl.non + elem0 + v * 4u) = __byte_perm(r0, r1, 0x6420);
    }
  }
};
template <> struct EncIn<kKindF32toF16> : EncInNarrow<kKindF32toF16> {};
template <> struct EncIn<kKindF32toBF16> : EncInNarrow<kKindF32toBF16> {};

// Error-feedback kinds: the narrowing kind's coder on y = x + e.  storeGroup runs on a ring slot before encodeGroup
// reads it; here it also loads the residual vectors beside the slot's input vectors, forms y, writes y back over x in
// the slot (so the narrowing tabOffset codes round(y)), stores round(y)'s stored bytes and writes each residual
// y - float(round(y)) over e.  The scalar paths do the same per word (loadWordEf).  Every element is visited once,
// by one lane, which reads its e before it writes e'.  The ring is the cp.async one only: a TMA bulk copy into a slot
// these generic-proxy stores have written would need a proxy fence first (encodeMemberBlocks).
template <int KIND>
struct EncInNarrowEf : EncInNarrow<KIND & ~0x80> {
  static constexpr int NK = KIND & ~0x80;  // the narrowing kind
  static constexpr int AT = archiveKind(KIND);
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t elem0,
                                                    uint32_t lane) {
    float4* ep = reinterpret_cast<float4*>(pl.err + elem0);
    uint4 ev[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {  // all four residual loads in flight before the first is used
      const float4 f = __ldcs(ep + lane + 32u * h);
      ev[h] = make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const uint32_t v = lane + 32u * h;
      uint4 x;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(slot + v * 16u));
      const uint4 y = make_uint4(efSum(x.x, ev[h].x), efSum(x.y, ev[h].y), efSum(x.z, ev[h].z), efSum(x.w, ev[h].w));
      asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(slot + v * 16u), "r"(y.x), "r"(y.y), "r"(y.z), "r"(y.w)
                   : "memory");
      const uint32_t p0 = narrowPair<NK>(y.x, y.y), p1 = narrowPair<NK>(y.z, y.w);
      *reinterpret_cast<uint32_t*>(pl.non + elem0 + v * 4u) = __byte_perm(rot16x2<AT>(p0), rot16x2<AT>(p1), 0x6420);
      __stcs(ep + v, make_float4(__uint_as_float(efResidual<KIND>(y.x, p0 & 0xffffu)),
                                 __uint_as_float(efResidual<KIND>(y.y, p0 >> 16)),
                                 __uint_as_float(efResidual<KIND>(y.z, p1 & 0xffffu)),
                                 __uint_as_float(efResidual<KIND>(y.w, p1 >> 16))));
    }
    __syncwarp();  // encodeGroup's lanes read words other lanes have just written
  }
  // one word of the scalar paths: element e of the block, whose residual is err[e]; returns round(y)
  static __device__ __forceinline__ uint32_t loadWordEf(const uint8_t* in, uint32_t e, float* err) {
    const uint32_t y = efSum(__ldg(reinterpret_cast<const uint32_t*>(in) + e), __float_as_uint(err[e]));
    const uint32_t w = narrowWord<NK>(y);
    err[e] = __uint_as_float(efResidual<KIND>(y, w));
    return w;
  }
};
template <> struct EncIn<kKindF32toF16EF> : EncInNarrowEf<kKindF32toF16EF> {};
template <> struct EncIn<kKindF32toBF16EF> : EncInNarrowEf<kKindF32toBF16EF> {};

// the word the scalar paths code: EF kinds also form y and write its residual
template <int KIND>
__device__ __forceinline__ auto encLoadWord(const uint8_t* in, uint32_t e, const StoredPlanes& pl, uint32_t elem0) {
  if constexpr (isEfKind(KIND))
    return EncIn<KIND>::loadWordEf(in, e, pl.err + elem0);
  else
    return EncIn<KIND>::loadWord(in, e);
}

// Sparse fp32: a +0 / -0 word looks up table entry 256 / 257, every other word its exponent symbol.  The kept words'
// 16 + 8 stored bits are compacted into the u16 and u8 planes in element order.  A group of 16 rows (512 words in the
// ring slot) goes in two steps: lane l takes words 16 l .. 16 l + 15 and one warp scan of the lanes' kept counts
// places its kept words in the warp's run (shared memory after the ring: a u16 half and a u8 half); then every
// complete unit of 16 kept words in the run goes to the planes as aligned 16 B vector stores (one u8 vector, two u16
// vectors), and the last partial unit moves to the run's start, carried over to the next group.  Run position p holds
// the kept word with plane index (cur & ~15) + p, so units are 16-word aligned in both planes.  A warp stores only the
// bytes its block owns, kept words [lo, segment end) with lo = table[block]: segments are not 16-word aligned, so the
// unit that starts below lo is stored word by word, and so is the partial unit left after the last group (flushTail).
// The scalar paths (unaligned input, the remaining rows, the partial row) store word by word too.
template <>
struct EncIn<kKindF32S> {
  static constexpr uint32_t kWordBytes = 4, kRingSlots = 3;
  static constexpr uint32_t kRingGroupBytes = kRingSlots * kEncGroupRows * 128u;  // the run starts here
  static constexpr uint32_t kRun8 = 1056u;                                        // u8 half (u16 half: 528 x 2 B)
  static constexpr uint32_t kRunBytes = kRun8 + 528u;                             // a run holds < 16 + 512 words
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(uint32_t w) {
    return STRIDE * ((w & 0x7fffffffu) == 0u ? 256u + (w >> 31) : (w >> 23) & 0xffu);
  }
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    uint32_t w;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 128));
    return tabOffsetOf<STRIDE>(w);
  }
  static __device__ __forceinline__ uint32_t loadWord(const uint8_t* in, uint32_t e) {
    return __ldg(reinterpret_cast<const uint32_t*>(in) + e);
  }
  // kept word idx of the planes <- r's low 24 bits
  static __device__ __forceinline__ void storeWord(const StoredPlanes& pl, uint32_t idx, uint32_t r) {
    reinterpret_cast<uint16_t*>(pl.non)[idx] = (uint16_t)r;
    pl.non1[idx] = (uint8_t)(r >> 16);
  }
  // run position p as r's low 24 bits
  static __device__ __forceinline__ uint32_t runWord(uint32_t run, uint32_t p) {
    uint32_t lo16, hi8;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(lo16) : "r"(run + 2u * p));
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(hi8) : "r"(run + kRun8 + p));
    return lo16 | (hi8 << 16);
  }
  static __device__ __forceinline__ void setRunWord(uint32_t run, uint32_t p, uint32_t r) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(run + 2u * p), "h"((unsigned short)r) : "memory");
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(run + kRun8 + p), "r"(r >> 16) : "memory");
  }
  // one row of words, whole warp (lanes without a word pass valid = false)
  static __device__ __forceinline__ void storeRow(const StoredPlanes& pl, uint32_t& cur, uint32_t w, bool valid,
                                                  uint32_t ltMask) {
    const bool keep = valid && (pl.keepAll != 0u || (w & 0x7fffffffu) != 0u);
    const uint32_t b = __ballot_sync(0xffffffffu, keep);
    if (keep) storeWord(pl, cur + __popc(b & ltMask), __funnelshift_l(w, w, 1));
    cur += __popc(b);
  }
  // one group of 16 rows in the ring slot at `slot`; `run` = shared address of the warp's run
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t& cur, uint32_t lo,
                                                    uint32_t run, uint32_t lane) {
    uint32_t w[16];
#pragma unroll
    for (int h = 0; h < 4; ++h)
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(w[4 * h]), "=r"(w[4 * h + 1]), "=r"(w[4 * h + 2]), "=r"(w[4 * h + 3])
                   : "r"(slot + lane * 64u + h * 16u));
    uint32_t keep = 0xffffu;
    if (!pl.keepAll) {
      keep = 0;
#pragma unroll
      for (int j = 0; j < 16; ++j) keep |= (uint32_t)((w[j] & 0x7fffffffu) != 0u) << j;
    }
    const uint32_t c = __popc(keep);
    uint32_t incl = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t x = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= (uint32_t)d) incl += x;
    }
    const uint32_t k = __shfl_sync(0xffffffffu, incl, 31);
    // 1. compaction into the run
    const uint32_t p = (cur & 15u) + incl - c;
    uint32_t a16 = run + 2u * p, a8 = run + kRun8 + p;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if ((keep >> j) & 1u) {
        const uint32_t r = __funnelshift_l(w[j], w[j], 1);
        asm volatile("st.shared.u16 [%0], %1;" ::"r"(a16), "h"((unsigned short)r) : "memory");
        asm volatile("st.shared.u8 [%0], %1;" ::"r"(a8), "r"(r >> 16) : "memory");
        a16 += 2u;
        a8 += 1u;
      }
    }
    __syncwarp();
    // 2. complete units to the planes (lane u takes unit u); the partial unit's words into registers
    const uint32_t A = cur & ~15u, total = (cur & 15u) + k, units = total >> 4, tail = total & 15u;
    if (lane < units) {
      const uint32_t v = A + 16u * lane;
      if (v >= lo) {
        uint4 x, y, z;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(run + 32u * lane));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y.x), "=r"(y.y), "=r"(y.z), "=r"(y.w) : "r"(run + 32u * lane + 16u));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(z.x), "=r"(z.y), "=r"(z.z), "=r"(z.w) : "r"(run + kRun8 + 16u * lane));
        uint4* d16 = reinterpret_cast<uint4*>(pl.non + 2u * (size_t)v);
        d16[0] = x;
        d16[1] = y;
        *reinterpret_cast<uint4*>(pl.non1 + v) = z;
      } else {  // the block's first unit starts inside the previous block's segment
        for (uint32_t i = lo - v; i < 16u; ++i) storeWord(pl, v + i, runWord(run, 16u * lane + i));
      }
    }
    const bool move = units != 0u && lane < tail;
    const uint32_t carry = move ? runWord(run, 16u * units + lane) : 0u;
    __syncwarp();
    if (move) setRunWord(run, lane, carry);
    __syncwarp();
    cur += k;
  }
  // the partial unit left in the run after the last group: kept words [max(cur & ~15, lo), cur)
  static __device__ __forceinline__ void flushTail(const StoredPlanes& pl, uint32_t cur, uint32_t lo, uint32_t run,
                                                   uint32_t lane) {
    const uint32_t idx = (cur & ~15u) + lane;
    if (lane < (cur & 15u) && idx >= lo) storeWord(pl, idx, runWord(run, lane));
    __syncwarp();
  }
};

#ifndef DGB_ENC_RING64
#define DGB_ENC_RING64 3
#endif
// fp64: 16 rows x 32 lanes x 8 B = 4 KiB per group, so the ring bounds the coder CTAs per SM
template <>
struct EncIn<kKindF64> {
  static constexpr uint32_t kWordBytes = 8, kRingSlots = DGB_ENC_RING64;
  template <uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffsetOf(unsigned long long w) {
    return EncIn<kKindF32>::tabOffsetOf<STRIDE>((uint32_t)(w >> 32));
  }
  template <int J, uint32_t STRIDE>
  static __device__ __forceinline__ uint32_t tabOffset(uint32_t ringLane) {
    // only the high half of the lane's word holds coded bits
    uint32_t w;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(w) : "r"(ringLane), "n"(J * 256 + 4));
    return EncIn<kKindF32>::tabOffsetOf<STRIDE>(w);
  }
  static __device__ __forceinline__ unsigned long long loadWord(const uint8_t* in, uint32_t e) {
    return __ldg(reinterpret_cast<const unsigned long long*>(in) + e);
  }
  static __device__ __forceinline__ void storeScalar(const StoredPlanes& pl, uint32_t e, unsigned long long w) {
    const unsigned long long v = (w << 1) | (w >> 63);
    reinterpret_cast<uint32_t*>(pl.non)[e] = (uint32_t)v;
    reinterpret_cast<uint16_t*>(pl.non1)[e] = (uint16_t)(v >> 32);
    pl.non2[e] = (uint8_t)(v >> 48);
  }
  // one group of 16 rows = 512 words = 4 KiB in the ring slot: lane l handles words 4 (l + 32 h) .. +3, so
  // every plane gets one vector store per lane and step (16 B, 8 B, 4 B)
  static __device__ __forceinline__ void storeGroup(uint32_t slot, const StoredPlanes& pl, uint32_t elem0,
                                                    uint32_t lane) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const uint32_t q = lane + 32u * h;
      uint4 a, b;
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "r"(slot + q * 32u));
      asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "r"(slot + q * 32u + 16u));
      // rotl64 by one of (hi:lo): lo' = lo << 1 | hi >> 31, hi' = hi << 1 | lo >> 31
      const uint4 lo = make_uint4(__funnelshift_l(a.y, a.x, 1), __funnelshift_l(a.w, a.z, 1), __funnelshift_l(b.y, b.x, 1),
                                  __funnelshift_l(b.w, b.z, 1));
      const uint32_t h0 = __funnelshift_l(a.x, a.y, 1), h1 = __funnelshift_l(a.z, a.w, 1);
      const uint32_t h2 = __funnelshift_l(b.x, b.y, 1), h3 = __funnelshift_l(b.z, b.w, 1);
      const uint32_t e = elem0 + q * 4u;
      *reinterpret_cast<uint4*>(pl.non + 4u * (size_t)e) = lo;
      *reinterpret_cast<uint2*>(pl.non1 + 2u * (size_t)e) = make_uint2(__byte_perm(h0, h1, 0x5410), __byte_perm(h2, h3, 0x5410));
      *reinterpret_cast<uint32_t*>(pl.non2 + e) =
          __byte_perm(__byte_perm(h0, h1, 0x0062), __byte_perm(h2, h3, 0x0062), 0x5410);
    }
  }
};

__host__ __device__ constexpr uint32_t encRingBytes(int kind) {  // sparse fp32: the ring, then the warp's run
  return kind == kKindF32S ? EncIn<kKindF32S>::kRingGroupBytes + EncIn<kKindF32S>::kRunBytes
         : kind == kKindF64 ? (uint32_t)DGB_ENC_RING64 * kEncGroupRows * 256u
         : kind == kKindBytes
             ? 4u * kEncGroupRows * 32u
             : (kind == kKindF32 || isNarrowKind(kind) ? 3u * kEncGroupRows * 128u
                                                       : (uint32_t)DGB_ENC_RING16 * kEncGroupRows * 64u);
}

// One rANS step for a full row (ans/GpuANSEncode.cuh:49-90 restated).  The
// update uses x' = (x / pdf) * (2^pb - pdf) + x + cdf, which equals
// (x / pdf) << pb + x % pdf + cdf, so the loop needs neither pdf nor pb.
// `wa` is the shared-memory BYTE address of the next free staging word.
// The emit half is PTX so that one predicate feeds the vote, the store and the
// shift (the compiler otherwise materialises the comparison twice).
// The emitted word gets its own register: the store waits for the POPC, and if it read the state
// register the in-place shift (and with it the whole serial chain) would wait too.  Two ways to
// make the copy, one per table format:
//   FMACOPY = false: plain copy, which ptxas folds into shift + select (wide entries: their rows are
//                    ALU-light, so the extra ALU work costs nothing)
//   FMACOPY = true : multiply by a 1 the compiler cannot see through (IMAD, FMA pipe) and shift the
//                    state in place under the predicate (packed entries: their unpacking already loads
//                    the ALU pipe, so the copy moves to the FMA pipe)
template <bool FMACOPY>
__device__ __forceinline__ void emitWords(uint32_t& state, uint32_t thr, uint32_t& wa, uint32_t ltMask,
                                          uint32_t one) {
  if (FMACOPY) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b32 v, t, a, w;\n"
        ".reg .b16 h;\n"
        "setp.ge.u32 p, %0, %2;\n"
        "mul.lo.u32 w, %0, %4;\n"
        "@p shr.u32 %0, %0, 16;\n"
        "vote.sync.ballot.b32 v, p, 0xffffffff;\n"
        "and.b32 t, v, %3;\n"
        "popc.b32 t, t;\n"
        "mad.lo.u32 a, t, 2, %1;\n"
        "cvt.u16.u32 h, w;\n"
        "@p st.shared.u16 [a], h;\n"
        "popc.b32 t, v;\n"
        "mad.lo.u32 %1, t, 2, %1;\n"
        "}\n"
        : "+r"(state), "+r"(wa)
        : "r"(thr), "r"(ltMask), "r"(one)
        : "memory");
  } else {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .b32 v, t, a, w;\n"
        ".reg .b16 h;\n"
        "setp.ge.u32 p, %0, %2;\n"
        "mov.b32 w, %0;\n"
        "shr.u32 t, %0, 16;\n"
        "selp.b32 %0, t, %0, p;\n"
        "vote.sync.ballot.b32 v, p, 0xffffffff;\n"
        "and.b32 t, v, %3;\n"
        "popc.b32 t, t;\n"
        "mad.lo.u32 a, t, 2, %1;\n"
        "cvt.u16.u32 h, w;\n"
        "@p st.shared.u16 [a], h;\n"
        "popc.b32 t, v;\n"
        "mad.lo.u32 %1, t, 2, %1;\n"
        "}\n"
        : "+r"(state), "+r"(wa)
        : "r"(thr), "r"(ltMask)
        : "memory");
  }
}

// Table entry -> the values a row needs.  Two formats (common.cuh), chosen per call by what the
// ANS input is:
//  * EncEntryWide (16 B, LDS.128, four shared-memory wavefronts per row): every field is stored, the
//    row needs the fewest instructions.  Right when a row touches few distinct symbols, i.e. the
//    exponent bytes of bf16 / fp32 data (mostly broadcast reads).
//  * EncEntry (8 B, LDS.64, two wavefronts): the threshold pdf << (31 - pb) is rebuilt from 2^pb - pdf
//    with one multiply-add and the fields are unpacked with shifts and masks.  Right for byte data
//    and fp16, where the bank conflicts of the wide entry dominate (encode call on an H100 at 700 W,
//    tools/walltime.py, packed vs wide: c2 397 vs 506 us, c4 286 vs 304 us; c3 270 us with either,
//    so bf16 keeps the wide entry).
// (Unpacking with IMAD.HI to move work from the ALU to the FMA pipe was tried and not kept.)
// Everything here is independent of the coder state, so it runs ahead of the serial chain.
struct EncRegs {
  uint32_t tabAddr, ltMask, thrNegScale;  // thrNegScale = -(2^(31 - pb)), packed format only
  uint32_t one;                           // 1, but not a compile-time constant (see emitWords)
};
__device__ __forceinline__ EncRegs makeEncRegs(uint32_t tabAddr, int pb) {
  EncRegs r;
  r.tabAddr = tabAddr;
  r.ltMask = laneMaskLt();
  r.thrNegScale = 0u - (1u << (31 - pb));
  r.one = 1u + ((uint32_t)pb >> 31);  // pb is a kernel argument
  return r;
}

template <bool WIDE>
struct EncSym;
template <>
struct EncSym<true> {
  static constexpr uint32_t kStride = 16;
  uint32_t thr, magic, kmpv, cdfShift;
  __device__ __forceinline__ void load(uint32_t addr, const EncRegs&) {
    // not volatile: the table is read-only while a block is encoded, so the scheduler may hoist it
    asm("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(thr), "=r"(magic), "=r"(kmpv), "=r"(cdfShift) : "r"(addr));
  }
  __device__ __forceinline__ uint32_t shiftReg() const { return cdfShift; }  // low 5 bits count
  __device__ __forceinline__ uint32_t kmp() const { return kmpv; }
  __device__ __forceinline__ uint32_t plusCdf(uint32_t x) const { return x + (cdfShift >> 5); }  // one LEA.HI
};
template <>
struct EncSym<false> {
  static constexpr uint32_t kStride = 8;
  uint32_t thr, magic, pack, kmpv;
  __device__ __forceinline__ void load(uint32_t addr, const EncRegs& rc) {
    asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(magic), "=r"(pack) : "r"(addr));
    kmpv = (pack >> kEncKmpShift) & kEncKmpMask;
    thr = kmpv * rc.thrNegScale + 0x80000000u;                                          // pdf << (31 - pb)
  }
  __device__ __forceinline__ uint32_t shiftReg() const { return pack; }
  __device__ __forceinline__ uint32_t kmp() const { return kmpv; }
  __device__ __forceinline__ uint32_t plusCdf(uint32_t x) const { return x + (pack >> kEncCdfShift); }
};

template <bool WIDE>
__device__ __forceinline__ void encodeUpdate(uint32_t& state, const EncSym<WIDE>& e) {
  const uint32_t div = __funnelshift_r(__umulhi(state, e.magic), 0u, e.shiftReg());
  state = div * e.kmp() + e.plusCdf(state);
}

template <bool WIDE>
__device__ __forceinline__ void encodeStep(uint32_t& state, uint32_t tabOff, const EncRegs& rc, uint32_t& wa) {
  EncSym<WIDE> e;
  e.load(rc.tabAddr + tabOff, rc);
  emitWords<!WIDE>(state, e.thr, wa, rc.ltMask, rc.one);
  encodeUpdate(state, e);
}

template <bool WIDE>
__device__ __forceinline__ void encodeStepPartial(bool valid, uint32_t& state, uint32_t tabOff,
                                                  const EncRegs& rc, uint32_t& wa) {
  EncSym<WIDE> e;
  e.load(rc.tabAddr + tabOff, rc);
  // invalid lanes never emit: compare against an unreachable threshold
  emitWords<!WIDE>(state, valid ? e.thr : 0xffffffffu, wa, rc.ltMask, rc.one);
  uint32_t next = state;
  encodeUpdate(next, e);
  state = valid ? next : state;
}

// One group of kEncGroupRows rows.  The symbol bytes and the table entries do not depend on
// the coder state, so they are fetched ahead of the serial state chain: all symbols of the
// group first, then table entries kept kDepth rows ahead of the row being coded.
template <int KIND, int J, uint32_t STRIDE>
struct EncLoad {
  static __device__ __forceinline__ void syms(uint32_t ringLane, uint32_t tabAddr, uint32_t* addr) {
    EncLoad<KIND, J - 1, STRIDE>::syms(ringLane, tabAddr, addr);
    addr[J - 1] = tabAddr + EncIn<KIND>::template tabOffset<J - 1, STRIDE>(ringLane);
  }
};
template <int KIND, uint32_t STRIDE>
struct EncLoad<KIND, 0, STRIDE> {
  static __device__ __forceinline__ void syms(uint32_t, uint32_t, uint32_t*) {}
};

template <bool WIDE, int KIND>
__device__ __forceinline__ void encodeGroup(uint32_t& state, uint32_t ringLane, const EncRegs& rc,
                                            uint32_t& wa) {
  constexpr int U = kEncGroupRows;
  constexpr int kDepth = 4;
  uint32_t addr[U];
  EncLoad<KIND, U, EncSym<WIDE>::kStride>::syms(ringLane, rc.tabAddr, addr);
  EncSym<WIDE> e[kDepth];
#pragma unroll
  for (int j = 0; j < kDepth; ++j) e[j].load(addr[j], rc);
#pragma unroll
  for (int j = 0; j < U; ++j) {
    const EncSym<WIDE> cur = e[j % kDepth];
    if (j + kDepth < U) e[j % kDepth].load(addr[j + kDepth], rc);
    emitWords<!WIDE>(state, cur.thr, wa, rc.ltMask, rc.one);
    encodeUpdate(state, cur);
  }
}

// Staging slot smaller than the worst case: when it runs low, the words staged so far are moved
// to this warp's global spill area (16 B granules; the < 8 leftover words slide to the slot start).
struct Spill {
  uint16_t* area;       // global, maxBlockWords(pb) words, 16 B aligned (nullptr: slot is worst-case sized)
  uint32_t limitBytes;  // spill when more than this many bytes are staged
  uint32_t spilled;     // words already in `area` (multiple of 8)
};

__device__ __forceinline__ void spillOut(Spill& sp, uint32_t stageAddr, uint16_t* stage, uint32_t& wa,
                                         uint32_t lane) {
  __syncwarp();
  const uint32_t used = (wa - stageAddr) >> 1;
  const uint32_t k = used & ~7u;
  uint4* dst = reinterpret_cast<uint4*>(sp.area + sp.spilled);
  const uint4* src = reinterpret_cast<const uint4*>(stage);
  for (uint32_t i = lane; i < k / 8u; i += 32u) dst[i] = src[i];
  const uint32_t left = used - k;
  uint16_t v = 0;
  if (lane < left) v = stage[k + lane];
  __syncwarp();
  if (lane < left) stage[lane] = v;
  __syncwarp();
  sp.spilled += k;
  wa = stageAddr + 2u * left;
}

// Encodes elements [0, n) of one block (raw words of data kind KIND at `in`; `elem0` = index of the
// block's first element in its member) with one warp into the staging slot at shared byte address
// `stageAddr` (spilling to sp.area when the slot is small); float kinds also write the block's
// stored plane(s).  Returns the TOTAL word count; the words not yet spilled are
// stage[0 .. total - sp.spilled).
template <bool WIDE, int KIND, bool TMA>
__device__ __forceinline__ uint32_t encodeBlockWarp(const uint8_t* __restrict__ in, uint32_t n, uint32_t elem0,
                                                    const StoredPlanes& planes, uint32_t tabAddr, int pb,
                                                    uint32_t stageAddr, uint16_t* stage, Spill& sp,
                                                    uint32_t ringAddr, uint32_t lane, uint32_t& stateOut,
                                                    uint32_t ringBar = 0, uint32_t* ringPhase = nullptr) {
  typedef EncIn<KIND> In;
  constexpr int U = kEncGroupRows;
  constexpr uint32_t WB = In::kWordBytes;
  constexpr uint32_t kGroupBytes = U * 32 * WB;     // 512 B, 1 KiB or 2 KiB
  constexpr uint32_t kChunks = kGroupBytes / 512u;  // 16 B copies per lane and group
  constexpr uint32_t kStride = EncSym<WIDE>::kStride;
  // groups in flight ahead of the one being coded: two, or one in a two-slot ring
  constexpr uint32_t kAhead = In::kRingSlots > 2 ? 2u : 1u;
  static_assert(In::kRingSlots >= 2 && (!TMA || kAhead == 2), "");
  static_assert(!TMA || !isEfKind(KIND), "the EF kinds write their ring slots: cp.async ring only");
  constexpr bool kSparse = isSparseKind(KIND);
  uint32_t state = kStateMin;
  uint32_t wa = stageAddr;
  const EncRegs rc = makeEncRegs(tabAddr, pb);
  const uint32_t fullRows = n >> 5;
  uint32_t r = 0;
  sp.spilled = 0;
  uint32_t pcur = 0;  // sparse kinds: plane offset of the block's next kept byte
  if constexpr (kSparse) pcur = __ldcg(planes.table + (elem0 >> 12));
  [[maybe_unused]] const uint32_t plo = pcur;  // sparse fp32: the block's first kept word, and the warp's run
  [[maybe_unused]] const uint32_t run = ringAddr + EncIn<kKindF32S>::kRingGroupBytes;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) == 0) {
    const uint32_t groups = fullRows / U;
    if (TMA) {
      // input rows arrive by TMA bulk copies (cp.async.bulk, one instruction of one lane per group of
      // 16 rows) into a ring of slots, each with its own mbarrier, two groups ahead of the coder
      auto issue = [&](uint32_t g, uint32_t slot) {
        if (lane == 0) {
          mbarExpectTx(ringBar + 8u * slot, kGroupBytes);
          bulkLoad(ringAddr + slot * kGroupBytes, in + (size_t)g * kGroupBytes, kGroupBytes, ringBar + 8u * slot);
        }
      };
      if (lane == 0) fenceProxyAsync();  // the ring was last touched through the generic proxy
      if (groups > 0) issue(0, 0);
      if (groups > 1) issue(1, 1);
      uint32_t slot = 0, slotNext = 2 % In::kRingSlots, phases = *ringPhase;
      for (uint32_t k = 0; k < groups; ++k) {
        __syncwarp();  // every lane is done with the group that last sat in slotNext
        if (k + 2 < groups) issue(k + 2, slotNext);
        if (sp.area && wa - stageAddr > sp.limitBytes) spillOut(sp, stageAddr, stage, wa, lane);
        mbarWait(ringBar + 8u * slot, (phases >> slot) & 1u);
        phases ^= 1u << slot;
        const uint32_t slotAddr = ringAddr + slot * kGroupBytes;
        if constexpr (KIND == kKindF32S)
          In::storeGroup(slotAddr, planes, pcur, plo, run, lane);
        else if constexpr (kSparse)
          In::storeGroup(slotAddr, planes, pcur, lane);
        else if (KIND != kKindBytes)
          In::storeGroup(slotAddr, planes, elem0 + k * (U * 32), lane);
        encodeGroup<WIDE, KIND>(state, slotAddr + lane * WB, rc, wa);
        slot = slot + 1 == In::kRingSlots ? 0u : slot + 1;
        slotNext = slotNext + 1 == In::kRingSlots ? 0u : slotNext + 1;
      }
      *ringPhase = phases;
    } else {
      // input rows stream through the cp.async ring, two groups ahead of the encoder
      const uint8_t* src = in + lane * 16u;
      const uint32_t dst = ringAddr + lane * 16u;
      auto issue = [&](uint32_t g, uint32_t slot) {
#pragma unroll
        for (uint32_t c = 0; c < kChunks; ++c)
          cpAsync16(dst + slot * kGroupBytes + c * 512u, src + (size_t)g * kGroupBytes + c * 512u);
      };
      if (groups > 0) issue(0, 0);
      cpAsyncCommit();
      if (kAhead > 1) {
        if (groups > 1) issue(1, 1);
        cpAsyncCommit();
      }
      uint32_t slot = 0, slotNext = kAhead % In::kRingSlots;
      for (uint32_t k = 0; k < groups; ++k) {
        if (sp.area && wa - stageAddr > sp.limitBytes) spillOut(sp, stageAddr, stage, wa, lane);
        cpAsyncWait<kAhead - 1>();  // group k has landed (group k + 1 may still be in flight)
        // one warp barrier does both jobs: every lane sees group k, and every lane is done reading group
        // k - 1, whose ring slot the request below overwrites
        __syncwarp();
        if (k + kAhead < groups) issue(k + kAhead, slotNext);
        cpAsyncCommit();
        const uint32_t slotAddr = ringAddr + slot * kGroupBytes;
        if constexpr (KIND == kKindF32S)
          In::storeGroup(slotAddr, planes, pcur, plo, run, lane);
        else if constexpr (kSparse)
          In::storeGroup(slotAddr, planes, pcur, lane);
        else if (KIND != kKindBytes)
          In::storeGroup(slotAddr, planes, elem0 + k * (U * 32), lane);
        encodeGroup<WIDE, KIND>(state, slotAddr + lane * WB, rc, wa);
        slot = slot + 1 == In::kRingSlots ? 0u : slot + 1;
        slotNext = slotNext + 1 == In::kRingSlots ? 0u : slotNext + 1;
      }
    }
    if constexpr (KIND == kKindF32S) In::flushTail(planes, pcur, plo, run, lane);
    r = groups * U;
  }
  // remaining rows (fewer than U, or all of them when the input is not 16 B aligned): every U rows
  // the same spill check as above
  uint32_t e = r * 32u + lane;
  for (uint32_t j = 0; r < fullRows; ++r, ++j, e += 32) {
    if (sp.area && (j % U) == 0 && wa - stageAddr > sp.limitBytes) spillOut(sp, stageAddr, stage, wa, lane);
    const auto w = encLoadWord<KIND>(in, e, planes, elem0);
    if constexpr (kSparse)
      In::storeRow(planes, pcur, w, true, rc.ltMask);
    else
      In::storeScalar(planes, elem0 + e, w);
    encodeStep<WIDE>(state, In::template tabOffsetOf<kStride>(w), rc, wa);
  }
  const uint32_t rem = n & 31u;
  if (rem) {
    if (sp.area && wa - stageAddr > sp.limitBytes) spillOut(sp, stageAddr, stage, wa, lane);
    const bool valid = lane < rem;
    const auto w = valid ? encLoadWord<KIND>(in, e, planes, elem0) : 0u;
    if constexpr (kSparse)
      In::storeRow(planes, pcur, w, valid, rc.ltMask);
    else if (valid)
      In::storeScalar(planes, elem0 + e, w);
    encodeStepPartial<WIDE>(valid, state, In::template tabOffsetOf<kStride>(w), rc, wa);
  }
  stateOut = state;
  return sp.spilled + ((wa - stageAddr) >> 1);
}

// Pads the block's stream to a multiple of 8 words and copies it to `dst` (global, 16 B aligned).
__device__ __forceinline__ void placeStream(uint16_t* stage, Spill& sp, uint32_t words, uint32_t padded,
                                            uint8_t* dst8, uint32_t lane) {
  const uint32_t local = words - sp.spilled;        // words still in the slot
  if (local + lane < padded - sp.spilled) stage[local + lane] = 0;  // pad < 8 words
  __syncwarp();
  uint4* dst = reinterpret_cast<uint4*>(dst8);
  if (sp.spilled) {
    const uint4* g = reinterpret_cast<const uint4*>(sp.area);
    for (uint32_t i = lane; i < sp.spilled / 8u; i += 32u) dst[i] = __ldcg(g + i);
    dst += sp.spilled / 8u;
  }
  const uint4* src = reinterpret_cast<const uint4*>(stage);
  for (uint32_t i = lane; i < (padded - sp.spilled) / 8u; i += 32u) dst[i] = src[i];
}

constexpr unsigned long long kFlagAgg = 1ull << 32;
constexpr unsigned long long kFlagPrefix = 2ull << 32;

// Exclusive prefix of the per-ticket totals of this member (decoupled
// look-back, one warp).  first = first ticket of the member.
__device__ __forceinline__ uint32_t lookbackWarp(volatile unsigned long long* desc, uint32_t ticket,
                                                 uint32_t first, uint32_t lane) {
  uint32_t base = 0;
  int64_t idx = (int64_t)ticket - 1;
  while (idx >= (int64_t)first) {
    const int64_t mine = idx - lane;
    unsigned long long d = kFlagPrefix;  // lanes before `first`: neutral, terminates the walk
    if (mine >= (int64_t)first) {
      do { d = desc[mine]; } while ((d >> 32) == 0ull);
    }
    const bool isPrefix = (d >> 32) == 2ull;
    const uint32_t pmask = __ballot_sync(0xffffffffu, isPrefix);
    // lanes 0..firstPrefixLane contribute (lane 0 is the nearest predecessor)
    const uint32_t stop = pmask ? (uint32_t)__ffs((int)pmask) - 1u : 31u;
    uint32_t v = lane <= stop ? (uint32_t)d : 0u;
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    base += v;
    if (pmask) break;
    idx -= 32;
  }
  return base;
}

// dynamic shared memory per warp: [table 2 KiB][input ring 2 KiB][staging slot]
__host__ __device__ constexpr uint32_t encWarpSmem(int pb, int kind) {
  return encTabBytes(kind) + encRingBytes(kind) + maxBlockWords(pb) * 2u;
}

// Sparse kinds: plane, table and keep flag of a member's archive from the header line the statistics pass
// wrote; returns the bytes in front of the ANS archive.
// (sparse fp32: `non` is the u16 plane and `non1` the u8 plane)
template <int KIND>
__device__ __forceinline__ uint32_t sparsePlanes(void* out, uint32_t size, StoredPlanes& pl) {
  uint8_t* a = static_cast<uint8_t*>(out);
  const uint4 h1 = __ldcg(reinterpret_cast<const uint4*>(a) + 1);  // S, esc
  pl.table = reinterpret_cast<const uint32_t*>(a + kSparseHeaderBytes);
  pl.non = a + kSparseHeaderBytes + sparseTableBytes<uint32_t>(size);
  pl.keepAll = (h1.y >> 16) == 0u ? 1u : 0u;
  __builtin_assume(__isGlobal(pl.non));
  __builtin_assume(__isGlobal(pl.table));
  if constexpr (KIND == kKindF32S) {
    pl.non1 = pl.non + 2u * roundUp(h1.x, 8u);
    __builtin_assume(__isGlobal(pl.non1));
    return sparseExtraBytes<uint32_t>(KIND, size, h1.x);
  } else {
    return sparseExtraBytes<uint32_t>(size, h1.x);
  }
}

// The body of encodeKernel; `ef` is the EF kinds' residual table (nullptr for every other kind)
template <int KIND>
__device__ __forceinline__ void encodeCanonical(const EncodeScratch& sc, int pb, bool useChecksum, uint32_t numMembers,
                                                uint32_t totalTickets, uint32_t* __restrict__ outSize,
                                                const EfMembers* ef) {
  constexpr int kind = KIND;
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t t = threadIdx.x, lane = t & 31u;
  // shuffle => provably warp-uniform (no divergence check around the votes in the hot loop)
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  uint8_t* mine = smem + (size_t)warp * encWarpSmem(pb, kind);
  uint4* myTab = reinterpret_cast<uint4*>(mine);
  const uint32_t tabAddr = smemAddr(mine);
  const uint32_t ringAddr = tabAddr + encTabBytes(kind);
  uint16_t* myStage = reinterpret_cast<uint16_t*>(mine + encTabBytes(kind) + encRingBytes(kind));
  const uint32_t stageAddr = smemAddr(myStage);
  volatile unsigned long long* desc = sc.lookback;
  uint32_t curMember = 0xffffffffu;

  for (;;) {
    uint32_t ticket = 0;
    if (lane == 0) ticket = atomicAdd(sc.ticket, 1u);
    ticket = __shfl_sync(0xffffffffu, ticket, 0);
    if (ticket >= totalTickets) break;
    // member m with work0[m] <= ticket < work0[m+1]  (uniform binary search, L1-cached)
    uint32_t lo = 0, hi = numMembers;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(&sc.members[mid].work0) <= ticket) lo = mid; else hi = mid;
    }
    const uint32_t m = lo;
    const MemberDesc md = sc.members[m];
    const uint32_t size = md.size;
    const uint32_t nb = divUp(size, kBlockBytes);
    const uint32_t block = ticket - md.work0;

    const uint8_t* ansIn;
    uint8_t* ansOut;
    uint32_t extraBytes = 0;
    StoredPlanes planes{nullptr, nullptr, nullptr};
    if constexpr (isEfKind(KIND)) planes.err = efAt(*ef, m);
    ansIn = static_cast<const uint8_t*>(md.in);
    if (kind == kKindBytes) {
      ansOut = static_cast<uint8_t*>(md.out);
    } else if constexpr (isSparseKind(KIND)) {
      extraBytes = sparsePlanes<KIND>(md.out, size, planes);
      ansOut = static_cast<uint8_t*>(md.out) + extraBytes;
    } else {
      extraBytes = kFloatHeaderBytes + floatNonCompBytes(archiveKind(kind), size);
      ansOut = static_cast<uint8_t*>(md.out) + extraBytes;
      planes.non = static_cast<uint8_t*>(md.out) + kFloatHeaderBytes;
      if (kind == kKindF64) {
        planes.non1 = planes.non + floatU16PlaneOffset<uint32_t>(kind, size);
        planes.non2 = planes.non + floatU8PlaneOffset<uint32_t>(kind, size);
        __builtin_assume(__isGlobal(planes.non2));
      } else {
        planes.non1 = planes.non + 2u * roundUp(size, 8u);
      }
      __builtin_assume(__isGlobal(planes.non));
      __builtin_assume(__isGlobal(planes.non1));
    }
    __builtin_assume(__isGlobal(ansIn));
    __builtin_assume(__isGlobal(ansOut));

    if (m != curMember) {
      // this member's encoder table -> my private copy (written by K1's epilogue)
      const uint4* src = sc.table + (size_t)m * tableSlots(KIND);
      if constexpr (isSparseKind(KIND)) {
        for (uint32_t i = lane; i < encTabVecs(false, KIND); i += 32u) myTab[i] = __ldcg(src + i);
      } else {
#pragma unroll
        for (uint32_t i = 0; i < kNumSymbols / 64; ++i) myTab[i * 32 + lane] = __ldcg(src + i * 32 + lane);
      }
      curMember = m;
      __syncwarp();
    }

    // ---- encode the block into my staging slot ----
    const uint32_t start = block * kBlockBytes;
    const uint32_t blockLen = min(kBlockBytes, size - start);
    uint32_t state;
    Spill sp{nullptr, 0u, 0u};  // worst-case sized slot: never spills
    const uint32_t words = encodeBlockWarp<false, KIND, false>(ansIn + (size_t)start * EncIn<KIND>::kWordBytes, blockLen, start, planes,
                                                               tabAddr, pb, stageAddr, myStage, sp, ringAddr, lane, state);
    const uint32_t padded = roundUp(words, 8u);

    // ---- packed offset of this block: look-back over the member's earlier tickets ----
    uint32_t base = 0;
    if (block != 0) {
      if (lane == 0) desc[ticket] = kFlagAgg | padded;
      base = lookbackWarp(desc, ticket, md.work0, lane);
    }
    if (lane == 0) desc[ticket] = kFlagPrefix | (unsigned long long)(base + padded);
    __syncwarp();

    // ---- final placement: states, blockWords, packed stream ----
    uint8_t* pStates = ansOut + kAnsHeaderBytes + kAnsPdfBytes;
    uint8_t* pBlockWords = pStates + 128u * nb;
    uint8_t* pData = pBlockWords + 8u * roundUp(nb, 2u);
    reinterpret_cast<uint32_t*>(pStates)[block * 32u + lane] = state;
    if (lane == 0)
      reinterpret_cast<uint2*>(pBlockWords)[block] = make_uint2((blockLen << 16) | words, base);
    placeStream(myStage, sp, words, padded, pData + 2u * (size_t)base, lane);
    if (block == nb - 1 && lane == 0) {
      // ans/GpuANSEncode.cuh:553-569 header (undefined bits zeroed)
      const uint32_t totalWords = base + padded;
      uint4* h = reinterpret_cast<uint4*>(ansOut);
      h[0] = make_uint4(kAnsMagicVersion, nb, size, totalWords);
      const bool ansChecksum = useChecksum && kind == kKindBytes;
      h[1] = make_uint4((uint32_t)pb | ((ansChecksum ? 1u : 0u) << 4),
                        ansChecksum ? __ldcg(sc.checksum + m) : 0u, 0u, 0u);
      if (nb & 1u) reinterpret_cast<uint2*>(pBlockWords)[nb] = make_uint2(0u, 0u);
      if (outSize) outSize[m] = ansOverhead(nb) + 2u * totalWords + extraBytes;
    }
    __syncwarp();  // staging and ring are reused by the next ticket
  }
}

template <int KIND>
__global__ void encodeKernel(EncodeScratch sc, int pb, bool useChecksum,
                             uint32_t numMembers, uint32_t totalTickets,
                             uint32_t* __restrict__ outSize) {
  encodeCanonical<KIND>(sc, pb, useChecksum, numMembers, totalTickets, outSize, nullptr);
}

// the canonical K2 of the EF kinds: encodeKernel plus the residual table
template <int KIND>
__global__ void encodeKernelEf(EncodeScratch sc, const __grid_constant__ EfMembers ef, int pb, bool useChecksum,
                               uint32_t numMembers, uint32_t totalTickets, uint32_t* __restrict__ outSize) {
  encodeCanonical<KIND>(sc, pb, useChecksum, numMembers, totalTickets, outSize, &ef);
}

// ---------------------------------------------------------------------------
// K2, default flavour: no inter-block dependency at all.  The archive format
// addresses every block's stream through blockWords[k].y, so streams may sit in
// the data section in ANY order; here a block takes its place with one
// atomicAdd on the member's word counter when it has been encoded.  Sizes, the
// pdf, every lane state and every stream are identical to the canonical
// encoder's (and to the reference's); only the ORDER of the streams inside the
// data section (and hence the .y offsets) depends on completion order.  The
// ordered, byte-for-byte canonical layout is available as option
// "encode_canonical" (encodeKernel above; c3 encode 360 vs 270 us on an H100 at
// 700 W: its warps wait on the look-back descriptors of slower predecessors).
//
// Work split is static: CTA c owns a contiguous range of flat blocks, walks it
// member by member (one shared table load per member) and its warps stride
// over the blocks of the member.
// ---------------------------------------------------------------------------
__host__ __device__ constexpr uint32_t encFastWarpSmem(uint32_t slotWords, int kind) {
  return encRingBytes(kind) + slotWords * 2u;  // ring + staging
}

// Per-warp view of the CTA's dynamic shared memory: [input ring | staging slot] per warp.
#ifndef DGB_ENC_TMA
#define DGB_ENC_TMA 0
#endif
// input rows by per-lane cp.async (0, default) or by TMA bulk copy (1).  The per-lane copy is the default: one lane
// issuing the bulk copy and 32 lanes polling the mbarrier cost more issue slots than the two LDGSTS per lane they replace.
constexpr bool kEncTma = DGB_ENC_TMA != 0;

struct WarpSmem {
  uint32_t ringAddr, stageAddr;
  uint16_t* stage;
  Spill sp;
  uint32_t ringBar;    // shared address of this warp's ring mbarriers (one per slot)
  uint32_t ringPhase;  // bit s = parity the next wait on slot s expects
};
__device__ __forceinline__ WarpSmem warpSmem(const EncodeScratch& sc, uint8_t* smem, uint32_t warp, uint32_t W,
                                             uint32_t slotWords, int pb, int kind, uint32_t spillWarpBase,
                                             unsigned long long (*ringBars)[4]) {
  WarpSmem ws;
  uint8_t* mine = smem + (size_t)warp * encFastWarpSmem(slotWords, kind);
  ws.ringAddr = smemAddr(mine);
  ws.sp.area = slotWords < maxBlockWords(pb)
                   ? reinterpret_cast<uint16_t*>(sc.spill) + (size_t)(spillWarpBase + blockIdx.x * W + warp) * maxBlockWords(pb)
                   : nullptr;
  ws.sp.limitBytes = (slotWords - kEncGroupRows * 32u - 8u) * 2u;  // a group emits at most 16*32 words
  ws.sp.spilled = 0;
  ws.stage = reinterpret_cast<uint16_t*>(mine + encRingBytes(kind));
  ws.stageAddr = smemAddr(ws.stage);
  ws.ringBar = smemAddr(&ringBars[warp][0]);  // static shared memory: the dynamic region is reused by statistics items
  ws.ringPhase = 0;
  if (kEncTma && (threadIdx.x & 31u) == 0) {
    for (uint32_t k = 0; k < 4; ++k) mbarInit(ws.ringBar + 8u * k, 1);
  }
  return ws;
}

// Loads member m's encoder table (written by the statistics epilogue) into the CTA's table slot.
template <bool WIDE, int KIND>
__device__ __forceinline__ void loadTable(const EncodeScratch& sc, uint4* sTab, uint32_t m) {
  const uint4* src = sc.table + (size_t)m * tableSlots(KIND);
  for (uint32_t i = threadIdx.x; i < encTabVecs(WIDE, KIND); i += blockDim.x) sTab[i] = __ldcg(src + i);
}

// Warps of the CTA encode blocks [first, last) of member m (block k by warp (k - first) % W): the
// 32-lane rANS state machine per block, then the block takes its place in the archive's data
// section with one 64-bit atomic.
template <bool WIDE, int KIND>
__device__ __forceinline__ void encodeMemberBlocks(const EncodeScratch& sc, const MemberDesc& md, uint32_t m,
                                                   uint32_t first, uint32_t last, int pb,
                                                   bool useChecksum, uint32_t tabAddr, WarpSmem& ws,
                                                   uint32_t warp, uint32_t W, uint32_t lane,
                                                   uint32_t* __restrict__ outSize, float* err = nullptr) {
  constexpr int kind = KIND;
  const uint32_t size = md.size;
  const uint32_t nb = divUp(size, kBlockBytes);
  const uint8_t* ansIn;
  uint8_t* ansOut;
  uint32_t extraBytes = 0;
  StoredPlanes planes{nullptr, nullptr, nullptr};
  if constexpr (isEfKind(KIND)) planes.err = err;
  ansIn = static_cast<const uint8_t*>(md.in);
  if (kind == kKindBytes) {
    ansOut = static_cast<uint8_t*>(md.out);
  } else if constexpr (isSparseKind(KIND)) {
    extraBytes = sparsePlanes<KIND>(md.out, size, planes);
    ansOut = static_cast<uint8_t*>(md.out) + extraBytes;
  } else {
    extraBytes = kFloatHeaderBytes + floatNonCompBytes(archiveKind(kind), size);
    ansOut = static_cast<uint8_t*>(md.out) + extraBytes;
    planes.non = static_cast<uint8_t*>(md.out) + kFloatHeaderBytes;
    if (kind == kKindF64) {
      planes.non1 = planes.non + floatU16PlaneOffset<uint32_t>(kind, size);
      planes.non2 = planes.non + floatU8PlaneOffset<uint32_t>(kind, size);
      __builtin_assume(__isGlobal(planes.non2));
    } else {
      planes.non1 = planes.non + 2u * roundUp(size, 8u);
    }
    __builtin_assume(__isGlobal(planes.non));
    __builtin_assume(__isGlobal(planes.non1));
  }
  __builtin_assume(__isGlobal(ansIn));
  __builtin_assume(__isGlobal(ansOut));
  uint8_t* pStates = ansOut + kAnsHeaderBytes + kAnsPdfBytes;
  uint8_t* pBlockWords = pStates + 128u * nb;
  uint8_t* pData = pBlockWords + 8u * roundUp(nb, 2u);

  for (uint32_t block = first + warp; block < last; block += W) {
    const uint32_t start = block * kBlockBytes;
    const uint32_t blockLen = min(kBlockBytes, size - start);
    uint32_t state;
    const uint32_t words = encodeBlockWarp<WIDE, KIND, kEncTma && !isEfKind(KIND)>(ansIn + (size_t)start * EncIn<KIND>::kWordBytes, blockLen, start,
                                                                planes, tabAddr, pb, ws.stageAddr, ws.stage, ws.sp, ws.ringAddr,
                                                                lane, state, ws.ringBar, &ws.ringPhase);
    const uint32_t padded = roundUp(words, 8u);
    // take a place in the data section: one 64-bit atomic hands out the word offset (low half)
    // and counts finished blocks (high half), so no fence is needed to order the two
    unsigned long long old = 0;
    if (lane == 0) old = atomicAdd(sc.allocDone + m, (1ull << 32) | (unsigned long long)padded);
    reinterpret_cast<uint32_t*>(pStates)[block * 32u + lane] = state;
    old = __shfl_sync(0xffffffffu, old, 0);
    const uint32_t base = (uint32_t)old;
    if (lane == 0)
      reinterpret_cast<uint2*>(pBlockWords)[block] = make_uint2((blockLen << 16) | words, base);
    placeStream(ws.stage, ws.sp, words, padded, pData + 2u * (size_t)base, lane);
    // the block that takes the last place knows the member's total and writes the header
    if (lane == 0 && (uint32_t)(old >> 32) == nb - 1u) {
      const uint32_t totalWords = base + padded;
      uint4* h = reinterpret_cast<uint4*>(ansOut);
      h[0] = make_uint4(kAnsMagicVersion, nb, size, totalWords);
      const bool ansChecksum = useChecksum && kind == kKindBytes;
      h[1] = make_uint4((uint32_t)pb | ((ansChecksum ? 1u : 0u) << 4),
                        ansChecksum ? __ldcg(sc.checksum + m) : 0u, 0u, 0u);
      if (nb & 1u) reinterpret_cast<uint2*>(pBlockWords)[nb] = make_uint2(0u, 0u);
      if (outSize) outSize[m] = ansOverhead(nb) + 2u * totalWords + extraBytes;
    }
    __syncwarp();  // staging and ring are reused by the next block
  }
}

// The body of encodeKernelFast; `ef` is the EF kinds' residual table (nullptr for every other kind)
template <bool WIDE, int KIND>
__device__ __forceinline__ void encodeFast(const EncodeScratch& sc, const InlineMembers& im, int pb, bool useChecksum,
                                           uint32_t numMembers, uint32_t blockBegin, uint32_t blockEnd,
                                           uint32_t slotWords, uint32_t spillWarpBase, uint32_t* __restrict__ outSize,
                                           const EfMembers* ef) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ __align__(16) uint4 sTab[encTabVecs(WIDE, KIND)];  // static: constant base for the hot LDS
  __shared__ uint32_t sMember;
  const uint32_t t = threadIdx.x, lane = t & 31u;
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  const uint32_t W = blockDim.x >> 5;
  __shared__ __align__(8) unsigned long long sRingBar[8][4];
  WarpSmem ws = warpSmem(sc, smem, warp, W, slotWords, pb, KIND, spillWarpBase, sRingBar);
  if (kEncTma) {
    fenceBarrierInit();
    __syncthreads();
  }
  const uint32_t tabAddr = smemAddr(sTab);

  const uint64_t g = gridDim.x, span = blockEnd - blockBegin;
  uint32_t cur = blockBegin + (uint32_t)(span * blockIdx.x / g);
  const uint32_t end = blockBegin + (uint32_t)(span * (blockIdx.x + 1) / g);

  while (cur < end) {
    if (t == 0) {
      uint32_t lo = 0, hi = numMembers;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (memberWork0(im, sc.members, mid) <= cur) lo = mid; else hi = mid;
      }
      sMember = lo;
    }
    __syncthreads();
    const uint32_t m = sMember;
    const MemberDesc md = memberAt(im, sc.members, m);
    const uint32_t nb = divUp(md.size, kBlockBytes);
    const uint32_t memberEnd = min(end, md.work0 + nb);
    loadTable<WIDE, KIND>(sc, sTab, m);
    __syncthreads();
    if constexpr (isEfKind(KIND))
      encodeMemberBlocks<WIDE, KIND>(sc, md, m, cur - md.work0, memberEnd - md.work0, pb, useChecksum, tabAddr, ws,
                                     warp, W, lane, outSize, efAt(*ef, m));
    else
      encodeMemberBlocks<WIDE, KIND>(sc, md, m, cur - md.work0, memberEnd - md.work0, pb, useChecksum, tabAddr, ws,
                                     warp, W, lane, outSize);
    cur = memberEnd;
    __syncthreads();  // table is replaced for the next member
  }
}

template <bool WIDE, int KIND>
__global__ void
encodeKernelFast(EncodeScratch sc, const __grid_constant__ InlineMembers im, int pb, bool useChecksum,
                                 uint32_t numMembers, uint32_t blockBegin, uint32_t blockEnd,
                                 uint32_t slotWords, uint32_t spillWarpBase,
                                 uint32_t* __restrict__ outSize) {
  encodeFast<WIDE, KIND>(sc, im, pb, useChecksum, numMembers, blockBegin, blockEnd, slotWords, spillWarpBase, outSize,
                         nullptr);
}

// K2 of the EF kinds: encodeKernelFast plus the residual table
template <bool WIDE, int KIND>
__global__ void
encodeKernelFastEf(EncodeScratch sc, const __grid_constant__ InlineMembers im, const __grid_constant__ EfMembers ef,
                   int pb, bool useChecksum, uint32_t numMembers, uint32_t blockBegin, uint32_t blockEnd,
                   uint32_t slotWords, uint32_t spillWarpBase, uint32_t* __restrict__ outSize) {
  encodeFast<WIDE, KIND>(sc, im, pb, useChecksum, numMembers, blockBegin, blockEnd, slotWords, spillWarpBase, outSize,
                         &ef);
}

// ---------------------------------------------------------------------------
// Fused single-launch encoder (option encode_fused=1; slower than the two-kernel path, c3 encode 313 vs 270 us
// on an H100 at 700 W, DESIGN.md section 4, so not the default).  One persistent grid; every CTA picks, at each step, one
// of two kinds of work from two global counters:
//   * a STATISTICS item  = one slab of one member (the body of K1 above: histogram (+ split, +
//     checksum); the CTA that finishes a member normalises, publishes pdf + table and sets the
//     member's `ready` flag), or
//   * an ENCODE chunk    = a run of 4 KiB blocks of one member (the body of K2), which needs the
//     member's flag.
// Chunks are claimed in member order, and a CTA whose chunk is not ready yet works on statistics
// items (which have no dependencies) instead of waiting, so the HBM-latency-bound statistics pass
// and the issue-bound coder share every SM and balance themselves; one CTA in `statsEvery` prefers
// statistics so that the tables stay ahead of the coders.  Progress never depends on co-residency:
// a claimed item is always held by a running CTA, and the only wait (chunk claimed, member not
// ready, no statistics left to claim) is for items other running CTAs hold.
// The reference runs 7-10 kernels for this (SURVEY.md 3.1); its README lists a single cooperative
// kernel as a next step (README.md:103).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ldAcquire(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void stRelease(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

enum FusedAct : uint32_t { kActExit = 0, kActWait = 1, kActStats = 2, kActEncode = 3 };
constexpr uint32_t kNoChunk = 0xffffffffu;

template <int KIND, bool WIDE, bool STAGED>
__global__ void __launch_bounds__(kStatsThreads, 4)
encodeFusedKernel(EncodeScratch sc, const uint32_t* __restrict__ histogramGiven, int pb, bool useChecksum,
                  uint32_t numMembers, uint32_t totalItems, uint32_t totalChunks, uint32_t slabVecs,
                  uint32_t chunkBlocks, uint32_t slotWords, uint32_t statsEvery,
                  uint32_t* __restrict__ outSize) {
  // dynamic shared memory: per-warp [ring | staging slot] while encoding, the per-warp histograms
  // while a statistics item runs (never both: the roles alternate between CTA-wide barriers)
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ __align__(16) uint4 sTab[WIDE ? kNumSymbols : kNumSymbols / 2];
  __shared__ uint32_t sCtl[8];
  __shared__ __align__(8) unsigned long long sStageBar;
  uint32_t (*sHist)[kNumSymbols] = reinterpret_cast<uint32_t (*)[kNumSymbols]>(smem);
  const uint32_t t = threadIdx.x, lane = t & 31u;
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  constexpr uint32_t W = kStatsThreads / 32;
  // statistics items: histograms in the first 8 KiB of the dynamic region, the slab's landing
  // buffer in the rest (the host sizes slabVecs to fit)
  uint32_t stagePhase = 0;
  StatsStage stage;
  stage.buf = reinterpret_cast<uint4*>(smem + sizeof(uint32_t) * kStatsWarps * kNumSymbols);
  stage.bar = smemAddr(&sStageBar);
  stage.phase = &stagePhase;
  if (STAGED) {
    if (t == 0) mbarInit(stage.bar, 1);
    fenceBarrierInit();
    __syncthreads();
  }
  __shared__ __align__(8) unsigned long long sRingBar[8][4];
  WarpSmem ws = warpSmem(sc, smem, warp, W, slotWords, pb, KIND, 0u, sRingBar);
  if (kEncTma) {
    fenceBarrierInit();
    __syncthreads();
  }
  const uint32_t tabAddr = smemAddr(sTab);
  const bool preferStats = statsEvery != 0u && (blockIdx.x % statsEvery) == 0u;

  // claim state (meaningful in thread 0; the decision is broadcast through sCtl)
  uint32_t chunk = kNoChunk, chunkMember = 0, itemMember = 0;
  bool chunksLeft = totalChunks != 0u, statsLeft = totalItems != 0u;
  uint32_t tabMember = 0xffffffffu;

  for (;;) {
    if (t == 0) {
      uint32_t act = kActWait, arg = 0, m = 0;
      uint32_t item = 0xffffffffu;
      if (preferStats && statsLeft) {
        item = atomicAdd(sc.ticket + 0, 1u);
        if (item >= totalItems) { statsLeft = false; item = 0xffffffffu; }
      }
      if (item == 0xffffffffu) {
        if (chunk == kNoChunk && chunksLeft) {
          chunk = atomicAdd(sc.ticket + 1, 1u);
          if (chunk >= totalChunks) { chunk = kNoChunk; chunksLeft = false; }
        }
        if (chunk != kNoChunk) {
          while (__ldg(&sc.workIdx[chunkMember + 1].y) <= chunk) ++chunkMember;  // claims only grow
          if (ldAcquire(sc.ready + chunkMember) != 0u) { act = kActEncode; arg = chunk; m = chunkMember; chunk = kNoChunk; }
        }
        if (act == kActWait && statsLeft) {
          item = atomicAdd(sc.ticket + 0, 1u);
          if (item >= totalItems) { statsLeft = false; item = 0xffffffffu; }
        }
        if (act == kActWait && item == 0xffffffffu && chunk == kNoChunk) act = kActExit;  // nothing left anywhere
      }
      if (item != 0xffffffffu) {
        while (__ldg(&sc.workIdx[itemMember + 1].x) <= item) ++itemMember;
        act = kActStats; arg = item; m = itemMember;
      }
      sCtl[0] = act; sCtl[1] = arg; sCtl[2] = m;
    }
    __syncthreads();
    const uint32_t act = sCtl[0], arg = sCtl[1], m = sCtl[2];
    if (act == kActExit) break;
    if (act == kActStats) {
      const uint2 w0 = __ldg(&sc.workIdx[m]), w1 = __ldg(&sc.workIdx[m + 1]);
      bool finished;
      if (KIND == kKindBytes) {
        finished = statsBytesItem<STAGED>(sc, sHist, histogramGiven, pb, useChecksum, slabVecs, sc.members[m], m, arg - w0.x,
                                          w1.x - w0.x, outSize, stage);
      } else {
        finished = statsFloatItem<KIND == kKindBytes ? DGB_FLOAT16 : KIND, STAGED>(
            sc, sHist, pb, useChecksum, slabVecs, sc.members[m], m, arg - w0.x, w1.x - w0.x, outSize, stage);
      }
      if (finished) {
        // table, pdf and (through the ticket chain) every comp / stored byte of the member are
        // visible before the flag
        __threadfence();
        __syncthreads();
        if (t == 0) stRelease(sc.ready + m, 1u);
      }
    } else if (act == kActEncode) {
      const MemberDesc md = sc.members[m];
      if (tabMember != m) {
        loadTable<WIDE, KIND>(sc, sTab, m);
        tabMember = m;
        __syncthreads();
      }
      const uint32_t nb = divUp(md.size, kBlockBytes);
      const uint32_t first = (arg - __ldg(&sc.workIdx[m].y)) * chunkBlocks;
      encodeMemberBlocks<WIDE, KIND>(sc, md, m, first, min(nb, first + chunkBlocks), pb, useChecksum, tabAddr, ws,
                                     warp, W, lane, outSize);
    } else {
      __nanosleep(256);
    }
    __syncthreads();  // sCtl, the table slot and the dynamic region are reused by the next step
  }
}

struct ScratchPlan {
  size_t members, workIdx, uploadEnd, zeroBegin, hist, histDone, checksum, ticket, allocDone, ready, zeroEnd,
      lookback, lookbackEnd, table, spill, total;
  uint32_t spillWarps;
  uint32_t blockZerosOff;
};

// Encoder warps that may need a spill slot (one slot = the worst-case stream of one block): never
// more than the device can hold resident (64 warps per SM), never more than the batch has work
// for, so small batches get small scratch (the reference's scratch scales with the batch too).
uint32_t spillWarpBound(uint32_t n, uint64_t totalBlocks) {
  const uint64_t resident = 64ull * (uint64_t)smCount();
  const uint64_t work = 8ull * ((uint64_t)n * 2ull + totalBlocks);  // 8 warps per CTA, <= items + chunks CTAs
  return (uint32_t)std::min(resident, work);
}

ScratchPlan planScratch(int kind, uint32_t n, uint32_t maxSize, uint32_t totalTickets, uint32_t spillWarps) {
  ScratchPlan p{};
  size_t o = 0;
  // uploaded together: member descriptors, then the fused launch's work index
  p.members = o; o += sizeof(MemberDesc) * (size_t)n;
  o = (o + 15) & ~size_t(15);
  p.workIdx = o; o += sizeof(uint2) * ((size_t)n + 1);
  p.uploadEnd = o;
  o = alignUp256(o);
  p.zeroBegin = o;
  p.hist = o; o = alignUp256(o + sizeof(uint32_t) * kNumSymbols * (size_t)n);
  p.histDone = o; o = alignUp256(o + sizeof(uint32_t) * (size_t)n);
  p.checksum = o; o = alignUp256(o + sizeof(uint32_t) * (size_t)n);
  p.ticket = o; o = alignUp256(o + 16);
  p.allocDone = o; o = alignUp256(o + sizeof(unsigned long long) * (size_t)n);
  // sparse kinds: [2n] +0 / -0 words per member, then [totalTickets] +-0 words per block (zeroCounts, blockZeros)
  p.blockZerosOff = isSparseKind(kind) ? roundUp(2u * n, 64u) : 0u;
  p.ready = o; o = alignUp256(o + sizeof(uint32_t) * (isSparseKind(kind) ? (size_t)p.blockZerosOff + totalTickets : (size_t)n));
  p.zeroEnd = o;
  // look-back descriptors: canonical (ordered) layout only; cleared only then
  p.lookback = o; o = alignUp256(o + sizeof(unsigned long long) * (size_t)totalTickets);
  p.lookbackEnd = o;
  p.table = o; o = alignUp256(o + sizeof(uint4) * tableSlots(kind) * (size_t)n);
  p.spillWarps = spillWarps;
  p.spill = o; o = alignUp256(o + (size_t)spillWarps * maxBlockWords(11) * 2u);
  p.total = o;
  return p;
}

uint32_t ticketsFor(uint32_t size) { return divUp(size, kBlockBytes); }

// withKind plus the encoder-only narrowing kinds (their kernels are instantiated here and nowhere else)
template <class F>
int withEncodeKind(int kind, F&& f) {
  switch (kind) {
    case kKindF32toF16: return f(IntC<kKindF32toF16>{});
    case kKindF32toBF16: return f(IntC<kKindF32toBF16>{});
    case kKindF32toF16EF: return f(IntC<kKindF32toF16EF>{});
    case kKindF32toBF16EF: return f(IntC<kKindF32toBF16EF>{});
    default: return withKind(kind, f);
  }
}

// fp64 staging slot of the fast coder: the smallest the coder allows.  The fp64 ring is 12 KiB per warp, and a
// smaller slot is what lets a second 8-warp CTA fit on an SM; fp64's coded byte (the high exponent byte)
// compresses so well that a block rarely emits more than the slot holds (those that do spill, see Spill).
constexpr uint32_t kEncSlotWordsF64 = kEncGroupRows * 32u + 264u;

}  // namespace

size_t encodeTempBytes(int kind, uint32_t n, uint32_t maxSize) {
  // worst case over warps-per-CTA choices: tickets with W = 1
  const uint64_t tickets = (uint64_t)n * divUp(maxSize, kBlockBytes);
  if (tickets > 0xffffffffull) return ~size_t(0);
  return planScratch(kind, n, maxSize, (uint32_t)tickets, spillWarpBound(n, tickets)).total + 256;
}

int encodeBatch(int kind, void* temp, size_t tempBytes, int pb, bool checksum, uint32_t n,
                const HostMember* members, const uint32_t* histogram_dev, uint32_t* outSize_dev,
                cudaStream_t stream, float* const* err) {
  if (n == 0) return DGB_OK;
  if (pb < 9 || pb > 11) return DGB_ERR_INVALID_ARG;
  if (kind != kKindBytes && histogram_dev) return DGB_ERR_INVALID_ARG;
  if (isEfKind(kind) != (err != nullptr)) return DGB_ERR_INVALID_ARG;
  const Options opt = options();  // one snapshot per call
  const uint32_t W = (uint32_t)std::max(1, std::min(opt.encode_warps, 8));  // warps per CTA (two-kernel path)
  const uint32_t elemBytes = wordBytes(kind);
  const bool canonical = opt.encode_canonical != 0;
  // the sparse and the narrowing kinds have neither the fused launch nor the staged statistics kernel: those
  // options run the default kernels for them (INTEGRATION.md section 4)
  const bool defaultOnly = isSparseKind(kind) || isNarrowKind(kind);
  const bool fused = !canonical && opt.encode_fused != 0 && !defaultOnly;
  // staging slot of the fast / fused encoder (spills to global scratch when a block needs more)
  uint32_t slotWords = opt.encode_slot_words > 0 ? (uint32_t)opt.encode_slot_words
                                                 : (kind == kKindBytes ? 2304u : (kind == kKindF64 ? kEncSlotWordsF64 : 1536u));
  slotWords = std::max<uint32_t>(roundUp(slotWords, 8u), kEncGroupRows * 32u + 264u);
  slotWords = std::min(slotWords, maxBlockWords(pb));
  // statistics slab: the two-kernel path streams it through registers; the fused launch lands it in
  // the part of the CTA's dynamic shared memory that the histograms do not use (TMA bulk copy)
  const bool staged = fused && opt.fused_stage != 0;
  uint32_t slabVecs = (uint32_t)std::max(1, opt.hist_slab_kb) * 1024u / 16u;
  if (staged) {
    const uint32_t stageBytes = (kStatsThreads / 32) * encFastWarpSmem(slotWords, kind) - (uint32_t)sizeof(uint32_t) * kStatsWarps * kNumSymbols;
    slabVecs = std::max(1u, std::min(slabVecs, stageBytes / 16u));
  }
  const uint32_t chunkBlocks = (uint32_t)std::max(1, std::min(opt.fused_chunk_blocks, 4096));
  const bool doPass = histogram_dev == nullptr || checksum;

  // ---- member table + work index (host staging, uploaded together) ----
  HostStage& hs = hostStage();
  const size_t descBytes = sizeof(MemberDesc) * (size_t)n;
  const size_t idxOff = (descBytes + 15) & ~size_t(15);
  hs.encodeUpload.resize(idxOff + sizeof(uint2) * ((size_t)n + 1));
  MemberDesc* desc = reinterpret_cast<MemberDesc*>(hs.encodeUpload.data());
  uint2* workIdx = reinterpret_cast<uint2*>(hs.encodeUpload.data() + idxOff);
  uint32_t maxSize = 0;
  uint64_t tickets = 0, items = 0, chunks = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const HostMember& hm = members[i];
    if ((hm.size && !hm.in) || !hm.out) return DGB_ERR_INVALID_ARG;
    if (reinterpret_cast<uintptr_t>(hm.out) & 15u) return DGB_ERR_INVALID_ARG;
    if (reinterpret_cast<uintptr_t>(hm.in) & (elemBytes - 1u)) return DGB_ERR_INVALID_ARG;
    // the reference refuses members whose worst-case archive does not fit 32 bits
    // (ans/GpuANSEncode.cu:13-25 CHECK_LE(rawSize, INT32_MAX)): the caller cannot have sized `out`
    if ((kind == kKindBytes ? dgb_ans_max_compressed_size(hm.size) : dgb_float_max_compressed_size(archiveKind(kind), hm.size)) == 0u)
      return DGB_ERR_TOO_LARGE;
    desc[i].in = hm.in;
    desc[i].out = hm.out;
    desc[i].size = hm.size;
    desc[i].work0 = (uint32_t)tickets;
    workIdx[i] = make_uint2((uint32_t)items, (uint32_t)chunks);
    const uint32_t nb = ticketsFor(hm.size);
    tickets += nb;
    chunks += divUp(nb, chunkBlocks);
    const uint32_t slabs = kind == kKindBytes ? bytesSlabs(hm.in, hm.size, slabVecs, doPass)
                                              : floatSlabs(hm.in, hm.size, elemBytes, slabVecs);
    items += std::max(1u, slabs);
    maxSize = std::max(maxSize, hm.size);
    if (tickets > 0x7fffffffull || items > 0x7fffffffull) return DGB_ERR_TOO_LARGE;
  }
  workIdx[n] = make_uint2((uint32_t)items, (uint32_t)chunks);
  if (err) {
    // the EF kinds never run the fused launch: their residual table takes its work index's place (8 n <= 8 (n + 1) B)
    float** et = reinterpret_cast<float**>(hs.encodeUpload.data() + idxOff);
    for (uint32_t i = 0; i < n; ++i) et[i] = err[i];
  }
  const uint32_t totalTickets = (uint32_t)tickets;
  const ScratchPlan sp = planScratch(kind, n, maxSize, totalTickets, spillWarpBound(n, tickets));
  if (!temp || tempBytes < sp.total || (reinterpret_cast<uintptr_t>(temp) & 255u))
    return temp && tempBytes >= sp.total ? DGB_ERR_INVALID_ARG : DGB_ERR_TEMP_TOO_SMALL;

  uint8_t* base = static_cast<uint8_t*>(temp);
  EncodeScratch sc;
  sc.members = reinterpret_cast<MemberDesc*>(base + sp.members);
  sc.workIdx = reinterpret_cast<const uint2*>(base + sp.workIdx);
  sc.hist = reinterpret_cast<uint32_t*>(base + sp.hist);
  sc.histDone = reinterpret_cast<uint32_t*>(base + sp.histDone);
  sc.checksum = reinterpret_cast<uint32_t*>(base + sp.checksum);
  sc.ticket = reinterpret_cast<uint32_t*>(base + sp.ticket);
  sc.lookback = reinterpret_cast<unsigned long long*>(base + sp.lookback);
  sc.allocDone = reinterpret_cast<unsigned long long*>(base + sp.allocDone);
  sc.ready = reinterpret_cast<uint32_t*>(base + sp.ready);
  sc.spill = base + sp.spill;
  sc.table = reinterpret_cast<uint4*>(base + sp.table);
  sc.blockZerosOff = sp.blockZerosOff;
  const bool stagedK1 = kind != kKindBytes && opt.stats_stage != 0 && !defaultOnly;

  // member table: inside the kernel parameters when it fits and the default kernels run, else uploaded to scratch
  static thread_local InlineMembers im;
  const bool inlined = opt.inline_members != 0 && n <= kInlineMembers && !fused && !canonical && !stagedK1;
  im.count = inlined ? n : 0u;
  // EF kinds: the residual table goes where the member table goes
  static thread_local EfMembers ef;
  ef.global = reinterpret_cast<float* const*>(base + sp.workIdx);
  ef.count = err && inlined ? n : 0u;
  if (err && inlined) std::memcpy(ef.e, err, sizeof(float*) * (size_t)n);
  if (inlined) {
    std::memcpy(im.m, desc, descBytes);
  } else {
    const int rc = uploadTable(base + sp.members, hs.encodeUpload.data(), hs.encodeUpload.size(), stream);
    if (rc != DGB_OK) return rc;
  }
  DGB_CUDA_TRY(cudaMemsetAsync(base + sp.zeroBegin, 0, (canonical ? sp.lookbackEnd : sp.zeroEnd) - sp.zeroBegin, stream));

  const int sms = smCount();
  // encoder table format (see EncSym in this file): wide entries for exponent-byte planes (by the archive type)
  const int ak = archiveKind(kind);
  const bool wideTable = !canonical && opt.encode_wide_table != 0 &&
                         (opt.encode_wide_table > 0 || ak == DGB_BFLOAT16 || ak == DGB_FLOAT32 || ak == DGB_FLOAT64 ||
                          ak == DGB_BFLOAT16_SPARSE || ak == DGB_FLOAT32_SPARSE);
  sc.wideTable = wideTable;

  if (fused) {
    // ---- one persistent launch: statistics items and encode chunks from two counters ----
    const uint32_t statsEvery = (uint32_t)std::max(0, opt.fused_stats_every);
    return withKind(kind, [&](auto K) { return withBool(wideTable, [&](auto WD) { return withBool(staged, [&](auto ST) {
      if constexpr (isSparseKind(decltype(K)::value)) {
        return (int)DGB_ERR_INVALID_ARG;  // not reached: `fused` is false for the sparse kinds
      } else {
      auto kern = encodeFusedKernel<decltype(K)::value, decltype(WD)::value, decltype(ST)::value>;
      constexpr uint32_t W = kStatsThreads / 32;
      const size_t smemBytes = (size_t)W * encFastWarpSmem(slotWords, kind);
      int perSm = 1;
      const int rc = residentCtasPerSm((const void*)kern, kStatsThreads, smemBytes, 200 * 1024, &perSm);
      if (rc != DGB_OK) return rc;
      uint64_t grid = (uint64_t)perSm * (uint64_t)sms;
      grid = std::min<uint64_t>(grid, items + chunks);
      grid = std::min<uint64_t>(grid, sp.spillWarps / W);  // every warp owns a spill slot
      grid = std::max<uint64_t>(grid, 1);
      timerBegin(opt, kSlotFused, stream);
      kern<<<(uint32_t)grid, kStatsThreads, smemBytes, stream>>>(sc, histogram_dev, pb, checksum, n, (uint32_t)items,
                                                                 (uint32_t)chunks, slabVecs, chunkBlocks, slotWords,
                                                                 statsEvery, outSize_dev);
      DGB_CUDA_TRY(cudaGetLastError());
      timerEnd(opt, kSlotFused, stream);
      return DGB_OK;
      }
    }); }); });
  }

  // ---- two-kernel path: sub-batches on internal streams (the ordered canonical encoder stays on one) ----
  // byte inputs gain nothing from splitting (their stats kernel is atomics-bound, not HBM-bound; capi.cu autoParts)
  SubBatches parts(kind, desc, n, opt, !canonical, stream);
  if (const int rc = parts.fork(); rc != DGB_OK) return rc;
  const uint32_t spillWarpsPerPart = sp.spillWarps / (uint32_t)parts.count();
  const uint32_t slabVecsK1 = stagedK1 ? std::min<uint32_t>(slabVecs, (uint32_t)std::max(1, opt.stats_stage_kb) * 64u) : slabVecs;
  // K2 launch configuration (same for every part)
  const size_t smemBytes = (size_t)W * (canonical ? encWarpSmem(pb, kind) : encFastWarpSmem(slotWords, kind));

  return withEncodeKind(kind, [&](auto K) { return withBool(wideTable, [&](auto WD) {
    constexpr int KIND = decltype(K)::value;
    constexpr bool WIDE = decltype(WD)::value;
    // K2: the canonical coder (ordered, packed table; wideTable is false) or the fast coder
    const void* coder;
    if constexpr (isEfKind(KIND))
      coder = canonical ? (const void*)encodeKernelEf<KIND> : (const void*)encodeKernelFastEf<WIDE, KIND>;
    else
      coder = canonical ? (const void*)encodeKernel<KIND> : (const void*)encodeKernelFast<WIDE, KIND>;
    int perSm = 1;
    int rc = residentCtasPerSm(coder, (int)(W * 32), smemBytes, 200 * 1024, &perSm);
    if (rc != DGB_OK) return rc;
    // option encode_k2_ctas caps the coder's CTAs per SM so that the statistics kernel of the next
    // sub-batch finds room beside it (0 = as many as fit)
    if (opt.encode_k2_ctas > 0) perSm = std::min(perSm, opt.encode_k2_ctas);
    const uint64_t resident = (uint64_t)perSm * sms;

    for (int part = 0; part < parts.count(); ++part) {
      const uint32_t m0 = parts.begin(part), m1 = parts.end(part);
      if (m1 == m0) continue;
      cudaStream_t ps;
      rc = parts.stream(part, &ps);
      if (rc != DGB_OK) return rc;
      // ---- K1 ----
      uint32_t partMax = 0;
      for (uint32_t i = m0; i < m1; ++i) partMax = std::max(partMax, desc[i].size);
      const uint64_t maxVecs = ((uint64_t)partMax * elemBytes) / 16u;
      uint32_t gridY = (uint32_t)std::max<uint64_t>(1, (maxVecs + slabVecsK1 - 1) / slabVecsK1);
      if (!stagedK1) {
        // enough CTAs to fill the machine a few times, never more than the slabs
        const uint32_t wantY = std::max(1u, (uint32_t)(std::max(1, opt.hist_ctas_per_sm) * sms) / (m1 - m0));
        gridY = std::min(gridY, wantY);
      }
      gridY = std::min(gridY, 65535u);
      dim3 grid1(m1 - m0, gridY);
      timerBegin(opt, kSlotStats, ps);
      if constexpr (KIND == kKindBytes) {
        statsBytesKernel<<<grid1, kStatsThreads, 0, ps>>>(sc, im, histogram_dev, pb, checksum, slabVecs, m0, outSize_dev);
      } else if constexpr (isEfKind(KIND)) {
        statsFloatEfKernel<KIND><<<grid1, kStatsThreads, 0, ps>>>(sc, im, ef, pb, checksum, slabVecs, m0, outSize_dev);
      } else if constexpr (isSparseKind(KIND) || isNarrowKind(KIND)) {
        statsFloatKernel<KIND><<<grid1, kStatsThreads, 0, ps>>>(sc, im, pb, checksum, slabVecs, m0, outSize_dev);
      } else if (stagedK1 && gridY * (uint64_t)slabVecsK1 >= maxVecs) {
        rc = residentCtasPerSm((const void*)statsFloatStagedKernel<KIND>, kStatsThreads, 0, 128 * 1024, nullptr);
        if (rc != DGB_OK) return rc;
        statsFloatStagedKernel<KIND><<<grid1, kStatsThreads, (size_t)slabVecsK1 * 16u, ps>>>(sc, pb, checksum, slabVecsK1, m0,
                                                                                            outSize_dev);
      } else {
        statsFloatKernel<KIND><<<grid1, kStatsThreads, 0, ps>>>(sc, im, pb, checksum, slabVecs, m0, outSize_dev);
      }
      DGB_CUDA_TRY(cudaGetLastError());
      timerEnd(opt, kSlotStats, ps);

      // ---- K2 ----
      const uint32_t blockBegin = desc[m0].work0;
      const uint32_t blockEnd = m1 < n ? desc[m1].work0 : totalTickets;
      const uint32_t partBlocks = blockEnd - blockBegin;
      if (partBlocks == 0) continue;
      timerBegin(opt, kSlotEncode, ps);
      if (canonical) {
        const uint32_t grid2 = std::min<uint32_t>(divUp(totalTickets, W), (uint32_t)resident);
        if constexpr (isEfKind(KIND))
          encodeKernelEf<KIND><<<grid2, W * 32, smemBytes, ps>>>(sc, ef, pb, checksum, n, totalTickets, outSize_dev);
        else
          encodeKernel<KIND><<<grid2, W * 32, smemBytes, ps>>>(sc, pb, checksum, n, totalTickets, outSize_dev);
      } else {
        // one resident wave, equal rounds per warp (see launchPlanDecode)
        const uint64_t rounds = std::max<uint64_t>(1, (partBlocks + resident * W - 1) / (resident * W));
        const uint64_t want = ((uint64_t)partBlocks + W * rounds - 1) / (W * rounds);
        uint32_t grid2 = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(want, resident));
        grid2 = std::max(1u, std::min(grid2, spillWarpsPerPart / W));  // every warp owns a spill slot
        if constexpr (isEfKind(KIND))
          encodeKernelFastEf<WIDE, KIND><<<grid2, W * 32, smemBytes, ps>>>(sc, im, ef, pb, checksum, n, blockBegin, blockEnd,
                                                                          slotWords, (uint32_t)part * spillWarpsPerPart,
                                                                          outSize_dev);
        else
          encodeKernelFast<WIDE, KIND><<<grid2, W * 32, smemBytes, ps>>>(sc, im, pb, checksum, n, blockBegin, blockEnd, slotWords,
                                                                        (uint32_t)part * spillWarpsPerPart, outSize_dev);
      }
      DGB_CUDA_TRY(cudaGetLastError());
      timerEnd(opt, kSlotEncode, ps);
    }
    return DGB_OK;  // ~SubBatches joins the helper streams
  }); });
}

}  // namespace dgb
