// decode.cu -- batched rANS decode (bytes) and fused float decompress
// (fp16/bf16/fp32/fp64, sparse fp16/bf16/fp32) for sm_90a (H100).  One launch per call (decodeFusedKernel, further down): a persistent grid
// whose CTAs lease members (header checks and the 2^pb LUT from the archive's own pdf happen inside the
// CTA) and whose warps claim 4 KiB blocks; lane states + compressed words of a block arrive by one TMA
// bulk copy (cp.async.bulk + mbarrier), the 32-lane interleaved rANS decode of ans/GpuANSDecode.cuh:55-217
// runs with table look-ups and the loop-carried refill load in shared memory, and float kinds join the
// decoded byte with the stored byte(s) (cp.async ring) and store the float word in the same loop, at any
// alignment (float/GpuFloatDecompress.cuh:22-179, float/GpuFloatUtils.cuh:100-204 join rules; the
// reference's two-pass path, float/GpuFloatDecompress.cuh:622-694, is not needed).
// The round-1 pair planKernel (header validation ans/GpuANSDecode.cuh:326-341, flat block offsets) +
// decodeKernel (static split of the blocks) is kept behind option decode_fused=0.
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"

// rows per software-pipelined group and the resident-warp target that caps registers
#ifndef DGB_DECODE_UNROLL
#define DGB_DECODE_UNROLL 8
#endif
#ifndef DGB_DECODE_WARPS_PER_SM
#define DGB_DECODE_WARPS_PER_SM 40
#endif

namespace dgb {

namespace {

struct DecodeScratch {
  MemberDesc* members;   // [n]; two-kernel path: planKernel fills work0 = first flat block;
                         //      single-launch path: work0 = upper bound of the member's block count (host, from capacity)
  uint32_t* next;        // [n] single-launch path: next unclaimed block of the member (zeroed)
  uint32_t* seen;        // [n] single-launch path: 1 once a CTA has reported the member (zeroed)
  uint32_t* totals;      // [0] = total blocks, [1] = unused
  uint32_t* checksum;    // [n] checksum of decoded output (use_checksum only; zeroed)
  uint32_t* archiveChecksum;  // [n]
  uint32_t* sizes;       // [n] decoded size in bytes (for the checksum pass)
};

// Where the ANS archive of member `md` starts, and the float-level fields.
struct ArchiveView {
  const uint8_t* ans;      // ANS archive base
  const uint8_t* non;      // float kinds: stored (non-compressed) plane(s)
  uint32_t floatWords;     // float kinds: size field of the float header
  bool ok;
  // sparse kinds: block table, stored bytes (`non`), escape word
  const uint32_t* table;
  uint32_t storedBytes;
  uint32_t esc;
};

template <int KIND>
__device__ __forceinline__ ArchiveView openArchive(const uint8_t* in) {
  ArchiveView v;
  if (KIND == kKindBytes) {
    v.ans = in;
    v.non = nullptr;
    v.floatWords = 0;
    v.ok = true;
  } else if constexpr (isFp8Kind(KIND)) {
    // a byte archive of fp8 words: floatWords is the ANS header's uncompressed size, one byte per word
    v.ans = in;
    v.non = nullptr;
    v.floatWords = __ldg(reinterpret_cast<const uint32_t*>(in) + 2);
    v.ok = true;
  } else if constexpr (isSparseKind(KIND)) {
    // the 32 B header: the dense 16 B, then S and esc (DESIGN.md section 0)
    const uint4 fh = __ldg(reinterpret_cast<const uint4*>(in));
    const uint4 sh = __ldg(reinterpret_cast<const uint4*>(in) + 1);
    v.ok = fh.x == kFloatMagicVersion && (int)(fh.z & 0xfu) == KIND && sh.x <= fh.y && sparseEscValid(sh.y);
    v.floatWords = fh.y;
    v.storedBytes = sh.x;
    v.esc = sh.y;
    v.table = reinterpret_cast<const uint32_t*>(in + kSparseHeaderBytes);
    v.non = in + kSparseHeaderBytes + sparseTableBytes<uint32_t>(fh.y);
    if constexpr (KIND == kKindF32S)
      v.ans = in + sparseExtraBytes<uint32_t>(KIND, fh.y, sh.x);
    else
      v.ans = in + sparseExtraBytes<uint32_t>(fh.y, sh.x);
  } else {
    // float/GpuFloatUtils.cuh:26-74 GpuFloatHeader
    const uint4 fh = __ldg(reinterpret_cast<const uint4*>(in));
    v.ok = fh.x == kFloatMagicVersion && (int)(fh.z & 0xfu) == KIND;
    v.floatWords = fh.y;
    v.non = in + kFloatHeaderBytes;
    v.ans = v.non + floatNonCompBytes(KIND, fh.y);
  }
  return v;
}

// (checksum flag, checksum) of a member archive: the ANS header's (at `ans`) for byte archives, the float
// header's (at `in`) otherwise.  With the flag clear the checksum word is undefined (the reference never writes
// it), so such a member is not verified.
template <int KIND>
__device__ __forceinline__ uint2 storedChecksumOf(const void* in, const uint8_t* ans) {
  const uint2 w = KIND == kKindBytes ? __ldg(reinterpret_cast<const uint2*>(ans + 16))
                                     : __ldg(reinterpret_cast<const uint2*>(in) + 1);
  return make_uint2(w.x & 0x10u, w.y);
}

// ---------------------------------------------------------------------------
// P: plan.  One CTA; member i handled by thread (i % blockDim) in rounds.
// ---------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(1024)
planKernel(DecodeScratch sc, uint32_t m0, uint32_t m1, uint32_t part, int pb,
           uint8_t* __restrict__ outSuccess, uint32_t* __restrict__ outSize, bool wantChecksum) {
  // members [m0, m1) form one sub-batch with its own flat block index space (totals[part])
  __shared__ uint32_t sWarp[32];
  uint32_t carry = 0;
  const uint32_t n = m1;
  for (uint32_t base = m0; base < n; base += blockDim.x) {
    const uint32_t i = base + threadIdx.x;
    uint32_t blocks = 0;
    if (i < n) {
      const MemberDesc md = sc.members[i];
      const ArchiveView av = openArchive<KIND>(static_cast<const uint8_t*>(md.in));
      bool ok = av.ok;
      uint32_t need = 0, nb = 0;
      if (ok) {
        const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(av.ans));
        const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(av.ans) + 1);
        nb = h0.y;
        need = h0.z;  // uncompressed bytes == float words for float kinds
        ok = h0.x == kAnsMagicVersion && (int)(h1.x & 0xfu) == pb && nb == divUp(need, kBlockBytes);
        if (KIND != kKindBytes) ok = ok && need == av.floatWords;
      }
      // ans/GpuANSDecode.cuh:326-337: success iff capacity suffices; size reported regardless
      const bool success = ok && md.size >= need;
      if (outSuccess) outSuccess[i] = success ? 1 : 0;
      if (outSize) outSize[i] = ok ? need : 0u;
      if (wantChecksum) {
        const uint2 ck = success ? storedChecksumOf<KIND>(md.in, av.ans) : make_uint2(0u, 0u);
        sc.archiveChecksum[i] = ck.y;
        sc.sizes[i] = ck.x ? need : 0u;
      }
      blocks = success ? nb : 0u;
    }
    uint32_t tot;
    const uint32_t excl = blockExclusiveScan<1024>(blocks, sWarp, &tot);
    if (i < n) sc.members[i].work0 = carry + excl;
    carry += tot;
  }
  if (threadIdx.x == 0) sc.totals[part] = carry;
}

// ---------------------------------------------------------------------------
// Output writers (ans/BatchProvider.cuh:16-37 BatchWriter, float/
// GpuFloatDecompress.cuh:391-486 JoinFloatWriter restated).  A writer is bound
// to one 4 KiB block.  The float kinds need the stored ("non-compressed")
// byte(s) of every element: those are streamed into a small per-warp
// shared-memory ring with cp.async (LDGSTS) -- one 16 B copy per lane covers a
// whole group of 8 rows -- two groups ahead of the row being decoded, so the
// join reads them with an LDS and the HBM latency of the stored plane never
// meets the dependent decode chain (per-row LDG.U8 of these bytes would put
// HBM latency on that chain; holding them in registers instead made ptxas sink
// the loads next to their use).
// ---------------------------------------------------------------------------
#ifndef DGB_DEC_GROUP_ROWS
#define DGB_DEC_GROUP_ROWS 16
#endif
constexpr int kGroupRows = DGB_DEC_GROUP_ROWS;  // rows per prefetch group (8 or 16)
constexpr uint32_t kRingSlots = 3;              // groups resident per warp: current + 2 in flight

// writer kinds of the decode-and-sum (further down): the archive kind | kAddWriter adds the decoded word to the
// output's word; | kWidenF32 writes (or adds into) fp32 outputs from fp16 / bf16 archives (dense or sparse);
// | kScaled multiplies every decoded word by the call's scale first (0x40 is the encoder's narrowing bit);
// | kDevScale (kernels only, with kScaled) reads that scale from device memory when the kernel runs;
// | kCheckFinite (writers only) also reports whether a word it stores is inf or NaN;
// | kNarrowOut (with kWidenF32) sums in fp32 from an fp32 accumulator and stores the sum rounded once to the
// archive's 16-bit type into a second output (the narrowing sums: kernels and the writer of a call's last archive);
// | kSqNorm (device-scale kinds only) also takes the squared norm of the words the call stores (kernels, and with
// kCheckFinite the writer of a call's last archive)
constexpr int kAddWriter = 0x10;
constexpr int kWidenF32 = 0x20;
constexpr int kScaled = 0x80;
constexpr int kDevScale = 0x100;
constexpr int kCheckFinite = 0x200;
constexpr int kNarrowOut = 0x400;
constexpr int kSqNorm = 0x800;
// the archive kind of a decode-and-sum kernel or writer kind
__host__ __device__ constexpr int reduceArchiveKind(int k) {
  return k & ~(kAddWriter | kWidenF32 | kScaled | kDevScale | kCheckFinite | kNarrowOut | kSqNorm);
}

template <int KIND>
struct RowWriter;

template <>
struct RowWriter<kKindBytes> {
  static constexpr uint32_t kRingSlotBytes = 0;
  uint8_t* out;
  struct Cursor { uint8_t* o; };
  __device__ __forceinline__ void setRing(uint32_t, uint32_t) {}
  __device__ __forceinline__ void setBlock(const ArchiveView&, void* outBase, uint32_t block, uint32_t lane) {
    out = static_cast<uint8_t*>(outBase) + (size_t)block * kBlockBytes + lane;
    __builtin_assume(__isGlobal(out));
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t) const { return Cursor{out + row * 32u}; }
  __device__ __forceinline__ void issue(uint32_t, uint32_t) const {}
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = (uint8_t)entry;
  }
  // rows outside the pipelined groups
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const { out[row * 32u] = (uint8_t)entry; }
};

template <int KIND>
struct RowWriter16 {
  static constexpr uint32_t kRingSlotBytes = kGroupRows * 32;  // one stored byte per element
  uint16_t* out;
  const uint8_t* non;      // this lane's byte of row 0 of the block
  const uint8_t* nonCopy;  // copy source of this lane (lanes 0..15 move 16 B each per group)
  uint32_t ring, lane;
  struct Cursor { uint16_t* o; uint32_t s; };
  __device__ __forceinline__ void setRing(uint32_t ringAddr, uint32_t l) { ring = ringAddr; lane = l; }
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    out = static_cast<uint16_t*>(outBase) + (size_t)block * kBlockBytes + l;
    non = av.non + (size_t)block * kBlockBytes + l;
    nonCopy = av.non + (size_t)block * kBlockBytes + l * 16u;
    __builtin_assume(__isGlobal(out));
    __builtin_assume(__isGlobal(non));
    __builtin_assume(__isGlobal(nonCopy));
  }
  // cursor of the group starting at `row`, resident in ring slot `slot`
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t slot) const {
    return Cursor{out + row * 32u, ring + slot * kRingSlotBytes + lane};
  }
  // request rows [row, row + 8) into ring slot `slot`
  __device__ __forceinline__ void issue(uint32_t row, uint32_t slot) const {
    if (lane < (uint32_t)(kGroupRows * 2)) cpAsync16(ring + slot * kRingSlotBytes + lane * 16u, nonCopy + row * 32u);
  }
  static __device__ __forceinline__ uint32_t join(uint32_t entry, uint32_t nc) {
    if (KIND == kKindF16) {
      // float/GpuFloatUtils.cuh:117-119: comp * 256 + nonComp  (bytes: [non, comp])
      return __byte_perm(entry, nc, 0x4404);
    }
    // float/GpuFloatUtils.cuh:149-159: (comp:non) rotated right by one within 16 bits.
    // x = comp<<24 | non<<16 ; (non : x) >> 17 leaves comp<<7 | non>>1 | (non&1)<<15 in the
    // low 16 bits (higher bits are dropped by the 16-bit store)
    return __funnelshift_r(__byte_perm(entry, nc, 0x0444), nc, 17);
  }
  // the joined word of row J of the cursor's group (from the ring), or of any row (from global memory)
  template <int J>
  __device__ __forceinline__ uint32_t word(const Cursor& c, uint32_t entry) const {
    return join(entry, ldsU8<J * 32>(c.s));
  }
  __device__ __forceinline__ uint32_t wordSlow(uint32_t row, uint32_t entry) const {
    return join(entry, __ldg(non + row * 32u));
  }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = (uint16_t)word<J>(c, entry);
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const {
    out[row * 32u] = (uint16_t)wordSlow(row, entry);
  }
};
template <> struct RowWriter<kKindF16> : RowWriter16<kKindF16> {};
template <> struct RowWriter<kKindBF16> : RowWriter16<kKindBF16> {};

// fp8 archives (decode-and-sum only, as the base of RowWriterSum): the decoded symbol is the whole fp8 word, so there
// is no stored plane and no ring
template <int KIND>
struct RowWriterFp8 {
  static constexpr uint32_t kRingSlotBytes = 0;
  struct Cursor {};
  __device__ __forceinline__ void setRing(uint32_t, uint32_t) {}
  __device__ __forceinline__ void setBlock(const ArchiveView&, void*, uint32_t, uint32_t) {}
  __device__ __forceinline__ Cursor at(uint32_t, uint32_t) const { return Cursor{}; }
  __device__ __forceinline__ void issue(uint32_t, uint32_t) const {}
  template <int J>
  __device__ __forceinline__ uint32_t word(const Cursor&, uint32_t entry) const { return entry & 0xffu; }
  __device__ __forceinline__ uint32_t wordSlow(uint32_t, uint32_t entry) const { return entry & 0xffu; }
};
template <> struct RowWriter<kKindE4M3> : RowWriterFp8<kKindE4M3> {};
template <> struct RowWriter<kKindE5M2> : RowWriterFp8<kKindE5M2> {};

// Sparse fp16 / bf16: the block's segment of stored bytes, [table[k], table[k + 1] or S), sits in the warp's ring
// (one copy per block, widened to 16 B bounds: at most 4112 bytes).  Rows are walked backwards, so the cursor
// starts one past the segment's last byte; per row it moves back by the number of kept lanes (symbol neither E+ nor
// E-), and a kept lane reads its byte at the cursor plus its rank among the kept lanes.  E+ / E- lanes write +0 / -0.
template <int KIND>
struct RowWriterSparse {
  static constexpr int BT = denseKind(KIND);
  static constexpr uint32_t kRingSlotBytes = 1376;  // 3 slots = 4128 bytes >= the widest segment
  uint16_t* out;
  const uint8_t* src;    // 16 B aligned start of the segment's copy
  uint32_t copyBytes;    // bytes to copy (multiple of 16)
  uint32_t ring, lane, ltMask;
  uint32_t ep, em;       // escape symbols; 0x100 / 0x101 (no symbol) when nothing is elided
  mutable uint32_t cur;  // shared address one past the next row's kept bytes
  struct Cursor { uint16_t* o; };
  __device__ __forceinline__ void setRing(uint32_t ringAddr, uint32_t l) {
    ring = ringAddr;
    lane = l;
    ltMask = laneMaskLt();
  }
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    out = static_cast<uint16_t*>(outBase) + (size_t)block * kBlockBytes + l;
    const uint32_t nb = divUp(av.floatWords, kBlockBytes);
    const uint32_t begin = __ldg(av.table + block);
    const uint32_t end = block + 1 < nb ? __ldg(av.table + block + 1) : av.storedBytes;
    const uint32_t a0 = begin & ~15u;
    src = av.non + a0;
    copyBytes = roundUp(end, 16u) - a0;
    cur = ring + (end - a0);
    const bool elide = av.esc != 0u;
    ep = elide ? (av.esc & 0xffu) : 0x100u;
    em = elide ? ((av.esc >> 8) & 0xffu) : 0x101u;
    __builtin_assume(__isGlobal(out));
    __builtin_assume(__isGlobal(src));
  }
  // the segment arrives by a bulk copy on the block's mbarrier (lane 0; bytes counted by the caller's expect_tx)
  __device__ __forceinline__ uint32_t bulkBytes() const { return copyBytes; }
  __device__ __forceinline__ void bulkIssue(uint32_t bar) const {
    if (copyBytes) {
      fenceProxyAsync();  // the ring may have been written through the generic proxy (copySync)
      bulkLoad(ring, src, copyBytes, bar);
    }
  }
  // ... or, when the block's stream is read from global memory, by the warp itself
  __device__ __forceinline__ void copySync() const {
    __syncwarp();
    for (uint32_t i = lane * 16u; i < copyBytes; i += 512u) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + i));
      asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(ring + i), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                   : "memory");
    }
    __syncwarp();
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t) const { return Cursor{out + row * 32u}; }
  __device__ __forceinline__ void issue(uint32_t, uint32_t) const {}
  // the word of this lane's element in the current row (whole warp; lanes with valid = false hold none)
  __device__ __forceinline__ uint32_t word(uint32_t entry, bool valid) const {
    const uint32_t s = entry & 0xffu;
    const bool keep = valid && s != ep && s != em;
    const uint32_t b = __ballot_sync(0xffffffffu, keep);
    cur -= __popc(b);
    uint32_t nc = 0;
    if (keep) asm volatile("ld.shared.u8 %0, [%1];" : "=r"(nc) : "r"(cur + __popc(b & ltMask)));
    return keep ? RowWriter16<BT>::join(entry, nc) : (s == ep ? 0u : 0x8000u);
  }
  template <int J>
  __device__ __forceinline__ uint32_t word(const Cursor&, uint32_t entry) const { return word(entry, true); }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = (uint16_t)word(entry, true);
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const { out[row * 32u] = (uint16_t)word(entry, true); }
  __device__ __forceinline__ void writePartial(uint32_t row, uint32_t entry, bool valid) const {
    const uint32_t w = word(entry, valid);
    if (valid) out[row * 32u] = (uint16_t)w;
  }
};
template <> struct RowWriter<kKindF16S> : RowWriterSparse<kKindF16S> {};
template <> struct RowWriter<kKindBF16S> : RowWriterSparse<kKindBF16S> {};
// the kinds whose writer loads a block's whole stored segment (bulkIssue / copySync)
__host__ __device__ constexpr bool copiesSegment(int kind) { return kind == kKindF16S || kind == kKindBF16S; }


template <>
struct RowWriter<kKindF64> {
  // per group: rows x 128 B of the u32 plane, rows x 64 B of the u16 plane, rows x 32 B of the u8 plane
  static constexpr uint32_t kRingSlotBytes = kGroupRows * 224;
  unsigned long long* out;
  const uint32_t* non4;
  const uint16_t* non2;
  const uint8_t* non1;
  const uint8_t* copy4;
  const uint8_t* copy2;
  const uint8_t* copy1;
  uint32_t ring, lane;
  struct Cursor { unsigned long long* o; uint32_t s4, s2, s1; };
  __device__ __forceinline__ void setRing(uint32_t ringAddr, uint32_t l) { ring = ringAddr; lane = l; }
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    out = static_cast<unsigned long long*>(outBase) + (size_t)block * kBlockBytes + l;
    const uint8_t* p4 = av.non + 4u * (size_t)block * kBlockBytes;
    const uint8_t* p2 = av.non + floatU16PlaneOffset<uint32_t>(kKindF64, av.floatWords) + 2u * (size_t)block * kBlockBytes;
    const uint8_t* p1 = av.non + floatU8PlaneOffset<uint32_t>(kKindF64, av.floatWords) + (size_t)block * kBlockBytes;
    non4 = reinterpret_cast<const uint32_t*>(p4) + l;
    non2 = reinterpret_cast<const uint16_t*>(p2) + l;
    non1 = p1 + l;
    copy4 = p4 + l * 16u;
    copy2 = p2 + l * 16u;
    copy1 = p1 + l * 16u;
    __builtin_assume(__isGlobal(out));
    __builtin_assume(__isGlobal(non4));
    __builtin_assume(__isGlobal(non2));
    __builtin_assume(__isGlobal(non1));
    __builtin_assume(__isGlobal(copy4));
    __builtin_assume(__isGlobal(copy2));
    __builtin_assume(__isGlobal(copy1));
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t slot) const {
    const uint32_t base = ring + slot * kRingSlotBytes;
    return Cursor{out + row * 32u, base + lane * 4u, base + kGroupRows * 128 + lane * 2u, base + kGroupRows * 192 + lane};
  }
  __device__ __forceinline__ void issue(uint32_t row, uint32_t slot) const {
    const uint32_t base = ring + slot * kRingSlotBytes;
#pragma unroll
    for (int h = 0; h < kGroupRows / 4; ++h)  // 32 lanes x 16 B = 4 rows x 128 B per copy
      cpAsync16(base + h * 512 + lane * 16u, copy4 + row * 128u + h * 512);
#pragma unroll
    for (int h = 0; h < kGroupRows / 8; ++h)
      cpAsync16(base + kGroupRows * 128 + h * 512 + lane * 16u, copy2 + row * 64u + h * 512);
    if (lane < (uint32_t)(kGroupRows * 2)) cpAsync16(base + kGroupRows * 192 + lane * 16u, copy1 + row * 32u);
  }
  static __device__ __forceinline__ unsigned long long join(uint32_t entry, uint32_t lo, uint32_t mid, uint32_t hi) {
    // (comp << 56 | stored 56 bits) rotated right by one; the high half is built as fp32's join builds its word
    const uint32_t h = __byte_perm(mid, __byte_perm(hi, entry, 0x0040), 0x5410);
    return ((unsigned long long)__funnelshift_r(h, lo, 1) << 32) | __funnelshift_r(lo, h, 1);
  }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = join(entry, ldsU32<J * 128>(c.s4), ldsU16<J * 64>(c.s2), ldsU8<J * 32>(c.s1));
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const {
    out[row * 32u] = join(entry, __ldg(non4 + row * 32u), __ldg(non2 + row * 32u), __ldg(non1 + row * 32u));
  }
};

template <>
struct RowWriter<kKindF32> {
  // per group: 8 rows x 64 B of the u16 plane, then 8 rows x 32 B of the u8 plane
  static constexpr uint32_t kRingSlotBytes = kGroupRows * 96;
  uint32_t* out;
  const uint16_t* non2;
  const uint8_t* non1;
  const uint8_t* copy2;
  const uint8_t* copy1;
  uint32_t ring, lane;
  struct Cursor { uint32_t* o; uint32_t s2, s1; };
  __device__ __forceinline__ void setRing(uint32_t ringAddr, uint32_t l) { ring = ringAddr; lane = l; }
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    out = static_cast<uint32_t*>(outBase) + (size_t)block * kBlockBytes + l;
    const uint8_t* p2 = av.non + 2u * (size_t)block * kBlockBytes;
    const uint8_t* p1 = av.non + 2u * (size_t)roundUp(av.floatWords, 8u) + (size_t)block * kBlockBytes;
    non2 = reinterpret_cast<const uint16_t*>(p2) + l;
    non1 = p1 + l;
    copy2 = p2 + l * 16u;
    copy1 = p1 + l * 16u;
    __builtin_assume(__isGlobal(out));
    __builtin_assume(__isGlobal(non2));
    __builtin_assume(__isGlobal(non1));
    __builtin_assume(__isGlobal(copy2));
    __builtin_assume(__isGlobal(copy1));
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t slot) const {
    const uint32_t base = ring + slot * kRingSlotBytes;
    return Cursor{out + row * 32u, base + lane * 2u, base + kGroupRows * 64 + lane};
  }
  __device__ __forceinline__ void issue(uint32_t row, uint32_t slot) const {
    const uint32_t base = ring + slot * kRingSlotBytes;
#pragma unroll
    for (int h = 0; h < kGroupRows / 8; ++h)  // 32 lanes x 16 B = 8 rows x 64 B per copy
      cpAsync16(base + h * 512 + lane * 16u, copy2 + row * 64u + h * 512);
    if (lane < (uint32_t)(kGroupRows * 2)) cpAsync16(base + kGroupRows * 64 + lane * 16u, copy1 + row * 32u);
  }
  static __device__ __forceinline__ uint32_t join(uint32_t entry, uint32_t lo, uint32_t hi) {
    // float/GpuFloatUtils.cuh:187-190: (comp << 24 | stored 24 bits) rotated right by one
    const uint32_t v = __byte_perm(lo, __byte_perm(hi, entry, 0x0040), 0x5410);
    return __funnelshift_r(v, v, 1);
  }
  template <int J>
  __device__ __forceinline__ uint32_t word(const Cursor& c, uint32_t entry) const {
    return join(entry, ldsU16<J * 64>(c.s2), ldsU8<J * 32>(c.s1));
  }
  __device__ __forceinline__ uint32_t wordSlow(uint32_t row, uint32_t entry) const {
    return join(entry, __ldg(non2 + row * 32u), __ldg(non1 + row * 32u));
  }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = word<J>(c, entry);
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const {
    out[row * 32u] = wordSlow(row, entry);
  }
};

// Sparse fp32: a block's kept words [begin, end) store 3 bytes each, up to 12 KiB per block, so the segment is
// streamed instead of copied whole: windows of 512 kept words anchored at the segment's end (window w holds kept
// words [max(begin, end - 512 (w + 1)), end - 512 w)), each as its u16 bytes and its u8 bytes widened to 16 B bounds
// (<= 1040 + 528 B), in a ring of three slots.  Rows are walked backwards with a kept-word cursor as in
// RowWriterSparse.  A row takes at most 32 kept words, so while the cursor is in window c the row reads windows c and
// c + 1 only; when it crosses into c + 1, window c's slot takes window c + 3 (cp.async, 16 B per lane) and window
// c + 2 must have landed.  The block starts with windows 0, 1 and 2 in flight (issued by setBlock, overlapping the
// stream's own load).  Whether a window has landed is tracked here alone (cp.async.wait_group 0 covers any group),
// so the generic loop's waits are only ever extra.
template <>
struct RowWriter<kKindF32S> {
  static constexpr uint32_t kWinWords = 512, kWin8 = 1040;  // u8 bytes start at slot + kWin8
  static constexpr uint32_t kRingSlotBytes = kWin8 + 528;    // 3 slots = 4704 bytes per warp
  uint32_t* out;
  const uint8_t* non16;  // u16 plane
  const uint8_t* non8;   // u8 plane
  uint32_t ring, lane, ltMask;
  uint32_t ep, em;  // escape symbols; 0x100 / 0x101 (no symbol) when nothing is elided
  uint32_t begin, end, numWin;
  mutable uint32_t cur;            // kept index one past the next row's kept words
  mutable uint32_t win, winLo;     // current window and its lowest kept index
  mutable uint32_t trig;           // the next row needs slowPath() when cur < trig
  mutable uint32_t issued, landed; // windows [0, issued) requested, [0, landed) known to be in shared memory
  mutable uint32_t b16c, b8c, b16n, b8n;  // shared address of kept index 0 (u16 / u8) in windows win and win + 1
  struct Cursor { uint32_t* o; };
  __device__ __forceinline__ void setRing(uint32_t ringAddr, uint32_t l) {
    ring = ringAddr;
    lane = l;
    ltMask = laneMaskLt();
  }
  __device__ __forceinline__ uint32_t winHi(uint32_t w) const { return end - kWinWords * w; }
  __device__ __forceinline__ uint32_t winLow(uint32_t w) const {
    const uint32_t hi = winHi(w);
    return hi - begin > kWinWords ? hi - kWinWords : begin;
  }
  __device__ __forceinline__ uint32_t slotOf(uint32_t w) const { return ring + (w % 3u) * kRingSlotBytes; }
  __device__ __forceinline__ void bases(uint32_t w, uint32_t& b16, uint32_t& b8) const {
    const uint32_t lo = winLow(w);
    b16 = slotOf(w) - ((2u * lo) & ~15u);
    b8 = slotOf(w) + kWin8 - (lo & ~15u);
  }
  // requests window w into its slot (whole warp; the slot's previous window is no longer read)
  __device__ __forceinline__ void issueWin(uint32_t w) const {
    const uint32_t lo = winLow(w), hi = winHi(w);
    const uint32_t a16 = (2u * lo) & ~15u, a8 = lo & ~15u;
    const uint32_t c16 = (roundUp(2u * hi, 16u) - a16) >> 4, c8 = (roundUp(hi, 16u) - a8) >> 4;
    const uint32_t slot = slotOf(w);
    for (uint32_t i = lane; i < c16 + c8; i += 32u) {
      if (i < c16)
        cpAsync16(slot + 16u * i, non16 + a16 + 16u * i);
      else
        cpAsync16(slot + kWin8 + 16u * (i - c16), non8 + a8 + 16u * (i - c16));
    }
  }
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    out = static_cast<uint32_t*>(outBase) + (size_t)block * kBlockBytes + l;
    const uint32_t nb = divUp(av.floatWords, kBlockBytes);
    begin = __ldg(av.table + block);
    end = block + 1 < nb ? __ldg(av.table + block + 1) : av.storedBytes;
    non16 = av.non;
    non8 = av.non + 2u * (size_t)roundUp(av.storedBytes, 8u);
    __builtin_assume(__isGlobal(out));
    __builtin_assume(__isGlobal(non16));
    __builtin_assume(__isGlobal(non8));
    const bool elide = av.esc != 0u;
    ep = elide ? (av.esc & 0xffu) : 0x100u;
    em = elide ? ((av.esc >> 8) & 0xffu) : 0x101u;
    // a malformed table (end < begin, or a segment longer than a block) must not send the copies past the ring
    if (end < begin || end - begin > kBlockBytes) end = begin;
    numWin = divUp(end - begin, kWinWords);
    cur = end;
    win = 0;
    winLo = winLow(0);
    trig = 0xffffffffu;  // the first row waits for windows 0 and 1
    // every window of the previous block has landed (its rows read them all); every lane is done reading the ring
    __syncwarp();
    issued = min(numWin, 3u);
    if (issued > 0u) issueWin(0);
    if (issued > 1u) issueWin(1);
    cpAsyncCommit();
    if (issued > 2u) issueWin(2);
    cpAsyncCommit();
    landed = 0;
    bases(0, b16c, b8c);
    bases(1, b16n, b8n);
  }
  __device__ __forceinline__ void slowPath() const {
    if (landed == 0u) {
      // windows 0 and 1 were committed before window 2's group and the decode loop's two (empty) groups
      cpAsyncWait<3>();
      __syncwarp();
      landed = min(issued, 2u);
    }
    if (cur <= winLo && win + 1u < numWin) {  // the next row starts in window win + 1
      ++win;
      winLo = winLow(win);
      b16c = b16n;
      b8c = b8n;
      if (win + 1u < numWin) {
        bases(win + 1u, b16n, b8n);
        if (landed <= win + 1u) {
          cpAsyncWait<0>();
          __syncwarp();
          landed = issued;
        }
      }
      if (issued < numWin && issued == win + 2u) {  // window win + 2 goes where window win - 1 was
        __syncwarp();
        issueWin(issued);
        cpAsyncCommit();
        ++issued;
      }
    }
    trig = win + 1u < numWin ? winLo + 1u : 0u;
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t) const { return Cursor{out + row * 32u}; }
  __device__ __forceinline__ void issue(uint32_t, uint32_t) const {}
  // the word of this lane's element in the current row (whole warp; lanes with valid = false hold none)
  __device__ __forceinline__ uint32_t word(uint32_t entry, bool valid) const {
    if (cur < trig) slowPath();
    const uint32_t s = entry & 0xffu;
    const bool keep = valid && s != ep && s != em;
    const uint32_t b = __ballot_sync(0xffffffffu, keep);
    cur -= __popc(b);
    const uint32_t idx = cur + __popc(b & ltMask);
    const bool inCur = idx >= winLo;
    uint32_t lo = 0, hi = 0;
    if (keep) {
      asm volatile("ld.shared.u16 %0, [%1];" : "=r"(lo) : "r"((inCur ? b16c : b16n) + 2u * idx));
      asm volatile("ld.shared.u8 %0, [%1];" : "=r"(hi) : "r"((inCur ? b8c : b8n) + idx));
    }
    return keep ? RowWriter<kKindF32>::join(entry, lo, hi) : (s == ep ? 0u : 0x80000000u);
  }
  template <int J>
  __device__ __forceinline__ uint32_t word(const Cursor&, uint32_t entry) const { return word(entry, true); }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    c.o[J * 32] = word(entry, true);
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const { out[row * 32u] = word(entry, true); }
  __device__ __forceinline__ void writePartial(uint32_t row, uint32_t entry, bool valid) const {
    const uint32_t w = word(entry, valid);
    if (valid) out[row * 32u] = w;
  }
};

// ---------------------------------------------------------------------------
// The compressed word stream of one block, read backwards.  Two flavours so the
// hot loop always knows the address space: staged in shared memory by the TMA
// bulk copy (LDS on the loop-carried path) or straight from global memory.
// ---------------------------------------------------------------------------
struct SmemStream {
  uint32_t addr;  // shared BYTE address one past the last unread word
  __device__ __forceinline__ uint32_t pop(uint32_t back) const {
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr - 2u * back));
    return v;
  }
  __device__ __forceinline__ void retreat(uint32_t cnt) { addr -= 2u * cnt; }
};
struct GmemStream {
  const uint16_t* p;  // one past the last unread word
  __device__ __forceinline__ uint32_t pop(uint32_t back) const { return __ldg(p - back); }
  __device__ __forceinline__ void retreat(uint32_t cnt) { p -= cnt; }
};

// ---------------------------------------------------------------------------
// Decode LUT, one entry per state residue (never leaves shared memory):
//   LUT64 = false: u32  [31:20] pdf  [19:8] s-cdf  [7:0] symbol
//   LUT64 = true : uint2 {pdf, (s-cdf) << 8 | symbol}   -- two fewer ALU ops per
//                  row for the unpack, twice the shared-memory footprint
// One decode step for a full row (ans/GpuANSDecode.cuh:55-105 restated); the
// returned word has the decoded symbol in its low byte.
// ---------------------------------------------------------------------------
template <int PB, bool LUT64>
struct Lut;
template <int PB>
struct Lut<PB, false> {
  typedef uint32_t Entry;
  static __device__ __forceinline__ Entry make(uint32_t pdf, uint32_t c, uint32_t sym) {
    return (pdf << 20) | (c << 8) | sym;
  }
  static __device__ __forceinline__ uint32_t step(uint32_t& state, const Entry* __restrict__ lut) {
    const uint32_t e = lut[state & ((1u << PB) - 1u)];
    // e >> 8 = pdf * 4096 + (s - cdf): the multiple of pdf is taken back out of the quotient, so the
    // (s - cdf) field needs no mask (all arithmetic mod 2^32); the -4096 folds into the shift (LEA.HI)
    state = (e >> 20) * ((state >> PB) - 4096u) + (e >> 8);
    return e;
  }
};
template <int PB>
struct Lut<PB, true> {
  typedef uint2 Entry;
  static __device__ __forceinline__ Entry make(uint32_t pdf, uint32_t c, uint32_t sym) {
    return make_uint2(pdf, (c << 8) | sym);
  }
  static __device__ __forceinline__ uint32_t step(uint32_t& state, const Entry* __restrict__ lut) {
    const uint2 e = lut[state & ((1u << PB) - 1u)];
    state = e.x * (state >> PB) + (e.y >> 8);
    return e.y;
  }
};

// refill (ans/GpuANSDecode.cuh:89-101 restated): lanes whose state dropped below 2^15 pop one
// word each, highest lane first
template <typename Stream>
__device__ __forceinline__ void refill(uint32_t& state, Stream& st, uint32_t geMask) {
  const bool rd = state < kStateMin;
  const uint32_t vote = __ballot_sync(0xffffffffu, rd);
  if (rd) state = (state << 16) + st.pop(__popc(vote & geMask));
  st.retreat(__popc(vote));
}
// shared-memory flavour in PTX: one predicate feeds the vote and the state update.  The load itself is NOT
// predicated: a predicated load leaves its destination "maybe written", which ptxas turns into one
// loop-carried register per unrolled row (16 registers of dead values in the round-1 kernel, spills in the
// free-running one).  Lanes that do not refill read at most 64 B below the stream, i.e. inside the slot's
// lane-state area, and drop the value.
template <>
__device__ __forceinline__ void refill<SmemStream>(uint32_t& state, SmemStream& st, uint32_t geMask) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .b32 v, t, a, w;\n"
      "setp.lt.u32 p, %0, 32768;\n"
      "vote.sync.ballot.b32 v, p, 0xffffffff;\n"
      "and.b32 t, v, %2;\n"
      "popc.b32 t, t;\n"
      "shl.b32 t, t, 1;\n"
      "sub.u32 a, %1, t;\n"
      "ld.shared.u16 w, [a];\n"  // unpredicated on purpose (see below)
      "@p mad.lo.u32 %0, %0, 65536, w;\n"
      "popc.b32 t, v;\n"
      "shl.b32 t, t, 1;\n"
      "sub.u32 %1, %1, t;\n"
      "}\n"
      : "+r"(state), "+r"(st.addr)
      : "r"(geMask));
}

template <int PB, bool LUT64, typename Stream>
__device__ __forceinline__ uint32_t decodeStep(uint32_t& state,
                                               const typename Lut<PB, LUT64>::Entry* __restrict__ lut,
                                               Stream& st, uint32_t geMask) {
  const uint32_t e = Lut<PB, LUT64>::step(state, lut);
  refill(state, st, geMask);
  return e;
}

template <int PB, bool LUT64, typename Stream>
__device__ __forceinline__ uint32_t decodeStepPartial(bool valid, uint32_t& state,
                                                      const typename Lut<PB, LUT64>::Entry* __restrict__ lut,
                                                      Stream& st, uint32_t geMask) {
  uint32_t s2 = state;
  const uint32_t e = Lut<PB, LUT64>::step(s2, lut);
  if (valid) state = s2;
  const bool rd = valid && state < kStateMin;
  const uint32_t vote = __ballot_sync(0xffffffffu, rd);
  if (rd) state = (state << 16) + st.pop(__popc(vote & geMask));
  st.retreat(__popc(vote));
  return e;
}

template <int KIND, int PB, bool LUT64, typename Stream, int J>
struct RowGroup {
  typedef RowWriter<KIND> W;
  // rows J-1 .. 0 of the group, highest first (the decoder walks rows backwards)
  static __device__ __forceinline__ void run(uint32_t& state,
                                             const typename Lut<PB, LUT64>::Entry* __restrict__ lut,
                                             Stream& st, uint32_t geMask, const W& wr,
                                             const typename W::Cursor& c) {
    const uint32_t e = decodeStep<PB, LUT64>(state, lut, st, geMask);
    wr.template write<J - 1>(c, e);
    RowGroup<KIND, PB, LUT64, Stream, J - 1>::run(state, lut, st, geMask, wr, c);
  }
};
template <int KIND, int PB, bool LUT64, typename Stream>
struct RowGroup<KIND, PB, LUT64, Stream, 0> {
  typedef RowWriter<KIND> W;
  static __device__ __forceinline__ void run(uint32_t&, const typename Lut<PB, LUT64>::Entry* __restrict__, Stream&,
                                             uint32_t, const W&, const typename W::Cursor&) {}
};

template <int KIND, int PB, bool LUT64, typename Stream>
__device__ __forceinline__ void decodeBlockWarp(uint32_t state, Stream st, uint32_t n,
                                                const typename Lut<PB, LUT64>::Entry* __restrict__ lut,
                                                const RowWriter<KIND>& wr, uint32_t lane) {
  typedef typename RowWriter<KIND>::Cursor Cursor;
  constexpr int U = kGroupRows;
  typedef RowGroup<KIND, PB, LUT64, Stream, U> G;
  const uint32_t geMask = laneMaskGe();
  uint32_t row = n >> 5;  // number of full rows; the partial row (if any) has this index
  const uint32_t rem = n & 31u;
  // groups of U full rows are walked from the top: group k covers rows [row0 - U*(k+1), row0 - U*k)
  const uint32_t row0 = row;
  const uint32_t groups = row0 / U;
  // stored bytes of the first two groups are requested before anything else (the barrier: every lane is done
  // reading the ring slots of the previous block)
  __syncwarp();
  if (groups > 0) wr.issue(row0 - U, 0);
  cpAsyncCommit();
  if (groups > 1) wr.issue(row0 - 2 * U, 1);
  cpAsyncCommit();
  if (rem) {
    const bool valid = lane < rem;
    const uint32_t e = decodeStepPartial<PB, LUT64>(valid, state, lut, st, geMask);
    if constexpr (isSparseKind(reduceArchiveKind(KIND)))
      wr.writePartial(row, e, valid);  // its ballot needs every lane
    else if (valid)
      wr.writeSlow(row, e);
  }
  uint32_t slot = 0, slotNext = 2;  // ring slots of group k and of group k + 2
  for (uint32_t k = 0; k < groups; ++k) {
    row -= U;
    cpAsyncWait<1>();  // group k has landed (group k + 1 may still be in flight)
    // one warp barrier does both jobs: every lane sees group k, and every lane is done reading group k - 1,
    // whose ring slot the request below overwrites (three slots: current + two in flight)
    __syncwarp();
    if (k + 2 < groups) wr.issue(row - 2 * U, slotNext);
    cpAsyncCommit();
    const Cursor c = wr.at(row, slot);
    G::run(state, lut, st, geMask, wr, c);
    slot = slot + 1 == kRingSlots ? 0u : slot + 1;
    slotNext = slotNext + 1 == kRingSlots ? 0u : slotNext + 1;
  }
  while (row > 0) {
    --row;
    const uint32_t e = decodeStep<PB, LUT64>(state, lut, st, geMask);
    wr.writeSlow(row, e);
  }
}

// LUT build from the archive's u16 pdf[256] (ans/GpuANSDecode.cuh:405-476
// restated; runs inside the decode CTA).  blockDim.x == WARPS*32.
template <int PB, bool LUT64, int WARPS>
__device__ void buildLut(const uint8_t* __restrict__ ans, typename Lut<PB, LUT64>::Entry* __restrict__ lut,
                         uint32_t* sPdf, uint32_t* sCdf, uint32_t* sWarp) {
  constexpr int T = WARPS * 32;
  constexpr int PER = (kNumSymbols + T - 1) / T;
  const uint16_t* pdfIn = reinterpret_cast<const uint16_t*>(ans + kAnsHeaderBytes);
  // contiguous PER symbols per thread so one block scan gives the cdf
  uint32_t p[PER];
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const uint32_t sym = threadIdx.x * PER + k;
    p[k] = sym < kNumSymbols ? (uint32_t)__ldg(pdfIn + sym) : 0u;
    s += p[k];
  }
  uint32_t tot;
  uint32_t c = blockExclusiveScan<T>(s, sWarp, &tot);
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const uint32_t sym = threadIdx.x * PER + k;
    if (sym < kNumSymbols) { sPdf[sym] = p[k]; sCdf[sym] = c; }
    c += p[k];
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  for (uint32_t sym = warp; sym < kNumSymbols; sym += WARPS) {
    const uint32_t pdf = sPdf[sym], begin = sCdf[sym];
    for (uint32_t j = lane; j < pdf; j += 32u) {
      if (begin + j < (1u << PB)) lut[begin + j] = Lut<PB, LUT64>::make(pdf, j, sym);
    }
  }
  __syncthreads();
}

template <int KIND, int PB, int WARPS, bool STAGE, bool LUT64>
__global__ void __launch_bounds__(WARPS * 32, DGB_DECODE_WARPS_PER_SM / WARPS)
decodeKernel(DecodeScratch sc, uint32_t m0, uint32_t m1, uint32_t part, uint32_t slotWords) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr uint32_t K = 1u << PB;
  typedef typename Lut<PB, LUT64>::Entry Entry;
  __shared__ __align__(16) Entry lut[K];  // static: constant base address for the hot LDS
  uint32_t* sPdf = reinterpret_cast<uint32_t*>(smem);
  uint32_t* sCdf = sPdf + kNumSymbols;
  uint32_t* sWarp = sCdf + kNumSymbols;           // 32 words
  uint32_t* sMisc = sWarp + 32;                   // 32 words
  unsigned long long* sBar = reinterpret_cast<unsigned long long*>(sMisc + 32);  // [WARPS]
  uint8_t* sRing = reinterpret_cast<uint8_t*>(sBar + ((WARPS + 1) & ~1));  // [WARPS] stored-byte rings
  constexpr uint32_t ringBytes = kRingSlots * RowWriter<KIND>::kRingSlotBytes;
  uint8_t* sSlots = sRing + WARPS * ringBytes;
  const uint32_t slotBytes = 128u + slotWords * 2u;  // lane states + stream

  const uint32_t t = threadIdx.x, lane = t & 31u;
  // shuffle makes the warp index provably warp-uniform, so the vote in the hot loop needs no
  // divergence check (BRA.DIV)
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  uint8_t* mySlot = sSlots + (size_t)warp * slotBytes;
  const uint32_t myBar = smemAddr(sBar + warp);
  uint32_t phase = 0;
  if (STAGE) {
    if (lane == 0) mbarInit(myBar, 1);
    fenceBarrierInit();
    __syncthreads();
  }

  const uint32_t total = __ldcg(sc.totals + part);
  // contiguous, balanced run of flat blocks for this CTA
  const uint64_t g = gridDim.x;
  uint32_t cur = (uint32_t)((uint64_t)total * blockIdx.x / g);
  const uint32_t end = (uint32_t)((uint64_t)total * (blockIdx.x + 1) / g);

  while (cur < end) {
    // member containing flat block `cur`: the last member whose first block <= cur (members
    // that contribute no blocks share their successor's start and are skipped by the search)
    if (t == 0) {
      uint32_t lo = m0, hi = m1;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldcg(&sc.members[mid].work0) <= cur) lo = mid; else hi = mid;
      }
      sMisc[0] = lo;
    }
    __syncthreads();
    const uint32_t m = sMisc[0];
    const MemberDesc md = sc.members[m];
    const ArchiveView av = openArchive<KIND>(static_cast<const uint8_t*>(md.in));
    const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(av.ans));
    const uint32_t nb = h0.y;
    const uint32_t memberFirst = __ldcg(&sc.members[m].work0);
    const uint32_t memberEnd = min(end, memberFirst + nb);
    buildLut<PB, LUT64, WARPS>(av.ans, lut, sPdf, sCdf, sWarp);

    const uint8_t* pStates = av.ans + kAnsHeaderBytes + kAnsPdfBytes;
    const uint2* pBlockWords = reinterpret_cast<const uint2*>(pStates + 128u * (size_t)nb);
    const uint16_t* pData = reinterpret_cast<const uint16_t*>(
        reinterpret_cast<const uint8_t*>(pBlockWords) + 8u * (size_t)roundUp(nb, 2u));
    const bool canStage = STAGE && ((reinterpret_cast<uintptr_t>(av.ans) & 15u) == 0);

    RowWriter<KIND> wr;
    wr.setRing(smemAddr(sRing + warp * ringBytes), lane);
    for (uint32_t fb = cur + warp; fb < memberEnd; fb += WARPS) {
      const uint32_t block = fb - memberFirst;
      const uint2 bw = __ldg(pBlockWords + block);
      const uint32_t blockLen = bw.x >> 16, words = bw.x & 0xffffu;
      const uint16_t* stream = pData + bw.y;
      wr.setBlock(av, md.out, block, lane);
      // two call sites on purpose: each knows the address space of the stream
      if (canStage && words <= slotWords && (bw.y & 7u) == 0u) {
        const uint32_t streamBytes = roundUp(words, 8u) * 2u;
        __syncwarp();
        if (lane == 0) {
          mbarExpectTx(myBar, 128u + streamBytes);
          bulkLoad(smemAddr(mySlot), pStates + 128u * (size_t)block, 128u, myBar);
          if (streamBytes) bulkLoad(smemAddr(mySlot + 128), stream, streamBytes, myBar);
        }
        mbarWait(myBar, phase);
        phase ^= 1u;
        const uint32_t state = reinterpret_cast<const uint32_t*>(mySlot)[lane];
        SmemStream st{smemAddr(mySlot + 128) + 2u * words};
        decodeBlockWarp<KIND, PB, LUT64>(state, st, blockLen, lut, wr, lane);
      } else {
        const uint32_t state = __ldg(reinterpret_cast<const uint32_t*>(pStates) + block * 32u + lane);
        GmemStream st{stream + words};
        decodeBlockWarp<KIND, PB, LUT64>(state, st, blockLen, lut, wr, lane);
      }
    }
    cur = memberEnd;
    __syncthreads();  // everyone done with this member's LUT before it is rebuilt
  }
}

// ---------------------------------------------------------------------------
// Single-launch decoder (default).  One persistent grid, no plan kernel, no sub-batches.  The host
// knows every member's capacity, hence an upper bound on its 4 KiB block count (work0; at least one
// so that every header is visited), and zeroes one claim counter per member.  A CTA LEASES a
// member: it reads and validates the header(s), builds the decode LUT once, and then each of its
// warps claims blocks of that member one at a time with an atomic (the next claim is issued before
// the current block is decoded, so its latency hides) until none are left; only then do the warps
// meet at a barrier and the CTA moves on to the next member that still has unclaimed blocks,
// starting from its home member.  Several CTAs lease the same member at once, so the work balances
// at block granularity and the kernel has no per-block or per-chunk CTA barrier (the static split
// of the two-kernel path leaves SMs idle while the longest members finish).  The first CTA to lease a
// member reports outSuccess / outSize (ans/GpuANSDecode.cuh:326-341 semantics); claims past the
// archive's real block count, or of a member that failed, are dropped.
// Tried and rejected: a variant without the lease-end barrier -- two LUT buffers per CTA, a generation
// counter, the first warp to run dry builds the next LUT alone while the others keep decoding -- was
// slower on every workload: a member runs dry for all of its warps within one block time, so they all
// arrive together anyway and then wait for a single-warp LUT build instead of sharing it.
// ---------------------------------------------------------------------------
constexpr uint32_t kNoMember = 0xffffffffu;

template <int KIND, int PB, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, DGB_DECODE_WARPS_PER_SM / WARPS)
decodeFusedKernel(DecodeScratch sc, const __grid_constant__ InlineMembers im, uint32_t n, uint32_t slotWords,
                  uint8_t* __restrict__ outSuccess, uint32_t* __restrict__ outSize, bool wantChecksum) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr uint32_t K = 1u << PB;
  typedef typename Lut<PB, false>::Entry Entry;
  __shared__ __align__(16) Entry lut[K];  // static: constant base address for the hot LDS
  uint32_t* sPdf = reinterpret_cast<uint32_t*>(smem);
  uint32_t* sCdf = sPdf + kNumSymbols;
  uint32_t* sWarp = sCdf + kNumSymbols;           // 32 words
  uint32_t* sMisc = sWarp + 32;                   // 32 words
  unsigned long long* sBar = reinterpret_cast<unsigned long long*>(sMisc + 32);  // [WARPS]
  uint8_t* sRing = reinterpret_cast<uint8_t*>(sBar + ((WARPS + 1) & ~1));  // [WARPS] stored-byte rings
  constexpr uint32_t ringBytes = kRingSlots * RowWriter<KIND>::kRingSlotBytes;
  uint8_t* sSlots = sRing + WARPS * ringBytes;
  const uint32_t slotBytes = 128u + slotWords * 2u;  // lane states + stream

  const uint32_t t = threadIdx.x, lane = t & 31u;
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  uint8_t* mySlot = sSlots + (size_t)warp * slotBytes;
  const uint32_t myBar = smemAddr(sBar + warp);
  uint32_t phase = 0;
  if (lane == 0) mbarInit(myBar, 1);
  fenceBarrierInit();
  __syncthreads();

  uint32_t cursor = (uint32_t)((uint64_t)blockIdx.x * n / gridDim.x);  // home member (used by warp 0)

  for (;;) {
    // ---- lease: the first member at or after the cursor of which this CTA can still claim a block
    //      (the claim comes first: a CTA that arrives when others have just taken the last blocks
    //      moves on without reading the header or building the LUT) ----
    if (warp == 0) {
      uint32_t pick = kNoMember, firstBlock = 0, tries = 0;
      while (tries < n) {
        // 32 members at a time
        uint32_t mm = cursor + lane;
        if (mm >= n) mm -= n;
        bool has = false;
        if (tries + lane < n) has = *reinterpret_cast<volatile uint32_t*>(sc.next + mm) < memberWork0(im, sc.members, mm);
        const uint32_t mask = __ballot_sync(0xffffffffu, has);
        if (mask == 0u) {
          tries += 32u;
          cursor = (cursor + 32u) % n;
          continue;
        }
        const uint32_t first = (uint32_t)__ffs((int)mask) - 1u;
        uint32_t cand = cursor + first;
        if (cand >= n) cand -= n;
        uint32_t c = 0;
        if (lane == 0) c = atomicAdd(sc.next + cand, 1u);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c < memberWork0(im, sc.members, cand)) {
          pick = cand;
          firstBlock = c;
          cursor = cand;
          break;
        }
        tries += first + 1u;  // lost the race for its last block
        cursor = cand + 1 == n ? 0u : cand + 1;
      }
      if (lane == 0) { sMisc[0] = pick; sMisc[1] = firstBlock; }
    }
    __syncthreads();
    const uint32_t m = sMisc[0];
    if (m == kNoMember) break;
    const MemberDesc md = memberAt(im, sc.members, m);
    const uint32_t blocksCap = md.work0;

    // ---- header(s), validity, LUT ----
    const ArchiveView av = openArchive<KIND>(static_cast<const uint8_t*>(md.in));
    bool ok = av.ok;
    uint32_t need = 0, nb = 0;
    if (ok) {
      const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(av.ans));
      const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(av.ans) + 1);
      nb = h0.y;
      need = h0.z;  // uncompressed bytes == float words for float kinds
      ok = h0.x == kAnsMagicVersion && (int)(h1.x & 0xfu) == PB && nb == divUp(need, kBlockBytes);
      if (KIND != kKindBytes) ok = ok && need == av.floatWords;
    }
    // ans/GpuANSDecode.cuh:326-337: success iff capacity suffices; size reported regardless
    const bool memberOk = ok && md.size >= need;
    if (t == 0 && atomicExch(sc.seen + m, 1u) == 0u) {
      if (outSuccess) outSuccess[m] = memberOk ? 1 : 0;
      if (outSize) outSize[m] = ok ? need : 0u;
      if (wantChecksum) {
        const uint2 ck = memberOk ? storedChecksumOf<KIND>(md.in, av.ans) : make_uint2(0u, 0u);
        sc.archiveChecksum[m] = ck.y;
        sc.sizes[m] = ck.x ? need : 0u;
      }
    }
    const bool work = memberOk && nb > 0;
    if (work) buildLut<PB, false, WARPS>(av.ans, lut, sPdf, sCdf, sWarp);

    const uint8_t* pStates = av.ans + kAnsHeaderBytes + kAnsPdfBytes;
    const uint2* pBlockWords = reinterpret_cast<const uint2*>(pStates + 128u * (size_t)nb);
    const uint16_t* pData = reinterpret_cast<const uint16_t*>(
        reinterpret_cast<const uint8_t*>(pBlockWords) + 8u * (size_t)roundUp(nb, 2u));
    const bool canStage = (reinterpret_cast<uintptr_t>(av.ans) & 15u) == 0;
    RowWriter<KIND> wr;
    wr.setRing(smemAddr(sRing + warp * ringBytes), lane);

    // ---- every warp claims blocks of the member until none are left ----
    uint32_t block = sMisc[1];  // warp 0 starts with the block claimed with the lease
    if (warp != 0) {
      if (lane == 0) block = atomicAdd(sc.next + m, 1u);
      block = __shfl_sync(0xffffffffu, block, 0);
    }
    while (block < blocksCap) {
      uint32_t nextBlock = 0;
      if (lane == 0) nextBlock = atomicAdd(sc.next + m, 1u);  // in flight while this block is decoded
      if (work && block < nb) {
        const uint2 bw = __ldg(pBlockWords + block);
        const uint32_t blockLen = bw.x >> 16, words = bw.x & 0xffffu;
        const uint16_t* stream = pData + bw.y;
        wr.setBlock(av, md.out, block, lane);
        // two call sites on purpose: each knows the address space of the stream
        if (canStage && words <= slotWords && (bw.y & 7u) == 0u) {
          const uint32_t streamBytes = roundUp(words, 8u) * 2u;
          __syncwarp();
          if (lane == 0) {
            if constexpr (copiesSegment(KIND)) {
              // the block's stored bytes ride on the same mbarrier
              mbarExpectTx(myBar, 128u + streamBytes + wr.bulkBytes());
              wr.bulkIssue(myBar);
            } else {
              mbarExpectTx(myBar, 128u + streamBytes);
            }
            bulkLoad(smemAddr(mySlot), pStates + 128u * (size_t)block, 128u, myBar);
            if (streamBytes) bulkLoad(smemAddr(mySlot + 128), stream, streamBytes, myBar);
          }
          mbarWait(myBar, phase);
          phase ^= 1u;
          const uint32_t state = reinterpret_cast<const uint32_t*>(mySlot)[lane];
          SmemStream st{smemAddr(mySlot + 128) + 2u * words};
          decodeBlockWarp<KIND, PB, false>(state, st, blockLen, lut, wr, lane);
        } else {
          if constexpr (copiesSegment(KIND)) wr.copySync();
          const uint32_t state = __ldg(reinterpret_cast<const uint32_t*>(pStates) + block * 32u + lane);
          GmemStream st{stream + words};
          decodeBlockWarp<KIND, PB, false>(state, st, blockLen, lut, wr, lane);
        }
      }
      block = __shfl_sync(0xffffffffu, nextBlock, 0);
    }
    __syncthreads();  // every warp is done with this member's LUT (and sMisc) before the next lease
  }
}

// XOR checksum of decoded outputs (ans/GpuChecksum.cuh:26-93 semantics: XOR of
// all bytes folded to 8 bits).  grid = (n, Y).
#if !defined(DGB_DECODE_NARROW_TU) && !defined(DGB_DECODE_NORM_TU) && !defined(DGB_DECODE_FP8_TU)
__global__ void __launch_bounds__(256)
checksumKernel(DecodeScratch sc) {
  const uint32_t m = blockIdx.x;
  const uint8_t* p = static_cast<const uint8_t*>(sc.members[m].out);
  const uint32_t size = sc.sizes[m];
  uint32_t x = 0;
  for (uint32_t i = blockIdx.y * blockDim.x + threadIdx.x; i < size; i += gridDim.y * blockDim.x)
    x ^= p[i];
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, d);
  if ((threadIdx.x & 31) == 0 && x) atomicXor(sc.checksum + m, x & 0xffu);
}
#endif

struct DecodePlan {
  size_t members, next, totals, checksum, archiveChecksum, sizes, total;
};

DecodePlan planDecodeScratch(uint32_t n) {
  DecodePlan p{};
  size_t o = 0;
  p.members = o; o = alignUp256(o + sizeof(MemberDesc) * (size_t)n);
  p.next = o; o = alignUp256(o + 8 * (size_t)n);  // next[n] then seen[n]
  p.totals = o; o = alignUp256(o + 4 * kMaxParts);
  p.checksum = o; o = alignUp256(o + 4 * (size_t)n);
  p.archiveChecksum = o; o = alignUp256(o + 4 * (size_t)n);
  p.sizes = o; o = alignUp256(o + 4 * (size_t)n);
  p.total = o;
  return p;
}

// Staging slot per warp (u16 words) and dynamic shared memory of a decoder CTA of `warps` warps.  The slot
// covers the worst case for raw bytes; float kinds code exponent-like bytes that compress well, so a
// smaller slot (more resident warps) covers them and rare larger blocks take the direct-from-global path
// inside the kernel.
template <int KIND, int PB>
size_t decoderSmem(int warps, const Options& opt, uint32_t* slotWords) {
  // fp64's stored-plane ring is 10.5 KiB per warp: with a 1024-word slot two 8-warp CTAs fit on an SM
  // fp8 archives code whole words, about 7 bits each for gradients: the worst-case slot, as for byte archives
  uint32_t slot = opt.decode_slot_words > 0 ? (uint32_t)opt.decode_slot_words
                                            : (KIND == kKindBytes || isFp8Kind(KIND) ? maxBlockWords(PB)
                                                                                    : (KIND == kKindF64 ? 1024u : 1536u));
  slot = std::min(roundUp(slot, 8u), maxBlockWords(PB));
  *slotWords = slot;
  return (2 * kNumSymbols + 64) * 4 + ((warps + 1) & ~1) * 8 + (size_t)warps * kRingSlots * RowWriter<KIND>::kRingSlotBytes +
         (size_t)warps * (128u + slot * 2u);
}

// Two-kernel path (option decode_fused=0) for members [m0, m1): planKernel, then decodeKernel.  One
// decoder variant is shipped per (kind, probBits): 8 warps per CTA, TMA-staged streams, 4-byte LUT
// entries (4 warps, direct-from-global streams and 8-byte LUT entries are not instantiated).
template <int KIND, int PB>
int launchPlanDecode(const Options& opt, const DecodeScratch& sc, bool checksum, uint32_t m0, uint32_t m1, uint32_t part,
                     uint64_t blockBound, uint8_t* outSuccess, uint32_t* outSize, cudaStream_t stream) {
  timerBegin(opt, kSlotPlan, stream);
  planKernel<KIND><<<1, 1024, 0, stream>>>(sc, m0, m1, part, PB, outSuccess, outSize, checksum);
  DGB_CUDA_TRY(cudaGetLastError());
  timerEnd(opt, kSlotPlan, stream);

  constexpr int kWarps = 8;
  auto kern = decodeKernel<KIND, PB, kWarps, true, false>;
  uint32_t slotWords;
  const size_t smemBytes = decoderSmem<KIND, PB>(kWarps, opt, &slotWords);
  int perSm = 1;
  const int rc = residentCtasPerSm((const void*)kern, kWarps * 32, smemBytes, 160 * 1024, &perSm);
  if (rc != DGB_OK) return rc;
  // one resident wave; every warp gets the same number of blocks (rounds) when the batch is
  // large, so no warp idles at the CTA barrier waiting for a neighbour's extra block
  const uint64_t resident = (uint64_t)perSm * smCount();
  const uint64_t rounds = std::max<uint64_t>(1, (blockBound + resident * kWarps - 1) / (resident * kWarps));
  const uint64_t want = (blockBound + kWarps * rounds - 1) / (kWarps * rounds);
  const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(want, resident));
  timerBegin(opt, kSlotDecode, stream);
  kern<<<grid, kWarps * 32, smemBytes, stream>>>(sc, m0, m1, part, slotWords);
  DGB_CUDA_TRY(cudaGetLastError());
  timerEnd(opt, kSlotDecode, stream);
  return DGB_OK;
}

// Single-launch decoder (the default) with WARPS warps per CTA.
template <int KIND, int PB, int WARPS>
int launchDecodeFused(const Options& opt, const DecodeScratch& sc, const InlineMembers& im, uint32_t n,
                      uint64_t totalChunks, uint8_t* outSuccess, uint32_t* outSize, bool checksum, cudaStream_t stream) {
  auto kern = decodeFusedKernel<KIND, PB, WARPS>;
  uint32_t slotWords;
  const size_t smemBytes = decoderSmem<KIND, PB>(WARPS, opt, &slotWords);
  int perSm = 1;
  const int rc = residentCtasPerSm((const void*)kern, WARPS * 32, smemBytes, 160 * 1024, &perSm);
  if (rc != DGB_OK) return rc;
  const uint64_t resident = (uint64_t)perSm * smCount();
  const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(resident, totalChunks));
  timerBegin(opt, kSlotDecode, stream);
  kern<<<grid, WARPS * 32, smemBytes, stream>>>(sc, im, n, slotWords, outSuccess, outSize, checksum);
  DGB_CUDA_TRY(cudaGetLastError());
  timerEnd(opt, kSlotDecode, stream);
  return DGB_OK;
}

// ---------------------------------------------------------------------------
// Decode-and-sum (dgb_float_decompress_reduce, no reference counterpart).  G groups of W archives of one dense
// fp16 / bf16 / fp32 kind; out[g] = (accumulate ? out[g] : x(g,0)) + x(g,1) + ... + x(g,W-1), left to right, each
// add one IEEE round-to-nearest-even add in the element type with subnormals kept.  A CTA leases a GROUP (the
// single-launch decoder's lease / claim / seen pattern over groups), checks the headers of all W archives, builds
// one LUT per archive of the current pass, and each warp claims a 4 KiB block index k and decodes block k of
// every archive of the pass in archive order.  Lane l owns the same elements of block k in every archive, so
// its running sums are its own earlier stores (program order, no atomics, no cross-lane traffic), and the sum
// order per element is fixed whatever the grid, the claims or the passes: the result is bit-reproducible.
// The first archive of an accumulate=0 call is stored verbatim (the archive kind's own writer); every later one
// goes through an add writer (RowWriterSum, below: one writer built from the kind's flags for every decode-and-sum
// writer kind), which loads the 16 running sums of a row group when the group starts (once per group instead of
// once per row on the decode loop), adds, and stores.
// LUTs cost shared memory, so at most kReducePass archives are decoded per launch; the host issues
// ceil(W / kReducePass) launches in order and every launch after the first accumulates (DESIGN.md section 3).
// Widening sums (dgb_float_decompress_reduce_to): fp16 / bf16 archives summed into fp32 outputs.  The kernel's
// kind is then the archive kind | kWidenF32; every decoded word is converted exactly to fp32 and each add is one
// fp32 round-to-nearest-even add, which is torch's acc.float() + x.float() fold.
// Sparse sums (dgb_float_decompress_reduce_sparse): archives of type 5, 6 or 8 into outputs of the dense type, or
// types 5 and 6 into fp32.  The kernel's kind is then the sparse kind (| kWidenF32); each word comes from the sparse
// decoder's writer and is added as a dense word is, so the result is the dense sum of the same words bit for bit.
// Scaled sums (dgb_float_decompress_reduce_scaled): any of the ten kinds above | kScaled.  Every writer, the store
// of archive 0 included, replaces the decoded word x by its term s(x) (scaleWord / scaleWiden) before it stores or
// adds it; the running sum an add writer loads is not scaled.  The scale is a kernel parameter (InlineMembers::scale)
// read by these kinds only.
// ---------------------------------------------------------------------------
#ifndef DGB_REDUCE_PASS_ARCHIVES
#define DGB_REDUCE_PASS_ARCHIVES 4
#endif
constexpr uint32_t kReducePass = DGB_REDUCE_PASS_ARCHIVES;
constexpr int kReduceWarps = 8;

template <int KIND>
__device__ __forceinline__ uint32_t addWord(uint32_t a, uint32_t b) {
  if constexpr (KIND == kKindF32) {
    return __float_as_uint(__fadd_rn(__uint_as_float(a), __uint_as_float(b)));
  } else {
    unsigned short r;
    if constexpr (KIND == kKindF16)
      asm("add.rn.f16 %0, %1, %2;" : "=h"(r) : "h"((unsigned short)a), "h"((unsigned short)b));
    else
      asm("add.rn.bf16 %0, %1, %2;" : "=h"(r) : "h"((unsigned short)a), "h"((unsigned short)b));
    return r;
  }
}
// running-sum loads of a row group, volatile so that they are issued when the group starts
__device__ __forceinline__ uint32_t ldGlobalU16(const uint16_t* p) {
  uint32_t v;
  asm volatile("ld.global.u16 %0, [%1];" : "=r"(v) : "l"(__cvta_generic_to_global(p)));
  return v;
}
__device__ __forceinline__ uint32_t ldGlobalU32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(__cvta_generic_to_global(p)));
  return v;
}

// The exact fp32 value of a joined fp16 / bf16 word.  join leaves garbage above bit 15 (the 16-bit store drops
// it), so the widening takes the low half only.
template <int KIND>
__device__ __forceinline__ uint32_t widenWord(uint32_t w) {
  if constexpr (KIND == kKindBF16) {
    return w << 16;
  } else if constexpr (isFp8Kind(KIND)) {
    // an fp8 word (low byte; the byte above it is dropped) to f16 and f16 to fp32, both exact
    uint32_t h;
    if constexpr (KIND == kKindE4M3)
      asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"((unsigned short)w));
    else
      asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h) : "h"((unsigned short)w));
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"((unsigned short)h));
    return __float_as_uint(f);
  } else {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"((unsigned short)w));
    return __float_as_uint(f);
  }
}

// The terms of the scaled sums.  __fmul_rn is one mul.rn.f32 that nvcc never contracts with the add that follows
// into an FFMA (a fused multiply-add rounds once, the contract twice).  scaleWord: a word of dense kind KIND times s,
// in that kind: fp32 products as they are, 16-bit words widened exactly and the fp32 product rounded back to the
// 16-bit type with round-to-nearest-even (narrowWord, which also rounds the narrowing sums' fp32 results).
// scaleWiden: a 16-bit word's fp32 product, left in fp32.
template <int KIND>
__device__ __forceinline__ uint32_t narrowWord(float p) {
  unsigned short r;
  if constexpr (KIND == kKindF16)
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(r) : "f"(p));
  else
    asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(p));
  return r;
}
template <int KIND>
__device__ __forceinline__ uint32_t scaleWord(uint32_t w, float s) {
  if constexpr (KIND == kKindF32) {
    return __float_as_uint(__fmul_rn(__uint_as_float(w), s));
  } else {
    return narrowWord<KIND>(__fmul_rn(__uint_as_float(widenWord<KIND>(w)), s));
  }
}
template <int KIND>
__device__ __forceinline__ uint32_t scaleWiden(uint32_t w, float s) {
  return __float_as_uint(__fmul_rn(__uint_as_float(widenWord<KIND>(w)), s));
}

// The non-finite check of the device-scale sums (| kCheckFinite): the writer of a call's last archive passes every
// word it stores through note(), which ORs into the lane's `bad` whether the word's exponent field is all ones (inf
// or NaN) in SK, the stored type; decodeReduceBlock votes over the warp once per block.  Lanes that store nothing
// (past the end of a partial row, or every lane of a group left unwritten) never call note().
template <int SK>
__device__ __forceinline__ bool nonFiniteWord(uint32_t w) {
  constexpr uint32_t e = SK == kKindF32 ? 0x7f800000u : SK == kKindF16 ? 0x7c00u : 0x7f80u;
  return (w & e) == e;
}
template <int SK>
struct FiniteCheck {
  mutable uint32_t bad = 0u;
  __device__ __forceinline__ uint32_t note(uint32_t w) const {
    bad |= nonFiniteWord<SK>(w) ? 1u : 0u;
    return w;
  }
};
struct NoFiniteCheck { static __device__ __forceinline__ uint32_t note(uint32_t w) { return w; } };
// The squared norm of the device-scale sums (| kSqNorm, with kCheckFinite): the same writer passes every word it
// stores, after note(), through noteSq(), which widens it exactly to fp64 (SK, the stored type) and adds its square
// to the lane's `sq` with one fma (v * v is exact in fp64, so this is sq + v * v).  The decoder stores a lane's
// words in descending row order, so that is the order of the lane's sum; decodeReduceBlock folds the lanes.
template <int SK>
__device__ __forceinline__ double wordF64(uint32_t w) {
  if constexpr (SK == kKindF32) return (double)__uint_as_float(w);
  else return (double)__uint_as_float(widenWord<SK>(w));
}
template <int SK>
struct SqNormSum {
  mutable double sq = 0.0;
  __device__ __forceinline__ uint32_t noteSq(uint32_t w) const {
    const double v = wordF64<SK>(w);
    sq = fma(v, v, sq);
    return w;
  }
};
struct NoSqNorm { static __device__ __forceinline__ uint32_t noteSq(uint32_t w) { return w; } };
template <bool SCALED>
struct SumScale { static constexpr float scale = 1.0f; };  // unscaled sums: combine ignores it
template <>
struct SumScale<true> { float scale; };  // the call's scale; decodeReduceBlock sets it
template <bool NARROW>
struct SumNarrowOut {};
template <>
struct SumNarrowOut<true> { uint16_t* dst; };  // this lane's element of the block in the 16-bit output

// the kind in which a decode-and-sum writer kind adds, which is the type it stores except for the narrowing writers
__host__ __device__ constexpr int reduceSumKind(int wk) {
  return (wk & kWidenF32) != 0 ? kKindF32 : denseKind(reduceArchiveKind(wk));
}
// the type a decode-and-sum writer kind stores: the sum kind, or the archive's 16-bit type (| kNarrowOut)
__host__ __device__ constexpr int reduceStoreKind(int wk) {
  return (wk & kNarrowOut) != 0 ? denseKind(reduceArchiveKind(wk)) : reduceSumKind(wk);
}

// The decode-and-sum writer of writer kind WK: the archive kind's writer B (its ring, copies and join; a sparse
// kind's segment copy or windows and kept-word cursor) and four steps on every word it decodes:
//   1. the word w from B: word<J> from the ring, wordSlow from global memory (a sparse kind's elided word is the
//      +0 or -0 it stands for and goes through the steps below like any other: -0 + -0 = -0, -0 + +0 = +0);
//   2. the term: w, or w widened exactly to fp32 (| kWidenF32: widenWord), or w times the call's scale
//      (| kScaled: scaleWord in the archive's dense type, scaleWiden when widening);
//   3. (| kAddWriter) the term added to the element's running sum with one addWord in the sum kind;
//   4. (| kNarrowOut) the fp32 result rounded once to the archive's 16-bit type (narrowWord);
//   5. (| kCheckFinite) the result noted by FiniteCheck before it is stored;
//   6. (| kSqNorm) its square added to the lane's fp64 sum by SqNormSum.
// It stores one u16 (same-type fp16 / bf16 sums, and the narrowing writers) or one u32 (fp32 and widening sums: a
// row is one 128 B store) per element.  Add writers load a row group's running sums when the group starts (volatile
// loads in at(), so they are issued there), writeSlow and writePartial the one sum they add to.  A narrowing writer
// loads its running sums from `sum`, the fp32 accumulator, and stores to `dst`, the 16-bit output; it never reads
// `dst` and never writes `sum`.  A sparse word votes across the warp, so sparse rows, the partial one too
// (writePartial), run on the whole warp, and the vote comes before the running sum is read.  The unscaled store of
// archive 0 (WK = the bare archive kind) is the archive kind's own writer.
template <int WK>
struct RowWriterSum : RowWriter<reduceArchiveKind(WK)>,
                      SumScale<(WK & kScaled) != 0>,
                      SumNarrowOut<(WK & kNarrowOut) != 0>,
                      std::conditional<(WK & kCheckFinite) != 0, FiniteCheck<reduceStoreKind(WK)>, NoFiniteCheck>::type,
                      std::conditional<(WK & kSqNorm) != 0, SqNormSum<reduceStoreKind(WK)>, NoSqNorm>::type {
  typedef RowWriter<reduceArchiveKind(WK)> B;
  static constexpr int AK = reduceArchiveKind(WK), kSumKind = reduceSumKind(WK);
  static constexpr bool kAdd = (WK & kAddWriter) != 0, kWiden = (WK & kWidenF32) != 0;
  static constexpr bool kScale = (WK & kScaled) != 0, kNarrow = (WK & kNarrowOut) != 0;
  static_assert(!kNarrow || kWiden, "a narrowing writer sums in fp32");
  static_assert((WK & kSqNorm) == 0 || (WK & kCheckFinite) != 0, "the squared norm is taken by the checking writer");
  typedef typename std::conditional<kSumKind == kKindF32, uint32_t, uint16_t>::type T;
  T* sum;
  struct Cursor {
    T* o;
    typename B::Cursor in;      // B's cursor of the group: its ring addresses (its output pointer goes unused)
    uint32_t prev[kGroupRows];  // add writers: the running sums of the group's rows
    uint16_t* d;                // narrowing writers: the group's first row in the 16-bit output
  };
  __device__ __forceinline__ void setBlock(const ArchiveView& av, void* outBase, uint32_t block, uint32_t l) {
    B::setBlock(av, outBase, block, l);
    sum = static_cast<T*>(outBase) + (size_t)block * kBlockBytes + l;
    __builtin_assume(__isGlobal(sum));
  }
  __device__ __forceinline__ Cursor at(uint32_t row, uint32_t slot) const {
    Cursor c{sum + row * 32u, B::at(row, slot)};
    if constexpr (kAdd) {
#pragma unroll
      for (int j = 0; j < kGroupRows; ++j) {
        if constexpr (sizeof(T) == 4) c.prev[j] = ldGlobalU32(c.o + j * 32);
        else c.prev[j] = ldGlobalU16(c.o + j * 32);
      }
    }
    if constexpr (kNarrow) c.d = this->dst + row * 32u;
    return c;
  }
  // steps 2 to 4 (prev: add writers only); this->note() around it is step 5.  Static, as are the unscaled scale and
  // the unchecked note: passing the writer into the store path makes the sparse fp32 add writer spill more
  static __device__ __forceinline__ uint32_t combine(uint32_t prev, uint32_t w, float s) {
    uint32_t v = w;
    if constexpr (kScale && kWiden) v = scaleWiden<denseKind(AK)>(w, s);
    else if constexpr (kScale) v = scaleWord<denseKind(AK)>(w, s);
    else if constexpr (kWiden) v = widenWord<denseKind(AK)>(w);
    if constexpr (kAdd) v = addWord<kSumKind>(prev, v);
    if constexpr (kNarrow) v = narrowWord<denseKind(AK)>(__uint_as_float(v));
    return v;
  }
  template <int J>
  __device__ __forceinline__ void write(const Cursor& c, uint32_t entry) const {
    if constexpr (kNarrow)
      c.d[J * 32] = (uint16_t)this->noteSq(this->note(combine(kAdd ? c.prev[J] : 0u, B::template word<J>(c.in, entry), this->scale)));
    else
      c.o[J * 32] = (T)this->noteSq(this->note(combine(kAdd ? c.prev[J] : 0u, B::template word<J>(c.in, entry), this->scale)));
  }
  __device__ __forceinline__ void writeSlow(uint32_t row, uint32_t entry) const {
    if constexpr (isSparseKind(AK)) {
      writePartial(row, entry, true);
    } else if constexpr (kNarrow) {
      this->dst[row * 32u] = (uint16_t)this->noteSq(this->note(combine(kAdd ? sum[row * 32u] : 0u, B::wordSlow(row, entry), this->scale)));
    } else if constexpr (kAdd) {
      T* o = sum + row * 32u;
      *o = (T)this->noteSq(this->note(combine(*o, B::wordSlow(row, entry), this->scale)));
    } else {
      sum[row * 32u] = (T)this->noteSq(this->note(combine(0u, B::wordSlow(row, entry), this->scale)));
    }
  }
  // sparse kinds: every lane takes part in the word's vote; lanes with valid = false store nothing
  __device__ __forceinline__ void writePartial(uint32_t row, uint32_t entry, bool valid) const {
    const uint32_t w = B::word(entry, valid);
    if (valid) {
      T* o = sum + row * 32u;
      if constexpr (kNarrow)
        this->dst[row * 32u] = (uint16_t)this->noteSq(this->note(combine(kAdd ? (uint32_t)*o : 0u, w, this->scale)));
      else
        *o = (T)this->noteSq(this->note(combine(kAdd ? (uint32_t)*o : 0u, w, this->scale)));
    }
  }
};
// every writer kind other than the bare archive kinds, whose own writers are above
template <int KIND>
struct RowWriter : RowWriterSum<KIND> {
  static_assert((KIND & (kAddWriter | kWidenF32 | kScaled | kCheckFinite | kNarrowOut)) != 0,
                "not a decode-and-sum writer kind");
};

// An archive may join group g iff its float header has the magic and KIND, its ANS header has PB and a block count
// consistent with its word count, and that word count is the group's output size.
template <int KIND, int PB>
__device__ __forceinline__ bool reduceArchiveOk(const void* in, uint32_t words) {
  const ArchiveView av = openArchive<KIND>(static_cast<const uint8_t*>(in));
  if (!av.ok || av.floatWords != words) return false;
  const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(av.ans));
  const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(av.ans) + 1);
  return h0.x == kAnsMagicVersion && (int)(h1.x & 0xfu) == PB && h0.z == words && h0.y == divUp(words, kBlockBytes);
}

// block `block` of one archive through writer kind WK (the single-launch decoder's block body); narrowOut: the
// group's 16-bit output, which only the narrowing writers (| kNarrowOut) store to; sqPart: the group's fp64 block
// partials, which only the squared-norm writers (| kSqNorm) store to
template <int WK, int PB>
__device__ __forceinline__ void decodeReduceBlock(const uint8_t* in, void* out, uint32_t block, uint32_t nb,
                                                  const typename Lut<PB, false>::Entry* __restrict__ lut,
                                                  uint32_t ring, uint8_t* mySlot, uint32_t myBar, uint32_t& phase,
                                                  uint32_t slotWords, uint32_t lane, float scale,
                                                  float* foundInf, void* narrowOut, double* sqPart = nullptr) {
  const ArchiveView av = openArchive<reduceArchiveKind(WK)>(in);
  const uint8_t* pStates = av.ans + kAnsHeaderBytes + kAnsPdfBytes;
  const uint2* pBlockWords = reinterpret_cast<const uint2*>(pStates + 128u * (size_t)nb);
  const uint16_t* pData = reinterpret_cast<const uint16_t*>(
      reinterpret_cast<const uint8_t*>(pBlockWords) + 8u * (size_t)roundUp(nb, 2u));
  RowWriter<WK> wr;
  wr.setRing(ring, lane);
  wr.setBlock(av, out, block, lane);
  if constexpr ((WK & kScaled) != 0) wr.scale = scale;
  if constexpr ((WK & kNarrowOut) != 0) {
    wr.dst = static_cast<uint16_t*>(narrowOut) + (size_t)block * kBlockBytes + lane;
    __builtin_assume(__isGlobal(wr.dst));
  }
  const uint2 bw = __ldg(pBlockWords + block);
  const uint32_t blockLen = bw.x >> 16, words = bw.x & 0xffffu;
  const uint16_t* stream = pData + bw.y;
  if ((reinterpret_cast<uintptr_t>(av.ans) & 15u) == 0 && words <= slotWords && (bw.y & 7u) == 0u) {
    const uint32_t streamBytes = roundUp(words, 8u) * 2u;
    __syncwarp();
    if (lane == 0) {
      if constexpr (copiesSegment(reduceArchiveKind(WK))) {
        // sparse fp16 / bf16: the block's stored bytes ride on the same mbarrier (decodeFusedKernel)
        mbarExpectTx(myBar, 128u + streamBytes + wr.bulkBytes());
        wr.bulkIssue(myBar);
      } else {
        mbarExpectTx(myBar, 128u + streamBytes);
      }
      bulkLoad(smemAddr(mySlot), pStates + 128u * (size_t)block, 128u, myBar);
      if (streamBytes) bulkLoad(smemAddr(mySlot + 128), stream, streamBytes, myBar);
    }
    mbarWait(myBar, phase);
    phase ^= 1u;
    const uint32_t state = reinterpret_cast<const uint32_t*>(mySlot)[lane];
    SmemStream st{smemAddr(mySlot + 128) + 2u * words};
    decodeBlockWarp<WK, PB, false>(state, st, blockLen, lut, wr, lane);
  } else {
    if constexpr (copiesSegment(reduceArchiveKind(WK))) wr.copySync();
    const uint32_t state = __ldg(reinterpret_cast<const uint32_t*>(pStates) + block * 32u + lane);
    GmemStream st{stream + words};
    decodeBlockWarp<WK, PB, false>(state, st, blockLen, lut, wr, lane);
  }
  if constexpr ((WK & kCheckFinite) != 0) {
    // one vote per block; every lane that saw a non-finite word would store the same 1.0f
    if (__any_sync(0xffffffffu, wr.bad != 0u) && lane == 0 && foundInf) *foundInf = 1.0f;
  }
  if constexpr ((WK & kSqNorm) != 0) {
    // the block's partial q: the xor butterfly p += shfl_xor(p, o), o = 16, 8, 4, 2, 1 (every lane ends with the
    // same value); the block is decoded once per call by this writer, so q is stored once
    double q = wr.sq;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (lane == 0) sqPart[block] = q;
  }
}

// f(std::integral_constant<int, K>()) with K the writer kind of one archive: WK when it is stored (archive a0 of a
// pass that does not add), WK | kAddWriter when it is added; | kNarrowOut as well for the last archive of a
// narrowing sum (NARROW kinds only), and | kCheckFinite for the last archive of a checked sum (CHECK kinds only, so
// the others instantiate no checking or narrowing writer), with | kSqNorm too in the squared-norm kinds (NORM)
template <int WK, bool CHECK, bool NARROW = false, bool NORM = false, typename F>
__device__ __forceinline__ void withWriterKind(bool store, bool last, F&& f) {
  if constexpr (NARROW) {
    if (last) return withWriterKind<WK | kNarrowOut, CHECK, false, NORM>(store, true, f);
  }
  if constexpr (CHECK) {
    if (last) return withWriterKind<WK | kCheckFinite | (NORM ? kSqNorm : 0), false>(store, false, f);
  }
  if (store) f(std::integral_constant<int, WK>());
  else f(std::integral_constant<int, WK | kAddWriter>());
}

// One pass: archives [a0, a1) of every group.  Member table entry g * width + j = {archive (g, j), out[g],
// out_size[g], block cap of group g}.  addFirst: archive a0 adds too (accumulate, or a later pass).  Only the
// first pass (a0 == 0) reports outSuccess.  KIND is the archive kind, | kWidenF32 for fp32 outputs, | kScaled for
// scaled sums (the scale is im.scale, in every pass), | kScaled | kDevScale for device-scale sums
// (decodeReduceDevScaleKernel: the scale is *scaleDev, read once per CTA in every pass; the writer of archive
// width - 1, the last pass's last, checks the words it stores and sets *foundInf, when not null, to 1.0f on inf or
// NaN).  The writers of a device-scale kind are the host-scaled ones: only where s comes from differs.
// | kNarrowOut (decodeReduceNarrowKernel, with kWidenF32): the members' out is the group's fp32 accumulator and
// narrowOut[g] its 16-bit output; archive width - 1 goes through the narrowing writer, which reads the accumulator
// and stores the rounded sum to narrowOut[g], and every other archive through the widening writers into the
// accumulator.
// | kSqNorm (decodeReduceNormKernel, device-scale kinds only): the writer of archive width - 1 also stores the fp64
// squared-norm partial of each block of group g to sqPart[sqOff[g] + block], and groupOk[g] records whether every
// archive of group g is valid (the fold kernel, decode_norm.cu, reads both).
template <int KIND, int PB>
__device__ __forceinline__ void decodeReduceBody(const DecodeScratch& sc, const InlineMembers& im, uint32_t groups,
                                                 uint32_t width, uint32_t a0, uint32_t a1, bool addFirst,
                                                 uint32_t slotWords, uint8_t* __restrict__ outSuccess,
                                                 const float* scaleDev, float* foundInf, void* const* narrowOut,
                                                 double* sqPart = nullptr, const uint32_t* sqOff = nullptr,
                                                 uint32_t* groupOk = nullptr) {
  constexpr int AK = reduceArchiveKind(KIND);
  constexpr bool DEV = (KIND & kDevScale) != 0;
  constexpr bool NARROW = (KIND & kNarrowOut) != 0;
  constexpr bool NORM = (KIND & kSqNorm) != 0;
  // the writer kind of archive 0; | kAddWriter for the others
  constexpr int WK = KIND & ~(kDevScale | kNarrowOut | kSqNorm);
  constexpr int WARPS = kReduceWarps;
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr uint32_t K = 1u << PB;
  typedef typename Lut<PB, false>::Entry Entry;
  static_assert(kReducePass * K * sizeof(Entry) <= 40 * 1024, "the pass's LUTs must fit static shared memory");
  __shared__ __align__(16) Entry lut[kReducePass][K];
  uint32_t* sPdf = reinterpret_cast<uint32_t*>(smem);
  uint32_t* sCdf = sPdf + kNumSymbols;
  uint32_t* sWarp = sCdf + kNumSymbols;
  uint32_t* sMisc = sWarp + 32;
  unsigned long long* sBar = reinterpret_cast<unsigned long long*>(sMisc + 32);
  uint8_t* sRing = reinterpret_cast<uint8_t*>(sBar + ((WARPS + 1) & ~1));
  constexpr uint32_t ringBytes = kRingSlots * RowWriter<AK>::kRingSlotBytes;  // every writer kind's: RowWriterSum's base
  uint8_t* sSlots = sRing + WARPS * ringBytes;
  const uint32_t slotBytes = 128u + slotWords * 2u;

  const uint32_t t = threadIdx.x, lane = t & 31u;
  const uint32_t warp = __shfl_sync(0xffffffffu, t >> 5, 0);
  uint8_t* mySlot = sSlots + (size_t)warp * slotBytes;
  const uint32_t myBar = smemAddr(sBar + warp);
  const uint32_t ring = smemAddr(sRing + warp * ringBytes);
  uint32_t phase = 0;
  if (lane == 0) mbarInit(myBar, 1);
  if constexpr (DEV) {
    if (t == 0) sMisc[3] = __float_as_uint(*scaleDev);  // the CTA's one load of the scale
  }
  fenceBarrierInit();
  __syncthreads();
  // the unscaled kinds never read it
  const float scale = DEV ? __uint_as_float(sMisc[3]) : (KIND & kScaled) != 0 ? im.scale : 1.0f;

  uint32_t cursor = (uint32_t)((uint64_t)blockIdx.x * groups / gridDim.x);
  for (;;) {
    // ---- lease a group (decodeFusedKernel's lease over groups); the first CTA to lease it reports its status ----
    if (warp == 0) {
      uint32_t pick = kNoMember, firstBlock = 0, tries = 0;
      while (tries < groups) {
        uint32_t gg = cursor + lane;
        if (gg >= groups) gg -= groups;
        bool has = false;
        if (tries + lane < groups)
          has = *reinterpret_cast<volatile uint32_t*>(sc.next + gg) < memberWork0(im, sc.members, gg * width);
        const uint32_t mask = __ballot_sync(0xffffffffu, has);
        if (mask == 0u) {
          tries += 32u;
          cursor = (cursor + 32u) % groups;
          continue;
        }
        const uint32_t first = (uint32_t)__ffs((int)mask) - 1u;
        uint32_t cand = cursor + first;
        if (cand >= groups) cand -= groups;
        uint32_t c = 0;
        if (lane == 0) c = atomicAdd(sc.next + cand, 1u);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c < memberWork0(im, sc.members, cand * width)) {
          pick = cand;
          firstBlock = c;
          cursor = cand;
          break;
        }
        tries += first + 1u;
        cursor = cand + 1 == groups ? 0u : cand + 1;
      }
      if (lane == 0) {
        sMisc[0] = pick;
        sMisc[1] = firstBlock;
        sMisc[2] = pick != kNoMember && a0 == 0 && outSuccess && atomicExch(sc.seen + pick, 1u) == 0u;
      }
    }
    __syncthreads();
    const uint32_t g = sMisc[0];
    if (g == kNoMember) break;
    const bool report = sMisc[2] != 0;
    const MemberDesc gd = memberAt(im, sc.members, g * width);
    const uint32_t blocksCap = gd.work0, nb = divUp(gd.size, kBlockBytes);
    void* nout = nullptr;
    if constexpr (NARROW) nout = narrowOut[g];
    double* gpart = nullptr;
    if constexpr (NORM) gpart = sqPart + sqOff[g];

    // ---- every archive of the group is checked before anything is stored to it: the decision depends on the
    //      headers and out_size alone, so every CTA and every pass takes the same one ----
    bool ok = true;
    for (uint32_t j = t; j < width; j += WARPS * 32) {
      const bool v = reduceArchiveOk<AK, PB>(memberAt(im, sc.members, g * width + j).in, gd.size);
      if (report) outSuccess[g * width + j] = v ? 1 : 0;
      ok = ok && v;
    }
    bool work;
    if constexpr (NORM) {
      // the same decision on every CTA and in every pass, so whichever CTA leased the group may record it
      const bool all = __syncthreads_and(ok);
      if (t == 0) groupOk[g] = all ? 1u : 0u;
      work = all && nb > 0;
    } else {
      work = __syncthreads_and(ok) && nb > 0;
    }
    if (work) {
      for (uint32_t a = a0; a < a1; ++a)
        buildLut<PB, false, WARPS>(openArchive<AK>(static_cast<const uint8_t*>(memberAt(im, sc.members, g * width + a).in)).ans,
                                   lut[a - a0], sPdf, sCdf, sWarp);
    }

    // ---- every warp claims block indices of the group until none are left; block k of every archive ----
    uint32_t block = sMisc[1];
    if (warp != 0) {
      if (lane == 0) block = atomicAdd(sc.next + g, 1u);
      block = __shfl_sync(0xffffffffu, block, 0);
    }
    while (block < blocksCap) {
      uint32_t nextBlock = 0;
      if (lane == 0) nextBlock = atomicAdd(sc.next + g, 1u);
      if (work && block < nb) {
        for (uint32_t a = a0; a < a1; ++a) {
          const uint8_t* in = static_cast<const uint8_t*>(memberAt(im, sc.members, g * width + a).in);
          // archive width - 1 writes the final value of every element: the device-scale sums check it there, and
          // the narrowing sums round it there
          withWriterKind<WK, DEV, NARROW, NORM>(a == a0 && !addFirst, a + 1 == width, [&](auto wk) {
            constexpr int W = decltype(wk)::value;
            decodeReduceBlock<W, PB>(in, gd.out, block, nb, lut[(W & kAddWriter) != 0 ? a - a0 : 0u], ring, mySlot,
                                     myBar, phase, slotWords, lane, scale, foundInf, nout, gpart);
          });
        }
      }
      block = __shfl_sync(0xffffffffu, nextBlock, 0);
    }
    __syncthreads();  // every warp is done with the LUTs (and sMisc) before the next lease
  }
}

template <int KIND, int PB>
__global__ void __launch_bounds__(kReduceWarps * 32, 4)
decodeReduceKernel(DecodeScratch sc, const __grid_constant__ InlineMembers im, uint32_t groups, uint32_t width,
                   uint32_t a0, uint32_t a1, bool addFirst, uint32_t slotWords, uint8_t* __restrict__ outSuccess) {
  static_assert((KIND & (kDevScale | kNarrowOut)) == 0, "");
  decodeReduceBody<KIND, PB>(sc, im, groups, width, a0, a1, addFirst, slotWords, outSuccess, nullptr, nullptr,
                             nullptr);
}
// the device-scale sums (KIND | kScaled | kDevScale): the same body with the scale's and the flag's pointers
template <int KIND, int PB>
__global__ void __launch_bounds__(kReduceWarps * 32, 4)
decodeReduceDevScaleKernel(DecodeScratch sc, const __grid_constant__ InlineMembers im, uint32_t groups,
                           uint32_t width, uint32_t a0, uint32_t a1, bool addFirst, uint32_t slotWords,
                           uint8_t* __restrict__ outSuccess, const float* __restrict__ scaleDev,
                           float* __restrict__ foundInf) {
  static_assert((KIND & (kScaled | kDevScale | kNarrowOut)) == (kScaled | kDevScale), "");
  decodeReduceBody<KIND, PB>(sc, im, groups, width, a0, a1, addFirst, slotWords, outSuccess, scaleDev, foundInf,
                             nullptr);
}
// the narrowing sums (archive kind | kWidenF32 | kNarrowOut, | kScaled, | kScaled | kDevScale): the same body with
// the device table of the groups' 16-bit outputs; scaleDev and foundInf are those of the device-scale kinds (null
// for the others)
template <int KIND, int PB>
__global__ void __launch_bounds__(kReduceWarps * 32, 4)
decodeReduceNarrowKernel(DecodeScratch sc, const __grid_constant__ InlineMembers im, uint32_t groups,
                         uint32_t width, uint32_t a0, uint32_t a1, bool addFirst, uint32_t slotWords,
                         uint8_t* __restrict__ outSuccess, const float* __restrict__ scaleDev,
                         float* __restrict__ foundInf, void* const* __restrict__ narrowOut) {
  static_assert((KIND & (kWidenF32 | kNarrowOut)) == (kWidenF32 | kNarrowOut), "");
  decodeReduceBody<KIND, PB>(sc, im, groups, width, a0, a1, addFirst, slotWords, outSuccess, scaleDev, foundInf,
                             narrowOut);
}
// the squared-norm sums (a device-scale kind | kSqNorm, narrowing or not; decode_norm.cu): the device-scale kernels'
// parameters, the narrowing table (null for the others), the block partials, their per-group offsets and the
// per-group validity flags
template <int KIND, int PB>
__global__ void __launch_bounds__(kReduceWarps * 32, 4)
decodeReduceNormKernel(DecodeScratch sc, const __grid_constant__ InlineMembers im, uint32_t groups,
                       uint32_t width, uint32_t a0, uint32_t a1, bool addFirst, uint32_t slotWords,
                       uint8_t* __restrict__ outSuccess, const float* __restrict__ scaleDev,
                       float* __restrict__ foundInf, void* const* __restrict__ narrowOut,
                       double* __restrict__ sqPart, const uint32_t* __restrict__ sqOff,
                       uint32_t* __restrict__ groupOk) {
  static_assert((KIND & (kScaled | kDevScale | kSqNorm)) == (kScaled | kDevScale | kSqNorm), "");
  decodeReduceBody<KIND, PB>(sc, im, groups, width, a0, a1, addFirst, slotWords, outSuccess, scaleDev, foundInf,
                             narrowOut, sqPart, sqOff, groupOk);
}

template <int KIND, int PB>
int launchDecodeReduce(const Options& opt, const DecodeScratch& sc, const InlineMembers& im, uint32_t groups,
                       uint32_t width, uint64_t totalChunks, bool accumulate, uint8_t* outSuccess, cudaStream_t stream,
                       const float* scaleDev = nullptr, float* foundInf = nullptr,
                       void* const* narrowOut = nullptr, const SqNormScratch* norm = nullptr) {
  constexpr bool DEV = (KIND & kDevScale) != 0, NARROW = (KIND & kNarrowOut) != 0, NORM = (KIND & kSqNorm) != 0;
  const void* kern;
  if constexpr (NORM) kern = (const void*)decodeReduceNormKernel<KIND, PB>;
  else if constexpr (NARROW) kern = (const void*)decodeReduceNarrowKernel<KIND, PB>;
  else if constexpr (DEV) kern = (const void*)decodeReduceDevScaleKernel<KIND, PB>;
  else kern = (const void*)decodeReduceKernel<KIND, PB>;
  uint32_t slotWords;
  const size_t smemBytes = decoderSmem<reduceArchiveKind(KIND), PB>(kReduceWarps, opt, &slotWords);
  int perSm = 1;
  const int rc = residentCtasPerSm(kern, kReduceWarps * 32, smemBytes, 160 * 1024, &perSm);
  if (rc != DGB_OK) return rc;
  const uint64_t resident = (uint64_t)perSm * smCount();
  const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(resident, totalChunks));
  for (uint32_t a0 = 0; a0 < width; a0 += kReducePass) {
    // claim counters and `seen` start at zero in every pass
    DGB_CUDA_TRY(cudaMemsetAsync(sc.next, 0, 8 * (size_t)groups * width, stream));
    timerBegin(opt, kSlotDecode, stream);
    const uint32_t a1 = std::min(width, a0 + kReducePass);
    if constexpr (NORM)
      decodeReduceNormKernel<KIND, PB><<<grid, kReduceWarps * 32, smemBytes, stream>>>(
          sc, im, groups, width, a0, a1, accumulate || a0 > 0, slotWords, outSuccess, scaleDev, foundInf, narrowOut,
          norm->part, norm->off, norm->ok);
    else if constexpr (NARROW)
      decodeReduceNarrowKernel<KIND, PB><<<grid, kReduceWarps * 32, smemBytes, stream>>>(
          sc, im, groups, width, a0, a1, accumulate || a0 > 0, slotWords, outSuccess, scaleDev, foundInf, narrowOut);
    else if constexpr (DEV)
      decodeReduceDevScaleKernel<KIND, PB><<<grid, kReduceWarps * 32, smemBytes, stream>>>(
          sc, im, groups, width, a0, a1, accumulate || a0 > 0, slotWords, outSuccess, scaleDev, foundInf);
    else
      decodeReduceKernel<KIND, PB><<<grid, kReduceWarps * 32, smemBytes, stream>>>(
          sc, im, groups, width, a0, a1, accumulate || a0 > 0, slotWords, outSuccess);
    DGB_CUDA_TRY(cudaGetLastError());
    timerEnd(opt, kSlotDecode, stream);
  }
  return DGB_OK;
}

}  // namespace

#if defined(DGB_DECODE_NARROW_TU)
// decode_narrow.cu compiles this file once more with DGB_DECODE_NARROW_TU: that module holds the narrowing sums'
// kernels and this launcher only.  In the main module their 36 kernels changed the code ptxas generated for the
// sparse fp32 decode-and-sum kernels (the same sources gave a different and longer schedule), so they are kept apart.
int launchDecodeReduceNarrow(int kind, int pb, bool scaled, const Options& opt, MemberDesc* members, uint32_t* next,
                             const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                             bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                             float* foundInf, void* const* narrowTable) {
  DecodeScratch sc{};
  sc.members = members;
  sc.next = next;
  sc.seen = next + (size_t)groups * width;
  return withKind(kind, [&](auto K) { return withPb(pb, [&](auto P) {
    constexpr int KIND = decltype(K)::value, PB = decltype(P)::value;
    if constexpr (denseKind(KIND) == kKindF16 || denseKind(KIND) == kKindBF16) {
      constexpr int NK = KIND | kWidenF32 | kNarrowOut;
      if (scaled)
        return launchDecodeReduce<NK | kScaled, PB>(opt, sc, im, groups, width, totalChunks, accumulate, outSuccess,
                                                    stream, nullptr, nullptr, narrowTable);
      if (!scaleDev)
        return launchDecodeReduce<NK, PB>(opt, sc, im, groups, width, totalChunks, accumulate, outSuccess, stream,
                                          nullptr, nullptr, narrowTable);
      return launchDecodeReduce<NK | kScaled | kDevScale, PB>(opt, sc, im, groups, width, totalChunks, accumulate,
                                                              outSuccess, stream, scaleDev, foundInf, narrowTable);
    } else {
      return (int)DGB_ERR_INVALID_ARG;  // not reached (decodeReduce checks the kind)
    }
  }); });
}
#elif !defined(DGB_DECODE_NORM_TU) && !defined(DGB_DECODE_FP8_TU)

size_t decodeTempBytes(int /*kind*/, uint32_t n) { return planDecodeScratch(n).total + 256; }

int decodeBatch(int kind, void* temp, size_t tempBytes, int pb, bool checksum, uint32_t n,
                const HostMember* members, uint8_t* outSuccess_dev, uint32_t* outSize_dev,
                uint8_t* mismatchHost, cudaStream_t stream) {
  if (n == 0) return DGB_OK;
  if (pb < 9 || pb > 11) return DGB_ERR_INVALID_ARG;
  const DecodePlan dp = planDecodeScratch(n);
  if (!temp || tempBytes < dp.total) return DGB_ERR_TEMP_TOO_SMALL;
  if (reinterpret_cast<uintptr_t>(temp) & 255u) return DGB_ERR_INVALID_ARG;
  if (checksum) {
    const int rc = checkNotCapturing(stream);  // the verification below synchronises the stream
    if (rc != DGB_OK) return rc;
  }

  const Options opt = options();  // one snapshot per call
  // the sparse kinds have only the single-launch decoder: decode_fused=0 runs it for them (INTEGRATION.md section 4)
  const bool fused = opt.decode_fused != 0 || isSparseKind(kind);
  HostStage& hs = hostStage();
  hs.decodeTable.resize(n);
  MemberDesc* desc = hs.decodeTable.data();
  const uint32_t elemBytes = wordBytes(kind);
  uint64_t totalChunks = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (!members[i].in || (members[i].size && !members[i].out)) return DGB_ERR_INVALID_ARG;
    // headers are read as 16 B vectors; the reference imposes the same alignment
    if (reinterpret_cast<uintptr_t>(members[i].in) & 15u) return DGB_ERR_INVALID_ARG;
    if (reinterpret_cast<uintptr_t>(members[i].out) & (elemBytes - 1u)) return DGB_ERR_INVALID_ARG;
    desc[i].in = members[i].in;
    desc[i].out = members[i].out;
    desc[i].size = members[i].size;  // capacity
    // single-launch path: block count bound from the capacity (>= 1: every header is visited once)
    const uint32_t blocks = std::max(1u, divUp(members[i].size, kBlockBytes));
    desc[i].work0 = fused ? blocks : 0u;
    totalChunks += divUp(blocks, 8u);
  }
  uint8_t* base = static_cast<uint8_t*>(temp);
  DecodeScratch sc;
  sc.members = reinterpret_cast<MemberDesc*>(base + dp.members);
  sc.next = reinterpret_cast<uint32_t*>(base + dp.next);
  sc.seen = sc.next + n;
  sc.totals = reinterpret_cast<uint32_t*>(base + dp.totals);
  sc.checksum = reinterpret_cast<uint32_t*>(base + dp.checksum);
  sc.archiveChecksum = reinterpret_cast<uint32_t*>(base + dp.archiveChecksum);
  sc.sizes = reinterpret_cast<uint32_t*>(base + dp.sizes);
  // member table: inside the kernel parameters when it fits (the checksum pass reads it from scratch)
  static thread_local InlineMembers im;
  const bool inlined = opt.inline_members != 0 && fused && !checksum && n <= kInlineMembers;
  im.count = inlined ? n : 0u;
  if (inlined) {
    std::memcpy(im.m, desc, sizeof(MemberDesc) * n);
  } else {
    const int rc = uploadTable(sc.members, desc, sizeof(MemberDesc) * n, stream);
    if (rc != DGB_OK) return rc;
  }
  if (checksum) DGB_CUDA_TRY(cudaMemsetAsync(sc.checksum, 0, 4 * (size_t)n, stream));

  if (fused) {
    DGB_CUDA_TRY(cudaMemsetAsync(sc.next, 0, 8 * (size_t)n, stream));
    const int rc = withKind(kind, [&](auto K) { return withPb(pb, [&](auto P) {
      constexpr int KIND = decltype(K)::value, PB = decltype(P)::value;
      // warps per CTA = warps that share one LUT and meet at the barrier when a lease ends.  Float kinds: 8 (4 is
      // equal: c3 decode 190 us either way on an H100 at 700 W, tools/walltime.py).  Byte archives need the worst-case
      // staging slot (5.1 KiB per warp), which caps 8-warp CTAs at 32 resident warps per SM; 20-warp CTAs reach 40
      // (same H100: c2 decode 249 us against 271 with 8 warps) -- used when the members are long enough to keep 20
      // warps busy through a lease.
      int w = opt.decode_warps;
      // (at 11 bits the LUT is 8 KiB and the slot 5.6 KiB per warp: a 20-warp CTA needs 126 KiB and fits once per
      // SM and gains nothing -- c2p11 decode 248 us with 20 or 8 warps on the same H100 -- so the wide CTA is used
      // up to 10 bits only)
      if (w == 0) w = (KIND == kKindBytes && PB <= 10 && totalChunks * 8u >= 160ull * n) ? 20 : 8;
      if (w == 4) return launchDecodeFused<KIND, PB, 4>(opt, sc, im, n, totalChunks, outSuccess_dev, outSize_dev, checksum, stream);
      if constexpr (KIND == kKindBytes) {
        if (w == 20)
          return launchDecodeFused<KIND, PB, 20>(opt, sc, im, n, totalChunks, outSuccess_dev, outSize_dev, checksum, stream);
      }
      return launchDecodeFused<KIND, PB, 8>(opt, sc, im, n, totalChunks, outSuccess_dev, outSize_dev, checksum, stream);
    }); });
    if (rc != DGB_OK) return rc;
  } else {
    // two-kernel path: sub-batches on internal streams: the plan kernel (pure latency) of one part
    // hides behind the decode kernel of another, and the tail of one decode kernel overlaps the next
    SubBatches parts(kind, desc, n, opt, true, stream);
    if (const int rc = parts.fork(); rc != DGB_OK) return rc;
    const int rc = withKind(kind, [&](auto K) { return withPb(pb, [&](auto P) {
      if constexpr (isSparseKind(decltype(K)::value)) {
        return (int)DGB_ERR_INVALID_ARG;  // not reached (`fused` above)
      } else {
        for (int part = 0; part < parts.count(); ++part) {
          const uint32_t m0 = parts.begin(part), m1 = parts.end(part);
          if (m1 == m0) continue;
          cudaStream_t ps;
          int prc = parts.stream(part, &ps);
          if (prc != DGB_OK) return prc;
          uint64_t partBound = 0;
          for (uint32_t i = m0; i < m1; ++i) partBound += divUp(desc[i].size, kBlockBytes);
          prc = launchPlanDecode<decltype(K)::value, decltype(P)::value>(opt, sc, checksum, m0, m1, part, partBound,
                                                                        outSuccess_dev, outSize_dev, ps);
          if (prc != DGB_OK) return prc;
        }
        return (int)DGB_OK;
      }
    }); });
    if (rc != DGB_OK) return rc;
  }  // ~SubBatches orders the helper streams before the caller's stream

  if (checksum) {
    // ans/GpuANSDecode.cuh:555-591 / float/GpuFloatDecompress.cuh:698-733: checksum the
    // output, compare with the archive's on the host (this path synchronises).
    // Float kinds: the checksum covers the first `size` BYTES (SURVEY A.6/B6); sc.sizes holds
    // the word count, which is exactly that byte count.
    const int sms = smCount();
    dim3 grid(n, std::max(1, std::min(64, 4 * sms / (int)std::max(1u, n))));
    checksumKernel<<<grid, 256, 0, stream>>>(sc);
    DGB_CUDA_TRY(cudaGetLastError());
    hs.checksum.resize(3 * (size_t)n);
    uint32_t* got = hs.checksum.data();
    uint32_t* want = got + n;
    uint32_t* sizes = want + n;
    DGB_CUDA_TRY(cudaMemcpyAsync(got, sc.checksum, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream));
    DGB_CUDA_TRY(cudaMemcpyAsync(want, sc.archiveChecksum, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream));
    DGB_CUDA_TRY(cudaMemcpyAsync(sizes, sc.sizes, 4 * (size_t)n, cudaMemcpyDeviceToHost, stream));
    DGB_CUDA_TRY(cudaStreamSynchronize(stream));
    bool bad = false;
    for (uint32_t i = 0; i < n; ++i) {
      // members that were skipped (capacity / bad header) are reported through outSuccess; members whose
      // archive has the checksum flag clear carry no checksum and have size 0 here
      const bool mm = sizes[i] != 0 && got[i] != want[i];
      if (mismatchHost) mismatchHost[i] = mm ? 1 : 0;
      bad = bad || mm;
    }
    if (bad) return DGB_ERR_CHECKSUM;
  }
  return DGB_OK;
}

int decodeReduce(int kind, int outKind, void* temp, size_t tempBytes, int pb, uint32_t groups, uint32_t width,
                 const void* const* in, void* const* out, const uint32_t* outSize, bool accumulate,
                 uint8_t* outSuccess_dev, bool sparse, const float* scale, const float* scaleDev, float* foundInf,
                 cudaStream_t stream, void* const* narrowOut, double* sqNorm) {
  // dense fp16 / bf16 / fp32 archives, or (sparse) their sparse types 5, 6 and 8; scale: null for a plain sum, else
  // the multiplier of the scaled kinds; scaleDev (device memory, read by the kernels) in place of scale for the
  // device-scale kinds, with the non-finite flag foundInf (may be null).  narrowOut (host array of G, or null): a
  // narrowing sum of fp16 / bf16 archives, whose out[g] (outKind fp32) is the group's accumulator and narrowOut[g]
  // its output of the archive's 16-bit type; out and out[g] may be null when the call reads no accumulator (W = 1
  // without accumulate).  sqNorm (device, G doubles; with scaleDev only): the squared-norm kernels (decode_norm.cu),
  // whose block partials take the scratch past the decode's own
  // fp8 byte archives (decode_fp8.cu): fp32 outputs, device scale only
  const bool fp8 = isFp8Kind(kind);
  if (fp8 ? (sparse || !scaleDev || narrowOut || outKind != kKindF32)
          : sparse ? !isSparseKind(kind) : (kind != kKindF16 && kind != kKindBF16 && kind != kKindF32))
    return DGB_ERR_INVALID_ARG;
  // outputs of the archive's dense kind, or fp32 sums of (sparse) fp16 / bf16 archives
  const int dk = denseKind(kind);
  const bool widen = outKind != dk;
  if (widen && !fp8 && !(outKind == kKindF32 && (dk == kKindF16 || dk == kKindBF16))) return DGB_ERR_INVALID_ARG;
  if (narrowOut && !widen) return DGB_ERR_INVALID_ARG;
  if (pb < 9 || pb > 11 || width == 0) return DGB_ERR_INVALID_ARG;
  if (groups == 0) return DGB_OK;
  const bool readsAcc = !narrowOut || width > 1 || accumulate;
  if (!in || (readsAcc && !out) || !outSize) return DGB_ERR_INVALID_ARG;
  const uint64_t n64 = (uint64_t)groups * width;
  if (n64 > 0xffffffffull) return DGB_ERR_INVALID_ARG;
  const uint32_t n = (uint32_t)n64;
  const DecodePlan dp = planDecodeScratch(n);
  const size_t need = dp.total + (sqNorm ? sqNormScratchBytes(groups, sqNormBlocks(groups, outSize)) : 0u);
  if (!temp || tempBytes < need) return DGB_ERR_TEMP_TOO_SMALL;
  if (reinterpret_cast<uintptr_t>(temp) & 255u) return DGB_ERR_INVALID_ARG;

  const Options opt = options();  // one snapshot per call
  HostStage& hs = hostStage();
  hs.decodeTable.resize(n);
  MemberDesc* desc = hs.decodeTable.data();
  const uint32_t elemBytes = wordBytes(outKind);
  uint64_t totalChunks = 0;
  for (uint32_t g = 0; g < groups; ++g) {
    if (narrowOut && ((outSize[g] && !narrowOut[g]) || (reinterpret_cast<uintptr_t>(narrowOut[g]) & 1u)))
      return DGB_ERR_INVALID_ARG;
    // a narrowing call that reads no accumulator never touches the members' out: the 16-bit output stands in for it
    // (any global pointer does)
    void* o = readsAcc ? out[g] : narrowOut[g];
    if (readsAcc && ((outSize[g] && !o) || (reinterpret_cast<uintptr_t>(o) & (elemBytes - 1u)))) return DGB_ERR_INVALID_ARG;
    // block cap >= 1: every group's headers are visited, so its status is reported
    const uint32_t blocks = std::max(1u, divUp(outSize[g], kBlockBytes));
    totalChunks += divUp(blocks, 8u);
    for (uint32_t j = 0; j < width; ++j) {
      const void* a = in[(size_t)g * width + j];
      if (!a || (reinterpret_cast<uintptr_t>(a) & 15u)) return DGB_ERR_INVALID_ARG;
      desc[(size_t)g * width + j] = MemberDesc{a, o, outSize[g], blocks};
    }
  }
  uint8_t* base = static_cast<uint8_t*>(temp);
  DecodeScratch sc{};
  sc.members = reinterpret_cast<MemberDesc*>(base + dp.members);
  sc.next = reinterpret_cast<uint32_t*>(base + dp.next);
  sc.seen = sc.next + n;
  static thread_local InlineMembers im;
  const bool inlined = opt.inline_members != 0 && n <= kInlineMembers;
  im.count = inlined ? n : 0u;
  if (inlined) {
    std::memcpy(im.m, desc, sizeof(MemberDesc) * n);
  } else {
    const int rc = uploadTable(sc.members, desc, sizeof(MemberDesc) * n, stream);
    if (rc != DGB_OK) return rc;
  }
  // the narrowing sums' table of 16-bit outputs: G pointers in the scratch the checksum pass of a plain decode uses,
  // 3 * 4 * n >= 8 * G bytes that no decode-and-sum touches otherwise
  im.scale = scale ? *scale : 1.0f;  // a kernel parameter: a captured launch keeps the value it was captured with
  void** t = nullptr;
  if (narrowOut) {
    t = reinterpret_cast<void**>(base + dp.checksum);
    const int rc = uploadTable(t, narrowOut, sizeof(void*) * (size_t)groups, stream);
    if (rc != DGB_OK) return rc;
  }
  if (fp8) {
    SqNormScratch ns;
    if (sqNorm) {
      const int rc = sqNormPrepare(base + dp.total, groups, outSize, &ns, stream);
      if (rc != DGB_OK) return rc;
    }
    return launchDecodeReduceFp8(kind, pb, opt, sc.members, sc.next, im, groups, width, totalChunks, accumulate,
                                 outSuccess_dev, stream, scaleDev, foundInf, sqNorm ? &ns : nullptr, sqNorm);
  }
  if (sqNorm) {
    SqNormScratch ns;
    const int rc = sqNormPrepare(base + dp.total, groups, outSize, &ns, stream);
    if (rc != DGB_OK) return rc;
    return launchDecodeReduceNorm(kind, pb, widen, opt, sc.members, sc.next, im, groups, width, totalChunks,
                                  accumulate, outSuccess_dev, stream, scaleDev, foundInf, t, ns, sqNorm);
  }
  if (narrowOut) {
    return launchDecodeReduceNarrow(kind, pb, scale != nullptr, opt, sc.members, sc.next, im, groups, width,
                                    totalChunks, accumulate, outSuccess_dev, stream, scaleDev, foundInf, t);
  }
  return withKind(kind, [&](auto K) { return withPb(pb, [&](auto P) {
    constexpr int KIND = decltype(K)::value;
    constexpr int DK = denseKind(KIND);
    // the kernel of writer kind WK, or of WK | kScaled (| kDevScale)
    // (the device-scale kernels are named last, so that every other kernel is instantiated, and compiled, in the
    // order it had before they existed)
    auto launch = [&](auto WK) {
      if (scale)
        return launchDecodeReduce<decltype(WK)::value | kScaled, decltype(P)::value>(
            opt, sc, im, groups, width, totalChunks, accumulate, outSuccess_dev, stream);
      if (!scaleDev)
        return launchDecodeReduce<decltype(WK)::value, decltype(P)::value>(opt, sc, im, groups, width, totalChunks,
                                                                          accumulate, outSuccess_dev, stream);
      return launchDecodeReduce<decltype(WK)::value | kScaled | kDevScale, decltype(P)::value>(
          opt, sc, im, groups, width, totalChunks, accumulate, outSuccess_dev, stream, scaleDev, foundInf);
    };
    if constexpr (DK == kKindF16 || DK == kKindBF16) {
      if (widen) return launch(std::integral_constant<int, KIND | kWidenF32>());
      return launch(std::integral_constant<int, KIND>());
    } else if constexpr (DK == kKindF32)
      return launch(std::integral_constant<int, KIND>());
    else
      return (int)DGB_ERR_INVALID_ARG;  // not reached (checked above)
  }); });
}

// ---------------------------------------------------------------------------
// Header queries (ans/GpuANSInfo.cuh:16-37, float/GpuFloatInfo.cuh:19-41)
// ---------------------------------------------------------------------------
namespace {
__global__ void infoKernel(int kind, const void* const* in, uint32_t n, uint32_t* outSizes,
                           uint32_t* outTypes, uint32_t* outChecksum) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* h = static_cast<const uint32_t*>(in[i]);
  if (kind == kKindBytes) {
    const bool ok = h[0] == kAnsMagicVersion;
    if (outSizes) outSizes[i] = ok ? h[2] : 0u;  // UNCOMPRESSED bytes (ans/GpuANSInfo.cuh:27-29)
    if (outChecksum) outChecksum[i] = ok ? h[5] : 0u;
  } else {
    const bool ok = h[0] == kFloatMagicVersion;
    if (outSizes) outSizes[i] = ok ? h[1] : 0u;  // float words
    if (outTypes) outTypes[i] = ok ? (h[2] & 0xfu) : 0u;
    if (outChecksum) outChecksum[i] = ok ? h[3] : 0u;
  }
}
}  // namespace

// ---------------------------------------------------------------------------
// Archive mover: copies each archive EXACTLY as long as its own header says (float header + stored planes +
// ANS header .. data section), never the padded row it sits in.  Meant for sources in peer memory
// (NVLink): the sizes never travel to the host, every thread keeps four 16 B loads in flight, and a
// small persistent grid (option "pull_ctas") saturates the link while the decode kernel of the
// previous group owns the rest of the SMs.  An archive with a bad header is copied as its first 32
// bytes, so the decoder that follows reports it; one that exceeds the destination capacity is cut
// (the decoder then fails its bounds checks on the member, never reads past the row).
// ---------------------------------------------------------------------------
namespace {
__device__ __forceinline__ uint4 ldgNc(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
constexpr uint32_t kPullThreads = 512;
constexpr uint32_t kPullChunkVecs = 4096;  // 64 KiB work units

// SPARSE: 0 for the dense kinds, else the sparse kind (fp16 and bf16 lay out their sections alike)
template <int SPARSE>
__device__ __forceinline__ uint32_t archiveBytes(int kind, const uint8_t* a) {  // inlined: kind folds where it is constant
  uint32_t extra = 0;
  if constexpr (SPARSE == kKindF32S) {
    const uint4 fh = __ldg(reinterpret_cast<const uint4*>(a));
    const uint4 sh = __ldg(reinterpret_cast<const uint4*>(a) + 1);
    if (fh.x != kFloatMagicVersion || sh.x > fh.y) return 32u;
    extra = sparseExtraBytes<uint32_t>(SPARSE, fh.y, sh.x);
  } else if constexpr (SPARSE != 0) {
    const uint4 fh = __ldg(reinterpret_cast<const uint4*>(a));
    const uint4 sh = __ldg(reinterpret_cast<const uint4*>(a) + 1);
    if (fh.x != kFloatMagicVersion || sh.x > fh.y) return 32u;
    extra = sparseExtraBytes<uint32_t>(fh.y, sh.x);
  } else if (kind != kKindBytes) {
    const uint4 fh = __ldg(reinterpret_cast<const uint4*>(a));
    if (fh.x != kFloatMagicVersion) return 32u;
    extra = kFloatHeaderBytes + floatNonCompBytes(kind, fh.y);
  }
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(a + extra));
  if (h.x != kAnsMagicVersion) return extra + 32u;
  const uint64_t total = (uint64_t)extra + ansOverhead(h.y) + 2ull * h.w;
  return total > 0xfffffff0ull ? 32u : (uint32_t)total;
}

template <int SPARSE>
__device__ __forceinline__ void pullArchivesBody(const InlineMembers& im, int kind, uint32_t* __restrict__ outBytes) {
  __shared__ uint32_t sFirst[kInlineMembers + 1];  // first chunk of member i
  __shared__ uint32_t sBytes[kInlineMembers];
  const uint32_t t = threadIdx.x, n = im.count;
  if (t < n) {
    const uint32_t want = archiveBytes<SPARSE>(kind, static_cast<const uint8_t*>(im.m[t].in));
    const uint32_t b = min(want, im.m[t].size & ~15u);
    sBytes[t] = b;
    if (outBytes && blockIdx.x == 0) outBytes[t] = want;
  }
  __syncthreads();
  if (t == 0) {
    uint32_t c = 0;
    for (uint32_t i = 0; i < n; ++i) { sFirst[i] = c; c += divUp(sBytes[i] / 16u, kPullChunkVecs); }
    sFirst[n] = c;
  }
  __syncthreads();
  const uint32_t total = sFirst[n];
  uint32_t m = 0;
  for (uint32_t c = blockIdx.x; c < total; c += gridDim.x) {
    while (sFirst[m + 1] <= c) ++m;
    const uint32_t v0 = (c - sFirst[m]) * kPullChunkVecs;
    const uint32_t v1 = min(sBytes[m] / 16u, v0 + kPullChunkVecs);
    const uint4* __restrict__ src = static_cast<const uint4*>(im.m[m].in);
    uint4* __restrict__ dst = static_cast<uint4*>(im.m[m].out);
    uint32_t v = v0 + t;
    for (; v + 3u * kPullThreads < v1; v += 4u * kPullThreads) {
      const uint4 a = ldgNc(src + v), b = ldgNc(src + v + kPullThreads), cc = ldgNc(src + v + 2u * kPullThreads),
                  d = ldgNc(src + v + 3u * kPullThreads);
      dst[v] = a; dst[v + kPullThreads] = b; dst[v + 2u * kPullThreads] = cc; dst[v + 3u * kPullThreads] = d;
    }
    for (; v < v1; v += kPullThreads) dst[v] = ldgNc(src + v);
  }
}

// byte, fp16, bf16 and fp32 archives (kind at run time)
__global__ void __launch_bounds__(kPullThreads)
pullArchivesKernel(const __grid_constant__ InlineMembers im, int kind, uint32_t* __restrict__ outBytes) {
  __builtin_assume(kind != kKindF64);
  pullArchivesBody<0>(im, kind, outBytes);
}
// fp64 archives: their own instantiation, so the kernel above keeps its plane-size arithmetic
__global__ void __launch_bounds__(kPullThreads)
pullArchivesF64Kernel(const __grid_constant__ InlineMembers im, uint32_t* __restrict__ outBytes) {
  pullArchivesBody<0>(im, kKindF64, outBytes);
}
// sparse fp16 / bf16 archives: sizes from the 32 B header
__global__ void __launch_bounds__(kPullThreads)
pullArchivesSparseKernel(const __grid_constant__ InlineMembers im, uint32_t* __restrict__ outBytes) {
  pullArchivesBody<kKindF16S>(im, kKindF16S, outBytes);
}
// sparse fp32 archives: the same header, two stored planes
__global__ void __launch_bounds__(kPullThreads)
pullArchivesSparse32Kernel(const __grid_constant__ InlineMembers im, uint32_t* __restrict__ outBytes) {
  pullArchivesBody<kKindF32S>(im, kKindF32S, outBytes);
}
}  // namespace

int pullArchives(int kind, uint32_t n, const void* const* src, void* const* dst, const uint32_t* capacity,
                 uint32_t* outBytes_dev, cudaStream_t stream) {
  if (n == 0) return DGB_OK;
  if (!src || !dst || !capacity) return DGB_ERR_INVALID_ARG;
  const Options opt = options();  // one snapshot per call
  const int ctas = std::max(1, opt.pull_ctas);
  static thread_local InlineMembers im;
  for (uint32_t i0 = 0; i0 < n; i0 += kInlineMembers) {
    const uint32_t k = std::min(kInlineMembers, n - i0);
    im.count = k;
    for (uint32_t i = 0; i < k; ++i) {
      if (!src[i0 + i] || !dst[i0 + i]) return DGB_ERR_INVALID_ARG;
      if ((reinterpret_cast<uintptr_t>(src[i0 + i]) | reinterpret_cast<uintptr_t>(dst[i0 + i])) & 15u) return DGB_ERR_INVALID_ARG;
      im.m[i].in = src[i0 + i];
      im.m[i].out = dst[i0 + i];
      im.m[i].size = capacity[i0 + i];
      im.m[i].work0 = 0;
    }
    timerBegin(opt, kSlotPull, stream);
    uint32_t* ob = outBytes_dev ? outBytes_dev + i0 : nullptr;
    if (kind == kKindF64)
      pullArchivesF64Kernel<<<ctas, kPullThreads, 0, stream>>>(im, ob);
    else if (kind == kKindF32S)
      pullArchivesSparse32Kernel<<<ctas, kPullThreads, 0, stream>>>(im, ob);
    else if (isSparseKind(kind))
      pullArchivesSparseKernel<<<ctas, kPullThreads, 0, stream>>>(im, ob);
    else
      pullArchivesKernel<<<ctas, kPullThreads, 0, stream>>>(im, kind, ob);
    DGB_CUDA_TRY(cudaGetLastError());
    timerEnd(opt, kSlotPull, stream);
  }
  return DGB_OK;
}

int getInfo(int kind, void* temp, size_t tempBytes, const void* const* in, bool inIsDevice,
            uint32_t n, uint32_t* outSizes, uint32_t* outTypes, uint32_t* outChecksum,
            cudaStream_t stream) {
  if (n == 0) return DGB_OK;
  if (!in) return DGB_ERR_INVALID_ARG;
  const void* const* in_dev = in;
  if (!inIsDevice) {
    if (!temp || tempBytes < sizeof(void*) * (size_t)n) return DGB_ERR_TEMP_TOO_SMALL;
    const int rc = uploadTable(temp, in, sizeof(void*) * (size_t)n, stream);
    if (rc != DGB_OK) return rc;
    in_dev = static_cast<const void* const*>(temp);
  }
  infoKernel<<<divUp(n, 128), 128, 0, stream>>>(kind, in_dev, n, outSizes, outTypes, outChecksum);
  DGB_CUDA_TRY(cudaGetLastError());
  return DGB_OK;
}

#endif  // DGB_DECODE_NARROW_TU, DGB_DECODE_NORM_TU, DGB_DECODE_FP8_TU

}  // namespace dgb
