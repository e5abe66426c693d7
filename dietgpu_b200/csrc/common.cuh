// common.cuh -- wire-format constants, device helpers and the internal host
// interface shared by the codec translation units.
//
// Wire format: identical to the reference's (ans/GpuANSUtils.cuh:67-227 and
// float/GpuFloatUtils.cuh:26-74, paths relative to /root/reference/dietgpu/).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>
#include <vector>

#include "../../include/dietgpu_b200.h"

namespace dgb {

// ---- format constants ------------------------------------------------------
constexpr uint32_t kBlockBytes = 4096;   // ans/GpuANSUtils.cuh:37
constexpr uint32_t kRowsPerBlock = kBlockBytes / 32;
constexpr uint32_t kNumSymbols = 256;
constexpr uint32_t kStateMin = 1u << 15; // ans/GpuANSUtils.cuh:46-49
constexpr uint32_t kAnsMagicVersion = (0xd00du << 16) | 1u;   // :52-55,105-107
constexpr uint32_t kFloatMagicVersion = (0xf00fu << 16) | 1u; // float/GpuFloatUtils.cuh:20-29
constexpr uint32_t kAnsHeaderBytes = 32;
constexpr uint32_t kAnsPdfBytes = 512;
constexpr uint32_t kFloatHeaderBytes = 16;

__host__ __device__ constexpr uint32_t divUp(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
__host__ __device__ constexpr uint32_t roundUp(uint32_t a, uint32_t b) { return divUp(a, b) * b; }
__host__ __device__ constexpr uint64_t roundUp64(uint64_t a, uint64_t b) { return (a + b - 1) / b * b; }

// ans/GpuANSUtils.cuh:68-81
__host__ __device__ constexpr uint32_t ansOverhead(uint32_t numBlocks) {
  return kAnsHeaderBytes + kAnsPdfBytes + 128u * numBlocks + 8u * roundUp(numBlocks, 2u);
}

// Stored ("non-compressed") planes of a float archive, in this order after the 16 B float header, each
// starting 16 B aligned and zero padded (float/GpuFloatUtils.cuh:123-127,163-167,194-203 for types 1-3):
//   fp16, bf16 : u8 plane
//   fp32       : u16 plane, u8 plane
//   fp64       : u32 plane, u16 plane, u8 plane  (type 4, an extension the reference does not have)
// Byte offsets relative to the first plane, in T: uint32_t on the device (every offset inside an archive
// fits 32 bits), uint64_t for the host's size bounds, which must see totals that do not.
template <class T>
__host__ __device__ constexpr T roundUpT(T a, T b) { return (a + b - 1) / b * b; }
template <class T>
__host__ __device__ constexpr T floatU16PlaneOffset(int ft, T n) {  // fp32, fp64
  return ft == DGB_FLOAT64 ? T(4) * roundUpT<T>(n, 4) : T(0);
}
template <class T>
__host__ __device__ constexpr T floatU8PlaneOffset(int ft, T n) {
  return ft == DGB_FLOAT64   ? T(4) * roundUpT<T>(n, 4) + T(2) * roundUpT<T>(n, 8)
         : ft == DGB_FLOAT32 ? T(2) * roundUpT<T>(n, 8)
                             : T(0);
}
template <class T>
__host__ __device__ constexpr T floatPlanesBytes(int ft, T n) {
  return ft == DGB_FLOAT64   ? T(4) * roundUpT<T>(n, 4) + T(2) * roundUpT<T>(n, 8) + roundUpT<T>(n, 16)
         : ft == DGB_FLOAT32 ? T(2) * roundUpT<T>(n, 8) + roundUpT<T>(n, 16)
                             : roundUpT<T>(n, 16);
}
__host__ __device__ constexpr uint32_t floatNonCompBytes(int ft, uint32_t n) { return floatPlanesBytes<uint32_t>(ft, n); }

// Sparse fp16 / bf16 archives (types 5 and 6, an extension the reference does not have): the dense type's coded
// symbol and stored byte, but +0 and -0 words are coded as two symbols no other word uses (E+, E-) and store
// nothing.  After the 32 B header (the dense 16 B, then S = words that store a byte, esc = E+ | E- << 8 | 1 << 16
// or 0 when nothing is elided, 0, 0) come a u32 per 4 KiB block (stored bytes of all earlier blocks), the S
// stored bytes in element order, and the ANS archive; every section starts 16 B aligned and is zero padded.
// Sparse fp32 (type 8) is the same layout with the dense fp32 symbol (r >> 24, r = rotl32(w, 1)) and stored bits:
// S counts the kept words, and the stored section is a u16 plane (2 roundUp(S, 8) B, r & 0xffff) followed by a u8
// plane (roundUp(S, 16) B, bits 16..23 of r), both compacted in element order; the table counts kept words.
constexpr uint32_t kSparseHeaderBytes = 32;
__host__ __device__ constexpr bool isSparseKind(int ft) {
  return ft == DGB_FLOAT16_SPARSE || ft == DGB_BFLOAT16_SPARSE || ft == DGB_FLOAT32_SPARSE;
}
__host__ __device__ constexpr int denseKind(int ft) {  // the dense type whose symbol and stored byte(s) a kind uses
  return ft == DGB_FLOAT16_SPARSE    ? DGB_FLOAT16
         : ft == DGB_BFLOAT16_SPARSE ? DGB_BFLOAT16
         : ft == DGB_FLOAT32_SPARSE  ? DGB_FLOAT32
                                     : ft;
}
template <class T>
__host__ __device__ constexpr T sparseTableBytes(T n) { return T(4) * roundUpT<T>((n + 4095) / 4096, 4); }
// header + block table + stored bytes in front of the ANS archive of a sparse fp16 / bf16 archive (S = stored bytes)
template <class T>
__host__ __device__ constexpr T sparseExtraBytes(T n, T S) {
  return T(kSparseHeaderBytes) + sparseTableBytes<T>(n) + roundUpT<T>(S, 16);
}
// the same for any sparse kind ft (S = kept words): the stored section depends on the stored width
template <class T>
__host__ __device__ constexpr T sparseStoredBytes(int ft, T S) {
  return ft == DGB_FLOAT32_SPARSE ? T(2) * roundUpT<T>(S, 8) + roundUpT<T>(S, 16) : roundUpT<T>(S, 16);
}
template <class T>
__host__ __device__ constexpr T sparseExtraBytes(int ft, T n, T S) {
  return T(kSparseHeaderBytes) + sparseTableBytes<T>(n) + sparseStoredBytes<T>(ft, S);
}
__host__ __device__ constexpr bool sparseEscValid(uint32_t esc) {
  return esc == 0u || ((esc >> 16) == 1u && (esc & 0xffu) < ((esc >> 8) & 0xffu));
}

// Worst-case u16 words one 4 KiB block can emit: every symbol costs at most
// probBits bits (a symbol of pdf 1), so 4096*pb/16 words; +8 for 16 B padding.
__host__ __device__ constexpr uint32_t maxBlockWords(int pb) { return 256u * (uint32_t)pb + 8u; }

// ---- per-member descriptor (device), built on the host ----------------------
enum CodecKind : int {
  kKindBytes = 0,
  kKindF16 = DGB_FLOAT16,
  kKindBF16 = DGB_BFLOAT16,
  kKindF32 = DGB_FLOAT32,
  kKindF64 = DGB_FLOAT64,
  kKindF16S = DGB_FLOAT16_SPARSE,
  kKindBF16S = DGB_BFLOAT16_SPARSE,
  kKindF32S = DGB_FLOAT32_SPARSE,
  // Narrowing encoder kinds (dgb_float_compress_to), 0x40 | the archive type, never written to the wire: the
  // encoder reads float32 words and rounds each to the archive type's 16-bit word (cvt.rn, torch's CUDA cast)
  // before it takes the coded and stored bytes out of it, so the archive is an ordinary fp16 / bf16 archive.
  // Encoder only: decode.cu never dispatches them.
  kKindF32toF16 = 0x40 | DGB_FLOAT16,
  kKindF32toBF16 = 0x40 | DGB_BFLOAT16,
  // The same with error feedback (dgb_float_compress_to_ef), 0x80 | the narrowing kind: each word is y = x + e, with
  // e the member's float32 residual word, and the coder overwrites e with y - float(round(y)) (+0 where the rounded
  // word is not finite).  Encoder only, never on the wire; their kernels also take the residual table (EfMembers).
  kKindF32toF16EF = 0x80 | kKindF32toF16,
  kKindF32toBF16EF = 0x80 | kKindF32toBF16,
  // fp8 words: their archives are byte archives, so only the fp8 decode-and-sum (decode_fp8.cu) dispatches them
  kKindE4M3 = DGB_FLOAT8_E4M3,
  kKindE5M2 = DGB_FLOAT8_E5M2
};
__host__ __device__ constexpr bool isFp8Kind(int k) { return k == kKindE4M3 || k == kKindE5M2; }
__host__ __device__ constexpr bool isEfKind(int k) { return k == kKindF32toF16EF || k == kKindF32toBF16EF; }
__host__ __device__ constexpr bool isNarrowKind(int k) {
  return k == kKindF32toF16 || k == kKindF32toBF16 || isEfKind(k);
}
// the float type a kind's archives carry (header, size bound, plane layout, table format)
__host__ __device__ constexpr int archiveKind(int k) { return isNarrowKind(k) ? (k & ~0xc0) : k; }

struct MemberDesc {
  const void* in;     // encode: raw input (bytes / float words); decode: archive
  void* out;          // encode: archive; decode: output
  uint32_t size;      // encode: input size (bytes, or float WORDS); decode: capacity (same unit)
  uint32_t work0;     // first flat work item (chunk / ticket) of this member
};
static_assert(sizeof(MemberDesc) == 24, "");

// Batches of up to kInlineMembers members travel to the default kernels INSIDE the kernel parameters
// (constant bank, 1.5 KB) instead of through a copy in front of the first launch: one dependent
// operation less per call.  Larger batches (and the optional kernel flavours) read the same table from the
// scratch buffer, where uploadTable puts it; either way no host memory is read after the call returns.
constexpr uint32_t kInlineMembers = 64;
struct InlineMembers {
  uint32_t count;  // 0: the table is in global memory (scratch)
  float scale;     // the scaled decode-and-sum kernels' multiplier (decode.cu kScaled); no other kernel reads it
  MemberDesc m[kInlineMembers];
};
__device__ __forceinline__ MemberDesc memberAt(const InlineMembers& im, const MemberDesc* global, uint32_t i) {
  return im.count ? im.m[i] : global[i];
}
__device__ __forceinline__ uint32_t memberWork0(const InlineMembers& im, const MemberDesc* global, uint32_t i) {
  return im.count ? im.m[i].work0 : __ldg(&global[i].work0);
}

// The residual buffers of the error-feedback kinds, member by member.  Only their kernels take this table, so the
// member table every other kernel receives keeps its layout.  Up to kInlineMembers pointers travel inside the
// kernel parameters (when the member table does); otherwise `global` is a copy in the scratch, uploaded with the
// member table (uploadTable), so no host memory is read after the call returns.
struct EfMembers {
  float* const* global;  // used when count == 0
  uint32_t count;
  float* e[kInlineMembers];
};
__device__ __forceinline__ float* efAt(const EfMembers& ef, uint32_t i) { return ef.count ? ef.e[i] : ef.global[i]; }

// ---- encoder symbol table entry (one per symbol, 8 B, shared memory) -------
// magic = ceil(2^(32+shift)/pdf): state / pdf == hi32(state * magic) >> shift for state < 2^31
//         (the quotient ans/GpuANSStatistics.cuh:343-358 computes, without its add; pdf == 1 uses
//         2^32 - 1, i.e. state - 1, and carries the missing 2^pb - 1 in the cdf term)
// pack  = shift (bits 0..4, consumed by shf.wrap) | 2^pb - pdf (bits 5..16) | cdf term (bits 20..31)
// The renormalisation threshold pdf << (31 - pb) is rebuilt from 2^pb - pdf (encode.cu ldsEntry).
struct __align__(8) EncEntry {
  uint32_t magic, pack;
};
constexpr uint32_t kEncKmpShift = 5, kEncKmpMask = 0xfffu, kEncCdfShift = 20;
// Wide form of the same entry: nothing to unpack, four wavefronts per lookup (see EncSym in encode.cu).
//   thr = pdf << (31 - pb), kmp = 2^pb - pdf, cdfShift = shift | cdf term << 5
struct __align__(16) EncEntryWide {
  uint32_t thr, magic, kmp, cdfShift;
};

// ---- tuning options (dgb_set_option) ---------------------------------------
struct Options {
  int decode_fused = 1;      // 1: one persistent launch, CTAs lease members and warps claim blocks; 0: plan + decode kernels
  int decode_warps = 0;      // single-launch decoder: warps per CTA (4, 8, 20 = byte archives only; 0 = auto)
  int decode_slot_words = 0; // TMA staging slot per warp in u16 words; 0 = auto
  int encode_warps = 8;      // warps per encode CTA (each warp is an independent worker)
  int encode_slot_words = 0; // staging slot of the fast encoder in u16 words; 0 = auto
  int encode_canonical = 0;  // 1: streams packed in block order (byte-identical archives, slower)
  int encode_fused = 0;      // 1: one persistent launch (statistics items + encode chunks), 0: two kernels (default: faster, DESIGN.md section 4)
  int fused_stage = 1;       // fused launch: statistics slabs land in shared memory by TMA bulk copy (0: register loads)
  int fused_stats_every = 4; // fused launch: one CTA in this many prefers statistics items (0: none does)
  int fused_chunk_blocks = 16;  // fused launch: 4 KiB blocks per encode chunk
  int encode_wide_table = -1;  // encoder table entries: 1 = 16 B, 0 = 8 B, -1 = by data kind (bf16/fp32 wide)
  int stats_stage = 0;       // two-kernel path, float kinds: 1 = statistics slab lands in shared memory by TMA (one slab per CTA)
  int stats_stage_kb = 32;   // ... slab size for that
  int encode_k2_ctas = 0;    // cap of coder CTAs per SM (0 = as many as fit)
  int hist_slab_kb = 64;     // bytes of input per histogram CTA iteration
  int hist_ctas_per_sm = 32; // stats grid = this many CTAs per SM (each CTA loops over slabs)
  int parts = 0;             // sub-batches run on internal streams (0 = auto, 1 = off, max 4)
  int first_part_pct = 100;  // size of the first / last sub-batch relative to an equal share (capi.cu splitParts)
  int last_part_pct = 100;
  int pull_ctas = 64;        // grid of the archive mover (dgb_archives_pull): enough loads in flight for NVLink, few SMs
  int inline_members = 1;   // 1: member table inside the kernel parameters when the batch has <= 64 members
  int timing = 0;            // 1: bracket every kernel launch with CUDA events (bench.py roofline pass)
};
Options& options();

// ---- host-side internal API (capi.cu -> *.cu) --------------------------------
struct HostMember {
  const void* in;
  void* out;
  uint32_t size;  // see MemberDesc::size
};

// err: the error-feedback kinds' residual buffers, one per member (nullptr for every other kind)
int encodeBatch(int kind, void* temp, size_t tempBytes, int pb, bool checksum, uint32_t n,
                const HostMember* members, const uint32_t* histogram_dev, uint32_t* outSize_dev,
                cudaStream_t stream, float* const* err = nullptr);
int decodeBatch(int kind, void* temp, size_t tempBytes, int pb, bool checksum, uint32_t n,
                const HostMember* members, uint8_t* outSuccess_dev, uint32_t* outSize_dev,
                uint8_t* mismatchHost, cudaStream_t stream);
int decodeReduce(int kind, int outKind, void* temp, size_t tempBytes, int pb, uint32_t groups, uint32_t width,
                 const void* const* in, void* const* out, const uint32_t* outSize, bool accumulate,
                 uint8_t* outSuccess_dev, bool sparse, const float* scale, const float* scaleDev, float* foundInf,
                 cudaStream_t stream, void* const* narrowOut = nullptr, double* sqNorm = nullptr);
// the narrowing sums' kernels (decode_narrow.cu): decodeReduce's launches of kind | kWidenF32 | kNarrowOut, scaled
// (host scale) or with scaleDev / foundInf, reading the groups' 16-bit outputs from the device table narrowTable
int launchDecodeReduceNarrow(int kind, int pb, bool scaled, const Options& opt, MemberDesc* members, uint32_t* next,
                             const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                             bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                             float* foundInf, void* const* narrowTable);
size_t encodeTempBytes(int kind, uint32_t n, uint32_t maxSize);
size_t decodeTempBytes(int kind, uint32_t n);
int getInfo(int kind, void* temp, size_t tempBytes, const void* const* in, bool inIsDevice,
            uint32_t n, uint32_t* outSizes, uint32_t* outTypes, uint32_t* outChecksum,
            cudaStream_t stream);
int pullArchives(int kind, uint32_t n, const void* const* src, void* const* dst, const uint32_t* capacity,
                 uint32_t* outBytes_dev, cudaStream_t stream);

void setLastCudaError(cudaError_t e);

inline uint32_t wordBytes(int kind) {  // the narrowing kinds: their float32 input words
  return kind == kKindF64 ? 8u
                          : (kind == kKindF32 || kind == kKindF32S || isNarrowKind(kind) ? 4u : (kind == kKindBytes ? 1u : 2u));
}
inline size_t alignUp256(size_t v) { return (v + 255) & ~size_t(255); }

// Squared norms (decode_norm.cu): the fp64 squared norm of each of G groups of float words, in the fixed order of
// include/dietgpu_b200.h (lane, warp, group).  One fp64 partial per 4096-word block goes to scratch, and a fold
// kernel (one CTA per group) writes sq_norm[g].
struct SqNormScratch {
  uint32_t* off;  // [G + 1] index of group g's first partial; off[G] = every group's blocks
  uint32_t* size; // [G] the groups' word counts (right after off)
  uint32_t* ok;   // [G] the decode-and-sum's verdict on group g (1: every archive valid); unused by floatSqNorm
  double* part;   // [off[G]] one partial per block
};
inline uint64_t sqNormBlocks(uint32_t groups, const uint32_t* size) {
  uint64_t b = 0;
  for (uint32_t g = 0; g < groups; ++g) b += (size[g] + 4095u) / 4096u;
  return b;
}
inline size_t sqNormScratchBytes(uint32_t groups, uint64_t blocks) {
  return alignUp256(8 * (size_t)groups + 8) + alignUp256(4 * (size_t)groups) + alignUp256(8 * blocks);
}
// lays SqNormScratch out at `base` (256 B aligned) and uploads the offsets and sizes of size[0 .. G-1]
int sqNormPrepare(uint8_t* base, uint32_t groups, const uint32_t* size, SqNormScratch* out, cudaStream_t stream);
// decodeReduce's launches of the device-scale kinds | kSqNorm (narrowing ones when narrowTable is set), then the
// fold into sqNorm[g] for the groups the reduce kernels found valid
int launchDecodeReduceNorm(int kind, int pb, bool widen, const Options& opt, MemberDesc* members, uint32_t* next,
                           const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                           bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                           float* foundInf, void* const* narrowTable, const SqNormScratch& norm, double* sqNorm);
// the fold of the block partials into sqNorm[g] for the groups the decode-and-sum kernels found valid (decode_norm.cu)
int sqNormFoldValid(const Options& opt, const SqNormScratch& norm, uint32_t groups, double* sqNorm, cudaStream_t stream);
// decodeReduce's launches of the fp8 kinds (decode_fp8.cu): fp8 byte archives summed into fp32 with the device scale,
// | kSqNorm when norm is not null (then followed by the fold into sqNorm)
int launchDecodeReduceFp8(int kind, int pb, const Options& opt, MemberDesc* members, uint32_t* next,
                          const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                          bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                          float* foundInf, const SqNormScratch* norm, double* sqNorm);
// dgb_float_cast_fp8 (cast_fp8.cu): inKind fp32 or bf16, fp8Kind e4m3 or e5m2 (checked by the entry point)
int castFp8(int inKind, int fp8Kind, uint32_t n, const void* const* in, const uint32_t* size, const float* scaleDev,
            void* const* out, uint32_t* histogram, cudaStream_t stream);
// dgb_float_sq_norm: dense fp16 / bf16 / fp32 words
size_t floatSqNormTempBytes(uint32_t groups, const uint32_t* size);
int floatSqNorm(int kind, void* temp, size_t tempBytes, uint32_t groups, const void* const* in, const uint32_t* size,
                double* sqNorm, cudaStream_t stream);
int smCount();  // SMs of the current device, cached per device

// Resident CTAs per SM of `kernel` with `threads` threads and `smemBytes` of dynamic shared memory, into
// *out.  The kernel's dynamic shared-memory limit is raised to `maxDynamicSmem` once per (kernel, device);
// with out == nullptr that is all it does.  Cached per host thread: once warm it makes no CUDA call
// beyond cudaGetDevice and allocates nothing.
int residentCtasPerSm(const void* kernel, int threads, size_t smemBytes, int maxDynamicSmem, int* out);

// Per-thread host staging of the codec calls, reused: no allocation on the steady-state call path.
// Nothing here is read after the call returns (uploadTable), so a later call, or a graph capture, may
// overwrite every buffer.
struct HostStage {
  std::vector<HostMember> members;      // the entry point's member list (capi.cu)
  std::vector<uint8_t> encodeUpload;    // encoder member table + work index, uploaded together
  std::vector<MemberDesc> decodeTable;  // decoder member table
  std::vector<uint32_t> checksum;       // decoder checksum pass: computed, stored and decoded size per member
  std::vector<uint32_t> sqNormOff;      // squared norms: first block partial of each group, and the total
};
HostStage& hostStage();

// Enqueues on `stream` a copy of `bytes` (a multiple of 8) of host memory at `src` to `dst` (device, 8 B
// aligned).  `src` is read before this returns, so the caller may reuse it at once: an ordinary call copies
// from pageable memory, which stages the bytes; on a capturing stream the bytes travel inside the parameters
// of small copy kernels, so a graph replays the bytes it captured, not whatever `src` holds at replay time.
int uploadTable(void* dst, const void* src, size_t bytes, cudaStream_t stream);

// DGB_ERR_CAPTURING when `stream` is being captured into a CUDA graph, else DGB_OK; for calls that
// synchronise the stream, which a capture cannot hold
int checkNotCapturing(cudaStream_t stream);

// Per-kernel timing (Options::timing of the call): slots are stable indices reported by
// dgb_kernel_times().  No-ops when timing is off.
enum TimerSlot : int { kSlotStats = 0, kSlotEncode = 1, kSlotPlan = 2, kSlotDecode = 3, kSlotChecksum = 4, kSlotFused = 5, kSlotPull = 6, kNumSlots = 7 };
void timerBegin(const Options& opt, int slot, cudaStream_t stream);
void timerEnd(const Options& opt, int slot, cudaStream_t stream);

// Sub-batches of one call: a large batch is cut into up to kMaxParts contiguous member ranges of
// roughly equal bytes whose kernels run on internal streams forked from the caller's stream, so the
// HBM-bound and the issue-bound kernels of different sub-batches overlap and launch gaps hide.  The
// destructor joins every forked stream back to the caller's stream, on every exit path: the caller
// frees / reuses its scratch when the call returns, so work queued on a helper stream must be ordered
// before whatever it enqueues next -- also when a later launch of the same call failed.
constexpr int kMaxParts = 8;
struct StreamPool;
class SubBatches {
 public:
  // `split` false: one sub-batch on the caller's stream
  SubBatches(int kind, const MemberDesc* members, uint32_t n, const Options& opt, bool split, cudaStream_t stream);
  ~SubBatches();
  SubBatches(const SubBatches&) = delete;
  SubBatches& operator=(const SubBatches&) = delete;
  int fork();  // records the fork point on the caller's stream (nothing to do for one sub-batch)
  int count() const { return parts_; }
  uint32_t begin(int k) const { return bounds_[k]; }
  uint32_t end(int k) const { return bounds_[k + 1]; }
  int stream(int k, cudaStream_t* out);  // the stream of sub-batch k, forked on first use

 private:
  int parts_;
  uint32_t bounds_[kMaxParts + 1];
  cudaStream_t stream_;
  StreamPool* pool_ = nullptr;
  bool forked_[kMaxParts] = {};
};

// Runtime data kind / probBits / flag turned into a template argument: f(std::integral_constant)
// with the matching value (read it as decltype(arg)::value).
template <int V>
using IntC = std::integral_constant<int, V>;
template <class F>
int withKind(int kind, F&& f) {
  switch (kind) {
    case kKindBytes: return f(IntC<kKindBytes>{});
    case kKindF16: return f(IntC<kKindF16>{});
    case kKindBF16: return f(IntC<kKindBF16>{});
    case kKindF32: return f(IntC<kKindF32>{});
    case kKindF64: return f(IntC<kKindF64>{});
    case kKindF16S: return f(IntC<kKindF16S>{});
    case kKindBF16S: return f(IntC<kKindBF16S>{});
    case kKindF32S: return f(IntC<kKindF32S>{});
    default: return DGB_ERR_INVALID_ARG;
  }
}
template <class F>
int withPb(int pb, F&& f) {
  switch (pb) {
    case 9: return f(IntC<9>{});
    case 10: return f(IntC<10>{});
    case 11: return f(IntC<11>{});
    default: return DGB_ERR_INVALID_ARG;
  }
}
template <class F>
int withBool(bool b, F&& f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}

#define DGB_CUDA_TRY(expr)                    \
  do {                                        \
    cudaError_t _e = (expr);                  \
    if (_e != cudaSuccess) {                  \
      ::dgb::setLastCudaError(_e);            \
      return DGB_ERR_CUDA;                    \
    }                                         \
  } while (0)

#ifdef __CUDACC__
// ---- small device helpers ---------------------------------------------------
__device__ __forceinline__ uint32_t laneId() {
  uint32_t l;
  asm("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}
__device__ __forceinline__ uint32_t laneMaskLt() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
__device__ __forceinline__ uint32_t laneMaskGe() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_ge;" : "=r"(m));
  return m;
}
__device__ __forceinline__ uint32_t smemAddr(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- mbarrier + TMA 1-D bulk copy (cp.async.bulk), sm_90+ ------------
__device__ __forceinline__ void mbarInit(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fenceBarrierInit() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fenceProxyAsync() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbarExpectTx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbarWait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "DGB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DGB_DONE_%=;\n"
      "bra DGB_WAIT_%=;\n"
      "DGB_DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16 B aligned.
__device__ __forceinline__ void bulkLoad(uint32_t dstSmem, const void* src, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(dstSmem),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// ---- cp.async (LDGSTS) 16 B copies and shared-memory loads at a constant offset ----
__device__ __forceinline__ void cpAsync16(uint32_t dstSmem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dstSmem), "l"(src) : "memory");
}
__device__ __forceinline__ void cpAsyncCommit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cpAsyncWait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
template <int OFF>
__device__ __forceinline__ uint32_t ldsU8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
  return v;
}
template <int OFF>
__device__ __forceinline__ uint32_t ldsU16(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
  return v;
}
template <int OFF>
__device__ __forceinline__ uint32_t ldsU32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF));
  return v;
}
// block-wide exclusive scan of one value per thread for THREADS threads
// (THREADS multiple of 32, <= 1024).  `warpSums` is smem of THREADS/32 words.
template <int THREADS>
__device__ __forceinline__ uint32_t blockExclusiveScan(uint32_t v, uint32_t* warpSums,
                                                       uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= (uint32_t)d) incl += t;
  }
  if (lane == 31) warpSums[warp] = incl;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < THREADS / 32; ++w) {
    uint32_t s = warpSums[w];
    if ((uint32_t)w < warp) base += s;
    tot += s;
  }
  if (total) *total = tot;
  __syncthreads();
  return base + incl - v;
}
#endif  // __CUDACC__

}  // namespace dgb
