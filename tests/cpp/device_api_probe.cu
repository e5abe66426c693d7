// Test vehicle for include/dietgpu_b200_device.cuh: small kernels that each call one entry point of
// the header directly, so that tests/test_gpu_device_api.py can compare its results with the CPU
// oracle one function at a time (the example kernels in device_api_example.cu only exercise the
// header through whole tiles).
//
//   probe_normalise     blockNormalizedPdf + blockBuildEncodeTable, several histograms per CTA
//   probe_encode_entry  makeEncodeEntry on a list of (pdf, cdf, probBits)
//   probe_block_encode  warpEncodeBlock, one warp per block, shared or global in / out
//   probe_block_decode  blockBuildDecodeLut<PB, 32> + warpDecodeBlock, one warp per block
//   probe_decode_lut    blockBuildDecodeLut<PB, THREADS>, several pdfs per CTA, every return value
//   probe_archive_overhead / probe_max_block_words: the host-callable layout constants
//
// Outputs go to caller-provided buffers that the tests prefill with a sentinel; in the shared-memory
// variants the kernels prefill their shared buffers with the same sentinel and copy them back whole
// (including the part past the data) so that stray writes show up in either memory space.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dietgpu_b200_device.cuh"

namespace dd = dietgpu_b200::device;

namespace {

constexpr uint16_t kSentinel16 = 0xa5a5u;
constexpr uint8_t kSentinel8 = 0xa5u;
constexpr uint32_t kSentinel32 = 0xa5a5a5a5u;
constexpr uint32_t kMaxDecodeWords = 4608;  // stream words a shared-memory decode can hold
constexpr uint32_t kOutGuard = 64;          // bytes past n copied back by the shared-memory decode
constexpr uint32_t kLutGuard = 32;          // u32 past 2^PB copied back by the LUT probe
constexpr uint32_t kMaxLutsPerCta = 4;

// ---- normalisation --------------------------------------------------------------------------------
// CTA c normalises histograms [c * perCta, min((c + 1) * perCta, numHist)) one after the other, each
// through both entry points, with no barrier of its own in between.
__global__ void __launch_bounds__(256)
normaliseKernel(const uint32_t* counts, const uint32_t* totals, uint32_t numHist, uint32_t perCta, int probBits,
                uint32_t* pdfOut, uint32_t* cdfOut, uint16_t* pdf16Out, uint32_t* tableOut) {
  __shared__ dd::EncodeTable table;
  const uint32_t t = threadIdx.x;
  const uint32_t first = blockIdx.x * perCta;
  const uint32_t last = min(first + perCta, numHist);
  for (uint32_t h = first; h < last; ++h) {
    uint32_t cdf;
    const uint32_t pdf = dd::blockNormalizedPdf(counts[h * 256 + t], totals[h], probBits, &cdf);
    pdfOut[h * 256 + t] = pdf;
    cdfOut[h * 256 + t] = cdf;
    dd::blockBuildEncodeTable(counts + h * 256, totals[h], probBits, &table, pdf16Out + h * 256);
    tableOut[(h * 256 + t) * 2] = table.e[t].magic;
    tableOut[(h * 256 + t) * 2 + 1] = table.e[t].pack;
  }
}

__global__ void encodeEntryKernel(const uint32_t* pdf, const uint32_t* cdf, const int32_t* probBits, uint32_t count,
                                  uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const dd::EncodeEntry e = dd::makeEncodeEntry(pdf[i], cdf[i], probBits[i]);
  out[2 * i] = e.magic;
  out[2 * i + 1] = e.pack;
}

// ---- block coder ----------------------------------------------------------------------------------
// The warp's encode table from a u16 pdf: exclusive scan, then makeEncodeEntry per symbol.
template <int PB>
__device__ void warpTableFromPdf(const uint16_t* pdf, dd::EncodeTable* table) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t p[8], s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) { p[k] = pdf[lane * 8 + k]; s += p[k]; }
  uint32_t inc = s;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= (uint32_t)d) inc += v;
  }
  uint32_t c = inc - s;
#pragma unroll
  for (int k = 0; k < 8; ++k) { table->e[lane * 8 + k] = dd::makeEncodeEntry(p[k], c, PB); c += p[k]; }
  __syncwarp();
}

// Block b: bytes in[inOff[b], + n[b]) under pdf[b * 256, + 256) -> words[wordsOff[b], + n[b] + 8),
// numWords[b], states[b * 32, + 32).  SMEM: the bytes and the stream live in shared memory.
template <int PB, bool SMEM>
__global__ void __launch_bounds__(32)
blockEncodeKernel(const uint8_t* in, const uint32_t* inOff, const uint32_t* nIn, const uint16_t* pdf, uint16_t* words,
                  const uint32_t* wordsOff, uint32_t* numWords, uint32_t* states) {
  __shared__ dd::EncodeTable table;
  __shared__ alignas(16) uint8_t sIn[dd::kBlockBytes];
  __shared__ alignas(16) uint16_t sWords[dd::kBlockBytes + 8];
  const uint32_t b = blockIdx.x, lane = threadIdx.x;
  const uint32_t n = nIn[b];
  if (n == 0 || n > dd::kBlockBytes) {
    if (lane == 0) numWords[b] = 0xffffffffu;
    return;
  }
  warpTableFromPdf<PB>(pdf + b * 256, &table);
  const uint8_t* src = in + inOff[b];
  uint16_t* dst = words + wordsOff[b];
  if (SMEM) {
    for (uint32_t i = lane; i < n; i += 32) sIn[i] = src[i];
    for (uint32_t i = lane; i < n + 8; i += 32) sWords[i] = kSentinel16;
    __syncwarp();
  }
  uint32_t state;
  const uint32_t cnt = dd::warpEncodeBlock(SMEM ? sIn : src, n, &table, PB, SMEM ? sWords : dst, &state);
  states[b * 32 + lane] = state;
  if (lane == 0) numWords[b] = cnt;
  if (SMEM) {
    __syncwarp();
    for (uint32_t i = lane; i < n + 8; i += 32) dst[i] = sWords[i];
  }
}

// Block b: lane states states[b * 32, + 32), stream words + wordsOff[b] with numWords[b] words, n[b]
// bytes under pdf[b * 256, + 256) -> out[outOff[b], + n[b]) and every lane's return in ok[b * 32, + 32)
// (2 if the LUT was rejected, 3 for arguments the probe cannot hold).  SMEM: the stream and the output
// live in shared memory; the output is copied back with kOutGuard bytes past n.
template <int PB, bool SMEM>
__global__ void __launch_bounds__(32)
blockDecodeKernel(const uint16_t* pdf, const uint32_t* states, const uint16_t* words, const uint32_t* wordsOff,
                  const uint32_t* numWords, const uint32_t* nIn, uint8_t* out, const uint32_t* outOff, uint32_t* ok) {
  __shared__ uint32_t lut[1u << PB];
  __shared__ alignas(16) uint16_t sWords[kMaxDecodeWords];
  __shared__ alignas(16) uint8_t sOut[dd::kBlockBytes + kOutGuard];
  const uint32_t b = blockIdx.x, lane = threadIdx.x;
  const uint32_t n = nIn[b], nw = numWords[b];
  if (n == 0 || n > dd::kBlockBytes || (SMEM && nw > kMaxDecodeWords)) {
    ok[b * 32 + lane] = 3u;
    return;
  }
  if (!dd::blockBuildDecodeLut<PB, 32>(pdf + b * 256, lut)) {
    ok[b * 32 + lane] = 2u;
    return;
  }
  const uint16_t* src = words + wordsOff[b];
  uint8_t* dst = out + outOff[b];
  if (SMEM) {
    for (uint32_t i = lane; i < nw; i += 32) sWords[i] = src[i];
    for (uint32_t i = lane; i < n + kOutGuard; i += 32) sOut[i] = kSentinel8;
    __syncwarp();
  }
  const bool r = dd::warpDecodeBlock<PB>(states[b * 32 + lane], SMEM ? sWords : src, nw, n, lut, SMEM ? sOut : dst);
  ok[b * 32 + lane] = r ? 1u : 0u;
  if (SMEM) {
    __syncwarp();
    for (uint32_t i = lane; i < n + kOutGuard; i += 32) dst[i] = sOut[i];
  }
}

// ---- decode LUT -----------------------------------------------------------------------------------
// CTA c builds the LUTs of pdfs [c * perCta, + perCta) back to back into separate shared slots, with
// no barrier of its own between the calls, then copies every slot (2^PB + kLutGuard words) and every
// thread's return value out.
template <int PB, int THREADS>
__global__ void __launch_bounds__(THREADS)
decodeLutKernel(const uint16_t* pdf, uint32_t perCta, uint32_t* lutOut, uint32_t* retOut) {
  constexpr uint32_t kSlot = (1u << PB) + kLutGuard;
  __shared__ uint32_t slots[kMaxLutsPerCta][kSlot];
  const uint32_t t = threadIdx.x;
  for (uint32_t i = t; i < perCta * kSlot; i += THREADS) slots[i / kSlot][i % kSlot] = kSentinel32;
  bool ret[kMaxLutsPerCta];
#pragma unroll
  for (uint32_t k = 0; k < kMaxLutsPerCta; ++k)
    if (k < perCta) ret[k] = dd::blockBuildDecodeLut<PB, THREADS>(pdf + (blockIdx.x * perCta + k) * 256, slots[k]);
  __syncthreads();
  for (uint32_t k = 0; k < perCta; ++k) {
    const uint32_t g = blockIdx.x * perCta + k;
    for (uint32_t i = t; i < kSlot; i += THREADS) lutOut[g * kSlot + i] = slots[k][i];
    retOut[g * THREADS + t] = ret[k] ? 1u : 0u;
  }
}

template <int PB, bool SMEM>
int launchBlockEncode(uint32_t numBlocks, const uint8_t* in, const uint32_t* inOff, const uint32_t* n,
                      const uint16_t* pdf, uint16_t* words, const uint32_t* wordsOff, uint32_t* numWords,
                      uint32_t* states, cudaStream_t st) {
  blockEncodeKernel<PB, SMEM><<<numBlocks, 32, 0, st>>>(in, inOff, n, pdf, words, wordsOff, numWords, states);
  return (int)cudaGetLastError();
}

template <int PB, bool SMEM>
int launchBlockDecode(uint32_t numBlocks, const uint16_t* pdf, const uint32_t* states, const uint16_t* words,
                      const uint32_t* wordsOff, const uint32_t* numWords, const uint32_t* n, uint8_t* out,
                      const uint32_t* outOff, uint32_t* ok, cudaStream_t st) {
  blockDecodeKernel<PB, SMEM><<<numBlocks, 32, 0, st>>>(pdf, states, words, wordsOff, numWords, n, out, outOff, ok);
  return (int)cudaGetLastError();
}

template <int PB, int THREADS>
int launchDecodeLut(uint32_t numCtas, uint32_t perCta, const uint16_t* pdf, uint32_t* lutOut, uint32_t* retOut,
                    cudaStream_t st) {
  decodeLutKernel<PB, THREADS><<<numCtas, THREADS, 0, st>>>(pdf, perCta, lutOut, retOut);
  return (int)cudaGetLastError();
}

template <int PB>
int dispatchLutThreads(int threads, uint32_t numCtas, uint32_t perCta, const uint16_t* pdf, uint32_t* lutOut,
                       uint32_t* retOut, cudaStream_t st) {
  switch (threads) {
    case 32: return launchDecodeLut<PB, 32>(numCtas, perCta, pdf, lutOut, retOut, st);
    case 96: return launchDecodeLut<PB, 96>(numCtas, perCta, pdf, lutOut, retOut, st);
    case 256: return launchDecodeLut<PB, 256>(numCtas, perCta, pdf, lutOut, retOut, st);
    case 1024: return launchDecodeLut<PB, 1024>(numCtas, perCta, pdf, lutOut, retOut, st);
    default: return 1;
  }
}

}  // namespace

// Every launcher returns 0 on success, nonzero for arguments it does not support (nothing launched)
// or the launch error.

extern "C" int probe_normalise(const uint32_t* counts, const uint32_t* totals, uint32_t numHist, uint32_t perCta,
                               int probBits, uint32_t* pdfOut, uint32_t* cdfOut, uint16_t* pdf16Out,
                               uint32_t* tableOut, void* stream) {
  if (numHist == 0 || perCta == 0 || probBits < 9 || probBits > 11) return 1;
  normaliseKernel<<<(numHist + perCta - 1) / perCta, 256, 0, (cudaStream_t)stream>>>(
      counts, totals, numHist, perCta, probBits, pdfOut, cdfOut, pdf16Out, tableOut);
  return (int)cudaGetLastError();
}

extern "C" int probe_encode_entry(const uint32_t* pdf, const uint32_t* cdf, const int32_t* probBits, uint32_t count,
                                  uint32_t* out, void* stream) {
  if (count == 0) return 1;
  encodeEntryKernel<<<(count + 255) / 256, 256, 0, (cudaStream_t)stream>>>(pdf, cdf, probBits, count, out);
  return (int)cudaGetLastError();
}

extern "C" int probe_block_encode(int probBits, int smem, uint32_t numBlocks, const void* in, const uint32_t* inOff,
                                  const uint32_t* n, const uint16_t* pdf, uint16_t* words, const uint32_t* wordsOff,
                                  uint32_t* numWords, uint32_t* states, void* stream) {
  if (numBlocks == 0) return 1;
  const uint8_t* b = static_cast<const uint8_t*>(in);
  const cudaStream_t st = (cudaStream_t)stream;
#define DGB_ENC(PB, S) launchBlockEncode<PB, S>(numBlocks, b, inOff, n, pdf, words, wordsOff, numWords, states, st)
  switch (probBits) {
    case 9: return smem ? DGB_ENC(9, true) : DGB_ENC(9, false);
    case 10: return smem ? DGB_ENC(10, true) : DGB_ENC(10, false);
    case 11: return smem ? DGB_ENC(11, true) : DGB_ENC(11, false);
    default: return 1;
  }
#undef DGB_ENC
}

extern "C" int probe_block_decode(int probBits, int smem, uint32_t numBlocks, const uint16_t* pdf,
                                  const uint32_t* states, const uint16_t* words, const uint32_t* wordsOff,
                                  const uint32_t* numWords, const uint32_t* n, void* out, const uint32_t* outOff,
                                  uint32_t* ok, void* stream) {
  if (numBlocks == 0) return 1;
  uint8_t* o = static_cast<uint8_t*>(out);
  const cudaStream_t st = (cudaStream_t)stream;
#define DGB_DEC(PB, S) launchBlockDecode<PB, S>(numBlocks, pdf, states, words, wordsOff, numWords, n, o, outOff, ok, st)
  switch (probBits) {
    case 9: return smem ? DGB_DEC(9, true) : DGB_DEC(9, false);
    case 10: return smem ? DGB_DEC(10, true) : DGB_DEC(10, false);
    case 11: return smem ? DGB_DEC(11, true) : DGB_DEC(11, false);
    default: return 1;
  }
#undef DGB_DEC
}

// lutOut: numCtas * perCta slots of 2^probBits + 32 words; retOut: numCtas * perCta * threads words.
extern "C" int probe_decode_lut(int probBits, int threads, uint32_t numCtas, uint32_t perCta, const uint16_t* pdf,
                                uint32_t* lutOut, uint32_t* retOut, void* stream) {
  if (numCtas == 0 || perCta == 0 || perCta > kMaxLutsPerCta) return 1;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (probBits) {
    case 9: return dispatchLutThreads<9>(threads, numCtas, perCta, pdf, lutOut, retOut, st);
    case 10: return dispatchLutThreads<10>(threads, numCtas, perCta, pdf, lutOut, retOut, st);
    case 11: return dispatchLutThreads<11>(threads, numCtas, perCta, pdf, lutOut, retOut, st);
    default: return 1;
  }
}

extern "C" uint32_t probe_archive_overhead(uint32_t numBlocks) { return dd::archiveOverhead(numBlocks); }
extern "C" uint32_t probe_max_block_words(int probBits) { return dd::maxBlockWords(probBits); }
extern "C" uint32_t probe_out_guard() { return kOutGuard; }
extern "C" uint32_t probe_lut_guard() { return kLutGuard; }
