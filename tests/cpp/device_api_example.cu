// Example + test vehicle for include/dietgpu_b200_device.cuh: a user kernel that entropy-codes the
// tile it has just produced, without leaving the SM, and a kernel that consumes such archives.
//
//   tileCompress   : CTA c owns bytes [c * tileBytes, ...) of `in` (tileBytes <= 8 x 4096): it brings
//                    the tile into shared memory (standing in for "the tile this kernel computed"),
//                    histograms it, normalises, codes one 4 KiB block per warp from shared memory
//                    into shared memory, and writes a complete ANS archive (reference wire format,
//                    blocks in order) to out + c * outStride.  Any ansDecode -- this library's or the
//                    reference's -- reads it.
//   tileDecompress : the inverse, one CTA per archive, decoded tile handed on through shared memory.
//
// Both are templates on the probability precision PB (9, 10 or 11, the archive's probBits); the
// extern "C" launchers below take it at run time and dispatch.  tests/test_gpu_device_api.py drives
// them and checks the archives byte for byte against the CPU oracle and through the library's own
// decoder.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dietgpu_b200_device.cuh"

namespace dd = dietgpu_b200::device;

constexpr int kWarps = 8;
constexpr uint32_t kTileMax = kWarps * dd::kBlockBytes;

template <int PB>
struct TileSmem {
  uint32_t hist[dd::kNumSymbols];
  dd::EncodeTable table;
  uint16_t pdf[dd::kNumSymbols];
  uint32_t words[kWarps];
  uint32_t offset[kWarps + 1];
  uint32_t lut[1u << PB];
  alignas(16) uint8_t tile[kTileMax];
  alignas(16) uint16_t stream[kWarps][dd::maxBlockWords(PB)];
};

template <int PB>
__global__ void __launch_bounds__(kWarps * 32)
tileCompress(const uint8_t* __restrict__ in, uint32_t totalBytes, uint32_t tileBytes, uint8_t* __restrict__ out,
             uint32_t outStride, uint32_t* __restrict__ outSize) {
  extern __shared__ __align__(16) uint8_t raw[];
  TileSmem<PB>& s = *reinterpret_cast<TileSmem<PB>*>(raw);
  const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  const uint32_t begin = blockIdx.x * tileBytes;
  const uint32_t n = min(tileBytes, totalBytes - begin);
  const uint32_t nb = (n + dd::kBlockBytes - 1) / dd::kBlockBytes;

  // "produce" the tile in shared memory and histogram it
  s.hist[t] = 0;
  __syncthreads();
  for (uint32_t i = t; i < n; i += blockDim.x) {
    const uint8_t b = in[begin + i];
    s.tile[i] = b;
    atomicAdd(&s.hist[b], 1u);
  }
  __syncthreads();
  dd::blockBuildEncodeTable(s.hist, n, PB, &s.table, s.pdf);

  // one 4 KiB block per warp, shared memory to shared memory
  uint32_t state = 0, words = 0;
  const uint32_t blockLen = warp < nb ? min(dd::kBlockBytes, n - warp * dd::kBlockBytes) : 0u;
  if (warp < nb) {
    words = dd::warpEncodeBlock(s.tile + warp * dd::kBlockBytes, blockLen, &s.table, PB, s.stream[warp], &state);
    if (lane == 0) s.words[warp] = words;
  }
  __syncthreads();
  if (t == 0) {
    uint32_t off = 0;
    for (uint32_t k = 0; k < nb; ++k) { s.offset[k] = off; off += (s.words[k] + 7u) / 8u * 8u; }
    s.offset[nb] = off;
  }
  __syncthreads();

  // archive: header | pdf | lane states | blockWords | streams padded to 8 words
  uint8_t* archive = out + (size_t)blockIdx.x * outStride;
  const dd::ArchiveLayout a = dd::archiveLayout(archive, nb);
  a.pdf[t] = s.pdf[t];
  if (warp < nb) {
    a.states[warp * 32 + lane] = state;
    if (lane == 0) a.blockWords[warp] = make_uint2((blockLen << 16) | words, s.offset[warp]);
    uint16_t* dst = a.data + s.offset[warp];
    const uint32_t padded = (words + 7u) / 8u * 8u;
    for (uint32_t i = lane; i < padded; i += 32) dst[i] = i < words ? s.stream[warp][i] : (uint16_t)0;
  }
  if (t == 0) {
    if (nb & 1u) a.blockWords[nb] = make_uint2(0u, 0u);
    dd::writeArchiveHeader(archive, nb, n, s.offset[nb], PB);
    outSize[blockIdx.x] = dd::archiveOverhead(nb) + 2u * s.offset[nb];
  }
}

template <int PB>
__global__ void __launch_bounds__(kWarps * 32)
tileDecompress(const uint8_t* __restrict__ in, uint32_t inStride, uint8_t* __restrict__ out, uint32_t tileBytes,
               uint32_t* __restrict__ okOut) {
  extern __shared__ __align__(16) uint8_t raw[];
  TileSmem<PB>& s = *reinterpret_cast<TileSmem<PB>*>(raw);
  const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
  const uint8_t* archive = in + (size_t)blockIdx.x * inStride;
  const uint4 h0 = *reinterpret_cast<const uint4*>(archive);
  const uint32_t nb = h0.y, n = h0.z;
  bool ok = h0.x == dd::kAnsMagicVersion && nb <= kWarps && n <= kTileMax;
  const dd::ArchiveLayout a = dd::archiveLayout(const_cast<uint8_t*>(archive), ok ? nb : 0u);
  ok = ok && dd::blockBuildDecodeLut<PB, kWarps * 32>(a.pdf, s.lut);
  if (ok && warp < nb) {
    const uint2 bw = a.blockWords[warp];
    ok = dd::warpDecodeBlock<PB>(a.states[warp * 32 + lane], a.data + bw.y, bw.x & 0xffffu, bw.x >> 16, s.lut,
                                        s.tile + warp * dd::kBlockBytes);
  }
  const int allOk = __syncthreads_and(ok ? 1 : 0);
  // "consume" the decoded tile
  if (allOk)
    for (uint32_t i = t; i < n; i += blockDim.x) out[(size_t)blockIdx.x * tileBytes + i] = s.tile[i];
  if (t == 0) okOut[blockIdx.x] = (uint32_t)allOk;
}

template <int PB>
int launchCompress(const void* in, uint32_t totalBytes, uint32_t tileBytes, void* out, uint32_t outStride,
                   uint32_t* outSize, cudaStream_t stream) {
  const uint32_t tiles = (totalBytes + tileBytes - 1) / tileBytes;
  cudaFuncSetAttribute(tileCompress<PB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem<PB>));
  tileCompress<PB><<<tiles, kWarps * 32, sizeof(TileSmem<PB>), stream>>>(
      static_cast<const uint8_t*>(in), totalBytes, tileBytes, static_cast<uint8_t*>(out), outStride, outSize);
  return (int)cudaGetLastError();
}

template <int PB>
int launchDecompress(const void* in, uint32_t inStride, uint32_t tiles, void* out, uint32_t tileBytes,
                     uint32_t* okOut, cudaStream_t stream) {
  cudaFuncSetAttribute(tileDecompress<PB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem<PB>));
  tileDecompress<PB><<<tiles, kWarps * 32, sizeof(TileSmem<PB>), stream>>>(
      static_cast<const uint8_t*>(in), inStride, static_cast<uint8_t*>(out), tileBytes, okOut);
  return (int)cudaGetLastError();
}

// probBits: 9, 10 or 11 (the archive's); anything else returns nonzero without launching.
extern "C" int example_tile_compress(const void* in, uint32_t totalBytes, uint32_t tileBytes, void* out,
                                     uint32_t outStride, uint32_t* outSize, int probBits, void* stream) {
  if (tileBytes == 0 || tileBytes > kTileMax || totalBytes == 0) return 1;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (probBits) {
    case 9: return launchCompress<9>(in, totalBytes, tileBytes, out, outStride, outSize, st);
    case 10: return launchCompress<10>(in, totalBytes, tileBytes, out, outStride, outSize, st);
    case 11: return launchCompress<11>(in, totalBytes, tileBytes, out, outStride, outSize, st);
    default: return 1;
  }
}

extern "C" int example_tile_decompress(const void* in, uint32_t inStride, uint32_t tiles, void* out, uint32_t tileBytes,
                                       uint32_t* okOut, int probBits, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  switch (probBits) {
    case 9: return launchDecompress<9>(in, inStride, tiles, out, tileBytes, okOut, st);
    case 10: return launchDecompress<10>(in, inStride, tiles, out, tileBytes, okOut, st);
    case 11: return launchDecompress<11>(in, inStride, tiles, out, tileBytes, okOut, st);
    default: return 1;
  }
}
