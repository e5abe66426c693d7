// Round trip of three ReLU-like fp32 members through the C++ compatibility layer (include/dietgpu_b200_compat.hpp)
// with FloatType::kFloat32Sparse: floatCompress, floatGetCompressedInfo, floatDecompress with checksum verification.
// Plain asserts; run by tests/test_gpu_sparse_fp32.py.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../include/dietgpu_b200_compat.hpp"

using namespace dietgpu;

#define REQUIRE(c)                                                                \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::fprintf(stderr, "%s:%d REQUIRE(%s) failed\n", __FILE__, __LINE__, #c); \
      std::exit(1);                                                               \
    }                                                                             \
  } while (0)

int main() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    std::fprintf(stderr, "no CUDA device\n");
    return 2;
  }
  auto res = makeStackMemory(64 << 20);
  const std::vector<uint32_t> sizes = {1, 4097, 70001};
  const uint32_t n = (uint32_t)sizes.size();
  const uint32_t stride = getMaxFloatCompressedSize(FloatType::kFloat32Sparse, 70001);
  REQUIRE(stride != 0 && stride % 16 == 0);
  std::mt19937 gen(32);
  std::normal_distribution<float> dist;
  std::vector<std::vector<uint32_t>> orig(n);
  std::vector<uint32_t*> in(n), out(n);
  uint8_t* enc = nullptr;
  REQUIRE(cudaMalloc(&enc, (size_t)n * stride) == cudaSuccess);
  std::vector<const void*> inPtr(n), encPtrC(n);
  std::vector<void*> encPtr(n), outPtr(n);
  for (uint32_t i = 0; i < n; ++i) {
    for (uint32_t k = 0; k < sizes[i]; ++k) {
      const float x = dist(gen);  // ReLU, with a -0 for every fourth negative draw (a masked product)
      const uint32_t neg = (k % 4 == 0) ? 0x80000000u : 0u;
      uint32_t bits;
      std::memcpy(&bits, &x, 4);
      orig[i].push_back(x > 0.f ? bits : neg);
    }
    REQUIRE(cudaMalloc(&in[i], sizes[i] * sizeof(uint32_t)) == cudaSuccess);
    REQUIRE(cudaMalloc(&out[i], sizes[i] * sizeof(uint32_t)) == cudaSuccess);
    cudaMemcpy(in[i], orig[i].data(), sizes[i] * sizeof(uint32_t), cudaMemcpyHostToDevice);
    inPtr[i] = in[i];
    outPtr[i] = out[i];
    encPtr[i] = enc + (size_t)i * stride;
    encPtrC[i] = encPtr[i];
  }
  uint32_t *encSize = nullptr, *decSize = nullptr, *infoSize = nullptr, *infoType = nullptr;
  uint8_t* ok = nullptr;
  REQUIRE(cudaMalloc(&encSize, 4 * n) == cudaSuccess && cudaMalloc(&decSize, 4 * n) == cudaSuccess);
  REQUIRE(cudaMalloc(&infoSize, 4 * n) == cudaSuccess && cudaMalloc(&infoType, 4 * n) == cudaSuccess);
  REQUIRE(cudaMalloc(&ok, n) == cudaSuccess);

  FloatCodecConfig cfg(FloatType::kFloat32Sparse, ANSCodecConfig(10, false), true, true);
  floatCompress(res, cfg, n, inPtr.data(), sizes.data(), encPtr.data(), encSize, 0);
  floatGetCompressedInfo(res, encPtrC.data(), n, infoSize, infoType, nullptr, 0);
  auto st = floatDecompress(res, cfg, n, encPtrC.data(), outPtr.data(), sizes.data(), ok, decSize, 0);
  REQUIRE(st.error == FloatDecompressError::None);

  std::vector<uint32_t> es(n), ds(n), is(n), it(n);
  std::vector<uint8_t> oks(n);
  cudaMemcpy(es.data(), encSize, 4 * n, cudaMemcpyDeviceToHost);
  cudaMemcpy(ds.data(), decSize, 4 * n, cudaMemcpyDeviceToHost);
  cudaMemcpy(is.data(), infoSize, 4 * n, cudaMemcpyDeviceToHost);
  cudaMemcpy(it.data(), infoType, 4 * n, cudaMemcpyDeviceToHost);
  cudaMemcpy(oks.data(), ok, n, cudaMemcpyDeviceToHost);
  for (uint32_t i = 0; i < n; ++i) {
    REQUIRE(es[i] > 32 && es[i] <= stride);
    REQUIRE(oks[i] == 1 && ds[i] == sizes[i]);
    REQUIRE(is[i] == sizes[i] && it[i] == (uint32_t)FloatType::kFloat32Sparse);
    std::vector<uint32_t> got(sizes[i]);
    cudaMemcpy(got.data(), out[i], sizes[i] * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    REQUIRE(std::memcmp(got.data(), orig[i].data(), sizes[i] * sizeof(uint32_t)) == 0);
    cudaFree(in[i]);
    cudaFree(out[i]);
  }
  cudaFree(enc);
  cudaFree(encSize);
  cudaFree(decSize);
  cudaFree(infoSize);
  cudaFree(infoType);
  cudaFree(ok);
  std::printf("sparse32_roundtrip: all passed\n");
  return 0;
}
