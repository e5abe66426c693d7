// decode_fp8.cu -- the fp8 decode-and-sum kernels and their launcher, in a module of their own: decode.cu compiled once
// more with DGB_DECODE_FP8_TU for the device-scale decode-and-sum kernels of the fp8 kinds (fp8 byte archives summed
// into fp32, | kSqNorm for the squared-norm entry).  Apart from the other decode modules, so that the kernels there
// keep their code.
#define DGB_DECODE_FP8_TU
#include "decode.cu"

namespace dgb {

int launchDecodeReduceFp8(int kind, int pb, const Options& opt, MemberDesc* members, uint32_t* next,
                          const InlineMembers& im, uint32_t groups, uint32_t width, uint64_t totalChunks,
                          bool accumulate, uint8_t* outSuccess, cudaStream_t stream, const float* scaleDev,
                          float* foundInf, const SqNormScratch* norm, double* sqNorm) {
  DecodeScratch sc{};
  sc.members = members;
  sc.next = next;
  sc.seen = next + (size_t)groups * width;
  // every fp8 sum widens to fp32 and takes the device scale: term(q) = fp32(q) * *scaleDev (RowWriterSum, scaleWiden)
  auto run = [&](auto K) {
    return withPb(pb, [&](auto P) {
      constexpr int WK = decltype(K)::value | kWidenF32 | kScaled | kDevScale, PB = decltype(P)::value;
      if (norm)
        return launchDecodeReduce<WK | kSqNorm, PB>(opt, sc, im, groups, width, totalChunks, accumulate, outSuccess,
                                                    stream, scaleDev, foundInf, nullptr, norm);
      return launchDecodeReduce<WK, PB>(opt, sc, im, groups, width, totalChunks, accumulate, outSuccess, stream,
                                        scaleDev, foundInf);
    });
  };
  const int rc = kind == kKindE4M3 ? run(IntC<kKindE4M3>()) : run(IntC<kKindE5M2>());
  if (rc != DGB_OK || !norm) return rc;
  return sqNormFoldValid(opt, *norm, groups, sqNorm, stream);
}

}  // namespace dgb
