// decode_narrow.cu -- the narrowing decode-and-sum kernels (decode.cu, kNarrowOut: fp16 / bf16 archives summed in
// fp32 and rounded once to 16 bits) and their launcher, in a module of their own (see launchDecodeReduceNarrow)
#define DGB_DECODE_NARROW_TU
#include "decode.cu"
