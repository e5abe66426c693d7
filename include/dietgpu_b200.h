/*
 * dietgpu_b200.h -- C ABI of the H100-native batched rANS + float codec.
 *
 * This is the drop-in boundary for DietGPU's codec hot path.  The reference
 * (facebookresearch/dietgpu) has no C ABI of its own: its public surface is
 * the C++ API in dietgpu/ans/GpuANSCodec.h and dietgpu/float/GpuFloatCodec.h
 * plus torch.ops.dietgpu.* (dietgpu/DietGpu.cpp).  Each entry point below
 * names the reference C++ function it replaces (file:line relative to
 * /root/reference/dietgpu/); include/dietgpu_b200_compat.hpp re-creates those
 * exact C++ signatures on top of this ABI and INTEGRATION.md shows the
 * binding a maintainer would add.
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; no C++ or torch types;
 *   - "host array" = an array in host memory, consumed before the call
 *     returns; "_dev" = device memory; `stream` is a cudaStream_t passed as
 *     void* (NULL = the legacy default stream);
 *   - all device work is enqueued on `stream`; calls are asynchronous unless
 *     a checksum has to be verified (decode with use_checksum != 0).  No
 *     device work reads a host array after the call returns, so every call
 *     but checksum-verifying decodes can be captured into a CUDA graph;
 *   - temp_dev/temp_bytes: caller-owned device scratch, 256 B aligned, at
 *     least dgb_*_temp_bytes(...) bytes; it may be reused by the next call on
 *     the same stream.  The library allocates nothing (no cudaMalloc);
 *   - compressed buffers must be 16 B aligned (as in the reference,
 *     ans/GpuANSEncode.cu:19-21); raw ANS inputs 4 B aligned
 *     (ans/GpuANSCodec.h:16); float data aligned to its word size;
 *   - return value: DGB_OK or a DGB_ERR_* code; never aborts, never throws.
 *     There is NO CPU fallback: without a usable CUDA device the calls fail
 *     with DGB_ERR_CUDA.
 *   - wire format: identical to the reference's (ans/GpuANSUtils.cuh:67-227,
 *     float/GpuFloatUtils.cuh:26-74); archives are interchangeable in both
 *     directions.  Bits the reference leaves undefined are written as zero.
 */
#ifndef DIETGPU_B200_H_
#define DIETGPU_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGB_OK 0
#define DGB_ERR_INVALID_ARG 1     /* bad prob_bits / float type / alignment / NULL */
#define DGB_ERR_TEMP_TOO_SMALL 2  /* temp_bytes < dgb_*_temp_bytes(...) */
#define DGB_ERR_CUDA 3            /* a CUDA runtime call failed (see dgb_last_cuda_error) */
#define DGB_ERR_CHECKSUM 4        /* decode: stored checksum != recomputed checksum */
#define DGB_ERR_TOO_LARGE 5       /* a size exceeds the format's 32-bit limits */
#define DGB_ERR_CAPTURING 6       /* decode with checksum verification on a stream that is being captured */

/* float/GpuFloatCodec.h:18-23 FloatType; DGB_FLOAT64 is this library's extension: its archives (float type 4)
 * carry the high exponent byte of each double in the ANS part and the other 56 bits in a u32, a u16 and a
 * u8 plane (DESIGN.md section 0).  The reference cannot read them. */
#define DGB_FLOAT16 1
#define DGB_BFLOAT16 2
#define DGB_FLOAT32 3
#define DGB_FLOAT64 4
/* Sparse fp16 / bf16 (also this library's extension; the reference cannot read these archives either): the
 * dense type's archive, except that +0 and -0 words are coded as two otherwise unused symbols and store no
 * byte, so zero-heavy data (ReLU activations, masked or pruned tensors) compresses further.  The header is
 * 32 B (the dense 16 B, then the stored-byte count and the two escape symbols), followed by a u32 per 4 KiB
 * block, the stored bytes and the ANS archive (DESIGN.md section 0). */
#define DGB_FLOAT16_SPARSE 5
#define DGB_BFLOAT16_SPARSE 6
/* Sparse fp32 (the same extension for float32 words): +0 and -0 words are coded as two otherwise unused exponent
 * symbols and store none of their 24 low bits; every other word stores them as in DGB_FLOAT32, in a compacted u16
 * plane and a compacted u8 plane.  Same 32 B header and block table as the 16-bit sparse types (DESIGN.md
 * section 0).  7 stays unassigned. */
#define DGB_FLOAT32_SPARSE 8
/* fp8 words (OCP FP8: E4M3 with no infinities and max 448, E5M2 with max 57344).  An fp8 archive is an ordinary
 * byte archive (dgb_ans_encode_pointer of the fp8 bytes; the 256-symbol coder codes each word whole), so there is no
 * float header for these types: only dgb_float_cast_fp8 and the device-scale decode-and-sum entries take them, and
 * every other float entry refuses them.  9 stays unassigned. */
#define DGB_FLOAT8_E4M3 10
#define DGB_FLOAT8_E5M2 11

/* ans/GpuANSCodec.h:16,20 */
#define DGB_ANS_REQUIRED_ALIGNMENT 4
#define DGB_ANS_DEFAULT_PROB_BITS 10

int dgb_version(void);
const char* dgb_error_string(int code);
/* cudaError_t of the most recent DGB_ERR_CUDA on this thread (0 if none). */
int dgb_last_cuda_error(void);

/* ---- size bounds -------------------------------------------------------- */

/* ans/GpuANSEncode.cu:13-25 getMaxCompressedSize (same value, same quirk). */
uint32_t dgb_ans_max_compressed_size(uint32_t uncompressed_bytes);
/* float/GpuFloatCompress.cu:23-45 getMaxFloatCompressedSize; for DGB_FLOAT64, 16 + the ANS bound + the three
 * planes; for the sparse fp16 / bf16 types, 32 + 4 * roundUp(ceil(n / 4096), 4) + roundUp(n, 16) + the ANS bound;
 * for DGB_FLOAT32_SPARSE, 32 + 4 * roundUp(ceil(n / 4096), 4) + 2 * roundUp(n, 8) + roundUp(n, 16) + the ANS
 * bound.  0 when the bound does not fit 32 bits (encode then returns DGB_ERR_TOO_LARGE). */
uint32_t dgb_float_max_compressed_size(int float_type, uint32_t num_floats);

/* ---- scratch sizing (new; the reference sizes scratch implicitly through
 *      StackDeviceMemory and falls back to cudaMalloc) ---------------------- */
size_t dgb_ans_encode_temp_bytes(uint32_t num_in_batch, uint32_t max_uncompressed_bytes);
size_t dgb_ans_decode_temp_bytes(uint32_t num_in_batch);
size_t dgb_float_compress_temp_bytes(int float_type, uint32_t num_in_batch, uint32_t max_num_floats);
size_t dgb_float_decompress_temp_bytes(int float_type, uint32_t num_in_batch, uint32_t max_num_floats);

/* ---- byte rANS encode --------------------------------------------------- */

/* ans/GpuANSCodec.h:100-128 / ans/GpuANSEncode.cu:55-113 ansEncodeBatchPointer.
 * in/out: host arrays of num_in_batch device pointers; in_size: host array of
 * byte counts; out[i] must hold dgb_ans_max_compressed_size(in_size[i]) bytes.
 * histogram_dev: optional device [num_in_batch][256] u32 pre-computed counts.
 * out_size_dev: optional device u32[num_in_batch], receives archive sizes. */
int dgb_ans_encode_pointer(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                           uint32_t num_in_batch, const void* const* in, const uint32_t* in_size,
                           const uint32_t* histogram_dev, void* const* out,
                           uint32_t* out_size_dev, void* stream);

/* ans/GpuANSCodec.h:65-98 / ans/GpuANSEncode.cu:27-53 ansEncodeBatchStride. */
int dgb_ans_encode_stride(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                          uint32_t num_in_batch, const void* in_dev, uint32_t in_per_batch_size,
                          uint32_t in_per_batch_stride, const uint32_t* histogram_dev,
                          void* out_dev, uint32_t out_per_batch_stride,
                          uint32_t* out_size_dev, void* stream);

/* ans/GpuANSCodec.h:130-164 / ans/GpuANSEncode.cu:115-179 ansEncodeBatchSplitSize.
 * in_split_sizes: host array; member i starts at sum_{j<i} in_split_sizes[j];
 * interior sizes must be multiples of 4. */
int dgb_ans_encode_split_size(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                              uint32_t num_in_batch, const void* in_dev,
                              const uint32_t* in_split_sizes, const uint32_t* histogram_dev,
                              void* out_dev, uint32_t out_stride, uint32_t* out_size_dev,
                              void* stream);

/* ---- byte rANS decode --------------------------------------------------- */

/* ans/GpuANSCodec.h:228-263 / ans/GpuANSDecode.cu:47-120 ansDecodeBatchPointer.
 * out_capacity: host array (bytes).  out_success_dev (u8[n]) / out_size_dev
 * (u32[n]): optional device arrays; a member whose capacity is too small, or
 * whose header is not a valid archive of `prob_bits`, gets success=0 and is
 * skipped (size = required bytes, or 0 for an invalid header).
 * With use_checksum != 0 the call synchronises `stream`, compares checksums
 * and returns DGB_ERR_CHECKSUM on mismatch; checksum_mismatch_host (optional
 * host u8[n]) then flags the failing members.  A member whose archive was
 * written without a checksum (flag bit 4 of its options clear) is not
 * verified: its checksum word is undefined.  That synchronisation cannot be
 * captured into a CUDA graph: on a capturing stream such a call returns
 * DGB_ERR_CAPTURING before it enqueues anything, and the capture stays valid. */
int dgb_ans_decode_pointer(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                           uint32_t num_in_batch, const void* const* in, void* const* out,
                           const uint32_t* out_capacity, uint8_t* out_success_dev,
                           uint32_t* out_size_dev, uint8_t* checksum_mismatch_host, void* stream);

/* ans/GpuANSCodec.h:170-226 / ans/GpuANSDecode.cu:20-45 ansDecodeBatchStride. */
int dgb_ans_decode_stride(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                          uint32_t num_in_batch, const void* in_dev, uint32_t in_per_batch_stride,
                          void* out_dev, uint32_t out_per_batch_stride,
                          uint32_t out_per_batch_capacity, uint8_t* out_success_dev,
                          uint32_t* out_size_dev, uint8_t* checksum_mismatch_host, void* stream);

/* ans/GpuANSCodec.h:265-303 / ans/GpuANSDecode.cu:122-193 ansDecodeBatchSplitSize. */
int dgb_ans_decode_split_size(void* temp_dev, size_t temp_bytes, int prob_bits, int use_checksum,
                              uint32_t num_in_batch, const void* const* in, void* out_dev,
                              const uint32_t* out_split_sizes, uint8_t* out_success_dev,
                              uint32_t* out_size_dev, uint8_t* checksum_mismatch_host,
                              void* stream);

/* ans/GpuANSCodec.h:309-341 / ans/GpuANSInfo.cu:14-49 ansGetCompressedInfo{,Device}.
 * out_sizes_dev receives each archive's UNCOMPRESSED size in bytes (what the
 * reference kernel reports, ans/GpuANSInfo.cuh:27-29), 0 for a bad header.
 * in_is_device_array != 0: `in` is a device array of device pointers. */
int dgb_ans_get_compressed_info(void* temp_dev, size_t temp_bytes, const void* const* in,
                                int in_is_device_array, uint32_t num_in_batch,
                                uint32_t* out_sizes_dev, uint32_t* out_checksum_dev, void* stream);

/* ---- float codec (fp16 / bf16 / fp32 / fp64) ------------------------------ */

/* float/GpuFloatCodec.h:103-139 / float/GpuFloatCompress.cu:47-101 floatCompress.
 * in_size counts float WORDS.  out[i] must hold
 * dgb_float_max_compressed_size(float_type, in_size[i]) bytes.  The checksum covers the first in_size[i]
 * BYTES of the input, the reference's float rule (for DGB_FLOAT64, the first in_size[i] / 8 words). */
int dgb_float_compress_pointer(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                               int use_checksum, uint32_t num_in_batch, const void* const* in,
                               const uint32_t* in_size, void* const* out, uint32_t* out_size_dev,
                               void* stream);

/* Scaled fp8 cast with a fused histogram (new; no reference counterpart), the first half of an fp8 compress.
 * in_float_type: DGB_FLOAT32 or DGB_BFLOAT16; fp8_type: DGB_FLOAT8_E4M3 or DGB_FLOAT8_E5M2; any other pair returns
 * DGB_ERR_INVALID_ARG before any CUDA call.  in[i] (aligned to its word size) holds in_size[i] words; out[i]
 * receives in_size[i] bytes, q = cvt.rn.satfinite.fp8(fp32(x) * s), with s = *scale_dev (4 B aligned; NULL means
 * 1.0f), the product one round-to-nearest-even fp32 multiply (never contracted) and the bf16 widening exact.  For
 * every x whose product is not NaN this is torch's (x.float() * s).clamp(-M, M).to(fp8) byte for byte (M = 448 for
 * E4M3, 57344 for E5M2): out-of-range products and infinities saturate to +-M, products too small for the fp8
 * type's subnormals round to +-0 and keep their sign.  A NaN product gives the byte 0x7F whatever its sign (the
 * H100's F2FP.SATFINITE writes the positive canonical NaN).
 * histogram_dev (may be NULL): num_in_batch x 256 u32 counts, overwritten (not accumulated) with the histogram of
 * each out[i]: exactly what the byte encoder's statistics pass counts, so that
 *   dgb_float_cast_fp8(..., out, hist, stream); dgb_ans_encode_pointer(..., out, in_size, hist, archives, ...)
 * is the fp8 compress, whose archives are byte archives of q, bit-identical to dgb_ans_encode_pointer of q without a
 * histogram.  With the histogram and no checksum the encoder skips its own statistics pass, so the input is read once
 * and q is written once and read once.  out[i] may have any alignment, but the byte encoder wants it 4 B aligned
 * (DGB_ANS_REQUIRED_ALIGNMENT).  in and out must not overlap.  Never synchronises; capturable into a CUDA graph (a
 * replay reads *scale_dev's value then). */
int dgb_float_cast_fp8(int in_float_type, int fp8_type, uint32_t num_in_batch, const void* const* in,
                       const uint32_t* in_size, const float* scale_dev, void* const* out, uint32_t* histogram_dev,
                       void* stream);

/* Compress with a narrowing cast (new; no reference counterpart).  The allowed pairs (in_float_type, float_type)
 * are (DGB_FLOAT16, DGB_FLOAT16), (DGB_BFLOAT16, DGB_BFLOAT16) and (DGB_FLOAT32, DGB_FLOAT32), which are exactly
 * dgb_float_compress_pointer, and the narrowing pairs (DGB_FLOAT32, DGB_FLOAT16) and (DGB_FLOAT32, DGB_BFLOAT16);
 * any other pair returns DGB_ERR_INVALID_ARG before any CUDA call.
 * Narrowing: in[i] holds in_size[i] float32 words (4 B aligned), and out[i] receives exactly the archive
 * dgb_float_compress_pointer(float_type, ...) writes for r = the words rounded to float_type, round to nearest
 * even as torch's CUDA cast rounds (cvt.rn.f16.f32 / cvt.rn.bf16.f32, NaNs included):
 * the same size, header, pdf, lane states, block table and streams (with encode_canonical = 1 the same bytes;
 * by default the streams are in completion order, as for every type), and the checksum of r (its first
 * in_size[i] bytes).  The archive is an ordinary float_type archive: every decoder, the decode-and-sum and the
 * reference read it.  No temporary of r exists; the input is not modified.  out[i] must hold
 * dgb_float_max_compressed_size(float_type, in_size[i]) bytes, the scratch is
 * dgb_float_compress_temp_bytes(float_type, n, max in_size), and the refusals and error codes are
 * dgb_float_compress_pointer's.  Never synchronises; capturable into a CUDA graph. */
int dgb_float_compress_to(void* temp_dev, size_t temp_bytes, int in_float_type, int float_type, int prob_bits,
                          int use_checksum, uint32_t num_in_batch, const void* const* in, const uint32_t* in_size,
                          void* const* out, uint32_t* out_size_dev, void* stream);

/* Narrowing compress with error feedback (new; no reference counterpart).  The allowed pairs are the narrowing
 * ones, (DGB_FLOAT32, DGB_FLOAT16) and (DGB_FLOAT32, DGB_BFLOAT16).  err is a host array of num_in_batch device
 * pointers: err[i] holds in_size[i] float32 residual words, one per input word.  For each input word x, its
 * residual word e and the archive type T:
 *   y  = x + e                            one round-to-nearest float32 add, subnormals kept (torch's CUDA add)
 *   w  = round_T(y)                       cvt.rn.f16.f32 / cvt.rn.bf16.f32, as dgb_float_compress_to rounds
 *   e' = y - float(w) if w is finite, else +0   (one float32 subtraction, exact for a finite w; no fused multiply-add)
 * out[i] receives exactly the archive dgb_float_compress_to(DGB_FLOAT32, float_type, ...) writes for the words y
 * (with encode_canonical = 1 the same bytes; by default the same fields, size and decoded words, with the streams in
 * completion order), and the checksum option covers w.  err[i] is overwritten with e'; the input is not modified.
 * The residual of a word that rounds to inf or NaN is +0 so that the buffer never holds an inf or a NaN: that step
 * still carries the non-finite word, and the next starts clean.  So e' is bit for bit the torch expression
 * torch.where(w.isfinite(), y - w.float(), 0) with y = x + e and w = y.to(T).
 * err[i] must have the same address modulo 16 as in[i], and the err buffers must not overlap each other, any input,
 * any output or the scratch.  A pair other than the two above, a NULL err, a NULL err[i] for a non-empty member, or
 * an err[i] whose address modulo 16 differs from in[i]'s returns DGB_ERR_INVALID_ARG before any CUDA call, as do
 * dgb_float_compress_to's refusals.  Scratch: dgb_float_compress_temp_bytes(float_type, n, max in_size); output
 * bounds: dgb_float_compress_to's.  Never synchronises; capturable into a CUDA graph (a replay reads the residuals
 * the previous replay wrote). */
int dgb_float_compress_to_ef(void* temp_dev, size_t temp_bytes, int in_float_type, int float_type, int prob_bits,
                             int use_checksum, uint32_t num_in_batch, const void* const* in, const uint32_t* in_size,
                             float* const* err, void* const* out, uint32_t* out_size_dev, void* stream);

/* float/GpuFloatCodec.h:141-170 / float/GpuFloatCompress.cu:103-159 floatCompressSplitSize. */
int dgb_float_compress_split_size(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                                  int use_checksum, uint32_t num_in_batch, const void* in_dev,
                                  const uint32_t* in_split_sizes, void* out_dev,
                                  uint32_t out_stride, uint32_t* out_size_dev, void* stream);

/* float/GpuFloatCodec.h:176-208 / float/GpuFloatDecompress.cu:22-115 floatDecompress.
 * out_capacity / out_size_dev are in float WORDS.  The reference's
 * is16ByteAligned switch is not needed: one fused decode+join kernel handles
 * any word-aligned output. */
int dgb_float_decompress_pointer(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                                 int use_checksum, uint32_t num_in_batch, const void* const* in,
                                 void* const* out, const uint32_t* out_capacity,
                                 uint8_t* out_success_dev, uint32_t* out_size_dev,
                                 uint8_t* checksum_mismatch_host, void* stream);

/* float/GpuFloatCodec.h:210-246 / float/GpuFloatDecompress.cu:117-179 floatDecompressSplitSize. */
int dgb_float_decompress_split_size(void* temp_dev, size_t temp_bytes, int float_type,
                                    int prob_bits, int use_checksum, uint32_t num_in_batch,
                                    const void* const* in, void* out_dev,
                                    const uint32_t* out_split_sizes, uint8_t* out_success_dev,
                                    uint32_t* out_size_dev, uint8_t* checksum_mismatch_host,
                                    void* stream);

/* Decode-and-sum (new; no reference counterpart): out[g] = (accumulate ? out[g] : x(g,0)) + x(g,1) + ... +
 * x(g,W-1) in archive order, where x(g,j) is the decoded content of archive (g, j) = in[g * W + j] and each + is
 * one IEEE-754 round-to-nearest-even addition in the element type, subnormals kept (for fp16 / bf16 the same
 * result as torch's a + b).  Without accumulate and with W = 1 this is a plain decode (NaN payloads and -0 kept).
 * float_type: DGB_FLOAT16, DGB_BFLOAT16 or DGB_FLOAT32 (else DGB_ERR_INVALID_ARG).  in: host array of G * W
 * device pointers (16 B aligned), group-major; out / out_size: host arrays of G (out_size in words, outputs
 * aligned to the word size; outputs must not overlap each other or any archive).  An archive is valid when its
 * headers have float_type and prob_bits, a consistent block count and exactly out_size[g] words;
 * out_success_dev (optional, device u8[G * W]) receives 1 or 0 per archive, and a group with an invalid archive
 * is not written at all.  Stored checksums are not verified.  num_groups = 0 returns DGB_OK and does nothing.
 * Never synchronises; capturable into a CUDA graph.  Scratch: dgb_float_decompress_temp_bytes(float_type,
 * G * W, 0). */
int dgb_float_decompress_reduce(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                                uint32_t num_groups, uint32_t archives_per_group, const void* const* in,
                                void* const* out, const uint32_t* out_size, int accumulate,
                                uint8_t* out_success_dev, void* stream);

/* Decode-and-sum into outputs of out_float_type (new; no reference counterpart).  The allowed pairs
 * (float_type, out_float_type) are (DGB_FLOAT16, DGB_FLOAT16), (DGB_BFLOAT16, DGB_BFLOAT16) and
 * (DGB_FLOAT32, DGB_FLOAT32), which give exactly what dgb_float_decompress_reduce gives, and the widening pairs
 * (DGB_FLOAT16, DGB_FLOAT32) and (DGB_BFLOAT16, DGB_FLOAT32); any other pair returns DGB_ERR_INVALID_ARG.
 * Widening: out[g] = (accumulate ? out[g] : f(x(g,0))) + f(x(g,1)) + ... + f(x(g,W-1)) in archive order, where
 * f is the exact conversion of a 16-bit word to fp32 and each + is one fp32 round-to-nearest-even addition,
 * subnormals kept: bit-identical to torch's fold acc = x0.float(); acc = acc + x1.float(); ...  With W = 1 and
 * no accumulate this is a plain decode widened to fp32 (-0, infinities and subnormals exact; a NaN stays a
 * NaN).  Outputs are fp32 (4 B aligned) and out_size counts their elements, which must equal every archive's
 * word count.  Everything else is as in dgb_float_decompress_reduce: the validity rule (the archives have
 * float_type), statuses, groups with an invalid archive left unwritten, no synchronisation, graph capture and
 * the scratch size dgb_float_decompress_temp_bytes(float_type, G * W, 0). */
int dgb_float_decompress_reduce_to(void* temp_dev, size_t temp_bytes, int float_type, int out_float_type,
                                   int prob_bits, uint32_t num_groups, uint32_t archives_per_group,
                                   const void* const* in, void* const* out, const uint32_t* out_size,
                                   int accumulate, uint8_t* out_success_dev, void* stream);

/* Decode-and-sum of sparse archives (new; no reference counterpart).  The allowed pairs (float_type,
 * out_float_type) are (DGB_FLOAT16_SPARSE, DGB_FLOAT16), (DGB_BFLOAT16_SPARSE, DGB_BFLOAT16),
 * (DGB_FLOAT32_SPARSE, DGB_FLOAT32), (DGB_FLOAT16_SPARSE, DGB_FLOAT32) and (DGB_BFLOAT16_SPARSE, DGB_FLOAT32); any
 * other pair returns DGB_ERR_INVALID_ARG.  For every input the result is bit-identical to
 * dgb_float_decompress_reduce_to(float_type's dense type, out_float_type) on dense archives of the same words:
 * an elided word is the +0 or -0 it stands for and is added as such.  An archive is valid when its headers have
 * float_type (a dense archive in a sparse group is invalid) and prob_bits, a consistent block count and exactly
 * out_size[g] words.  Everything else is as in dgb_float_decompress_reduce_to: the sum order, statuses, groups
 * with an invalid archive left unwritten, no synchronisation, graph capture, num_groups = 0 returning DGB_OK and
 * the scratch size dgb_float_decompress_temp_bytes(float_type, G * W, 0). */
int dgb_float_decompress_reduce_sparse(void* temp_dev, size_t temp_bytes, int float_type, int out_float_type,
                                       int prob_bits, uint32_t num_groups, uint32_t archives_per_group,
                                       const void* const* in, void* const* out, const uint32_t* out_size,
                                       int accumulate, uint8_t* out_success_dev, void* stream);

/* Pre-multiplied decode-and-sum (new; no reference counterpart): every decoded word x is multiplied by `scale`
 * before it is summed, as an average over ranks (scale = 1 / W) or a gradient pre-division needs, without a scaled
 * copy of any input.  The allowed pairs (float_type, out_float_type) are the five of dgb_float_decompress_reduce_to
 * and the five of dgb_float_decompress_reduce_sparse; any other pair returns DGB_ERR_INVALID_ARG before any CUDA
 * call.  The term of a word is
 *   fp16 / bf16 archives, outputs of the same type:  round_T(fp32(x) * scale), one fp32 round-to-nearest-even
 *                                                     multiply, then one round-to-nearest-even conversion to T;
 *   fp32 archives:                                   x * scale, one fp32 round-to-nearest-even multiply;
 *   fp16 / bf16 archives, fp32 outputs:              fp32(x) * scale, left in fp32;
 * sparse archives take the rule of their dense type for the word they stand for: an elided word is the +0 or -0 it
 * stands for and is multiplied like any other (a negative scale turns +0 into -0; an infinite or NaN scale makes it
 * NaN).  out[g] = (accumulate ? out[g] : term(x(g,0))) + term(x(g,1)) + ... + term(x(g,W-1)) in archive order with
 * the output type's add; the value taken in by accumulate is not scaled, so a sum may be split over several calls.
 * This is torch's fold with term(x) = (x.float() * s).to(out dtype) for a float32 tensor s, bit for bit (NaN
 * payloads aside); with scale = 1 it is exactly the unscaled entries' result.  Everything else is as in
 * dgb_float_decompress_reduce_to / dgb_float_decompress_reduce_sparse: the validity rule, statuses, groups with an
 * invalid archive left unwritten, no synchronisation, num_groups = 0 returning DGB_OK and the scratch size
 * dgb_float_decompress_temp_bytes(float_type, G * W, 0).  The scale travels by value in the kernels' parameters: a
 * call captured into a CUDA graph replays with the scale it was captured with. */
int dgb_float_decompress_reduce_scaled(void* temp_dev, size_t temp_bytes, int float_type, int out_float_type,
                                       int prob_bits, uint32_t num_groups, uint32_t archives_per_group,
                                       const void* const* in, void* const* out, const uint32_t* out_size,
                                       int accumulate, float scale, uint8_t* out_success_dev, void* stream);

/* Device-scale decode-and-sum (new; no reference counterpart): dgb_float_decompress_reduce_scaled with the scale
 * read from device memory, *scale_dev, by the kernels when they run, and an optional non-finite flag.  For mixed-
 * precision loss scaling (an inverse loss scale that lives on the device), a per-token normalisation whose token
 * count comes out of an all-reduce, or a CUDA graph whose scale changes between replays: the host never reads the
 * scale, the call never synchronises and may be captured, and a replay reads the value *scale_dev holds then.
 * Everything else is dgb_float_decompress_reduce_scaled's contract with s = *scale_dev: the ten type pairs, the
 * terms, the fold, the validity rule, statuses, groups with an invalid archive left unwritten, num_groups = 0
 * returning DGB_OK with nothing written, and the scratch size; the result is bit-identical to that entry called
 * with the same float.  Every launch of a call (one per 4 archives of a group) reads *scale_dev.
 * found_inf_dev (may be NULL): set to 1.0f when any output word this call writes ends up inf or NaN (exponent field
 * all ones).  Only final values are checked: the words the writer of archive W - 1 stores.  Output words this call
 * leaves alone (past out_size[g], or in a group with an invalid archive) never count.  The flag is never cleared,
 * as torch.amp's found_inf is not; a non-finite input word, a finite word times an infinite or NaN scale, inf * 0, a
 * sum that overflows and a non-finite running value taken in by accumulate all set it, since no later term turns
 * inf or NaN finite.
 * DGB_ERR_INVALID_ARG before any CUDA call: scale_dev NULL or not 4 B aligned, found_inf_dev not 4 B aligned, and
 * every argument dgb_float_decompress_reduce_scaled refuses.
 * fp8 sums: this entry and dgb_float_decompress_reduce_scaled_dev_norm also take the pairs (DGB_FLOAT8_E4M3,
 * DGB_FLOAT32) and (DGB_FLOAT8_E5M2, DGB_FLOAT32), which no other decode-and-sum entry takes.  Their archives are
 * byte archives (dgb_float_cast_fp8 + dgb_ans_encode_pointer) of out_size[g] fp8 words; one is valid iff its ANS
 * header has the magic, prob_bits, ceil(out_size[g] / 4096) blocks and out_size[g] uncompressed bytes.  The term is
 * fp32(q) * s (the fp8 word widened exactly, one fp32 multiply), so out[g] = (accumulate ? out[g] : term(q(g,0))) +
 * term(q(g,1)) + ... in fp32 in archive order: torch's acc = q0.float() * d; acc = acc + q1.float() * d; ... bit for
 * bit.  Statuses, found_inf_dev, groups left unwritten, graph capture and num_groups = 0 are as above; the scratch
 * is dgb_float_decompress_temp_bytes(fp8 type, G * W, 0). */
int dgb_float_decompress_reduce_scaled_dev(void* temp_dev, size_t temp_bytes, int float_type, int out_float_type,
                                           int prob_bits, uint32_t num_groups, uint32_t archives_per_group,
                                           const void* const* in, void* const* out, const uint32_t* out_size,
                                           int accumulate, const float* scale_dev, float* found_inf_dev,
                                           uint8_t* out_success_dev, void* stream);

/* Narrowing decode-and-sum (new; no reference counterpart): fp16 / bf16 archives summed in fp32 and rounded once to
 * the archives' 16-bit type, so a 16-bit result carries one rounding instead of one per add and needs no fp32
 * output.  float_type: DGB_FLOAT16, DGB_BFLOAT16, DGB_FLOAT16_SPARSE or DGB_BFLOAT16_SPARSE; out[g] (2 B aligned)
 * has that dense type, acc[g] (4 B aligned) is an fp32 accumulator of out_size[g] elements.
 * out[g] = round(S) with S = (accumulate ? acc[g] : term(x(g,0))) + term(x(g,1)) + ... + term(x(g,W-1)) taken in
 * fp32 in archive order, each + one fp32 round-to-nearest-even add, and round one round-to-nearest-even conversion
 * to the 16-bit type: bit-identical to dgb_float_decompress_reduce_to (or _scaled / _scaled_dev) into fp32 outputs
 * followed by torch's .to(dtype).  term is the widening entries' term: fp32(x), or fp32(x) * s with the host
 * `scale` or the device scale *scale_dev (at most one of them).  The running sums of every archive but the last go
 * through acc[g], which ends up unspecified; out[g] is only written, never read.  acc (the array, and each acc[g] with
 * out_size[g] > 0) may be NULL when the call reads no accumulator: W = 1 without accumulate.  found_inf_dev (with
 * scale_dev only; may be NULL): set to 1.0f when a 16-bit word this call stores is inf or NaN, so an fp32 sum that
 * rounds to an fp16 infinity counts.  Everything else is as in dgb_float_decompress_reduce_scaled_dev: the validity
 * rule, statuses, groups with an invalid archive left unwritten (acc[g] and out[g] both), num_groups = 0 returning
 * DGB_OK, no synchronisation, graph capture (a replay reads *scale_dev's value then) and the scratch size
 * dgb_float_decompress_temp_bytes(float_type, G * W, 0).  DGB_ERR_INVALID_ARG before any CUDA call: any other
 * float_type, scale with scale_dev, found_inf_dev without scale_dev, a misaligned scale_dev or found_inf_dev, a NULL
 * or misaligned acc[g] or out[g] where it is needed, and every argument the other decode-and-sum entries refuse. */
int dgb_float_decompress_reduce_narrow(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                                       uint32_t num_groups, uint32_t archives_per_group, const void* const* in,
                                       float* const* acc, void* const* out, const uint32_t* out_size,
                                       int accumulate, const float* scale, const float* scale_dev,
                                       float* found_inf_dev, uint8_t* out_success_dev, void* stream);

/* Squared norms (new; no reference counterpart), for clipping a reduced gradient by its global norm without reading
 * it again.  The squared norm of a group is an fp64 value over the float words v[0 .. n-1] of the group (for a
 * decode-and-sum: the words the call stores, after scaling and after the narrowing sums' 16-bit rounding), taken in
 * this order, whatever the grid or the order in which blocks were claimed:
 *   1. lane: word i lies in block k = i / 4096, row r = (i mod 4096) / 32 and lane l = i mod 32.  Each lane starts
 *      from +0 and adds, for its words of block k in DESCENDING row order (the decoder's order: a partial last row
 *      first), v * v with v the word widened exactly to fp64 (v * v is exact, so this is one fp64 add; fma(v, v, p)).
 *      A lane past the end of a partial row adds nothing; an elided sparse word is the +0 or -0 it stands for.
 *   2. warp: the 32 lane sums p are combined by the xor butterfly p = p + shfl_xor(p, o) for o = 16, 8, 4, 2, 1,
 *      which leaves every lane with the same value q[k], the block's partial.
 *   3. group: thread t (0 <= t < 256) of one 256-thread CTA sums q[t], q[t + 256], q[t + 512], ... from +0 in
 *      increasing block order; each of the 8 warps applies the butterfly of step 2 to its 32 sums, and the result is
 *      ((w[0] + w[1]) + w[2]) + ... + w[7] over the warp sums w in warp order.
 * Every add is one fp64 round-to-nearest-even add.  An inf or NaN word gives an inf or NaN norm; an empty group gets
 * +0.  tests/sq_norm_reference.py restates the order in numpy. */

/* dgb_float_decompress_reduce_scaled_dev, and sq_norm_dev[g] (device, G doubles, 8 B aligned; required) overwritten
 * with the squared norm above of the out_size[g] words the call stores to out[g].  Only the writer of archive W - 1
 * contributes, so a call of several launches (W > 4) takes the norm in its last.  A group with an invalid archive
 * leaves sq_norm_dev[g] untouched, as it leaves out[g].  Outputs, statuses and found_inf_dev are bit-identical to
 * dgb_float_decompress_reduce_scaled_dev's.  An unscaled caller passes a device 1.0f as scale_dev.
 * Scratch: dgb_float_decompress_reduce_norm_temp_bytes(float_type, G, W, out_size).
 * DGB_ERR_INVALID_ARG before any CUDA call: sq_norm_dev NULL or not 8 B aligned, and everything
 * dgb_float_decompress_reduce_scaled_dev refuses.  num_groups = 0 returns DGB_OK and writes nothing; the call never
 * synchronises and may be captured into a CUDA graph. */
int dgb_float_decompress_reduce_scaled_dev_norm(void* temp_dev, size_t temp_bytes, int float_type,
                                                int out_float_type, int prob_bits, uint32_t num_groups,
                                                uint32_t archives_per_group, const void* const* in, void* const* out,
                                                const uint32_t* out_size, int accumulate, const float* scale_dev,
                                                float* found_inf_dev, double* sq_norm_dev, uint8_t* out_success_dev,
                                                void* stream);

/* dgb_float_decompress_reduce_narrow with the device scale (scale_dev required; there is no host scale), and
 * sq_norm_dev[g] as in dgb_float_decompress_reduce_scaled_dev_norm, over the 16-bit words stored to out[g] (the
 * rounded sums).  Scratch: dgb_float_decompress_reduce_norm_temp_bytes(float_type, G, W, out_size).
 * DGB_ERR_INVALID_ARG before any CUDA call: scale_dev NULL or not 4 B aligned, sq_norm_dev NULL or not 8 B aligned,
 * and everything dgb_float_decompress_reduce_narrow refuses. */
int dgb_float_decompress_reduce_narrow_norm(void* temp_dev, size_t temp_bytes, int float_type, int prob_bits,
                                            uint32_t num_groups, uint32_t archives_per_group, const void* const* in,
                                            float* const* acc, void* const* out, const uint32_t* out_size,
                                            int accumulate, const float* scale_dev, float* found_inf_dev,
                                            double* sq_norm_dev, uint8_t* out_success_dev, void* stream);

/* Scratch of the two entries above: dgb_float_decompress_temp_bytes(float_type, G * W, 0) plus the squared norm's own
 * part, 8 B per 4096-word block of every group (8 * sum of ceil(out_size[g] / 4096)) and 12 B per group for the block
 * offsets, sizes and validity flags, each rounded up to 256 B.  0 for an invalid float_type (the fp8 types are
 * valid here). */
size_t dgb_float_decompress_reduce_norm_temp_bytes(int float_type, uint32_t num_groups, uint32_t archives_per_group,
                                                   const uint32_t* out_size);

/* The squared norm above of G dense float tensors already in device memory: in[g] (host array of G device
 * pointers, aligned to the word size) holds size[g] words of float_type (DGB_FLOAT16, DGB_BFLOAT16 or DGB_FLOAT32),
 * and sq_norm_dev[g] (device, 8 B aligned, required) is overwritten with their squared norm, bit-identical to what
 * the decode-and-sum norm entries give for the same stored words.  A plain read of the words (one warp per 4096-word
 * block).  Scratch: dgb_float_sq_norm_temp_bytes(G, size), 256 B aligned.  DGB_ERR_INVALID_ARG before any CUDA
 * call for another float_type, sq_norm_dev NULL or misaligned, in or size NULL, or in[g] NULL or misaligned with
 * size[g] > 0; num_groups = 0 returns DGB_OK and writes nothing.  Never synchronises; capturable. */
int dgb_float_sq_norm(void* temp_dev, size_t temp_bytes, int float_type, uint32_t num_groups, const void* const* in,
                      const uint32_t* size, double* sq_norm_dev, void* stream);
/* 8 B per group for the pointer table, plus the squared norm's part of dgb_float_decompress_reduce_norm_temp_bytes. */
size_t dgb_float_sq_norm_temp_bytes(uint32_t num_groups, const uint32_t* size);

/* float/GpuFloatCodec.h:252-292 / float/GpuFloatInfo.cu:17-64 floatGetCompressedInfo{,Device}. */
int dgb_float_get_compressed_info(void* temp_dev, size_t temp_bytes, const void* const* in,
                                  int in_is_device_array, uint32_t num_in_batch,
                                  uint32_t* out_sizes_dev, uint32_t* out_types_dev,
                                  uint32_t* out_checksum_dev, void* stream);

/* ---- host front end helpers (new) ----------------------------------------- */
/* Plain asynchronous copies on `stream`, used by the host-buffer front end (dietgpu_b200.HostCodec)
 * to move whole member groups in one DMA each instead of one call per member.  dgb_copy_async is
 * cudaMemcpyAsync(cudaMemcpyDefault); dgb_copy_rows_async copies `rows` rows of `width_bytes` between
 * two pitched matrices (cudaMemcpy2DAsync), e.g. archives [n, cols] device <-> pinned host. */
int dgb_copy_async(void* dst, const void* src, size_t bytes, void* stream);
int dgb_copy_rows_async(void* dst, size_t dst_pitch, const void* src, size_t src_pitch,
                        size_t width_bytes, size_t rows, void* stream);

/* ---- archive mover (new; for the compressed collectives) -------------------- */
/* Copies num_in_batch archives from src[i] to dst[i] (host arrays of device pointers, 16 B aligned), each
 * exactly as long as its own header says and at most dst_capacity[i] bytes: float_type 0 = ANS archives
 * (ans/GpuANSUtils.cuh:67-227 header), DGB_FLOAT16/BFLOAT16/FLOAT32/FLOAT64 and the sparse types = float archives
 * (float/GpuFloatUtils.cuh:26-74).  src may be memory of a peer GPU mapped into this process (NVLink):
 * sizes are read on the device, nothing travels to the host; out_bytes_dev (optional, device, [n]) receives
 * the archive sizes.  An archive with a bad header is copied as its first 32 bytes so that the decoder
 * which follows reports it.  The reference has no counterpart (it names the use, README.md:72,103-104). */
int dgb_archives_pull(int float_type, uint32_t num_in_batch, const void* const* src, void* const* dst,
                      const uint32_t* dst_capacity, uint32_t* out_bytes_dev, void* stream);

/* ---- tuning knob (benchmarks / tests only) ------------------------------- */
/* Selects an internal kernel variant by name ("parts", "encode_canonical", "decode_warps" ...; the list
 * is in INTEGRATION.md section 4).  Unknown names return DGB_ERR_INVALID_ARG.  Defaults are the tuned choice. */
int dgb_set_option(const char* name, int value);
int dgb_get_option(const char* name, int* value);
/* Per-thread override: the first call copies the process-wide set into a copy that only codec calls made by
 * THIS thread see (and dgb_get_option on this thread reports); dgb_clear_thread_options drops the copy.  Every
 * codec call snapshots its effective set at entry, so changing options never affects a call in flight. */
int dgb_set_thread_option(const char* name, int value);
int dgb_clear_thread_options(void);
/* With option "timing" = 1 every kernel launch is bracketed by CUDA events on the caller's
 * stream; this returns (and resets) the summed durations in ms and launch counts per kernel:
 * slot 0 stats (K1), 1 encode (K2), 2 plan, 3 decode, 4 checksum, 5 fused encode, 6 archive mover.  Synchronises the device. */
int dgb_kernel_times(float* ms, int* counts, int nslots);

#ifdef __cplusplus
}
#endif
#endif /* DIETGPU_B200_H_ */
