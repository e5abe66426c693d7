"""Host-side mirror of the reference's PyTorch operator surface
(torch.ops.dietgpu.*, /root/reference/dietgpu/DietGpu.cpp:915-972) on top of
the C ABI: same names, same argument meaning, same return values, same error
behaviour (TORCH_CHECK -> RuntimeError).  Tensors are only used for device
memory, streams and dtypes; all compute is in libdietgpu_b200.so.

    compress_data(compress_as_float, ts_in, checksum=False, temp_mem=None,
                  out_compressed=None, out_compressed_bytes=None)
        -> (Tensor [B, maxCols] u8, Tensor [B] i32, int temp_bytes_used)   DietGpu.cpp:277-308
    decompress_data(compress_as_float, ts_in, ts_out, checksum=False, temp_mem=None,
                    out_status=None, out_decompressed_words=None) -> int     DietGpu.cpp:646-677
    ... and the *_split_size / *_simple / max_* variants.

Python's precision is fixed at 10 bits as in the reference (DietGpu.cpp:114);
`prob_bits=` is an extension used by the parity tests (C++ API parity).

Where the reference would write or read memory the caller did not hand over, this layer (and the C++
operators, which raise for the same inputs) differs on purpose: byte batches of mixed dtypes get rows sized
by their largest member in bytes, split sizes must fit the tensor they index, float outputs must share one
dtype, and archives and output rows must be 16 B aligned.
"""
from __future__ import annotations

import ctypes as C
import numbers
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import capi

K_DEFAULT_PRECISION = 10  # DietGpu.cpp:114

_FLOAT_TYPES = {torch.float16: capi.FLOAT16, torch.bfloat16: capi.BFLOAT16, torch.float32: capi.FLOAT32,
                torch.float64: capi.FLOAT64}
_DTYPE_OF = {v: k for k, v in _FLOAT_TYPES.items()}
# sparse=True: fp16 / bf16 / fp32 archives that code +0 and -0 words as two spare symbols and store no bits for them
_SPARSE16_TYPES = {torch.float16: capi.FLOAT16_SPARSE, torch.bfloat16: capi.BFLOAT16_SPARSE}
_SPARSE_TYPES = {**_SPARSE16_TYPES, torch.float32: capi.FLOAT32_SPARSE}
_SPARSE_DTYPE_OF = {v: k for k, v in _SPARSE_TYPES.items()}


def _check(cond: bool, msg: str = "") -> None:
    if not cond:
        raise RuntimeError("dietgpu_b200 check failed" + (": " + msg if msg else ""))


def _float_type(t: torch.Tensor, sparse: bool = False) -> int:
    if sparse:
        if t.dtype not in _SPARSE_TYPES:
            raise ValueError(f"sparse=True needs float16, bfloat16 or float32 tensors, not {t.dtype}")
        return _SPARSE_TYPES[t.dtype]
    _check(t.dtype in _FLOAT_TYPES, f"unsupported float dtype {t.dtype}")
    return _FLOAT_TYPES[t.dtype]


def _check_sparse(compress_as_float: bool, sparse: bool) -> None:
    if sparse and not compress_as_float:
        raise ValueError("sparse=True needs compress_as_float=True")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _max_numel_and_bytes(ts: Sequence[torch.Tensor]) -> Tuple[int, int]:
    """Largest member in elements and, separately, in bytes (a byte batch may mix dtypes)."""
    mx = mx_bytes = 0
    for t in ts:
        _check(t.numel() * t.element_size() <= 0xFFFFFFFF, "tensor exceeds 4 GiB - 1")
        mx = max(mx, t.numel())
        mx_bytes = max(mx_bytes, t.numel() * t.element_size())
    return mx, mx_bytes


def _check_archive_aligned(t: torch.Tensor) -> None:
    _check(t.data_ptr() % 16 == 0, "compressed input is not 16 B aligned")


def _split_total(splits: Sequence[int], capacity: int, what: str) -> None:
    total = sum(splits)
    _check(total <= capacity, f"split sizes sum to {total}, more than {what} holds ({capacity})")


class _Temp:
    """Scratch handling: use the caller's temp_mem when it is large enough, else a
    stream-ordered torch allocation (the reference falls back to a synchronous
    cudaMalloc with a warning, utils/StackDeviceMemory.cpp:119-139)."""

    def __init__(self, temp_mem: Optional[torch.Tensor], need: int, device):
        self.need = need
        self.tensor = None
        if temp_mem is not None:
            _check(temp_mem.is_cuda and temp_mem.is_contiguous(), "temp_mem must be a contiguous CUDA tensor")
            base = temp_mem.data_ptr()
            pad = (-base) % 256
            avail = temp_mem.numel() * temp_mem.element_size() - pad
            if avail >= need:
                self.ptr, self.bytes = base + pad, avail
                return
        self.tensor = torch.empty(need + 256, dtype=torch.uint8, device=device)
        base = self.tensor.data_ptr()
        pad = (-base) % 256
        self.ptr, self.bytes = base + pad, need


# ---------------------------------------------------------------- sizes ----

def _bound(v: int, size: int) -> int:
    """The C ABI returns 0 when the worst-case archive does not fit the format's 32-bit sizes (the
    reference CHECK-aborts there, ans/GpuANSEncode.cu:22): raise instead of sizing a buffer from 0."""
    _check(v != 0 or size == 0, f"input of {size} elements is too large for one archive (32-bit format limit)")
    return v


def max_float_compressed_output_size(ts: Sequence[torch.Tensor], *, sparse: bool = False) -> Tuple[int, int]:
    mx, _ = _max_numel_and_bytes(ts)
    return len(ts), _bound(capi.lib().dgb_float_max_compressed_size(_float_type(ts[0], sparse), mx), mx)


def max_float_compressed_size(dtype: torch.Tensor, size: int, *, sparse: bool = False) -> int:
    """The single-size bound keeps its original `sparse=True` contract, float16 / bfloat16 only; the bound of a
    sparse float32 archive comes from max_float_compressed_output_size(ts, sparse=True) (or, for a size alone, from
    capi.lib().dgb_float_max_compressed_size(capi.FLOAT32_SPARSE, size))."""
    if sparse and dtype.dtype not in _SPARSE16_TYPES:
        raise ValueError(f"max_float_compressed_size(sparse=True) takes float16 or bfloat16, not {dtype.dtype}; "
                         "size sparse float32 archives with max_float_compressed_output_size(ts, sparse=True)")
    return _bound(capi.lib().dgb_float_max_compressed_size(_float_type(dtype, sparse), size), size)


def max_any_compressed_output_size(ts: Sequence[torch.Tensor]) -> Tuple[int, int]:
    # rows sized by the largest member in bytes; the reference multiplies the largest element count by
    # the first member's element size (DietGpu.cpp:134), too small for a batch of mixed dtypes
    _, mx_bytes = _max_numel_and_bytes(ts)
    return len(ts), _bound(capi.lib().dgb_ans_max_compressed_size(mx_bytes), mx_bytes)


def max_any_compressed_size(nbytes: int) -> int:
    return _bound(capi.lib().dgb_ans_max_compressed_size(nbytes), nbytes)


# ------------------------------------------------------------- compress ----

def _validate_out(out_compressed, out_sizes, n: int, cols: int, dev):
    if out_compressed is not None:
        _check(out_compressed.dtype == torch.uint8 and out_compressed.is_cuda
               and out_compressed.is_contiguous() and out_compressed.dim() == 2)
        _check(out_compressed.size(0) >= n and out_compressed.size(1) >= cols)
        _check(out_compressed.device == dev)
        _check(out_compressed.data_ptr() % 16 == 0 and (n <= 1 or out_compressed.size(1) % 16 == 0),
               "out_compressed rows are not 16 B aligned")
        comp = out_compressed
    else:
        comp = torch.empty((n, cols), dtype=torch.uint8, device=dev)
    if out_sizes is not None:
        _check(out_sizes.dtype == torch.int32 and out_sizes.is_cuda and out_sizes.dim() == 1
               and out_sizes.is_contiguous() and out_sizes.size(0) >= n and out_sizes.device == dev)
        sizes = out_sizes
    else:
        sizes = torch.empty((n,), dtype=torch.int32, device=dev)
    return comp, sizes


_NARROW_TYPES = {torch.float16: capi.FLOAT16, torch.bfloat16: capi.BFLOAT16}
# fp8 archives: byte archives of the scaled fp8 cast (dgb_float_cast_fp8) of float32 / bfloat16 inputs
FP8_TYPES = {torch.float8_e4m3fn: capi.FLOAT8_E4M3, torch.float8_e5m2: capi.FLOAT8_E5M2}
_FP8_INPUT_TYPES = {torch.float32: capi.FLOAT32, torch.bfloat16: capi.BFLOAT16}


def _check_fp8_inputs(what: str, ts_in: Sequence[torch.Tensor], dtype, scale_tensor) -> None:
    """The arguments of a scaled fp8 cast: an fp8 dtype, a non-empty list of contiguous CUDA tensors of one dtype
    (float32 or bfloat16) on one device, and scale_tensor None or a one-element float32 CUDA tensor on that device.
    Reads metadata only."""
    if dtype not in FP8_TYPES:
        raise ValueError(f"{what}: the fp8 dtype is torch.float8_e4m3fn or torch.float8_e5m2, not {dtype}")
    if isinstance(ts_in, torch.Tensor) or len(ts_in) == 0:
        raise ValueError(f"{what}: a non-empty list of tensors expected")
    d0, dev = ts_in[0].dtype, ts_in[0].device
    for t in ts_in:
        if getattr(t, "dtype", None) not in _FP8_INPUT_TYPES or t.dtype != d0 or not t.is_cuda \
                or t.device != dev or not t.is_contiguous():
            raise ValueError(f"{what}: contiguous float32 or bfloat16 CUDA tensors of one dtype on one device expected")
        if t.numel() > 0xFFFFFFFF:
            raise ValueError(f"{what}: a tensor of more than 2^32 - 1 elements")
    if scale_tensor is not None:
        _check_flag_tensor(f"{what}: scale_tensor", scale_tensor, dev)


def _cast_fp8_ptrs(ts_in: Sequence[torch.Tensor], ft: int, scale_tensor, out_ptrs, hist_ptr) -> None:
    L = capi.lib()
    with torch.cuda.device(ts_in[0].device):
        rc = L.dgb_float_cast_fp8(_FP8_INPUT_TYPES[ts_in[0].dtype], ft, len(ts_in),
                                  capi.ptr_array([t.data_ptr() for t in ts_in]),
                                  capi.u32_array([t.numel() for t in ts_in]),
                                  None if scale_tensor is None else scale_tensor.data_ptr(), out_ptrs, hist_ptr,
                                  _stream())
    capi.check(rc, "cast_fp8")


def cast_fp8(ts_in: Sequence[torch.Tensor], dtype: torch.dtype,
             scale_tensor: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """The scaled fp8 cast (dgb_float_cast_fp8) of contiguous float32 or bfloat16 CUDA tensors of one dtype on one
    device: returns one tensor of `dtype` (torch.float8_e4m3fn or torch.float8_e5m2) per input, shaped like it,
    holding (t.float() * s).clamp(-M, M).to(dtype) byte for byte, with s = scale_tensor (a one-element float32 CUDA
    tensor read by the kernel, never by the host; None means 1) and M the dtype's largest finite value (448 or 57344).
    A NaN product gives the byte 0x7F.  One pass over each input.  Misuse raises ValueError before any device work."""
    _check_fp8_inputs("cast_fp8", ts_in, dtype, scale_tensor)
    outs = [torch.empty(t.shape, dtype=dtype, device=t.device) for t in ts_in]
    _cast_fp8_ptrs(ts_in, FP8_TYPES[dtype], scale_tensor, capi.ptr_array([o.data_ptr() for o in outs]), None)
    return outs


def _compress_fp8(ts_in, dtype, checksum, temp_mem, out_compressed, out_compressed_bytes, prob_bits, scale_tensor):
    """compress_data(True, ts_in, archive_dtype=<fp8>): the cast with its histogram into a 16 B-aligned temporary,
    then the byte encoder given that histogram."""
    n = len(ts_in)
    dev = ts_in[0].device
    mx, _ = _max_numel_and_bytes(ts_in)
    L = capi.lib()
    cols = _bound(L.dgb_ans_max_compressed_size(mx), mx)
    comp, sizes = _validate_out(out_compressed, out_compressed_bytes, n, cols, dev)
    row = comp.size(1)
    offs, o = [], 0
    for t in ts_in:
        offs.append(o)
        o += (t.numel() + 15) // 16 * 16
    with torch.cuda.device(dev):
        q = torch.empty(max(o, 16), dtype=torch.uint8, device=dev)
        hist = torch.empty(n * 256, dtype=torch.int32, device=dev)
        q_ptrs = capi.ptr_array([q.data_ptr() + k for k in offs])
        _cast_fp8_ptrs(ts_in, FP8_TYPES[dtype], scale_tensor, q_ptrs, hist.data_ptr())
        tmp = _Temp(temp_mem, L.dgb_ans_encode_temp_bytes(n, mx), dev)
        rc = L.dgb_ans_encode_pointer(tmp.ptr, tmp.bytes, prob_bits, int(checksum), n, q_ptrs,
                                      capi.u32_array([t.numel() for t in ts_in]), hist.data_ptr(),
                                      capi.ptr_array([comp.data_ptr() + i * row for i in range(n)]), sizes.data_ptr(),
                                      _stream())
    capi.check(rc, "compress_data")
    return comp, sizes, tmp.need


def _narrow_type(compress_as_float: bool, ts_in: Sequence[torch.Tensor], sparse: bool,
                 archive_dtype: Optional[torch.dtype]) -> Optional[int]:
    """The archive float type of a narrowing compress, or None for an ordinary one (archive_dtype None or the
    inputs' dtype).  Decided from dtypes alone, before any tensor is touched."""
    if archive_dtype is None or (len(ts_in) > 0 and archive_dtype == ts_in[0].dtype):
        return None
    if not compress_as_float or sparse or len(ts_in) == 0 or ts_in[0].dtype != torch.float32 \
            or archive_dtype not in _NARROW_TYPES:
        raise ValueError("compress_data: archive_dtype narrows float32 inputs to float16 or bfloat16 archives "
                         "(compress_as_float=True, sparse=False); got "
                         f"{ts_in[0].dtype if len(ts_in) else None} inputs, archive_dtype={archive_dtype}, "
                         f"compress_as_float={compress_as_float}, sparse={sparse}")
    return _NARROW_TYPES[archive_dtype]


def compress_data(compress_as_float: bool, ts_in: Sequence[torch.Tensor], checksum: bool = False,
                  temp_mem: Optional[torch.Tensor] = None, out_compressed: Optional[torch.Tensor] = None,
                  out_compressed_bytes: Optional[torch.Tensor] = None, *,
                  prob_bits: int = K_DEFAULT_PRECISION, sparse: bool = False,
                  archive_dtype: Optional[torch.dtype] = None,
                  error_feedback: Optional[Sequence[torch.Tensor]] = None,
                  scale_tensor: Optional[torch.Tensor] = None):
    """archive_dtype (float16 / bfloat16, with float32 inputs): narrowing compress (dgb_float_compress_to).
    Every member's archive is exactly the archive of t.to(archive_dtype) (torch's CUDA cast), with rows sized by
    that type's bound, and no 16-bit temporary is made.  None, or the inputs' dtype, is the ordinary call; any
    other combination raises ValueError.

    error_feedback=[e_0, ...] (narrowing compress only; dgb_float_compress_to_ef): one contiguous float32 CUDA
    tensor per input, with its numel, on its device and at its address modulo 16, holding the rounding error the
    previous call left.  Member i is compressed as y = ts_in[i] + e_i (torch's add), so its archive is exactly the
    archive of y.to(archive_dtype), and e_i is overwritten in place with
    torch.where(w.isfinite(), y - w.float(), 0) for w = y.to(archive_dtype), bit for bit, in the same kernels.
    Error buffers must not overlap the inputs or each other.  Any misuse raises ValueError before any device work.

    archive_dtype=torch.float8_e4m3fn / torch.float8_e5m2 (float32 or bfloat16 inputs, compress_as_float=True,
    sparse=False, no error_feedback): fp8 compress.  Member i's archive is the byte archive (compress_data(False, ...))
    of cast_fp8([ts_in[i]], archive_dtype, scale_tensor)[0] viewed as uint8, rows sized by
    max_any_compressed_output_size: the cast writes the fp8 bytes and their histogram into a temporary in one pass,
    and the byte encoder, given that histogram, skips its own statistics pass.  Decode with
    decompress_data(False, [archive], [out.view(torch.uint8)]) or sum with decompress_data_reduce(archive_dtype=).
    scale_tensor (fp8 compress only): the cast's scale, a one-element float32 CUDA tensor (None means 1)."""
    if archive_dtype in FP8_TYPES:
        if not compress_as_float or sparse or error_feedback is not None:
            raise ValueError("compress_data: an fp8 archive_dtype needs compress_as_float=True, sparse=False and no "
                             f"error_feedback; got compress_as_float={compress_as_float}, sparse={sparse}, "
                             f"error_feedback={'set' if error_feedback is not None else None}")
        _check_fp8_inputs("compress_data", ts_in, archive_dtype, scale_tensor)
        return _compress_fp8(ts_in, archive_dtype, checksum, temp_mem, out_compressed, out_compressed_bytes, prob_bits,
                             scale_tensor)
    if scale_tensor is not None:
        raise ValueError("compress_data: scale_tensor is the scale of an fp8 compress (archive_dtype "
                         f"torch.float8_e4m3fn or torch.float8_e5m2), not of archive_dtype={archive_dtype}")
    narrow = _narrow_type(compress_as_float, ts_in, sparse, archive_dtype)
    if error_feedback is not None and narrow is None:
        raise ValueError("compress_data: error_feedback needs a narrowing compress (float32 inputs, archive_dtype "
                         "float16 or bfloat16, compress_as_float=True, sparse=False); got "
                         f"{ts_in[0].dtype if len(ts_in) else None} inputs, archive_dtype={archive_dtype}, "
                         f"compress_as_float={compress_as_float}, sparse={sparse}")
    if narrow is not None:
        return _compress_narrow(ts_in, narrow, checksum, temp_mem, out_compressed, out_compressed_bytes, prob_bits,
                                error_feedback)
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_in) > 0, "empty batch")
    dev = ts_in[0].device
    for t in ts_in:
        _check(t.is_cuda and t.is_contiguous() and t.device == dev)
        if compress_as_float:
            _check(t.dtype == ts_in[0].dtype)
            _float_type(t, sparse)
    n = len(ts_in)
    _, cols = (max_float_compressed_output_size(ts_in, sparse=sparse) if compress_as_float
               else max_any_compressed_output_size(ts_in))
    comp, sizes = _validate_out(out_compressed, out_compressed_bytes, n, cols, dev)
    row = comp.size(1)
    in_ptrs = capi.ptr_array([t.data_ptr() for t in ts_in])
    out_ptrs = capi.ptr_array([comp.data_ptr() + i * row for i in range(n)])
    L = capi.lib()
    with torch.cuda.device(dev):
        if compress_as_float:
            ft = _float_type(ts_in[0], sparse)
            in_sizes = capi.u32_array([t.numel() for t in ts_in])
            need = L.dgb_float_compress_temp_bytes(ft, n, max(t.numel() for t in ts_in))
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_float_compress_pointer(tmp.ptr, tmp.bytes, ft, prob_bits, int(checksum), n,
                                              in_ptrs, in_sizes, out_ptrs, sizes.data_ptr(), _stream())
        else:
            in_sizes = capi.u32_array([t.numel() * t.element_size() for t in ts_in])
            need = L.dgb_ans_encode_temp_bytes(n, max(t.numel() * t.element_size() for t in ts_in))
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_ans_encode_pointer(tmp.ptr, tmp.bytes, prob_bits, int(checksum), n, in_ptrs,
                                          in_sizes, None, out_ptrs, sizes.data_ptr(), _stream())
    capi.check(rc, "compress_data")
    return comp, sizes, tmp.need


def _byte_range(t: torch.Tensor) -> Tuple[int, int]:
    return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()


def _check_error_feedback(ts_in: Sequence[torch.Tensor], errs, others: Sequence[Optional[torch.Tensor]]) -> None:
    """error_feedback of a narrowing compress: one float32 residual buffer per input, laid out like it (numel,
    device, contiguity, address modulo 16), overlapping no input, no other residual buffer and none of `others`
    (the caller's output and scratch).  Reads metadata only."""
    if isinstance(errs, torch.Tensor) or not isinstance(errs, (list, tuple)) or len(errs) != len(ts_in):
        raise ValueError(f"compress_data: error_feedback is a list of {len(ts_in)} tensors, one per input")
    for i, (t, e) in enumerate(zip(ts_in, errs)):
        if getattr(e, "dtype", None) != torch.float32 or not getattr(e, "is_cuda", False) or e.device != t.device:
            raise ValueError(f"compress_data: error_feedback[{i}] must be a float32 CUDA tensor on {t.device}; got "
                             f"{getattr(e, 'dtype', type(e))} on {getattr(e, 'device', None)}")
        if e.numel() != t.numel() or not e.is_contiguous():
            raise ValueError(f"compress_data: error_feedback[{i}] must be contiguous with {t.numel()} elements; got "
                             f"{e.numel()} elements, contiguous={e.is_contiguous()}")
        if e.numel() and e.data_ptr() % 16 != t.data_ptr() % 16:
            raise ValueError(f"compress_data: error_feedback[{i}] starts at {e.data_ptr() % 16} B modulo 16, its input "
                             f"at {t.data_ptr() % 16} B: the two must match")
    # sweep in address order: a residual buffer may touch nothing else, inputs may overlap each other
    spans = sorted([(*_byte_range(e), True) for e in errs if e.numel()]
                   + [(*_byte_range(t), False) for t in list(ts_in) + [o for o in others if o is not None]
                      if t.numel()])
    end_any = end_err = 0
    for lo, hi, is_err in spans:
        if lo < (end_any if is_err else end_err):
            raise ValueError("compress_data: an error_feedback buffer overlaps an input, the output, the scratch or "
                             "another error_feedback buffer")
        end_any = max(end_any, hi)
        if is_err:
            end_err = max(end_err, hi)


def _compress_narrow(ts_in, ft: int, checksum, temp_mem, out_compressed, out_compressed_bytes, prob_bits,
                     error_feedback=None):
    dev = ts_in[0].device
    for t in ts_in:
        _check(t.is_cuda and t.is_contiguous() and t.device == dev and t.dtype == torch.float32)
    if error_feedback is not None:
        _check_error_feedback(ts_in, error_feedback, (out_compressed, temp_mem))
    n = len(ts_in)
    mx, _ = _max_numel_and_bytes(ts_in)
    L = capi.lib()
    cols = _bound(L.dgb_float_max_compressed_size(ft, mx), mx)
    comp, sizes = _validate_out(out_compressed, out_compressed_bytes, n, cols, dev)
    row = comp.size(1)
    with torch.cuda.device(dev):
        need = L.dgb_float_compress_temp_bytes(ft, n, mx)
        tmp = _Temp(temp_mem, need, dev)
        args = (capi.ptr_array([t.data_ptr() for t in ts_in]), capi.u32_array([t.numel() for t in ts_in]))
        if error_feedback is not None:
            args += (capi.ptr_array([e.data_ptr() for e in error_feedback]),)
        args += (capi.ptr_array([comp.data_ptr() + i * row for i in range(n)]), sizes.data_ptr(), _stream())
        f = L.dgb_float_compress_to if error_feedback is None else L.dgb_float_compress_to_ef
        rc = f(tmp.ptr, tmp.bytes, capi.FLOAT32, ft, prob_bits, int(checksum), n, *args)
    capi.check(rc, "compress_data")
    return comp, sizes, tmp.need


def _matrix_to_tensors(n: int, matrix: torch.Tensor, sizes: torch.Tensor) -> List[torch.Tensor]:
    host = sizes[:n].cpu().tolist()  # syncs, like compressedMatrixToTensors (DietGpu.cpp:75-103)
    flat = matrix.view(-1)
    cols = matrix.size(1)
    return [flat.narrow(0, i * cols, host[i]) for i in range(n)]


def compress_data_split_size(compress_as_float: bool, t_in: torch.Tensor, t_in_split_sizes: torch.Tensor,
                             checksum: bool = False, temp_mem: Optional[torch.Tensor] = None,
                             out_compressed: Optional[torch.Tensor] = None,
                             out_compressed_bytes: Optional[torch.Tensor] = None, *,
                             prob_bits: int = K_DEFAULT_PRECISION, sparse: bool = False):
    _check_sparse(compress_as_float, sparse)
    dev = t_in.device
    _check(t_in.is_cuda and t_in.is_contiguous())
    ft = _float_type(t_in, sparse) if compress_as_float else 0
    if not compress_as_float:
        _check(t_in.data_ptr() % 4 == 0, "start pointer is not aligned")
    _check(t_in_split_sizes.is_contiguous() and t_in_split_sizes.device.type == "cpu"
           and t_in_split_sizes.dtype == torch.int32)
    splits = t_in_split_sizes.tolist()
    n = len(splits)
    for i, s in enumerate(splits):
        _check(s > 0)
        if not compress_as_float and i != n - 1:
            _check(s % 4 == 0, "the size of an interior split is not a multiple of 4 bytes")
    # splits count words of t_in's dtype for floats, bytes otherwise
    _split_total(splits, t_in.numel() if compress_as_float else t_in.numel() * t_in.element_size(), "t_in")
    mx = max(splits)
    L = capi.lib()
    cols = _bound(L.dgb_float_max_compressed_size(ft, mx) if compress_as_float else L.dgb_ans_max_compressed_size(mx), mx)
    comp, sizes = _validate_out(out_compressed, out_compressed_bytes, n, cols, dev)
    arr = capi.u32_array(splits)
    with torch.cuda.device(dev):
        if compress_as_float:
            need = L.dgb_float_compress_temp_bytes(ft, n, mx)
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_float_compress_split_size(tmp.ptr, tmp.bytes, ft, prob_bits, int(checksum), n,
                                                 t_in.data_ptr(), arr, comp.data_ptr(), comp.size(1),
                                                 sizes.data_ptr(), _stream())
        else:
            need = L.dgb_ans_encode_temp_bytes(n, mx)
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_ans_encode_split_size(tmp.ptr, tmp.bytes, prob_bits, int(checksum), n,
                                             t_in.data_ptr(), arr, None, comp.data_ptr(), comp.size(1),
                                             sizes.data_ptr(), _stream())
    capi.check(rc, "compress_data_split_size")
    return _matrix_to_tensors(n, comp, sizes), sizes, tmp.need


def compress_data_simple(compress_as_float: bool, ts_in: Sequence[torch.Tensor], checksum: bool = False,
                         temp_mem: Optional[int] = 64 * 1024 * 1024, *, sparse: bool = False) -> List[torch.Tensor]:
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_in) > 0)
    scratch = None
    if temp_mem and temp_mem > 0:
        scratch = torch.empty(temp_mem, dtype=torch.uint8, device=ts_in[0].device)
    comp, sizes, _ = compress_data(compress_as_float, ts_in, checksum, scratch, None, None, sparse=sparse)
    host = sizes.cpu().tolist()
    return [comp[i, :host[i]].clone() for i in range(len(ts_in))]


def pull_archives(compress_as_float: bool, ts_src: Sequence[torch.Tensor], ts_dst: Sequence[torch.Tensor],
                  float_dtype: Optional[torch.dtype] = None, out_bytes: Optional[torch.Tensor] = None, *,
                  sparse: bool = False) -> None:
    """Copies each archive of ts_src (uint8 rows, e.g. views of a peer GPU's memory) into the matching row of
    ts_dst, exactly as long as its header says (dgb_archives_pull): the transfer step of the compressed
    collectives.  `float_dtype` names the float kind of the archives when compress_as_float (`sparse`: archives
    made with sparse=True)."""
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_src) > 0 and len(ts_src) == len(ts_dst))
    dev = ts_dst[0].device
    for a, b in zip(ts_src, ts_dst):
        _check(a.is_cuda and b.is_cuda and b.device == dev and a.dtype == torch.uint8 and b.dtype == torch.uint8)
        _check(a.is_contiguous() and b.is_contiguous())
    ft = _float_type(torch.empty(0, dtype=float_dtype), sparse) if compress_as_float else 0
    if out_bytes is not None:
        _check(out_bytes.is_cuda and out_bytes.dtype == torch.int32 and out_bytes.numel() >= len(ts_src))
    with torch.cuda.device(dev):
        rc = capi.lib().dgb_archives_pull(ft, len(ts_src), capi.ptr_array([t.data_ptr() for t in ts_src]),
                                          capi.ptr_array([t.data_ptr() for t in ts_dst]),
                                          capi.u32_array([t.numel() for t in ts_dst]),
                                          out_bytes.data_ptr() if out_bytes is not None else None, _stream())
    capi.check(rc, "pull_archives")


# ----------------------------------------------------------- decompress ----

def _validate_status(out_status, out_sizes, n, dev):
    if out_status is not None:
        _check(out_status.is_contiguous() and out_status.is_cuda and out_status.dtype == torch.uint8
               and out_status.numel() == n and out_status.device == dev)
    if out_sizes is not None:
        _check(out_sizes.is_contiguous() and out_sizes.is_cuda and out_sizes.dtype == torch.int32
               and out_sizes.numel() == n and out_sizes.device == dev)
    return (out_status.data_ptr() if out_status is not None else None,
            out_sizes.data_ptr() if out_sizes is not None else None)


def _raise_checksum(rc: int, what: str, as_float: bool):
    if rc == capi.ERR_CHECKSUM:
        raise RuntimeError(("floatDecompress" if as_float else "ANSDecode")
                           + ": checksum mismatch seen on decoded data; archive cannot be unpacked")
    capi.check(rc, what)


def decompress_data(compress_as_float: bool, ts_in: Sequence[torch.Tensor], ts_out: Sequence[torch.Tensor],
                    checksum: bool = False, temp_mem: Optional[torch.Tensor] = None,
                    out_status: Optional[torch.Tensor] = None,
                    out_decompressed_words: Optional[torch.Tensor] = None, *,
                    prob_bits: int = K_DEFAULT_PRECISION, sparse: bool = False) -> int:
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_in) > 0 and len(ts_in) == len(ts_out))
    dev = ts_in[0].device
    n = len(ts_in)
    caps = []
    for ti, to in zip(ts_in, ts_out):
        _check(ti.is_cuda and ti.device == dev and ti.is_contiguous() and ti.dtype == torch.uint8)
        _check_archive_aligned(ti)
        _check(to.is_cuda and to.device == dev and to.is_contiguous())
        if compress_as_float:
            _float_type(to, sparse)
            # capacities are counted in words of one float type
            _check(to.dtype == ts_out[0].dtype, "float outputs must all have the same dtype")
        cap = to.numel() if compress_as_float else to.numel() * to.element_size()
        _check(cap <= 0xFFFFFFFF)
        caps.append(cap)
    st_ptr, sz_ptr = _validate_status(out_status, out_decompressed_words, n, dev)
    L = capi.lib()
    in_ptrs = capi.ptr_array([t.data_ptr() for t in ts_in])
    out_ptrs = capi.ptr_array([t.data_ptr() for t in ts_out])
    cap_arr = capi.u32_array(caps)
    with torch.cuda.device(dev):
        if compress_as_float:
            ft = _float_type(ts_out[0], sparse)
            need = L.dgb_float_decompress_temp_bytes(ft, n, max(caps))
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_float_decompress_pointer(tmp.ptr, tmp.bytes, ft, prob_bits, int(checksum), n, in_ptrs,
                                                out_ptrs, cap_arr, st_ptr, sz_ptr, None, _stream())
        else:
            need = L.dgb_ans_decode_temp_bytes(n)
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_ans_decode_pointer(tmp.ptr, tmp.bytes, prob_bits, int(checksum), n, in_ptrs, out_ptrs,
                                          cap_arr, st_ptr, sz_ptr, None, _stream())
    _raise_checksum(rc, "decompress_data", compress_as_float)
    return tmp.need


_REDUCE_TYPES = {torch.float16: capi.FLOAT16, torch.bfloat16: capi.BFLOAT16, torch.float32: capi.FLOAT32}


def _scale32(scale) -> Optional[np.float32]:
    """None, or a host real number rounded once to float32 (the scale of the scaled decode-and-sum)."""
    if scale is None:
        return None
    if isinstance(scale, bool) or not isinstance(scale, numbers.Real):
        raise TypeError(f"scale is None or a real number (a host value, rounded to float32), not {type(scale).__name__}")
    return np.float32(scale)


def _check_flag_tensor(what: str, t, dev) -> None:
    """A one-element contiguous float32 CUDA tensor on dev (a device-resident scale, or a non-finite flag)."""
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{what} is a one-element float32 CUDA tensor, not {type(t).__name__}")
    if t.dtype != torch.float32 or t.numel() != 1 or not t.is_contiguous():
        raise ValueError(f"{what} is a one-element contiguous float32 tensor, not {t.dtype} with {t.numel()} "
                         f"element(s){'' if t.is_contiguous() else ', non-contiguous'}")
    if not t.is_cuda or t.device != dev:
        raise ValueError(f"{what} must be on the outputs' device {dev}, not {t.device}")


def _check_dev_scale(scale32, scale_tensor, found_inf, dev) -> None:
    """The device-scale keywords of decompress_data_reduce: scale_tensor replaces scale, found_inf needs it."""
    if scale_tensor is not None and scale32 is not None:
        raise ValueError("decompress_data_reduce: pass scale or scale_tensor, not both")
    if found_inf is not None and scale_tensor is None:
        raise ValueError("decompress_data_reduce: found_inf needs scale_tensor (torch.ones(1) for the unscaled sum)")
    if scale_tensor is not None:
        _check_flag_tensor("scale_tensor", scale_tensor, dev)
    if found_inf is not None:
        _check_flag_tensor("found_inf", found_inf, dev)


def _check_sq_norm(what: str, t, groups: int, dev) -> None:
    """A contiguous float64 CUDA tensor of `groups` elements on dev (the squared norms of a call)."""
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{what} is a float64 CUDA tensor, not {type(t).__name__}")
    if t.dtype != torch.float64 or t.numel() != groups or not t.is_contiguous():
        raise ValueError(f"{what} is a contiguous float64 tensor of {groups} element(s), not {t.dtype} with "
                         f"{t.numel()} element(s){'' if t.is_contiguous() else ', non-contiguous'}")
    if not t.is_cuda or t.device != dev:
        raise ValueError(f"{what} must be on the device {dev}, not {t.device}")


def decompress_data_reduce(ts_in: Sequence[Sequence[torch.Tensor]], ts_out: Sequence[torch.Tensor],
                           accumulate: bool = False, temp_mem: Optional[torch.Tensor] = None,
                           out_status: Optional[torch.Tensor] = None, *,
                           prob_bits: int = K_DEFAULT_PRECISION,
                           archive_dtype: Optional[torch.dtype] = None, sparse: bool = False,
                           scale: Optional[float] = None, scale_tensor: Optional[torch.Tensor] = None,
                           found_inf: Optional[torch.Tensor] = None, reduce_dtype: Optional[torch.dtype] = None,
                           acc: Optional[Sequence[torch.Tensor]] = None,
                           sq_norm: Optional[torch.Tensor] = None) -> int:
    """Decode-and-sum (dgb_float_decompress_reduce_to): ts_in is G lists of W uint8 float archives each, ts_out G
    contiguous CUDA tensors of one dtype (float16, bfloat16 or float32).  ts_out[g] becomes
    (ts_out[g] if accumulate else x(g, 0)) + x(g, 1) + ... + x(g, W - 1), added left to right with torch's adds in
    that dtype, where x(g, j) is archive ts_in[g][j] decoded; each archive must hold exactly ts_out[g].numel()
    words.  A group with an invalid archive is left untouched; out_status (CUDA uint8, G * W entries, group-major)
    receives 1 / 0 per archive.  Returns the scratch bytes used.

    archive_dtype: the archives' dtype; None (or the outputs' dtype) means the outputs' dtype.  float16 or
    bfloat16 archives with float32 outputs are summed in float32: the result is
    torch's fold acc = x(g, 0).float(); acc = acc + x(g, 1).float(); ... bit for bit.  Any other pair raises
    ValueError.

    sparse=True: the archives were made with compress_data(..., sparse=True) from archive_dtype tensors
    (dgb_float_decompress_reduce_sparse).  The same dtype pairs are allowed, and the result is bit-identical to this
    call on dense archives of the same words; a dense archive in such a group is invalid.

    scale (dgb_float_decompress_reduce_scaled): a real number s, rounded once to float32 (np.float32(s)).  Every
    decoded word x is multiplied by s before it is added: its term is (x.float() * s32).to(out dtype) with s32 =
    torch.tensor(s, dtype=torch.float32), so a 16-bit same-type sum rounds each product to the 16-bit type first,
    while float32 and widening sums keep it in float32.  The result is torch's fold acc = term(x(g, 0)) (or
    ts_out[g] unscaled when accumulating); acc = acc + term(x(g, 1)); ... bit for bit, with archive_dtype and sparse
    too (an elided zero is scaled like any other word, so s < 0 turns +0 into -0).  scale=1.0 gives the unscaled
    result; None (the default) calls the unscaled entries.  A scale is a host value: a tensor raises TypeError.

    scale_tensor (dgb_float_decompress_reduce_scaled_dev): the scale as a one-element float32 CUDA tensor on the
    outputs' device, e.g. a GradScaler's inverse scale or 1 / the token count of an all-reduce.  The kernels read it
    when they run, so the host never reads it (no synchronisation) and a CUDA graph replays with its current value.
    The result is bit for bit this call with scale=float(scale_tensor).  Not with scale.
    found_inf (with scale_tensor only): a one-element float32 CUDA tensor on the same device, set to 1.0 when any
    element this call writes ends up inf or NaN, and never cleared (torch.amp's found_inf); with
    scale_tensor=torch.ones(1) it flags the unscaled sum.  Elements of a group left untouched never count.
    These keywords raise ValueError before any archive is read.

    reduce_dtype=torch.float32 with float16 / bfloat16 outputs of archive_dtype (dense, or sparse=True)
    (dgb_float_decompress_reduce_narrow): the sum is taken in float32 and rounded once to the outputs' dtype, so
    ts_out[g] becomes S.to(dtype) with S = (acc[g] if accumulate else term(x(g, 0))) + term(x(g, 1)) + ... in
    float32, term being the widening sum's term (x.float(), or (x.float() * s32) with scale / scale_tensor): bit for
    bit the widening call into float32 outputs followed by torch's .to(dtype).  found_inf sees the rounded 16-bit
    results, so a float32 sum that rounds to an fp16 infinity counts.  acc: G contiguous float32 CUDA tensors on the
    outputs' device with ts_out[g].numel() elements each, holding the running sums accumulate starts from and taking
    the intermediate sums of the call (their contents afterwards are unspecified); ts_out[g] is only written.  acc
    is required with accumulate=True; otherwise None takes a stream-ordered temporary when W > 1.  reduce_dtype
    None or the outputs' dtype is the call described above; any other reduce_dtype, an acc without this path, or an
    acc of the wrong dtype, size or device raises ValueError before any archive is read.

    sq_norm (with scale_tensor only; dgb_float_decompress_reduce_scaled_dev_norm / _narrow_norm): a contiguous float64
    CUDA tensor of G elements on the outputs' device.  sq_norm[g] is overwritten with the squared norm of the
    elements the call stores to ts_out[g] (after scaling, and after the 16-bit rounding with reduce_dtype), taken in
    fp64 in the fixed order of include/dietgpu_b200.h, so it is bit-reproducible and equals sq_norm() of the
    outputs.  A group with an invalid archive leaves sq_norm[g] untouched.  Works with archive_dtype, sparse,
    reduce_dtype=torch.float32 / acc and found_inf; outputs and found_inf are bit-identical to the call without it.
    Without scale_tensor, with scale, or of the wrong dtype, size or device it raises ValueError before any archive
    is read.

    archive_dtype=torch.float8_e4m3fn / torch.float8_e5m2: fp8 archives (compress_data(archive_dtype=) or the byte
    archives of fp8 words) summed into float32 outputs with the device scale d = scale_tensor, which is required: the
    result is torch's fold acc = q(g, 0).float() * d (or ts_out[g] when accumulating); acc = acc + q(g, 1).float() * d;
    ... bit for bit, with found_inf and sq_norm as above.  Float32 outputs only; scale, sparse, acc and a reduce_dtype
    other than None or float32 raise ValueError before any archive is read."""
    scale32 = _scale32(scale)
    _check_dev_scale(scale32, scale_tensor, found_inf, ts_out[0].device if len(ts_out) else None)
    if sq_norm is not None:
        if scale_tensor is None:
            raise ValueError("decompress_data_reduce: sq_norm needs scale_tensor (torch.ones(1) for the unscaled sum)")
        _check_sq_norm("decompress_data_reduce: sq_norm", sq_norm, len(ts_out), ts_out[0].device if len(ts_out) else None)
    if archive_dtype in FP8_TYPES:
        return _reduce_fp8(ts_in, ts_out, accumulate, temp_mem, out_status, prob_bits, archive_dtype, sparse,
                           scale32, scale_tensor, found_inf, reduce_dtype, acc, sq_norm)
    _check(len(ts_in) > 0 and len(ts_in) == len(ts_out), "one output per group")
    width = len(ts_in[0])
    _check(width > 0, "a group needs at least one archive")
    dtype = ts_out[0].dtype
    if dtype not in _REDUCE_TYPES:
        raise ValueError(f"decompress_data_reduce sums float16, bfloat16 or float32 outputs, not {dtype}")
    if archive_dtype is None:
        archive_dtype = dtype
    if archive_dtype != dtype and not (dtype == torch.float32 and archive_dtype in (torch.float16, torch.bfloat16)):
        raise ValueError(f"decompress_data_reduce sums {archive_dtype} archives into {archive_dtype} outputs, or "
                         f"float16 / bfloat16 archives into float32 outputs; not into {dtype}")
    narrow = reduce_dtype is not None and reduce_dtype != dtype
    if narrow and not (reduce_dtype == torch.float32 and dtype in (torch.float16, torch.bfloat16)
                       and archive_dtype == dtype):
        raise ValueError(f"decompress_data_reduce: reduce_dtype is None, the outputs' dtype, or float32 for float16 / "
                         f"bfloat16 outputs of the archives' dtype; not {reduce_dtype} for {archive_dtype} archives "
                         f"into {dtype} outputs")
    dev = ts_out[0].device
    if acc is not None:
        if not narrow:
            raise ValueError("decompress_data_reduce: acc needs reduce_dtype=torch.float32 with float16 / bfloat16 "
                             "outputs")
        if len(acc) != len(ts_out):
            raise ValueError(f"decompress_data_reduce: acc needs one tensor per group ({len(ts_out)}), not {len(acc)}")
        for a, to in zip(acc, ts_out):
            if not isinstance(a, torch.Tensor) or a.dtype != torch.float32 or not a.is_contiguous():
                raise ValueError("decompress_data_reduce: acc holds contiguous float32 tensors")
            if not a.is_cuda or a.device != dev:
                raise ValueError(f"decompress_data_reduce: acc must be on the outputs' device {dev}, not {a.device}")
            if a.numel() != to.numel():
                raise ValueError(f"decompress_data_reduce: acc[g] needs ts_out[g].numel() = {to.numel()} elements, "
                                 f"not {a.numel()}")
    elif narrow and accumulate:
        raise ValueError("decompress_data_reduce: accumulate=True with reduce_dtype=torch.float32 needs acc (the "
                         "float32 running sums)")
    ins = []
    for group, to in zip(ts_in, ts_out):
        _check(len(group) == width, "every group needs the same number of archives")
        _check(to.is_cuda and to.device == dev and to.is_contiguous() and to.dtype == dtype,
               "outputs must be contiguous CUDA tensors of one dtype on one device")
        _check(to.numel() <= 0xFFFFFFFF)
        for ti in group:
            _check(ti.is_cuda and ti.device == dev and ti.is_contiguous() and ti.dtype == torch.uint8)
            _check_archive_aligned(ti)
            ins.append(ti)
    g, n = len(ts_out), len(ins)
    st_ptr, _ = _validate_status(out_status, None, n, dev)
    ft, out_ft = (_SPARSE_TYPES if sparse else _REDUCE_TYPES)[archive_dtype], _REDUCE_TYPES[dtype]
    L = capi.lib()
    if narrow:
        if acc is None and width > 1:
            flat = torch.empty(sum(t.numel() for t in ts_out), dtype=torch.float32, device=dev)
            acc, o = [], 0
            for to in ts_out:
                acc.append(flat[o:o + to.numel()])
                o += to.numel()
        s = None if scale32 is None else C.c_float(float(scale32))
        if sq_norm is not None:
            sizes = capi.u32_array([t.numel() for t in ts_out])
            with torch.cuda.device(dev):
                need = L.dgb_float_decompress_reduce_norm_temp_bytes(ft, g, width, sizes)
                tmp = _Temp(temp_mem, need, dev)
                rc = L.dgb_float_decompress_reduce_narrow_norm(
                    tmp.ptr, tmp.bytes, ft, prob_bits, g, width, capi.ptr_array([t.data_ptr() for t in ins]),
                    None if acc is None else capi.ptr_array([a.data_ptr() for a in acc]),
                    capi.ptr_array([t.data_ptr() for t in ts_out]), sizes, int(bool(accumulate)),
                    scale_tensor.data_ptr(), None if found_inf is None else found_inf.data_ptr(), sq_norm.data_ptr(),
                    st_ptr, _stream())
            capi.check(rc, "decompress_data_reduce")
            return tmp.need
        with torch.cuda.device(dev):
            need = L.dgb_float_decompress_temp_bytes(ft, n, 0)
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_float_decompress_reduce_narrow(
                tmp.ptr, tmp.bytes, ft, prob_bits, g, width, capi.ptr_array([t.data_ptr() for t in ins]),
                None if acc is None else capi.ptr_array([a.data_ptr() for a in acc]),
                capi.ptr_array([t.data_ptr() for t in ts_out]), capi.u32_array([t.numel() for t in ts_out]),
                int(bool(accumulate)), None if s is None else C.addressof(s),
                None if scale_tensor is None else scale_tensor.data_ptr(),
                None if found_inf is None else found_inf.data_ptr(), st_ptr, _stream())
        capi.check(rc, "decompress_data_reduce")
        return tmp.need
    entry = L.dgb_float_decompress_reduce_sparse if sparse else L.dgb_float_decompress_reduce_to
    extra = ()
    if scale32 is not None:
        entry, extra = L.dgb_float_decompress_reduce_scaled, (float(scale32),)
    elif scale_tensor is not None:
        entry = L.dgb_float_decompress_reduce_scaled_dev
        extra = (scale_tensor.data_ptr(), found_inf.data_ptr() if found_inf is not None else None)
        if sq_norm is not None:
            entry, extra = L.dgb_float_decompress_reduce_scaled_dev_norm, extra + (sq_norm.data_ptr(),)
    with torch.cuda.device(dev):
        if sq_norm is not None:
            need = L.dgb_float_decompress_reduce_norm_temp_bytes(ft, g, width,
                                                                 capi.u32_array([t.numel() for t in ts_out]))
        else:
            need = L.dgb_float_decompress_temp_bytes(ft, n, 0)
        tmp = _Temp(temp_mem, need, dev)
        rc = entry(tmp.ptr, tmp.bytes, ft, out_ft, prob_bits, g, width,
                   capi.ptr_array([t.data_ptr() for t in ins]),
                   capi.ptr_array([t.data_ptr() for t in ts_out]),
                   capi.u32_array([t.numel() for t in ts_out]), int(bool(accumulate)), *extra,
                   st_ptr, _stream())
    capi.check(rc, "decompress_data_reduce")
    return tmp.need


def _reduce_fp8(ts_in, ts_out, accumulate, temp_mem, out_status, prob_bits, archive_dtype, sparse, scale32,
                scale_tensor, found_inf, reduce_dtype, acc, sq_norm_out) -> int:
    """decompress_data_reduce of fp8 archives (dgb_float_decompress_reduce_scaled_dev / _norm)."""
    if scale_tensor is None or scale32 is not None or sparse or acc is not None \
            or reduce_dtype not in (None, torch.float32):
        raise ValueError("decompress_data_reduce: fp8 archives are summed into float32 with scale_tensor (the "
                         f"dequantisation scale), without scale, sparse or acc; got scale={scale32}, sparse={sparse}, "
                         f"reduce_dtype={reduce_dtype}, acc={'set' if acc is not None else None}")
    if len(ts_out) == 0 or any(not isinstance(o, torch.Tensor) or o.dtype != torch.float32 for o in ts_out):
        raise ValueError("decompress_data_reduce: fp8 archives are summed into float32 outputs")
    _check(len(ts_in) == len(ts_out), "one output per group")
    width = len(ts_in[0])
    _check(width > 0, "a group needs at least one archive")
    dev = ts_out[0].device
    ins = []
    for group, to in zip(ts_in, ts_out):
        _check(len(group) == width, "every group needs the same number of archives")
        _check(to.is_cuda and to.device == dev and to.is_contiguous(),
               "outputs must be contiguous CUDA tensors on one device")
        _check(to.numel() <= 0xFFFFFFFF)
        for ti in group:
            _check(ti.is_cuda and ti.device == dev and ti.is_contiguous() and ti.dtype == torch.uint8)
            _check_archive_aligned(ti)
            ins.append(ti)
    g, n = len(ts_out), len(ins)
    st_ptr, _ = _validate_status(out_status, None, n, dev)
    ft = FP8_TYPES[archive_dtype]
    L = capi.lib()
    sizes = capi.u32_array([t.numel() for t in ts_out])
    with torch.cuda.device(dev):
        if sq_norm_out is not None:
            tmp = _Temp(temp_mem, L.dgb_float_decompress_reduce_norm_temp_bytes(ft, g, width, sizes), dev)
            entry, extra = L.dgb_float_decompress_reduce_scaled_dev_norm, (sq_norm_out.data_ptr(),)
        else:
            tmp = _Temp(temp_mem, L.dgb_float_decompress_temp_bytes(ft, n, 0), dev)
            entry, extra = L.dgb_float_decompress_reduce_scaled_dev, ()
        rc = entry(tmp.ptr, tmp.bytes, ft, capi.FLOAT32, prob_bits, g, width,
                   capi.ptr_array([t.data_ptr() for t in ins]), capi.ptr_array([t.data_ptr() for t in ts_out]), sizes,
                   int(bool(accumulate)), scale_tensor.data_ptr(),
                   None if found_inf is None else found_inf.data_ptr(), *extra, st_ptr, _stream())
    capi.check(rc, "decompress_data_reduce")
    return tmp.need


def sq_norm(tensors: Sequence[torch.Tensor], out: Optional[torch.Tensor] = None,
            temp_mem: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The squared norm of each of G contiguous CUDA tensors of one dtype (float16, bfloat16 or float32) on one device,
    as a float64 tensor [G] (dgb_float_sq_norm): each element widened exactly to fp64 and its square summed in the
    fixed order of include/dietgpu_b200.h, the order decompress_data_reduce(sq_norm=) uses, so the two agree bit for
    bit on the same elements.  inf or NaN elements give an inf or NaN norm; an empty tensor gives +0.  out: a
    contiguous float64 CUDA tensor of G elements on the tensors' device, overwritten and returned.  Other inputs raise
    ValueError before any device work."""
    ts = list(tensors)
    if not ts:
        if out is not None:
            _check_sq_norm("sq_norm: out", out, 0, out.device)
            return out
        return torch.empty(0, dtype=torch.float64, device="cuda")
    dtype, dev = ts[0].dtype, ts[0].device
    if dtype not in _REDUCE_TYPES:
        raise ValueError(f"sq_norm takes float16, bfloat16 or float32 tensors, not {dtype}")
    for t in ts:
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_cuda or t.device != dev \
                or not t.is_contiguous():
            raise ValueError("sq_norm takes contiguous CUDA tensors of one dtype on one device")
        if t.numel() > 0xFFFFFFFF:
            raise ValueError("sq_norm: a tensor of more than 2^32 - 1 elements")
    if out is None:
        out = torch.empty(len(ts), dtype=torch.float64, device=dev)
    else:
        _check_sq_norm("sq_norm: out", out, len(ts), dev)
    L = capi.lib()
    sizes = capi.u32_array([t.numel() for t in ts])
    with torch.cuda.device(dev):
        tmp = _Temp(temp_mem, L.dgb_float_sq_norm_temp_bytes(len(ts), sizes), dev)
        rc = L.dgb_float_sq_norm(tmp.ptr, tmp.bytes, _REDUCE_TYPES[dtype], len(ts),
                                 capi.ptr_array([t.data_ptr() for t in ts]), sizes, out.data_ptr(), _stream())
    capi.check(rc, "sq_norm")
    return out


def decompress_data_split_size(compress_as_float: bool, ts_in: Sequence[torch.Tensor], t_out: torch.Tensor,
                               t_out_split_sizes: torch.Tensor, checksum: bool = False,
                               temp_mem: Optional[torch.Tensor] = None,
                               out_status: Optional[torch.Tensor] = None,
                               out_decompressed_words: Optional[torch.Tensor] = None, *,
                               prob_bits: int = K_DEFAULT_PRECISION, sparse: bool = False) -> int:
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_in) > 0)
    dev = ts_in[0].device
    n = t_out_split_sizes.numel()
    _check(t_out_split_sizes.device.type == "cpu" and t_out_split_sizes.dtype == torch.int32
           and t_out_split_sizes.is_contiguous())
    _check(n == len(ts_in))
    splits = t_out_split_sizes.tolist()
    for ti, s in zip(ts_in, splits):
        _check(ti.is_cuda and ti.device == dev and ti.is_contiguous() and ti.dtype == torch.uint8)
        _check_archive_aligned(ti)
        _check(s > 0)
    _check(t_out.is_cuda and t_out.is_contiguous())
    _check(t_out.device == dev, "t_out is not on the device of the compressed inputs")
    ft = _float_type(t_out, sparse) if compress_as_float else 0
    _split_total(splits, t_out.numel() if compress_as_float else t_out.numel() * t_out.element_size(), "t_out")
    st_ptr, sz_ptr = _validate_status(out_status, out_decompressed_words, n, dev)
    L = capi.lib()
    in_ptrs = capi.ptr_array([t.data_ptr() for t in ts_in])
    arr = capi.u32_array(splits)
    with torch.cuda.device(dev):
        if compress_as_float:
            need = L.dgb_float_decompress_temp_bytes(ft, n, max(splits))
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_float_decompress_split_size(tmp.ptr, tmp.bytes, ft, prob_bits, int(checksum), n, in_ptrs,
                                                   t_out.data_ptr(), arr, st_ptr, sz_ptr, None, _stream())
        else:
            need = L.dgb_ans_decode_temp_bytes(n)
            tmp = _Temp(temp_mem, need, dev)
            rc = L.dgb_ans_decode_split_size(tmp.ptr, tmp.bytes, prob_bits, int(checksum), n, in_ptrs,
                                             t_out.data_ptr(), arr, st_ptr, sz_ptr, None, _stream())
    _raise_checksum(rc, "decompress_data_split_size", compress_as_float)
    return tmp.need


def decompress_data_simple(compress_as_float: bool, ts_in: Sequence[torch.Tensor], checksum: bool = False,
                           temp_mem: Optional[int] = 64 * 1024 * 1024, *, sparse: bool = False) -> List[torch.Tensor]:
    _check_sparse(compress_as_float, sparse)
    _check(len(ts_in) > 0)
    dev = ts_in[0].device
    n = len(ts_in)
    for t in ts_in:
        _check(t.is_cuda and t.device == dev)
        _check_archive_aligned(t)
    L = capi.lib()
    sizes = torch.empty(n, dtype=torch.int32, device=dev)
    types = torch.zeros(n, dtype=torch.int32, device=dev)
    tmp = _Temp(None, 8 * n + 256, dev)
    in_ptrs = capi.ptr_array([t.data_ptr() for t in ts_in])
    with torch.cuda.device(dev):
        if compress_as_float:
            rc = L.dgb_float_get_compressed_info(tmp.ptr, tmp.bytes, in_ptrs, 0, n, sizes.data_ptr(),
                                                 types.data_ptr(), None, _stream())
        else:
            rc = L.dgb_ans_get_compressed_info(tmp.ptr, tmp.bytes, in_ptrs, 0, n, sizes.data_ptr(), None,
                                               _stream())
    capi.check(rc, "get_compressed_info")
    hs, ht = sizes.cpu().tolist(), types.cpu().tolist()
    dtype_of = _SPARSE_DTYPE_OF if sparse else _DTYPE_OF
    outs = []
    for i in range(n):
        if compress_as_float:
            _check(ht[i] == ht[0] and ht[i] in dtype_of, "inconsistent / invalid float type in archives")
            outs.append(torch.empty(hs[i], dtype=dtype_of[ht[i]], device=dev))
        else:
            outs.append(torch.empty(hs[i], dtype=torch.uint8, device=dev))
    scratch = None
    if temp_mem and temp_mem >= 256:
        scratch = torch.empty(temp_mem, dtype=torch.uint8, device=dev)
    decompress_data(compress_as_float, ts_in, outs, checksum, scratch, None, None, sparse=sparse)
    return outs
