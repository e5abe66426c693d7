"""The error-feedback contract of the narrowing compress (include/dietgpu_b200.h), restated in numpy:

    y = x + e (fp32, round to nearest)    w = round_T(y)    e' = y - float(w) if w is finite else +0

The CPU tests pin torch's expression to it; the GPU tests compare the kernels' words and residuals with it."""
import numpy as np
import torch


def _bf16_bits(y: np.ndarray) -> np.ndarray:
    """round to nearest even float32 -> bfloat16 (the high 16 bits), NaN kept a NaN"""
    u = y.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7fff + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(y), np.uint16(0x7fc0), r)


def _widen(w: np.ndarray, dt) -> np.ndarray:
    if dt == torch.float16:
        return w.astype(np.float32)
    return (w.astype(np.uint32) << 16).view(np.float32)


def np_step(x: np.ndarray, e: np.ndarray, dt):
    """(y, w as float32, e') of the contract for float32 arrays x and e"""
    with np.errstate(over="ignore", invalid="ignore"):
        y = (x + e).astype(np.float32)
        w = y.astype(np.float16) if dt == torch.float16 else _bf16_bits(y)
        wf = _widen(w, dt)
        res = np.where(np.isfinite(wf), (y - wf).astype(np.float32), np.float32(0.0)).astype(np.float32)
    return y, wf, res
