"""numpy restatement of the scaled fp8 cast (dgb_float_cast_fp8, ops.cast_fp8):

    q = cvt.rn.satfinite.fp8(fp32(x) * s)

The product is one float32 multiply rounded to nearest even.  A non-NaN product is clamped to [-M, M] and rounded to
the nearest finite fp8 value, ties to the even code, keeping its sign (so a product too small for the fp8 subnormals
becomes +0 or -0).  A NaN product gives 0x7F.  The fp8 values come from the formats' definitions (OCP FP8: E4M3 with
bias 7 and no infinities, E5M2 with bias 15), not from torch, so the tests can check torch and the kernel against it."""
import numpy as np

E4M3, E5M2 = "e4m3", "e5m2"
MAX = {E4M3: 448.0, E5M2: 57344.0}
NAN_BYTE = 0x7F


def code_values(kind):
    """float64 value of every fp8 code 0..255 (NaN for the NaN codes, +-inf for E5M2's infinities)."""
    mbits, bias = (3, 7) if kind == E4M3 else (2, 15)
    c = np.arange(256)
    sign = np.where(c & 0x80, -1.0, 1.0)
    e = (c >> mbits) & ((1 << (7 - mbits)) - 1)
    m = c & ((1 << mbits) - 1)
    v = np.where(e == 0, m / (1 << mbits) * 2.0 ** (1 - bias), (1 + m / (1 << mbits)) * 2.0 ** (e - bias))
    v = sign * v
    if kind == E4M3:
        v[(c & 0x7F) == 0x7F] = np.nan
    else:
        top = (c >> 2) & 0x1F
        v[(top == 0x1F) & (m == 0)] = sign[(top == 0x1F) & (m == 0)] * np.inf
        v[(top == 0x1F) & (m != 0)] = np.nan
    return v


def cast(x, s, kind):
    """uint8 codes of x (float32 array, or uint16 bf16 words) times the float32 scale s."""
    x = np.asarray(x)
    if x.dtype == np.uint16:
        x = (x.astype(np.uint32) << 16).view(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        p = (x.astype(np.float32) * np.float32(s)).astype(np.float32)
    vals = code_values(kind)[:0x80]
    top = int(np.nonzero(vals == MAX[kind])[0][0])  # the largest finite positive code
    pos = vals[:top + 1]  # increasing
    a = np.minimum(np.abs(p.astype(np.float64)), MAX[kind])
    nan = np.isnan(a)
    a = np.where(nan, 0.0, a)
    hi = np.minimum(np.searchsorted(pos, a, side="left"), top)
    lo = np.maximum(hi - 1, 0)
    lo = np.where(pos[hi] == a, hi, lo)
    dlo, dhi = a - pos[lo], pos[hi] - a
    pick = np.where(dlo < dhi, lo, np.where(dhi < dlo, hi, np.where(lo % 2 == 0, lo, hi)))
    code = pick.astype(np.uint8) | np.where(np.signbit(p), 0x80, 0).astype(np.uint8)
    return np.where(nan, np.uint8(NAN_BYTE), code).astype(np.uint8)


def edge_corpus(kind, s=1.0):
    """float32 inputs whose products with s sit on the cast's edges: every fp8 value and the midpoints between
    neighbours (ties) with their float32 neighbours, the subnormal boundaries, +-M and its neighbours, values beyond M,
    +-inf, NaN, +-0 and the float32 extremes.  Divided by s so that the products land there (s a power of two keeps
    them exact; another s moves them by an ulp, which the neighbours cover)."""
    v = code_values(kind)
    fin = np.unique(np.abs(v[np.isfinite(v)]))
    mids = (fin[:-1] + fin[1:]) / 2
    base = np.concatenate([fin, mids, fin[:1] / 2, fin[1:2] / 2, fin[1:2] / 4, [MAX[kind] * 1.0625, MAX[kind] * 2,
                                                                                    MAX[kind] + 8, 1e30, 3e38]])
    with np.errstate(over="ignore"):
        x = (base / np.float64(s)).astype(np.float32)
    x = np.concatenate([x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(0))])
    x = np.concatenate([x, -x, np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, 1e-45, -1e-45,
                                         np.finfo(np.float32).max, -np.finfo(np.float32).max], np.float32)])
    return x.astype(np.float32)
