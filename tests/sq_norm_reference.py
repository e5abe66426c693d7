"""numpy restatement of the squared norm of include/dietgpu_b200.h (dgb_float_sq_norm and the decode-and-sum norm
entries), step by step, so that tests can predict the kernels' fp64 value bit for bit.

values: the group's words as exact float64 values (a float16 / bfloat16 / float32 tensor's .double()).
  1. lane: word i is in block i // 4096, row (i % 4096) // 32, lane i % 32; each lane adds v * v (exact in fp64) to
     its sum from +0, rows in descending order (a partial last row first);
  2. warp: p = p + p[lane ^ o] for o = 16, 8, 4, 2, 1 gives the block's partial q[k];
  3. group: thread t of 256 sums q[t], q[t + 256], ... from +0; each warp of 32 threads applies step 2; the 8 warp
     sums are added in warp order.
Every + is one fp64 round-to-nearest-even add (numpy's float64 add)."""
import numpy as np

BLOCK, LANES, THREADS = 4096, 32, 256
_XOR = [np.arange(LANES) ^ o for o in (16, 8, 4, 2, 1)]


def butterfly(p):
    """Step 2 on the last axis (32 lanes): every lane's value after the xor butterfly."""
    p = np.asarray(p, dtype=np.float64)
    for idx in _XOR:
        p = p + p[..., idx]
    return p


def lane_sums(block):
    """Step 1: the 32 lane sums of one block of at most 4096 float64 values."""
    n = block.size
    rows, rem = divmod(n, LANES)
    s = np.zeros(LANES)
    if rem:
        tail = block[rows * LANES:]
        s[:rem] = s[:rem] + tail * tail
    full = block[:rows * LANES].reshape(rows, LANES)
    for r in range(rows - 1, -1, -1):
        s = s + full[r] * full[r]
    return s


def block_partials(values):
    """Steps 1 and 2 for every block: q[k]."""
    values = np.asarray(values, dtype=np.float64).reshape(-1)
    nb = -(-values.size // BLOCK)
    nfull = values.size // BLOCK
    q = np.zeros(nb)
    if nfull:
        x = values[:nfull * BLOCK].reshape(nfull, BLOCK // LANES, LANES)
        s = np.zeros((nfull, LANES))
        for r in range(BLOCK // LANES - 1, -1, -1):
            s = s + x[:, r] * x[:, r]
        q[:nfull] = butterfly(s)[:, 0]
    if nb > nfull:
        q[nfull] = butterfly(lane_sums(values[nfull * BLOCK:]))[0]
    return q


def fold_group(q):
    """Step 3: the group's value from its block partials."""
    q = np.asarray(q, dtype=np.float64)
    pad = (-q.size) % THREADS
    # a thread past the last block adds nothing; adding +0 to a sum of squares leaves it unchanged
    qq = np.concatenate([q, np.zeros(pad)]).reshape(-1, THREADS)
    t = np.zeros(THREADS)
    for row in qq:
        t = t + row
    w = butterfly(t.reshape(THREADS // LANES, LANES))[:, 0]
    r = w[0]
    for v in w[1:]:
        r = r + v
    return np.float64(r)


def sq_norm(values):
    """The squared norm of one group."""
    return fold_group(block_partials(values))


def fold(values):
    """((v[0] + v[1]) + v[2]) + ...: the collectives' member-order and rank-order folds."""
    values = np.asarray(values, dtype=np.float64).reshape(-1)
    r = values[0]
    for v in values[1:]:
        r = r + v
    return np.float64(r)


def same(a, b):
    """Bit equality of two fp64 values, any NaN matching any NaN."""
    a, b = np.float64(a), np.float64(b)
    return (np.isnan(a) and np.isnan(b)) or a.view(np.uint64) == b.view(np.uint64)


# ---- crafted order pins: each documented order gives a value its obvious alternatives do not ----------------------

def pin_rows(big, small):
    """One block: lane 0 holds `big` in its top row and `small` in its other rows (every other lane is 0).  Rows
    descending absorb every small square into big's; ascending rows would add them up first."""
    x = np.zeros(BLOCK)
    x[0::LANES] = small
    x[(BLOCK // LANES - 1) * LANES] = big
    return x


def pin_lanes(big, small):
    """One row: lane 0 holds `big`, lanes 1-31 `small`; the butterfly adds pair sums of growing size to big's."""
    x = np.full(LANES, small, dtype=np.float64)
    x[0] = big
    return x


def pin_blocks(big, small, blocks=600):
    """`blocks` blocks whose only non-zero word is the first: `big` in block 0, `small` in the others."""
    x = np.zeros(blocks * BLOCK)
    x[::BLOCK] = small
    x[0] = big
    return x
