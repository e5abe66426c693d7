"""Writes tests/golden/sparse32_golden.npz: small sparse fp32 members (float type 8) and their archives at prob bits
9, 10 and 11 with checksums, from the CPU restatement in tests/sparse32_oracle.py.  Run from the repository root:
python tests/golden/make_sparse32_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import sparse32_oracle as S  # noqa: E402
from test_oracle_sparse32 import all_but, masked_words, relu_words  # noqa: E402


def members():
    return {
        "empty": np.zeros(0, np.uint32),
        "relu_4097": relu_words(4097, 11),
        "relu_9000": relu_words(9000, 12),
        "masked_5000": masked_words(5000, 13),
        "one_free": all_but((99,)),  # nothing elided
        "two_free": all_but((17, 200)),
        "full_range": np.random.default_rng(8).integers(0, 1 << 32, 3001, dtype=np.uint32),
        "neg_zero_only": np.concatenate([np.full(40, S.NEG0, np.uint32), relu_words(600, 14)[relu_words(600, 14) != 0]]),
    }


def main():
    out = {}
    for name, w in members().items():
        key = f"sparse32/{name}"
        out[f"{key}/in"] = w
        for pb in (9, 10, 11):
            out[f"{key}/pb{pb}"] = S.compress(w, pb, True)
    np.savez_compressed(os.path.join(HERE, "sparse32_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
