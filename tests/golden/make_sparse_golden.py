"""Writes tests/golden/sparse_golden.npz: small sparse fp16 / bf16 members (float types 5 and 6) and their archives
at prob bits 9, 10 and 11 with checksums, from the CPU restatement in tests/sparse_oracle.py.  Run from the
repository root: python tests/golden/make_sparse_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import sparse_oracle as S  # noqa: E402
from test_oracle_sparse import all_but, masked_words, relu_words  # noqa: E402


def members(ft):
    return {
        "empty": np.zeros(0, np.uint16),
        "relu_4097": relu_words(4097, ft, 11),
        "relu_9000": relu_words(9000, ft, 12),
        "masked_5000": masked_words(5000, ft, 13),
        "one_free": all_but((99,), ft),            # nothing elided
        "two_free": all_but((17, 200), ft),
        "full_range": np.random.default_rng(ft).integers(0, 1 << 16, 3001, dtype=np.uint16),
    }


def main():
    out = {}
    for ft in (S.F16S, S.BF16S):
        for name, w in members(ft).items():
            key = f"sparse/{ft}/{name}"
            out[f"{key}/in"] = w
            for pb in (9, 10, 11):
                out[f"{key}/pb{pb}"] = S.compress(w, ft, pb, True)
    np.savez_compressed(os.path.join(HERE, "sparse_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
