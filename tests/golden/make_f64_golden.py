"""Generates tests/golden/f64_golden.npz: seeded float64 inputs with the float-type-4 archives the CPU
restatement (tests/f64_oracle.py) produces for them (the reference has no float64 codec, so there is no
reference archive to pin against).  tests/test_oracle_float64.py checks that they are still reproduced.
Run:  python tests/golden/make_f64_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import f64_oracle as F  # noqa: E402


def cases():
    rng = np.random.default_rng(64)
    return {
        "normal_1": rng.standard_normal(1).view(np.uint64),
        "normal_4099": rng.standard_normal(4099).view(np.uint64),
        "normal_8000": rng.standard_normal(8000).view(np.uint64),
        "full_range_2000": rng.integers(0, 2 ** 64, 2000, dtype=np.uint64),
        "empty": np.zeros(0, np.uint64),
    }


if __name__ == "__main__":
    out = {}
    for name, w in cases().items():
        out[f"f64/{name}/in"] = w
        for pb in (9, 10, 11):
            out[f"f64/{name}/pb{pb}"] = F.compress(w, pb, True)
    np.savez_compressed(os.path.join(HERE, "f64_golden.npz"), **out)
    print("wrote", len(out), "arrays")
