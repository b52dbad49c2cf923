"""Writes tests/golden/heffte_r2c_vectors.npz: forward (R2C) and backward (C2R) transforms of small real cubes computed by
the reference tree's heFFTe (heffte::fft3d_r2c, stock backend, r2c_direction 0 = our z) over P slab ranks, from
oracle/_ref/libheffte_r2c_ref.so, which build() compiles where the reference tree is present:

    python tests/golden/make_heffte_r2c_vectors.py

tests/test_heffte_r2c_vectors.py always checks the committed vectors against numpy's rfftn / irfftn convention and against
the library's recorded R2C / C2R schedules, and recomputes them with the live library where it is built."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

OUT = os.path.join(HERE, "heffte_r2c_vectors.npz")
# (n0, n1, n2, P): even and odd n2, P = 1, 2, 3 with uneven splits (5 over 2 and 3, 8 and 7 over 3)
CASES = [(6, 8, 10, 1), (6, 8, 10, 2), (6, 8, 10, 3), (5, 7, 9, 1), (5, 7, 9, 2), (5, 7, 9, 3), (7, 5, 16, 3)]


def case_input(n0, n1, n2, P):
    """the real cube of a case; the backward input is its numpy half spectrum (Hermitian where it must be)"""
    return np.random.default_rng(n0 * 100 + n1 * 10 + n2 + 1000 * P).standard_normal((n0, n1, n2))


def key(n0, n1, n2, P):
    return f"{n0}x{n1}x{n2}_P{P}"


def compute(ref, n0, n1, n2, P):
    A = case_input(n0, n1, n2, P)
    S = np.fft.rfftn(A)
    return {"fwd": ref.forward(A, P), "bwd": ref.backward(S, n2, P)}


def main():
    from oracle.heffte_r2c import HeffteR2CRef
    ref = HeffteR2CRef()
    out = {}
    for c in CASES:
        r = compute(ref, *c)
        out[key(*c) + "_fwd"] = r["fwd"]
        out[key(*c) + "_bwd"] = r["bwd"]
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
