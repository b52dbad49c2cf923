"""The reference tree's heFFTe real-to-complex transform (oracle/ref_heffte_r2c), TEST INFRASTRUCTURE ONLY.

build_ref_r2c() compiles oracle/_ref/libheffte_r2c_ref.so from the reference tree when that tree is present; elsewhere the
prebuilt file is used as is, and the tests fall back to the vectors recorded from it (tests/golden/heffte_r2c_vectors.npz,
written by tests/golden/make_heffte_r2c_vectors.py)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "_ref", "libheffte_r2c_ref.so")
_SRC = "/root/reference/heffte/heffteBenchmark"


def build_ref_r2c(force: bool = False):
    """path of oracle/_ref/libheffte_r2c_ref.so, built when the reference tree is present; None when it neither exists nor can
    be built"""
    rdir = os.path.join(_HERE, "ref_heffte_r2c")
    if os.path.isdir(_SRC):
        deps = [os.path.join(rdir, f) for f in ("heffte_r2c_ref.cpp", "Makefile")] + \
               [os.path.join(_HERE, "ref_heffte", f) for f in ("tmpi.cpp", "mpi.h", "heffte_config.h")]
        if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(d) for d in deps):
            subprocess.run(["make", "-C", rdir, "-s", f"REF={_SRC}"], check=True)
    return _LIB if os.path.exists(_LIB) else None


class HeffteR2CRef:
    """ctypes binding of heffte_ref_fft3d_r2c: world-array R2C / C2R by heFFTe over P slab ranks (threads)"""

    def __init__(self):
        path = build_ref_r2c()
        if path is None:
            raise FileNotFoundError("oracle/_ref/libheffte_r2c_ref.so is missing and the reference tree is not available to build it")
        self.lib = ctypes.CDLL(path)
        vp, i = ctypes.c_void_p, ctypes.c_int
        self.lib.heffte_ref_fft3d_r2c.argtypes = [i, i, i, i, vp, vp, i, i, i]

    def forward(self, A: np.ndarray, P: int) -> np.ndarray:
        """real A[x][y][z] (float64 / float32) -> half spectrum [x][y][n2//2+1], unnormalised"""
        A = np.ascontiguousarray(A)
        n0, n1, n2 = A.shape
        out = np.zeros((n0, n1, n2 // 2 + 1), dtype=np.complex128 if A.dtype == np.float64 else np.complex64)
        rc = self.lib.heffte_ref_fft3d_r2c(n0, n1, n2, P, A.ctypes.data, out.ctypes.data, 1, 0 if A.dtype == np.float64 else 1, 0)
        if rc != 0:
            raise ValueError(f"heffte_ref_fft3d_r2c failed ({rc})")
        return out

    def backward(self, S: np.ndarray, n2: int, P: int, scale_full: bool = False) -> np.ndarray:
        """half spectrum S[x][y][n2//2+1] -> real [x][y][n2], unnormalised unless scale_full"""
        S = np.ascontiguousarray(S)
        n0, n1, _ = S.shape
        out = np.zeros((n0, n1, n2), dtype=np.float64 if S.dtype == np.complex128 else np.float32)
        rc = self.lib.heffte_ref_fft3d_r2c(n0, n1, n2, P, S.ctypes.data, out.ctypes.data, -1, 0 if S.dtype == np.complex128 else 1, int(scale_full))
        if rc != 0:
            raise ValueError(f"heffte_ref_fft3d_r2c failed ({rc})")
        return out
