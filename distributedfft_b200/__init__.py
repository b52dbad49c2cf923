"""distributedfft_b200 -- H100-native slab-decomposed 3-D C2C FFT.

The product is `libdfft.so` (hand-written sm_90a CUDA kernels behind the C ABI of include/dfft.h)
and the `distFFT` driver.  This package is only the Python face of that library: a ctypes binding
with the reference's function names (3dmpifft_opt/include/fft_mpi_3d_api.h:68-74) used by the
tests and bench.py.  There is no CPU fallback: importing `distributedfft_b200.api` raises if the
library has not been built, and every call fails loudly without a CUDA device.
"""
from .api import *  # noqa: F401,F403
