"""phastft_b200 -- H100 (sm_90a) drop-in for PhastFT's 1-D power-of-two FFT path.

The package is a thin host-side mirror (api.py) of the reference's public API over the C ABI of
libphastft_cuda.so (csrc/, include/phastft_cuda.h).  Importing it requires the built shared
library; there is no CPU fallback.
"""
from .api import *  # noqa: F401,F403
from ._lib import LIB_PATH, device_count, last_launches, launch_count  # noqa: F401
