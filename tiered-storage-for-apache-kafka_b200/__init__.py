"""H100-native chunk-transform pipeline for Aiven's Kafka tiered-storage RemoteStorageManager.

Only the hot path of SURVEY.md §8 lives here: csrc/ (sm_90a CUDA kernels + the C-ABI of include/tsgpu.h),
binding.py (ctypes view of that C-ABI), host/ (C++ mirror of the reference's Transform/DetransformChunkEnumeration operator
surface and of the caller side of the copy path) and corpus.py (synthetic segment generators).
The directory name has a hyphen, so import it through the `tsgpu` shim at the repo root or importlib.
"""
from . import binding  # noqa: F401
from .binding import (FLAG_AES, FLAG_ZSTD, FLAG_ZSTD_DENSE, IV_SIZE, TAG_SIZE, Context, TsgpuError)  # noqa: F401
