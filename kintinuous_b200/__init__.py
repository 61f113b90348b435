"""kintinuous_b200 -- H100-native dense tracking-and-fusion hot path (Kintinuous frontend).

Python is only the test / bench harness language here: the product is the C-ABI shared library
``libkintinuous_b200.so`` (include/kintinuous_b200.h) built from ``csrc/*.cu`` for sm_90a.  This package
loads it with ctypes and mirrors the reference's operator / tracker interface (same names, argument
meaning and error behaviour).  There is NO CPU fallback: importing works without a GPU (so the symbol
table can be checked), but every compute call raises ``KtError`` when no CUDA device is present, and
``load()`` raises if the library has not been built.
"""
from .binding import KtError, load, lib_path, Config, Pose, Tracker, ops, cuda_available  # noqa: F401

__all__ = ["KtError", "load", "lib_path", "Config", "Pose", "Tracker", "ops", "cuda_available"]
