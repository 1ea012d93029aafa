"""super4pcs_b200 -- H100-native (sm_90a) Super4PCS congruent-set extraction + LCP verification.

The product is `lib/libs4g.so` (hand-written CUDA behind the C ABI of include/s4g.h) and the
header-compatible C++ layer in include/super4pcs/.  This Python package is the thin ctypes
binding the tests and bench.py drive the ABI through; it contains no algorithmic code and there
is NO CPU fallback: loading fails loudly if the CUDA library is missing.
"""
from .s4g import (S4GError, Context, TcsResult, PairFilters, lib_path, load_library,  # noqa: F401
                  exported_symbols, declared_symbols)
