"""triforce_b200 — H100-native (sm_90a) hot path of TriForce hierarchical speculative decoding.

Python host code (this package) → ctypes → `lib/libtriforce_b200.so` (C ABI in include/triforce_b200.h).
Importing the package does not load the library; the first kernel call does and fails loudly if it is missing.
"""
__version__ = "0.1.0"
