"""coach_b200 -- H100-native (sm_90a CUDA) implementation of IntelLabs/coach's replay-sample -> learn_from_batch
hot path, behind Coach's Memory / Filter / Agent plugin interface.  See DESIGN.md and INTEGRATION.md.

Compute lives in ``lib/libcoach_b200.so`` (hand-written CUDA, C ABI in ``include/coach_b200.h``); there is no CPU
fallback -- ``coach_b200._lib.load()`` raises if the library is missing.
"""
__version__ = "0.1.0"
