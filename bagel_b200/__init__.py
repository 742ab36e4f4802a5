"""bagel_b200 — H100-native (sm_90a) implementation of BAGEL's inference forward hot path.

Host side: Python mirroring the reference's API (ByteDance-Seed/Bagel: inferencer.py, modeling/bagel/*).
Compute: hand-written CUDA (wgmma / TMA / mbarrier) behind the C ABI in include/bagel_b200.h.
"""
__version__ = "0.1.0"
