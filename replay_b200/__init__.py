"""replay_b200 - H100-native (sm_90a) implementation of RePlay's sequential-recommender hot path.

Device work is hand-written CUDA in ``librp_b200.so`` (C ABI: include/rp_b200.h); this package is the thin
Python/PyTorch host side that mirrors the reference's interfaces for that path.  There is no CPU fallback: importing
the kernels' wrappers without the built library raises.
"""
__version__ = "0.1.0"
