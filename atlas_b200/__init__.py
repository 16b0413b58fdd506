"""atlas_b200 — Hopper-native (sm_90a, H100) implementation of Atlas' retrieve-then-read hot path.

Python here is host plumbing only (device memory, streams, torch.distributed); the arithmetic lives
in `csrc/` behind the C ABI declared in `include/atlas_b200.h`.  There is no CPU fallback.
"""
__version__ = "0.1"
