"""omni3d_b200 — H100-native (sm_90a) Cube R-CNN hot path behind the reference's interface.

Product code.  Never imports oracle/.  Every op fails loudly if libc3d.so (the hand-written
CUDA kernels, C ABI in include/c3d.h) is missing — there is no CPU or library fallback.
"""
__version__ = "0.1.0"
