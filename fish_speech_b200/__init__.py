"""fish_speech_b200 — H100-native (sm_90a) implementation of the Fish-Speech two-stage inference
hot path (Dual-AR text2semantic decode + DAC codec), behind the reference's own Python entry points.

The product path is the CUDA library `libfishb200.so` (hand-written sm_90a kernels behind the C-ABI
in include/fishb200.h).  There is no CPU or eager-PyTorch fallback: importing `_lib` raises if the
library is missing or cannot be loaded.
"""

__version__ = "0.1.0"
