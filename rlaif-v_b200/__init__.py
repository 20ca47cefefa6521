"""H100-native DPO training step for LLaVA-1.5 (drop-in for the RLAIF-V `muffin/train` hot path).

Python host code (this package) drives hand-written sm_90a CUDA kernels through the C-ABI
library declared in ``include/rlaifv_b200.h``.  Import as ``rlaifv_b200``.
"""
__version__ = "0.1.0"
