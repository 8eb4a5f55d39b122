"""visualcloze_b200 -- H100-native (sm_90a) implementation; the package name dates from its first target of the VisualCloze denoising hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic of the path runs in
hand-written CUDA kernels reached through the C ABI of ``libvcb200.so`` (``include/vcb200.h``).
There is no CPU fallback: importing the ops without the built library, or calling them without an H100,
raises.
"""
__version__ = "0.1.0"
