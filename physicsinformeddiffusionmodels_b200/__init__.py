"""H100-native engine for the physics-informed-diffusion hot path (see DESIGN.md).

Host code is Python/PyTorch (device memory, streams, autograd bookkeeping, torch.distributed);
every per-step operation is a hand-written sm_100a CUDA kernel in libpidm.so behind the C ABI of
include/pidm.h.  There is no CPU or PyTorch-op fallback on the product path."""
__version__ = '0.1.0'
