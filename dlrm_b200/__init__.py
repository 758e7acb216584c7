"""dlrm_b200 -- H100-native (sm_90a) DLRM forward/backward hot path behind the reference's
DLRM_Net module surface.  Host side: Python/PyTorch (device memory, streams, torch.distributed);
compute: hand-written CUDA in libdlrm_b200.so reached through the C ABI of include/dlrm_b200.h."""

__version__ = "0.1.0"
