"""retinanet-examples_b200 -- H100-native RetinaNet inference hot path (drop-in for ODTK's
odtk.infer / Model.forward / _C.decode / _C.nms).  Python host code over PyTorch tensors
(device memory, streams, torch.distributed) calling a C-ABI shared library of hand-written
sm_90a CUDA kernels through ctypes (include/odtk_b200.h).  There is no CPU fallback: every
op raises if the CUDA library is missing or a tensor is not on the GPU."""

__version__ = "0.1"
