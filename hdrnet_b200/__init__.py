"""hdrnet_b200 -- H100-native (sm_90a) implementation of google/hdrnet's bilateral-slice
hot path behind the reference's own ``hdrnet_ops`` / ``layers`` / ``models`` interface.

    from hdrnet_b200 import hdrnet_ops, layers, models
    out = hdrnet_ops.bilateral_slice_apply(grid, guide, image, has_offset=True)

Host code is Python over PyTorch tensors (device memory, streams, torch.distributed); the
compute is hand-written CUDA in ``csrc/`` reached through the C-ABI in
``include/hdrnet_b200.h``.  There is no CPU fallback.
"""
from . import _lib  # noqa: F401
from . import hdrnet_ops  # noqa: F401
from . import layers  # noqa: F401
from . import models  # noqa: F401

__all__ = ["hdrnet_ops", "layers", "models", "_lib"]
__version__ = "0.1.0"
