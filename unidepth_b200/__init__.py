"""unidepth_b200 -- CUDA-native (H100, sm_90a) implementation of UniDepth's inference forward pass.

Drop-in for `unidepth.models.UniDepthV2`, `unidepth.models.UniDepthV1` and `UniDepthV2old` on the `.infer()`
path (see unidepthv2.py / unidepthv1.py / unidepthv2old.py); the compute lives in libudb.so (csrc/, C ABI in include/udb.h), built by
`python -m unidepth_b200.build`.
"""
from . import camera  # noqa: F401  (Pinhole, BatchCamera, ... for infer(rgb, camera=...))
from .unidepthv1 import UniDepthV1  # noqa: F401
from .unidepthv2 import UniDepthV2  # noqa: F401
from .unidepthv2old import UniDepthV2old  # noqa: F401

__all__ = ["UniDepthV1", "UniDepthV2", "UniDepthV2old", "camera"]
