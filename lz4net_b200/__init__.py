"""lz4net_b200 -- an H100 (sm_90a) LZ4 r93 block codec behind lz4net's LZ4Codec / ILZ4Service / LZ4Stream surface.

Only the hot path lives here: hand-written CUDA kernels (csrc/), their C ABI (include/lz4b200.h, liblz4b200.so) and
the host-side mirror of the reference interface (codec.py).  There is no CPU codec in this package.
"""
from . import native, synth  # noqa: F401
from .codec import (Context, CudaLZ4Service, LZ4Codec, LZ4Stream, LZ4StreamFlags, LZ4StreamMode,  # noqa: F401
                    default_context)

__all__ = ["native", "synth", "Context", "CudaLZ4Service", "LZ4Codec", "LZ4Stream", "LZ4StreamFlags", "LZ4StreamMode",
           "default_context"]
