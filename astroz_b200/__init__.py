"""astroz_b200 -- H100-native batch SGP4/SDP4 propagation behind the astroz interface.

Only the propagation hot path of ATTron/astroz lives here (SURVEY.md section 8): hand-written sm_90a
CUDA kernels behind a C ABI (include/astroz_b200.h), plus host-side mirrors of the reference's
`Constellation` and python-sgp4-compatible `Satrec` / `SatrecArray`.  There is no CPU fallback.
"""
from ._lib import (AstrozCudaError, LIB_PATH, device_count, host_register, host_unregister, lib,  # noqa: F401
                   pinned_empty)
from .constellation import Constellation, Layout, OutputMode, fp64_peak_tflops, fp64_pipe_peak_tflops  # noqa: F401

__version__ = "0.1.0"
