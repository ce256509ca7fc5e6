"""femasr_b200: H100-native (sm_90a) implementation of FeMaSR's inference hot path.

  femasr_b200.lib    ctypes binding of libfemasr_b200.so (C ABI in include/femasr_b200.h)
  femasr_b200.net    host engine wrapper (workspace, test()/test_tile() scheduling)
  femasr_b200.module nn.Module base of the engine-backed networks (tensor tree, upload on change)
  femasr_b200.spec   parameter inventory + seeded random weights
  femasr_b200.build  nvcc build of the library (in-tree)
The reference-facing operator surface lives in `basicsr.archs.femasr_arch.FeMaSRNet`.
"""
import os

__version__ = "0.1.0"


def default_gemm_path() -> int:
    """1 = wgmma split-fp16 tensor-core GEMM (default), 0 = fp32 SIMT implicit GEMM (exact-arithmetic
    debug path); FEMASR_GEMM_PATH overrides."""
    return int(os.environ.get("FEMASR_GEMM_PATH", "1"))
