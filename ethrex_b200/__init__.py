"""ethrex_b200 -- host side of the H100-native BN254 MSM + Fr NTT backend for ethrex's L2 prover.

Everything numerical happens in libb200zk.so (hand-written sm_90a CUDA behind the C ABI of
include/b200zk.h); this package is the Python twin of the Rust shim in rust/ (the reference's
toolchain is absent from the build image).  There is no CPU fallback.
"""
from . import _ffi as ffi  # noqa: F401  (raises ImportError loudly if libb200zk.so is missing)
from ._ffi import (NTT_BE, NTT_CANONICAL, NTT_COSET, NTT_INVERSE, OUT_NATIVE, POINTS_BE, SCALARS_BE,  # noqa: F401
                   SCALARS_MONT)
from .backend import B200Backend, BackendType, ProofFormat, ProverType  # noqa: F401
from .context import Context  # noqa: F401
from .errors import B200Error, NoDeviceError  # noqa: F401

__all__ = ["Context", "B200Backend", "BackendType", "ProofFormat", "ProverType", "B200Error", "NoDeviceError", "ffi"]
