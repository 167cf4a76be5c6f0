"""renegade_b200 — H100-native proving backend for the PlonK prover behind renegade-fi/renegade's
crates/circuits: hand-written sm_90a CUDA (BN254 G1 Pippenger MSM, BN254-Fr radix-2 NTT) behind
a C ABI (include/b200prover.h), with this thin host-side mirror of the reference's interface.

Importing the package does not load the shared library; the first call does, and fails loudly if
it is missing or no CUDA device is visible (there is no CPU fallback)."""
from . import _lib  # noqa: F401
from .backend import (  # noqa: F401
    Bases, Context, Radix2EvaluationDomain, UnivariateKzgPCS, UnivariateUniversalParams,
    VariableBaseMSM, parse_ptau_file, MAX_SRS_DEGREE, SrsReport, check_srs, read_ptau_g2,
)

__version__ = "0.1.0"
