"""rusty_kaspa_b200 — H100-native transaction-validation hot path of rusty-kaspa.

Only what the path needs: `csrc/` (hand-written sm_90a CUDA + the C ABI of include/kgv.h, built
into libkgv.so) and the host-side mirror of the reference interface for this path.
"""
from ._lib import KgvError, LIB_PATH, SIG_INVALID, SIG_PK_PARSE_ERR, SIG_SIG_PARSE_ERR, SIG_VALID  # noqa: F401
from .verifier import GpuContext  # noqa: F401
from .validator import GpuUtxoSet, MempoolPolicy, Params, TransactionValidator, TxRules  # noqa: F401
from .muhash import MuHash  # noqa: F401
