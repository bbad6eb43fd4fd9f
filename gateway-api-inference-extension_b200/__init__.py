"""gateway-api-inference-extension_b200 — H100-native batched Endpoint-Picker scoring engine.

The product is the C-ABI shared library `libeppscore.so` (include/eppscore.h) built from the
hand-written sm_90a kernels under csrc/.  This package is the thin ctypes binding used by the
tests and bench.py (the host mirror of the reference's plugin interface is C++: host/); it holds no arithmetic of its
own and has no CPU fallback — loading fails loudly if the library has not been built, and `Engine()` fails
loudly without a CUDA device.

(The directory name contains hyphens, so it is registered under the import name `gaie_b200`
by `_pkg.py` at the repo root.)
"""
from ._capi import (  # noqa: F401
    ABI_SYMBOLS, Batch, Config, EppscoreError, LatencyInfo, LatencyParams, MAX_STREAMS, MAX_TOPK, SCORER, Snapshot, Stats, TopK, TIE_LOWEST_INDEX, TIE_SEEDED_RANDOM, PICK_MAX_SCORE, PICK_WEIGHTED_RANDOM, PICK_RANDOM, FILTER_PREFIX_AFFINITY, FILTER_SLO_HEADROOM_TIER,
    lib, lib_path,
)
from .engine import LATENCY_INFO_DTYPE, Engine, default_config, latency_params  # noqa: F401
