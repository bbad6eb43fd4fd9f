"""ctypes binding of tests/cpp/inflight_oracle.c: the inflight-load-producer restated on the CPU (test infrastructure only).

estimate(size, hint, chars) is SimpleTokenEstimator.Estimate for arrays; Tracker is the producer's pair of
concurrencyTrackers keyed by endpoint id (add / release / remove / get)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "inflight_oracle.c")
BUILD = os.path.join(ROOT, "tests", "cpp", "_build")
LIB = os.path.join(BUILD, "libinflight_oracle.so")

_lib = None


def build() -> str:
    """libinflight_oracle.so (gcc)"""
    if not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-ffp-contract=off", "-fPIC", "-shared", SRC, "-o", LIB, "-lm"])
    return LIB


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_estimate_tokens.restype = C.c_int64
        L.orc_estimate_tokens.argtypes = [C.c_int64, C.c_int32, C.c_int32]
        L.orc_inflight_new.restype = C.c_void_p
        L.orc_inflight_new.argtypes = []
        L.orc_inflight_free.argtypes = [C.c_void_p]
        for f in ("orc_inflight_add", "orc_inflight_release"):
            getattr(L, f).argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        L.orc_inflight_remove.argtypes = [C.c_void_p, C.c_int32]
        L.orc_inflight_get.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def estimate(size=None, hint=None, chars=None, R=None) -> np.ndarray:
    """int64[R] estimates; a missing array means size 0, hint -1, chars 0 (as eppscore_estimate_tokens)"""
    if R is None:
        R = len(next(a for a in (size, hint, chars) if a is not None))
    size = np.zeros(R, np.int64) if size is None else np.asarray(size, np.int64)
    hint = np.full(R, -1, np.int32) if hint is None else np.asarray(hint, np.int32)
    chars = np.zeros(R, np.int32) if chars is None else np.asarray(chars, np.int32)
    L = lib()
    return np.array([L.orc_estimate_tokens(int(size[r]), int(hint[r]), int(chars[r])) for r in range(R)], np.int64)


class Tracker:
    def __init__(self):
        self._h = lib().orc_inflight_new()

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:  # (at interpreter exit the module may be torn down first)
            _lib.orc_inflight_free(self._h)
            self._h = None

    def _call(self, fn, endpoint, tokens):
        ep = np.ascontiguousarray(endpoint, np.int32)
        tk = None if tokens is None else np.ascontiguousarray(tokens, np.int64)
        fn(self._h, len(ep), ep.ctypes.data, None if tk is None else tk.ctypes.data)

    def add(self, endpoint, tokens=None):
        self._call(lib().orc_inflight_add, endpoint, tokens)

    def release(self, endpoint, tokens=None):
        self._call(lib().orc_inflight_release, endpoint, tokens)

    def remove(self, endpoint: int):
        lib().orc_inflight_remove(self._h, endpoint)

    def get(self, M: int):
        req, tok = np.zeros(max(M, 1), np.int64), np.zeros(max(M, 1), np.int64)
        lib().orc_inflight_get(self._h, M, req.ctypes.data, tok.ctypes.data)
        return req[:M], tok[:M]
