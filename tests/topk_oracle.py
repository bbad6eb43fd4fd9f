"""ctypes binding of tests/cpp/topk_oracle.c: maxNumOfEndpoints restated on the CPU oracle (test infrastructure only).

pick_topk(weighted, profile, request_index, k) orders one request's candidates (weighted[m] not NaN) as the profile's
picker would; schedule_batch(...) is oracle_py.schedule_batch plus those lists for every request."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle_py as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "topk_oracle.c")
BUILD = os.path.join(ROOT, "tests", "cpp", "_build")
LIB = os.path.join(BUILD, "libtopk_oracle.so")
ORACLE_DIR = os.path.join(ROOT, "oracle", "_build")

_lib = None


def build() -> str:
    """libtopk_oracle.so (gcc, linked against oracle/_build/liboracle.so)"""
    oracle_lib = o.build()
    deps = [SRC, os.path.join(ROOT, "oracle", "oracle.h"), oracle_lib]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-ffp-contract=off", "-fPIC", "-shared", SRC, "-o", LIB,
                               "-L" + ORACLE_DIR, "-loracle", "-Wl,-rpath," + ORACLE_DIR, "-lm"])
    return LIB


def lib():
    global _lib
    if _lib is None:
        o.lib()  # liboracle.so first, so the dependency resolves
        L = C.CDLL(build())
        L.topk_oracle_pick.restype = C.c_int32
        L.topk_oracle_pick.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_int64, C.c_int32, C.c_void_p,
                                       C.c_void_p]
        _lib = L
    return _lib


def pick_topk(weighted, profile: o.Profile, request_index: int, k: int):
    """Returns (endpoints int32[k] padded with -1, scores float64[k] padded with 0.0)."""
    w = np.ascontiguousarray(weighted, np.float64)
    m_out = np.full(k, -1, np.int32)
    s_out = np.zeros(k, np.float64)
    lib().topk_oracle_pick(w.ctypes.data, len(w), profile.pick_mode, profile.tie_mode, profile.tie_seed, request_index, k,
                           m_out.ctypes.data, s_out.ctypes.data)
    return m_out, s_out


def lists(weighted, profile: o.Profile, k: int, request_base: int = 0):
    """pick_topk of every row of weighted [R, M]: (topk_pick int32[R, k], topk_score float64[R, k])"""
    R = weighted.shape[0]
    m = np.full((R, k), -1, np.int32)
    s = np.zeros((R, k), np.float64)
    for r in range(R):
        m[r], s[r] = pick_topk(weighted[r], profile, request_base + r, k)
    return m, s


def schedule_batch(snap, profile: o.Profile, index, R: int, *, topk: int, request_base: int = 0, **kw):
    """oracle_py.schedule_batch with the weighted score map, plus topk_pick / topk_score [R, k]"""
    out = o.schedule_batch(snap, profile, index, R, request_base=request_base, want_scores=True, **kw)
    out["topk_pick"], out["topk_score"] = lists(out["weighted_out"], profile, topk, request_base)
    return out
