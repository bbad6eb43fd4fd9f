"""ctypes binding of tests/cpp/running_oracle.c: the predicted-latency producer's running-request queues restated on the CPU
(test infrastructure only).  Queues(M) holds one requestPriorityQueue per endpoint id; add / remove apply a batch entry by
entry in request order; get(M) is the (min tpot, count) view the latency fold-in reads."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "running_oracle.c")
BUILD = os.path.join(ROOT, "tests", "cpp", "_build")
LIB = os.path.join(BUILD, "librunning_oracle.so")

_lib = None


def build() -> str:
    """librunning_oracle.so (gcc)"""
    if not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-ffp-contract=off", "-fPIC", "-shared", SRC, "-o", LIB])
    return LIB


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_running_new.restype = C.c_void_p
        L.orc_running_new.argtypes = [C.c_int32]
        L.orc_running_free.argtypes = [C.c_void_p]
        L.orc_running_add.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_running_remove.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_running_remove_endpoint.argtypes = [C.c_void_p, C.c_int32]
        L.orc_running_get.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def canonical(x):
    """-0.0 as +0.0: the engine stores a zero tpot as +0.0 (every consumer compares with > 0); the queue keeps the sign"""
    x = np.asarray(x, np.float64)
    return np.where(x == 0.0, 0.0, x)


class Queues:
    def __init__(self, n_ep: int):
        self.n_ep = n_ep
        self._h = lib().orc_running_new(n_ep)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:  # (at interpreter exit the module may be torn down first)
            _lib.orc_running_free(self._h)
            self._h = None

    def add(self, endpoint, key, tpot=None) -> np.ndarray:
        ep = np.ascontiguousarray(endpoint, np.int32)
        k = np.ascontiguousarray(key, np.uint64)
        t = None if tpot is None else np.ascontiguousarray(tpot, np.float64)
        out = np.zeros(max(len(ep), 1), np.uint8)
        lib().orc_running_add(self._h, len(ep), ep.ctypes.data, k.ctypes.data, None if t is None else t.ctypes.data, out.ctypes.data)
        return out[: len(ep)].astype(bool)

    def remove(self, endpoint, key) -> np.ndarray:
        ep = np.ascontiguousarray(endpoint, np.int32)
        k = np.ascontiguousarray(key, np.uint64)
        out = np.zeros(max(len(ep), 1), np.uint8)
        lib().orc_running_remove(self._h, len(ep), ep.ctypes.data, k.ctypes.data, out.ctypes.data)
        return out[: len(ep)].astype(bool)

    def remove_endpoint(self, endpoint: int):
        lib().orc_running_remove_endpoint(self._h, endpoint)

    def get(self, M: int | None = None):
        M = self.n_ep if M is None else M
        mn, cnt = np.zeros(max(M, 1), np.float64), np.zeros(max(M, 1), np.int32)
        lib().orc_running_get(self._h, M, mn.ctypes.data, cnt.ctypes.data)
        return mn[:M], cnt[:M]


def expand_case(case, ids):
    """A golden case as a list of ops ("add", ep, key, tpot, want) / ("remove", ep, key, want) / ("view", ep, min, count);
    `ids` maps request ids to keys (the empty id to 0).  A "large" case is generated as its Go test does."""
    if "large" in case:
        n = case["large"]["n"]
        ops = [("add", 0, ids(f"item{i}"), float(n - i), True) for i in range(n)]
        ops.append(("view", 0, 1.0, n))
        for i in range(n):  # Peek is item{n-1} (tpot 1.0), then item{n-2}, ...: the minimum never goes down
            ops.append(("remove", 0, ids(f"item{n - 1 - i}"), True))
            ops.append(("view", 0, float(i + 2) if i + 1 < n else 0.0, n - 1 - i))
        return ops
    out = []
    for op in case["ops"]:
        if op[0] == "add":
            out.append(("add", op[1], ids(op[2]), float(op[3]), op[4]))
        elif op[0] == "remove":
            out.append(("remove", op[1], ids(op[2]), op[3]))
        else:
            out.append(("view", op[1], float(op[2]), op[3]))
    return out


class KeyMap:
    """Request id -> exact uint64 key, from 1 in order of first use; the empty id is 0 (refused by Add)."""

    def __init__(self):
        self.k = {}

    def __call__(self, rid: str) -> int:
        if rid == "":
            return 0
        return self.k.setdefault(rid, len(self.k) + 1)
