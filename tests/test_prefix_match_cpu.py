"""eppscore_prefix_match's lookup and membership code (csrc/prefix_table.cuh table_find / slot_holds, what prefix_match_kernel
runs per lane) under the sequential execution policy (tests/cpp/index_match_emu.cpp), checked against the oracle's
matchLongestPrefix read at the listed endpoints.  The index is built with the emulator's commit code.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_py as o
from tests.prefix_match_scenarios import CHURN, churn_scenario, crafted_scenarios, expected

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
SRC = os.path.join(CPP, "index_match_emu.cpp")
OUT = os.path.join(CPP, "_build", "libindex_match_emu.so")


@pytest.fixture(scope="module")
def L():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    deps = [SRC, os.path.join(CPP, "index_emu.cpp"), os.path.join(ROOT, "gateway-api-inference-extension_b200", "csrc", "prefix_table.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-D_GLIBCXX_ASSERTIONS", SRC, "-o", OUT])
    lib = C.CDLL(OUT)
    P, LL = C.c_void_p, C.c_longlong
    for name, res, args in [
            ("emu_new", P, [C.c_int, LL, C.c_int, C.c_int]), ("emu_free", None, [P]),
            ("emu_commit", C.c_int, [P, C.c_int, P, P, P, C.c_int, P, C.c_int]),
            ("match_emu", None, [P, C.c_int, C.c_int, C.c_int, P, P, C.c_int, P, P]), ("emu_stat", LL, [P, C.c_int])]:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def _match(L, h, q, limit):
    R, k = q.endpoints.shape
    out = np.full((R, k), 0xBEEF, np.uint16)
    hs = np.ascontiguousarray(q.hashes)
    nh = np.ascontiguousarray(q.n_hashes)
    eps = np.ascontiguousarray(q.endpoints)
    L.match_emu(h, R, k, limit, hs.ctypes.data, nh.ctypes.data, hs.shape[1], eps.ctypes.data, out.ctypes.data)
    return out


def _run(L, sc):
    limit = sc.M
    h = L.emu_new(sc.M, 1 << 10, sc.lru, sc.lru_max)
    idx = o.Index(sc.lru)
    caps = None if sc.caps is None else np.ascontiguousarray(sc.caps, np.int32)
    asked = 0
    for b, queries in sc.steps:
        assert L.emu_commit(h, len(b.pick), b.pick.ctypes.data, b.hashes.ctypes.data, b.n_hashes.ctypes.data, b.hashes.shape[1],
                            None if caps is None else caps.ctypes.data, 0) == 0
        idx.commit(b.pick, b.hashes, b.n_hashes, caps)
        for q in queries:
            want = expected(idx, q, limit)
            got = _match(L, h, q, limit)
            assert np.array_equal(got, want), (sc.name, np.argwhere(got != want)[:5])
            asked += 1
    assert asked > 0
    L.emu_free(h)
    return want


@pytest.mark.parametrize("M,lru,R,nmax,seed", CHURN, ids=[f"lru{c[1]}" for c in CHURN])
def test_churn_matches_oracle(L, M, lru, R, nmax, seed):
    """Random commits with evictions: after every batch its prompts, cut prompts and fresh prompts match the oracle at k = 8
    random entries (some -1, some at or past max_endpoints)."""
    _run(L, churn_scenario(M, lru, R, nmax, seed, k=8, limit=M + 1))


@pytest.mark.parametrize("name", ["inline-to-row", "universal-prefix", "emptied-mid-prompt", "partial-holder", "long-prompts"])
def test_crafted_states_match_oracle(L, name):
    (sc,) = [s for s in crafted_scenarios(limit=10 ** 6) if s.name == name]
    # the entries at and past the limit are the crafted scenario's last two columns: 0 always
    sc_limit = sc.M
    for _, queries in sc.steps:
        for q in queries:
            q.endpoints[:, -2:] = [sc_limit, sc_limit + 7]
    got = _run(L, sc)
    assert not got[:, -3:].any()  # -1, max_endpoints and past it
    if name == "emptied-mid-prompt":  # endpoint 0 stops at the emptied block; endpoint 1's later hit does not count
        assert got[0].tolist()[:2] == [1, 0] and got[2].tolist()[:2] == [1, 1] and got[3].tolist()[:2] == [1, 0]
    if name == "partial-holder":
        assert got[0].tolist()[:3] == [8, 3, 1]
    if name == "long-prompts":
        assert got[0].tolist()[:4] == [1000, 300, 256, 0] and got[3].tolist()[:4] == [600, 300, 256, 0]
        assert not got[2].any()  # 0 hashes
