"""A reserved prefix index (eppscore_prefix_reserve): the room decision, the same-size rebuild into the spare table and the
swap (csrc/prefix_table.cuh RoomOps, the code the device kernels run) under the sequential execution policy
(tests/cpp/index_room_emu.cpp), checked against the oracle's indexer.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_py as o
from tests.index_scenarios import members_from_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
SRC = os.path.join(CPP, "index_room_emu.cpp")
OUT = os.path.join(CPP, "_build", "libindex_room_emu.so")
PROCEED, REBUILD, SKIP = 0, 1, 2
ERR_SKIPPED = 4


@pytest.fixture(scope="module")
def L():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    deps = [SRC, os.path.join(CPP, "index_emu.cpp"), os.path.join(ROOT, "gateway-api-inference-extension_b200", "csrc", "prefix_table.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-D_GLIBCXX_ASSERTIONS", SRC, "-o", OUT])
    lib = C.CDLL(OUT)
    P, LL, U = C.c_void_p, C.c_longlong, C.c_ulonglong
    for name, res, args in [
            ("room_emu_new", P, [C.c_int, LL, C.c_int, C.c_int, LL, LL, LL]), ("room_emu_free", None, [P]),
            ("room_emu_decision", C.c_int, [U] * 6), ("room_emu_commit", C.c_int, [P, C.c_int, P, P, P, C.c_int, P, C.c_int]),
            ("room_emu_apply", C.c_int, [P, LL, P, P, P]), ("room_emu_stat", LL, [P, C.c_int]), ("room_emu_digest", U, [P]),
            ("emu_lru_len", C.c_int, [P, C.c_int]), ("emu_lru_keys", C.c_int, [P, C.c_int, P, C.c_int]),
            ("emu_get_many", LL, [P, P, LL, P, C.c_int]), ("emu_stat", LL, [P, C.c_int])]:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def _commit(L, h, pick, hashes, nh):
    return L.room_emu_commit(h, len(pick), pick.ctypes.data, hashes.ctypes.data, nh.ctypes.data, hashes.shape[1], None, 0)


def _check(L, h, idx, M, keys):
    """Every LRU (oldest -> newest), len(hashToPods), canonical slots, and the sets of `keys`."""
    for e in range(M):
        n = idx.lru_len(e)
        assert L.emu_lru_len(h, e) == n, e
        if n > 0:
            out = np.zeros(n, np.uint64)
            assert L.emu_lru_keys(h, e, out.ctypes.data, n) == n
            assert [int(x) for x in out] == idx.lru_keys(e), e
    assert L.emu_stat(h, 0) == idx.num_hashes()
    assert L.emu_stat(h, 7) == 0  # every slot canonical: sorted members, 0xFFFF filler
    keys = np.ascontiguousarray(keys, np.uint64)
    words = (M + 31) // 32
    bits = np.zeros((len(keys), words), np.uint32)
    assert L.emu_get_many(h, keys.ctypes.data, len(keys), bits.ctypes.data, words) == 0, "slot count != size of its set"
    got = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :M].astype(bool)
    dh, ds = idx.dump()
    assert np.array_equal(got, members_from_pairs(keys, dh, ds, M))


def _batch(rng, M, R, nmax, groups):
    """R requests on M endpoints (some without a pick): a shared prefix from one of `groups`, then a unique tail."""
    pick = rng.integers(-1, M, size=R).astype(np.int32)
    hashes = np.zeros((R, nmax), np.uint64)
    nh = rng.integers(0, nmax + 1, size=R).astype(np.uint16)
    for r in range(R):
        n = int(nh[r])
        k = int(rng.integers(0, n + 1))
        hashes[r, :k] = groups[int(rng.integers(0, len(groups)))][:k]
        hashes[r, k:n] = rng.integers(1, 2 ** 63, size=n - k, dtype=np.uint64)
    return pick, hashes, nh


@pytest.mark.parametrize("M,lru,R,nmax,steps", [(6, 3, 40, 3, 200), (5, 40, 64, 24, 80), (4, 700, 96, 32, 90),
                                                (3, 31250, 512, 64, 120)])
def test_reserved_commits_under_churn_match_oracle(L, M, lru, R, nmax, steps):
    """Random commits on a table reserved for the live set: churn fills it with dead slots, so it is rebuilt into the spare
    again and again at the same size; after every step every LRU, len(hashToPods) and the slots match the oracle."""
    rng = np.random.Generator(np.random.PCG64(lru))
    live = M * lru + 64
    h = L.room_emu_new(M, 1 << 4, lru, 0, live, R * nmax, 2 * R * nmax)
    cap = L.emu_stat(h, 2)
    idx = o.Index(lru)
    groups = [rng.integers(1, 2 ** 63, size=nmax, dtype=np.uint64) for _ in range(6)]
    seen = [np.concatenate(groups)]
    for step in range(steps):
        pick, hashes, nh = _batch(rng, M, R, nmax, groups)
        assert _commit(L, h, pick, hashes, nh) != SKIP
        idx.commit(pick, hashes, nh)
        seen.append(hashes[pick >= 0].ravel())
        keys = np.unique(np.concatenate(seen[-3:] + seen[:1]))
        _check(L, h, idx, M, keys[keys != 0])
    assert L.room_emu_stat(h, 1) >= 2          # rebuilt on the device path, more than once ...
    assert L.emu_stat(h, 2) == cap             # ... and never resized
    assert L.room_emu_stat(h, 0) == 0 and L.room_emu_stat(h, 2) == 0
    L.room_emu_free(h)


def test_room_decision_edges(L):
    cap = 1024
    # proceed up to used + touches == cap / 2
    assert L.room_emu_decision(400, 100, cap, 0, 10 ** 6, 112) == PROCEED
    assert L.room_emu_decision(400, 100, cap, 0, 10 ** 6, 113) == REBUILD
    # past that: rebuild while live + touches <= cap / 4, skip one past it
    assert L.room_emu_decision(450, 100, cap, 0, 10 ** 6, cap // 4 - 100) == REBUILD
    assert L.room_emu_decision(450, 100, cap, 0, 10 ** 6, cap // 4 - 100 + 1) == SKIP
    # the overflow pool: rows in use + touches <= pool, whatever the table says
    assert L.room_emu_decision(0, 0, cap, 90, 100, 10) == PROCEED
    assert L.room_emu_decision(0, 0, cap, 90, 100, 11) == SKIP
    assert L.room_emu_decision(450, 100, cap, 90, 100, 11) == SKIP


def _filled(L, M, lru, seed):
    """A reserved index of 256 slots whose dead slots outnumber a quarter of the table, and the oracle beside it."""
    rng = np.random.Generator(np.random.PCG64(seed))
    h = L.room_emu_new(M, 1 << 4, lru, 0, 32, 32, 4096)
    assert L.emu_stat(h, 2) == 256
    idx = o.Index(lru)
    while True:
        live, used = L.emu_stat(h, 0), L.emu_stat(h, 1)
        if used > 256 // 4 + live:
            return h, idx
        pick = np.array([int(rng.integers(0, M))], np.int32)
        hs = rng.integers(1, 2 ** 63, size=(1, 4), dtype=np.uint64)
        nh = np.array([4], np.uint16)
        assert _commit(L, h, pick, hs, nh) != SKIP
        idx.commit(pick, hs, nh)


@pytest.mark.parametrize("extra", [0, 1], ids=["at-cap/4-live", "one-past"])
def test_commit_at_the_skip_edge(L, extra):
    """touches = cap/4 - live rebuilds and commits; one more touch skips the call whole: the index is bit-identical, the skip
    is counted and the sticky error bit is set."""
    M, lru = 3, 6
    h, idx = _filled(L, M, lru, seed=11)
    live = L.emu_stat(h, 0)
    t = 256 // 4 - live + extra
    rng = np.random.Generator(np.random.PCG64(99))
    pick = np.array([1], np.int32)
    hs = rng.integers(1, 2 ** 63, size=(1, t), dtype=np.uint64)
    nh = np.array([t], np.uint16)
    before, rebuilds = L.room_emu_digest(h), L.room_emu_stat(h, 1)
    d = _commit(L, h, pick, hs, nh)
    if extra == 0:
        assert d == REBUILD and L.room_emu_stat(h, 1) == rebuilds + 1 and L.room_emu_stat(h, 0) == 0
        idx.commit(pick, hs, nh)
    else:
        assert d == SKIP
        assert L.room_emu_digest(h) == before
        assert L.room_emu_stat(h, 0) == 1 and L.room_emu_stat(h, 2) & ERR_SKIPPED
    _check(L, h, idx, M, hs[0])
    L.room_emu_free(h)


def test_skipped_apply_and_pool_edge(L):
    """Raw deltas are all or nothing too, and the overflow pool bounds the room: rows in use + touches <= pool."""
    M = 64
    h = L.room_emu_new(M, 1 << 4, 100, 0, 256, 256, 12)
    for ep in range(11):  # the eleventh member moves the set to a bitset row
        one = (np.full(1, 77, np.uint64), np.full(1, ep, np.int32), np.zeros(1, np.uint8))
        assert L.room_emu_apply(h, 1, *(a.ctypes.data for a in one)) == PROCEED
    assert L.emu_stat(h, 3) == 1  # one row in use: 11 more touches fit the pool of 12, 12 do not
    before = L.room_emu_digest(h)
    hs = np.arange(1000, 1012, dtype=np.uint64)
    ep = np.full(12, 5, np.int32)
    op = np.zeros(12, np.uint8)
    assert L.room_emu_apply(h, 12, hs.ctypes.data, ep.ctypes.data, op.ctypes.data) == SKIP
    assert L.room_emu_digest(h) == before and L.room_emu_stat(h, 2) & ERR_SKIPPED
    assert L.room_emu_apply(h, 11, hs.ctypes.data, ep.ctypes.data, op.ctypes.data) == PROCEED
    assert L.emu_stat(h, 0) == 12
    L.room_emu_free(h)
