"""LoRA affinity past one 64-adapter word, on the CPU.

  - The oracle's lora-affinity scorer against a plain NumPy restatement of lora_affinity.go:84-99 that reads boolean
    active / waiting matrices (no bitmasks), at 1, 2, 3 and 16 words, for adapter ids on both sides of every word edge, past
    the dictionary and at 2^31 - 1, with endpoints in all four classes for each id.
  - Sensitivity: in the snapshots of wide_lora(), adapters a and a ^ 64 are in different classes on every endpoint, so a
    reading of word 0 only (id & 63) changes the expected output; tests/test_gpu_lora_width.py uses the same snapshots.
  - The host layer (tests/cpp/host_lora_width_test.cpp) on fleets with more adapter names than MaxAdapters, on the
    oracle-backed stand-in of the C ABI."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_py as o
from tests import topk_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")

LORA_WEIGHT = 2.5


def edge_ids(W, a_cap=None):
    """Adapter ids at every edge that matters for W words: -1, both sides of words 0/1/2, the last id, the first id past the
    dictionary, 2^31 - 1, and (given the engine's capacity) A_cap - 1 and A_cap."""
    ids = [-1, 0, 63, 64, 65, 127, 128, 64 * W - 1, 64 * W, 2 ** 31 - 1]
    if a_cap is not None:
        ids += [a_cap - 1, a_cap]
    return list(dict.fromkeys(ids))


def _alt(cls, cap):
    """another class the endpoint can have for an adapter: {2, 3} with room for one more adapter, {0, 1, 3} without"""
    return np.where(cap, 5 - cls, np.select([cls == 0, cls == 1], [1, 3], 0))


def wide_lora(M, W, seed, focus=(), tie_heavy=False):
    """A snapshot with W LoRA words (A = 64 W adapters) in which adapters a and a ^ 64 have different classes on every
    endpoint, and every id of `focus` below A has endpoints in each of the four classes (as far as M allows).
    Returns (snapshot kwargs for the engine and the oracle, dict of the boolean active / waiting [M, A] and class [M, A])."""
    rng = np.random.Generator(np.random.PCG64(seed))
    A = 64 * W
    cap = rng.random(M) < 0.25                 # room for one more adapter: class 2 unless active
    cls = np.where(cap[:, None], 2 + (rng.random((M, A)) < 0.15), rng.choice([0, 0, 0, 1, 3], size=(M, A)))
    lo = np.array([a for a in range(A) if not a & 64 and a | 64 < A], np.int64)
    if lo.size:
        hi = lo | 64
        same = cls[:, lo] == cls[:, hi]
        cls[:, hi] = np.where(same, _alt(cls[:, hi], cap[:, None]), cls[:, hi])
    # every focus id in every class, one focus cell per (endpoint, adapter pair)
    taken = np.zeros((M, max(A, 1)), bool)
    order = rng.permutation(M)
    k = 0
    for a in focus:
        if not 0 <= a < A:
            continue
        for c in (0, 1, 2, 3):
            for _ in range(M):
                e = int(order[k % M])
                k += 1
                p = a ^ 64
                ok = (c == 3 or cap[e] == (c == 2)) and not taken[e, a] and not (p < A and taken[e, p])
                if ok:
                    cls[e, a] = c
                    taken[e, a] = True
                    if p < A:
                        cls[e, p] = _alt(np.array(c), cap[e])
                    break
    active = cls == 3
    waiting = (cls == 1) | ((cls >= 2) & (rng.random((M, A)) < 0.2))
    extra = rng.integers(0, 3, M)
    nmodels = (active.sum(axis=1) + waiting.sum(axis=1) + extra).astype(np.int32)
    lmax = np.where(cap, nmodels + 1 + rng.integers(0, 3, M), np.maximum(nmodels - rng.integers(0, 3, M), 0)).astype(np.int32)
    kv = rng.random(M)
    kv = np.round(kv, 1) if tie_heavy else kv
    sd = dict(kv_usage=kv, queue=np.clip(rng.poisson(8, M), 0, 255).astype(np.int64), running=rng.poisson(16, M).astype(np.int64),
              lora_active=pack_bits(active, W), lora_waiting=pack_bits(waiting, W), lora_nmodels=nmodels, lora_max=lmax)
    return sd, dict(active=active, waiting=waiting, cls=cls, nmodels=nmodels, max=lmax)


def pack_bits(bits, W):
    """bool [M, 64 W] -> uint64 [M, W]: bit a of word a >> 6 (a & 63)"""
    M = bits.shape[0]
    if W == 0:
        return np.zeros((M, 0), np.uint64)
    return np.packbits(bits.reshape(M, W * 64), axis=1, bitorder="little").view("<u8").reshape(M, W).astype(np.uint64)


def lora_scores(truth, ids, word0_only=False):
    """lora_affinity.go:84-99 from the boolean matrices: [R, M] scores.  word0_only: the misreading that takes id & 63."""
    active, waiting = truth["active"], truth["waiting"]
    A = active.shape[1]
    room = truth["nmodels"] < truth["max"]
    out = np.zeros((len(ids), active.shape[0]))
    for r, a in enumerate(ids):
        col = (a & 63) if word0_only and a >= 0 else a
        known = 0 <= col < A
        act = active[:, col] if known else np.zeros(active.shape[0], bool)
        wait = waiting[:, col] if known else np.zeros(active.shape[0], bool)
        out[r] = np.where(act, 1.0, np.where(room, 0.8, np.where(wait, 0.6, 0.0)))
    return out


def weighted(scores):
    return 0.0 + LORA_WEIGHT * scores   # scheduler_profile.go:151-174: from 0.0, multiply then add


@pytest.mark.parametrize("W", [1, 2, 3, 16])
def test_oracle_lora_past_word_zero(W):
    M = 160
    ids = edge_ids(W)
    sd, truth = wide_lora(M, W, seed=W, focus=ids)
    A = 64 * W
    for a in ids:
        if 0 <= a < A:
            assert set(np.unique(truth["cls"][:, a])) == {0, 1, 2, 3}, a
    rng = np.random.Generator(np.random.PCG64(W + 50))
    req = np.array(ids * 3 + list(rng.integers(-1, A + 2, 77)), np.int32)
    R = len(req)
    snap = o.SnapshotData(**sd)
    prof = o.make_profile([(o.SCORER_LORA, LORA_WEIGHT)])
    got = o.schedule_batch(snap, prof, None, R, adapter_id=req, want_scores=True)
    want = weighted(lora_scores(truth, req))
    assert np.array_equal(got["weighted_out"].view(np.uint64), want.view(np.uint64))
    best = want.max(axis=1)
    assert np.array_equal(got["pick_score"], best)
    assert np.array_equal(got["pick"], np.argmax(want == best[:, None], axis=1))
    assert np.array_equal(got["tie_count"], (want == best[:, None]).sum(axis=1))
    # every class is reached by an id past word 0 (when there is one)
    if W > 1:
        past = want[(req >= 64) & (req < A)]
        assert set(np.unique(past)) == {0.0, LORA_WEIGHT * 0.6, LORA_WEIGHT * 0.8, LORA_WEIGHT * 1.0}


@pytest.mark.parametrize("W", [2, 3, 16])
def test_word_zero_reading_changes_the_answer(W):
    """On every endpoint a and a ^ 64 differ in class, so reading id & 63 moves every score of an id in [64, 128) on the
    endpoints without room for another adapter (where the class is not the capacity rule's), and moves picks."""
    M = 97
    A = 64 * W
    sd, truth = wide_lora(M, W, seed=100 + W, focus=edge_ids(W))
    lo = np.array([a for a in range(A) if not a & 64 and a | 64 < A])
    assert (truth["cls"][:, lo] != truth["cls"][:, lo | 64]).all()
    snap = o.SnapshotData(**sd)
    prof = o.make_profile([(o.SCORER_LORA, LORA_WEIGHT)])
    full = truth["nmodels"] >= truth["max"]
    second = np.arange(64, 128, dtype=np.int32)
    got = o.schedule_batch(snap, prof, None, len(second), adapter_id=second, want_scores=True)
    misread = weighted(lora_scores(truth, second, word0_only=True))
    assert (got["weighted_out"][:, full] != misread[:, full]).all()
    req = np.array([a for a in edge_ids(W) if 64 <= a < A] + list(range(64, A, 7)), np.int32)
    got = o.schedule_batch(snap, prof, None, len(req), adapter_id=req, want_scores=True)
    misread = weighted(lora_scores(truth, req, word0_only=True))
    assert (got["pick"] != np.argmax(misread == misread.max(axis=1)[:, None], axis=1)).mean() > 0.25


def _build_host_program():
    o.build()
    topk_lib = T.build()
    exe = os.path.join(BUILD, "host_lora_width_test")
    srcs = [os.path.join(CPP, "host_lora_width_test.cpp"), os.path.join(CPP, "oracle_backed_profiles_topk.cpp"),
            os.path.join(CPP, "oracle_backed_topk_wide.cpp")]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h")] + \
        [os.path.join(CPP, f) for f in ("oracle_backed_abi.cpp", "oracle_backed_profiles.cpp", "oracle_backed_topk.cpp")] + [topk_lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-ltopk_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def check_host_program_output(r):
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr
    lines = r.stdout.splitlines()
    assert lines[-1] == "host lora width: all checks passed"
    scen = [line for line in lines if line.startswith("scenario ")]
    assert scen and all(line.endswith(" ok") for line in scen)
    for want in ("two_profiles fleet=1000 max_adapters=64", "weighted_random fleet=200 max_adapters=100", "top12 fleet=65",
                 "max_score_seeded fleet=1000", "max_score_lowest fleet=65 max_adapters=64 threshold=8 targets=65 R=157",
                 "prerequest fleet=1000"):
        assert any(want in line for line in scen), want


def test_host_layer_fleets_past_max_adapters():
    """A fleet with more adapter names than MaxAdapters schedules (it used to fail every engine batch with ERR_CAPACITY), and a
    batch with more distinct targets than the engine holds returns what an unsplit batch returns."""
    exe = _build_host_program()
    check_host_program_output(subprocess.run([exe], capture_output=True, text=True, timeout=600))
