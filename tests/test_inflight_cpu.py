"""The inflight-load-producer on the CPU: the oracle (tests/cpp/inflight_oracle.c) against the reference's own test cases
(tests/golden/inflight_vectors.json), the engine's integer form of the estimator against the oracle's float form, the host
layer's InFlightLoadProducer on the oracle-backed stand-in of the C ABI, and the gathered update stream of two gloo ranks."""
import json
import os
import subprocess

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")


def golden():
    with open(os.path.join(ROOT, "tests", "golden", "inflight_vectors.json")) as f:
        return json.load(f)


def integer_estimate(size, hint, chars):
    """the engine's form (csrc/inflight_kernel.cu): (c + 2) >> 2 and (3i + 1) >> 1 for Go's half-away-from-zero rounds"""
    if size > 0:
        i = max(size // 4, 1)
    elif chars < 0:
        return 0
    elif hint >= 0:
        i = hint
    else:
        i = max((chars + 2) >> 2, 1)
    return i + ((3 * i + 1) >> 1)


def test_estimator_matches_reference_cases():
    for c in golden()["estimator"]:
        if "prompt_text" in c:
            assert len(c["prompt_text"]) == c["chars"], c["name"]
        got = int(I.estimate([c["size"]], [c["hint"]], [c["chars"]])[0])
        assert got == c["want"], (c["name"], got)
        assert integer_estimate(c["size"], c["hint"], c["chars"]) == c["want"], c["name"]


def test_integer_estimator_equals_float_form_at_rounding_boundaries():
    """chars = 0..4099 (every residue mod 4, c = 2 mod 4 is the half-way case), odd and even hints incl. 0, sizes 1..9 and
    large ones, body absent; plus random inputs"""
    rng = np.random.Generator(np.random.PCG64(7))
    cases = [(0, -1, c) for c in range(4100)]
    cases += [(0, h, c) for h in list(range(0, 64)) + [999, 1001, 2 ** 31 - 1] for c in (0, 2, 6, -1)]
    cases += [(s, -1, c) for s in list(range(1, 10)) + [2 ** 40 + 3, 2 ** 50 - 1] for c in (-1, 0, 7)]
    cases += [(0, -1, -1), (-5, 3, 10), (-5, -1, -1)]
    n = 3000
    size = np.where(rng.random(n) < 0.3, rng.integers(-10, 1 << 40, n), 0)
    hint = np.where(rng.random(n) < 0.3, rng.integers(0, 1 << 20, n), -1)
    cases += list(zip(size.tolist(), hint.tolist(), rng.integers(-1, 1 << 30, n).tolist()))
    s, h, c = (np.array(x) for x in zip(*cases))
    got = I.estimate(s, h, c)
    want = np.array([integer_estimate(*x) for x in cases], np.int64)
    assert np.array_equal(got, want)
    assert got[2] == 3 and got[6] == 5 and got[10] == 8  # c = 2, 6, 10: round(0.5) = 1, round(1.5) = 2, round(2.5) = 3


def apply_step(t, st, est):
    ep = [st["endpoint"]] * st.get("n", 1)
    if st["op"] == "remove":
        t.remove(st["endpoint"])
        return
    tok = [st["tokens"] if "tokens" in st else int(est(st["chars"]))] * len(ep)
    (t.add if st["op"] == "add" else t.release)(ep, tok)


def test_lifecycle_matches_reference_cases():
    for case in golden()["lifecycle"]:
        t = I.Tracker()
        n = len(case["endpoints"])
        for i, st in enumerate(case["steps"]):
            apply_step(t, st, lambda c: I.estimate([0], [-1], [c])[0])
            req, tok = t.get(n)
            assert req.tolist() == st["want_requests"] and tok.tolist() == st["want_tokens"], (case["name"], i)


def test_release_after_remove_goes_negative():
    """concurrencyTracker.add on a deleted key recreates the counter holding the delta (producer.go:226-236)"""
    t = I.Tracker()
    t.add([3, 3], [10, 20])
    t.remove(3)
    t.release([3], [10])
    req, tok = t.get(5)
    assert req.tolist() == [0, 0, 0, -1, 0] and tok.tolist() == [0, 0, 0, -10, 0]
    t.add([-1, 4], [99, 5])  # -1: no target endpoint
    assert t.get(5)[1].tolist() == [0, 0, 0, -10, 5]


def build_host_inflight_test():
    o.build()
    lib = I.build()
    exe = os.path.join(BUILD, "host_inflight_test_cpu")
    srcs = [os.path.join(CPP, "host_inflight_test.cpp"), os.path.join(CPP, "oracle_backed_abi.cpp"),
            os.path.join(CPP, "oracle_backed_inflight.cpp")]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-linflight_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def test_host_producer_on_the_oracle_backed_abi():
    exe = build_host_inflight_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host inflight: all checks passed" in r.stdout


M_EP, R_SHARD, K = 37, 500, 3


def _batches(world):
    """the same global batches on every rank: picks (some -1) and estimates"""
    rng = np.random.Generator(np.random.PCG64(11))
    out = []
    for _ in range(K):
        pick = rng.integers(-1, M_EP, world * R_SHARD).astype(np.int32)
        pick[: world * R_SHARD // 3] = 5  # dog-piling on one endpoint
        est = I.estimate(None, None, rng.integers(0, 5000, world * R_SHARD).astype(np.int32))
        out.append((pick, est))
    return out


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import importlib.util
    spec = importlib.util.spec_from_file_location("sharding", os.path.join(_pkg.PKG_DIR, "sharding.py"))
    sharding = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sharding)
    t = I.Tracker()               # this rank's replica (the oracle stands in for the engine's counters)
    ref = I.Tracker() if rank == 0 else None
    rng = np.random.Generator(np.random.PCG64(100 + rank))
    batches = _batches(world)
    for k, (pick, est) in enumerate(batches):
        lo, hi = rank * R_SHARD, (rank + 1) * R_SHARD
        g_ep = torch.empty(world * R_SHARD, dtype=torch.int32)
        g_tok = torch.empty(world * R_SHARD, dtype=torch.int64)
        sharding.gather_inflight_stream(dist, torch.from_numpy(pick[lo:hi]), torch.from_numpy(est[lo:hi]), g_ep, g_tok)
        perm = rng.permutation(world * R_SHARD)  # the order of the gathered stream does not matter
        t.add(g_ep.numpy()[perm], g_tok.numpy()[perm])
        if k >= 1:                               # batch k-1 completes: its shards release what they added
            ppick, pest = batches[k - 1]
            sharding.gather_inflight_stream(dist, torch.from_numpy(ppick[lo:hi]), torch.from_numpy(pest[lo:hi]), g_ep, g_tok)
            t.release(g_ep.numpy(), g_tok.numpy())
        if rank == 0:
            ref.add(pick, est)
            if k >= 1:
                ref.release(*batches[k - 1])
    mine = torch.from_numpy(np.concatenate(t.get(M_EP)))
    allc = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allc, mine)
    if rank == 0:
        want = np.concatenate(ref.get(M_EP))
        q.put((all(np.array_equal(c.numpy(), want) for c in allc), int(want[5]), int(want[:M_EP].sum())))
    dist.destroy_process_group()


def test_two_rank_gathered_updates_equal_one_process():
    port = 35500 + os.getpid() % 2000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    same, on_5, total = q.get(timeout=5)
    pick_last = _batches(2)[-1][0]
    assert same and total == int((pick_last >= 0).sum()) and on_5 >= 2 * R_SHARD // 3
