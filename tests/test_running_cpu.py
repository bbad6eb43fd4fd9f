"""The predicted-latency producer's running-request queues on the CPU: the oracle (tests/cpp/running_oracle.c) against the
reference's own test cases (tests/golden/running_queue_vectors.json), a tpot-0 entry turning the TPOT tightening off, the
host layer's TrackRunningRequests on the oracle-backed stand-in of the C ABI, and the gathered update stream of two gloo
ranks."""
import json
import os
import subprocess

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _pkg
from oracle import oracle_py as o
from tests import running_oracle as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")


def golden():
    with open(os.path.join(ROOT, "tests", "golden", "running_queue_vectors.json")) as f:
        return json.load(f)


def run_case(case, add, remove, view):
    """Drives one golden case through add(ep, key, tpot) -> bool, remove(ep, key) -> bool, view() -> (min, count)."""
    ids = Q.KeyMap()
    for op in Q.expand_case(case, ids):
        if op[0] == "add":
            assert add(op[1], op[2], op[3]) == op[4], (case["name"], op)
        elif op[0] == "remove":
            assert remove(op[1], op[2]) == op[3], (case["name"], op)
        else:
            mn, cnt = view()
            assert mn[op[1]] == op[2] and cnt[op[1]] == op[3], (case["name"], op, mn[op[1]], cnt[op[1]])


def test_oracle_matches_reference_cases():
    g = golden()
    assert len(g["cases"]) == 9
    for case in g["cases"]:
        q = Q.Queues(4)
        run_case(case, lambda m, k, t: bool(q.add([m], [k], [t])[0]), lambda m, k: bool(q.remove([m], [k])[0]), lambda: q.get(4))


def test_in_call_order_and_edge_values():
    q = Q.Queues(3)
    ep = np.array([0, 0, 0, 1, -1, 0, 2, 2], np.int32)
    key = np.array([7, 7, 0, 7, 9, 8, 5, 6], np.uint64)
    tpot = np.array([30.0, 10.0, 1.0, 20.0, 1.0, np.inf, -0.0, -1.0])
    # the first add of (0, 7) wins, key 0 and tpot < 0 are refused, -1 is skipped, the same key lives on endpoint 1 as well
    assert q.add(ep, key, tpot).tolist() == [True, False, False, True, False, True, True, False]
    mn, cnt = q.get()
    assert mn.tolist() == [30.0, 20.0, 0.0] and cnt.tolist() == [2, 1, 1]
    assert np.signbit(mn[2]) and Q.canonical(mn)[2] == 0.0 and not np.signbit(Q.canonical(mn)[2])
    assert q.remove([0, 0, 1], [7, 7, 8]).tolist() == [True, False, False]  # the second remove finds nothing
    mn, cnt = q.get()
    assert mn[0] == np.inf and cnt[0] == 1
    q.remove_endpoint(0)
    assert q.get()[1].tolist() == [0, 1, 1] and q.add([0], [7], [3.0]).tolist() == [True]


def test_zero_tpot_entry_turns_tightening_off():
    """A request without x-slo-tpot-ms is added with tpot 0 (requestcontrol_hooks.go:73-86): it becomes its endpoint's
    minimum, and validatePrediction only tightens bufferedTPOT when podMinTPOTSLO > 0 (prediction.go:152)."""
    q = Q.Queues(2)
    q.add([0, 0, 1], [1, 2, 3], [20.0, 0.0, 20.0])
    mn, cnt = q.get()
    assert mn.tolist() == [0.0, 20.0] and cnt.tolist() == [2, 1]
    lp = o.make_latency_params(streaming_mode=1)
    # TPOT 25 against an SLO of 30: valid unless the endpoint's minimum (20) tightens the buffered limit below 25
    loose = o.latency_validate(lp, 10.0, 25.0, 1000.0, 30.0, mn[0])
    tight = o.latency_validate(lp, 10.0, 25.0, 1000.0, 30.0, mn[1])
    assert loose["tpot_ok"] and not tight["tpot_ok"]
    assert loose == o.latency_validate(lp, 10.0, 25.0, 1000.0, 30.0, 0.0)


def build_host_running_test():
    o.build()
    lib = Q.build()
    exe = os.path.join(BUILD, "host_running_test_cpu")
    srcs = [os.path.join(CPP, "host_running_test.cpp"), os.path.join(CPP, "oracle_backed_abi.cpp"),
            os.path.join(CPP, "oracle_backed_running.cpp")]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-lrunning_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def test_host_track_running_requests_on_the_oracle_backed_abi():
    """the host layer with TrackRunningRequests against the same layer fed through State by the queue oracle"""
    exe = build_host_running_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host running: all checks passed" in r.stdout


M_EP, R_SHARD, K = 64, 500, 6


def _batches(world):
    """Per round: (endpoint, key, tpot) adds with keys repeating inside the round and across shards' rounds' removes."""
    rng = np.random.Generator(np.random.PCG64(7))
    out = []
    for k in range(K):
        n = world * R_SHARD
        ep = rng.integers(-1, M_EP, n).astype(np.int32)
        ep[: n // 4] = 3                                    # dog-piling on one endpoint
        key = rng.integers(1, 3 * n, n).astype(np.uint64)    # repeats: the first in global order wins
        key[rng.random(n) < 0.02] = 0
        tpot = rng.choice([0.0, 15.0, 22.0, 40.0], n)
        out.append((ep, key, tpot))
    return out


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import importlib.util
    spec = importlib.util.spec_from_file_location("sharding", os.path.join(_pkg.PKG_DIR, "sharding.py"))
    sharding = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sharding)
    mine = Q.Queues(M_EP)                     # this rank's replica (the oracle stands in for the engine's queues)
    ref = Q.Queues(M_EP) if rank == 0 else None
    batches = _batches(world)
    n = world * R_SHARD
    lo, hi = rank * R_SHARD, (rank + 1) * R_SHARD
    g_ep, g_key, g_t = torch.empty(n, dtype=torch.int32), torch.empty(n, dtype=torch.int64), torch.empty(n, dtype=torch.float64)
    for k, (ep, key, tpot) in enumerate(batches):
        sharding.gather_running_stream(dist, torch.from_numpy(ep[lo:hi]), torch.from_numpy(key[lo:hi].view(np.int64)), g_ep, g_key,
                                       torch.from_numpy(tpot[lo:hi]), g_t)
        mine.add(g_ep.numpy(), g_key.numpy().view(np.uint64), g_t.numpy())
        if k >= 2:                             # round k-2 completes
            pep, pkey, _ = batches[k - 2]
            sharding.gather_running_stream(dist, torch.from_numpy(pep[lo:hi]), torch.from_numpy(pkey[lo:hi].view(np.int64)), g_ep, g_key)
            mine.remove(g_ep.numpy(), g_key.numpy().view(np.uint64))
        if rank == 0:
            ref.add(ep, key, tpot)
            if k >= 2:
                ref.remove(batches[k - 2][0], batches[k - 2][1])
    mn, cnt = mine.get()
    got = torch.from_numpy(np.concatenate([mn, cnt.astype(np.float64)]))
    allc = [torch.empty_like(got) for _ in range(world)]
    dist.all_gather(allc, got)
    if rank == 0:
        wm, wc = ref.get()
        want = np.concatenate([wm, wc.astype(np.float64)])
        q.put((all(np.array_equal(c.numpy().view(np.uint64), want.view(np.uint64)) for c in allc), int(wc[3]), int(wc.sum())))
    dist.destroy_process_group()


def test_two_rank_gathered_updates_equal_one_process():
    port = 37500 + os.getpid() % 2000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    same, on_3, total = q.get(timeout=5)
    assert same and on_3 > 0 and total > 0
