"""The running-request queues of the predicted-latency producer at the headline shape (64K requests x 1024 endpoints): the
device time of eppscore_running_add and eppscore_running_remove (entries spread over every endpoint, and every entry on one
endpoint; with and without the snapshot terms prepared again behind them), of a remove where every removed entry was its
endpoint's minimum (the recompute pass runs), and of the closed-loop step schedule -> commit -> running_add (-> running_remove
two steps later) with a latency profile against the same step without the producer.  The queues are checked against the CPU
oracle.  Prints one JSON line with the GPU's name and power limit.  usage: prof_running.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests import running_oracle as Q  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
STEPS = 20
pkg = _pkg.load()
R, M, A = 65536, bench.M, bench.A
LAT = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5, ttft_prefix=-40.0,
           tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9, tpot_running=0.35, tpot_generated=0.01,
           streaming_mode=1)
SC_LAT = [("kv", 1.0), ("prefix", 1.0), ("latency", 2.0)]
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
del idx, prof, osnap
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream


def make_engine(scorers):
    e = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                      max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19))
    if ("latency", 2.0) in scorers:
        e.set_latency_params(pkg.latency_params(**LAT))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    e.running_reserve(4 * R)
    return e


def timed(calls, iters):
    """CUDA-event time of each of calls[i]() per iteration, eager launches on one stream (the calls restore the state)"""
    for c in calls:
        c()
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(len(calls) + 1)] for _ in range(iters)]
    for i in range(iters):
        for j, c in enumerate(calls):
            ev[i][j].record(stream)
            c()
        ev[i][-1].record(stream)
    torch.cuda.synchronize()
    return [float(np.median([ev[i][j].elapsed_time(ev[i][j + 1]) * 1e3 for i in range(iters)])) for j in range(len(calls))]


rng = np.random.Generator(np.random.PCG64(1))
keys = torch.from_numpy(np.arange(1, R + 1, dtype=np.uint64).view(np.int64)).to(dev)
tpot = torch.from_numpy(rng.choice([0.0, 18.0, 24.0, 30.0], R)).to(dev)
same_tpot = torch.full((R,), 24.0, dtype=torch.float64, device=dev)
spread = torch.from_numpy(rng.integers(0, M, R).astype(np.int32)).to(dev)
one = torch.full((R,), 17, dtype=torch.int32, device=dev)
arms, checks = {}, {}
for name, scorers in (("update", bench.SCORERS), ("update_and_prepare", SC_LAT)):
    e = make_engine(scorers)
    for dist, ep in (("spread", spread), ("one_endpoint", one)):
        add_us, rm_us = timed([lambda ep=ep, e=e: e.running_add(ep, keys, tpot, device=True, stream=sptr),
                               lambda ep=ep, e=e: e.running_remove(ep, keys, device=True, stream=sptr)], ITERS)
        arms[f"{name}_{dist}"] = {"running_add": add_us, "running_remove": rm_us}
        checks[f"{name}_{dist}_empty"] = bool((e.running_get(M)[1] == 0).all())
    # every removed entry is its endpoint's minimum: the last one of each endpoint's minimum class leaves, recompute runs
    add_us, rm_us = timed([lambda e=e: e.running_add(spread, keys, same_tpot, device=True, stream=sptr),
                           lambda e=e: e.running_remove(spread, keys, device=True, stream=sptr)], ITERS)
    arms[f"{name}_spread_all_minima"] = {"running_add": add_us, "running_remove": rm_us}
    e.running_add(spread, keys, tpot, device=True, stream=sptr)
    e.running_remove(spread[: R // 2], keys[: R // 2], device=True, stream=sptr)
    q = Q.Queues(M)
    q.add(spread.cpu().numpy(), keys.cpu().numpy().view(np.uint64), tpot.cpu().numpy())
    q.remove(spread[: R // 2].cpu().numpy(), keys[: R // 2].cpu().numpy().view(np.uint64))
    (gm, gc), (wm, wc) = e.running_get(M), q.get(M)
    checks[f"{name}_vs_oracle"] = bool(np.array_equal(gc, wc) and np.array_equal(gm, Q.canonical(wm)))
    checks[f"{name}_capacity_entries"] = e.running_reserve(0)
    e.close()

# ---- closed-loop step ----
sets = []
for i in range(3):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100 + i, prefix_seed=7)
    sets.append(dict(prompt_bytes=torch.from_numpy(p).to(dev), prompt_off=torch.from_numpy(off).to(dev),
                     model_seed=torch.from_numpy(np.full(R, seed, np.uint64).view(np.int64)).to(dev),
                     input_tokens=torch.from_numpy(rng.integers(0, 6000, R).astype(np.int32)).to(dev),
                     ttft_slo=torch.from_numpy(rng.choice([0.0, 140.0, 400.0], R)).to(dev),
                     tpot_slo=torch.from_numpy(rng.choice([0.0, 18.0, 24.0, 30.0], R)).to(dev)))
producer_us = []


def closed_loop(producer):
    e = make_engine(SC_LAT)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, bench.MAX_BLOCKS), dtype=torch.int64, device=dev))
    picks = [torch.empty(R, dtype=torch.int32, device=dev) for _ in range(STEPS + 3)]
    kk = [keys + k * R for k in range(STEPS + 3)]
    marks = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS + 3)]
    phase = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(STEPS + 3)]

    def step(k):
        d = sets[k % 3]
        phase[k][0].record(stream)
        e.schedule(R, device=True, stream=sptr, out=out, **d)
        phase[k][1].record(stream)
        e.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], touch_bound=R * 32, stream=sptr)
        picks[k].copy_(out["pick"])
        phase[k][2].record(stream)
        if producer:
            marks[k][0].record(stream)
            e.running_add(picks[k], kk[k], d["tpot_slo"], device=True, stream=sptr)
            if k >= 2:
                e.running_remove(picks[k - 2], kk[k - 2], device=True, stream=sptr)
            marks[k][1].record(stream)

    for k in range(3):
        step(k)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for k in range(3, STEPS + 3):
        step(k)
    b.record(stream)
    torch.cuda.synchronize()
    us = a.elapsed_time(b) / STEPS * 1e3
    phases.append({"schedule": sum(phase[k][0].elapsed_time(phase[k][1]) for k in range(3, STEPS + 3)) / STEPS * 1e3,
                   "commit": sum(phase[k][1].elapsed_time(phase[k][2]) for k in range(3, STEPS + 3)) / STEPS * 1e3,
                   "distinct_endpoints_last_batch": int(torch.unique(out["pick"]).numel())})
    ok = None
    if producer:
        producer_us.append(sum(marks[k][0].elapsed_time(marks[k][1]) for k in range(3, STEPS + 3)) / STEPS * 1e3)
        q = Q.Queues(M)
        for k in range(STEPS + 3):
            q.add(picks[k].cpu().numpy(), kk[k].cpu().numpy().view(np.uint64), sets[k % 3]["tpot_slo"].cpu().numpy())
            if k >= 2:
                q.remove(picks[k - 2].cpu().numpy(), kk[k - 2].cpu().numpy().view(np.uint64))
        (gm, gc), (wm, wc) = e.running_get(M), q.get(M)
        ok = bool(np.array_equal(gc, wc) and np.array_equal(gm, Q.canonical(wm)))
    e.close()
    return us, ok


phases = []
step_base, _ = closed_loop(False)
step_prod, ok_loop = closed_loop(True)
step_base2, _ = closed_loop(False)
checks["closed_loop_vs_oracle"] = ok_loop
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "running_queues", "R": R, "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "running_us": arms,
                  "closed_loop_step_us": {"without_producer": [step_base, step_base2], "with_producer": step_prod,
                                          "of_which_add_remove": producer_us[0],
                                          "phases_without_with_without": phases},
                  "checks": checks,
                  "note": "running_us: median CUDA-event time of one eppscore_running_add / _remove of 64K device entries, eager "
                          "launches; update: profile without the latency scorer (the queue kernels alone); update_and_prepare: "
                          "latency profile, so the snapshot terms are prepared again behind every call; spread_all_minima: one "
                          "tpot class, so every remove takes each endpoint's last minimum and the recompute pass runs. "
                          "closed_loop_step_us: schedule -> commit_picks_device -> [running_add -> running_remove of step k-2], "
                          "kv + prefix + latency profile, CUDA events over 20 steps; the run without the producer is timed before "
                          "and after the one with it"}))
