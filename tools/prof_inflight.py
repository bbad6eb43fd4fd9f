"""The in-flight load producer at the headline shape (64K requests x 1024 endpoints): the device time of
eppscore_inflight_add (picks spread over every endpoint, and every pick on one endpoint; with and without the snapshot terms
prepared again behind it), and of the closed-loop step schedule -> commit -> estimate -> add (-> release two steps later) with
a token-load profile against the same step without the producer.  The counters are checked against the CPU oracle's tracker.
Prints one JSON line with the GPU's name and power limit.  usage: prof_inflight.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests import inflight_oracle as I  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
STEPS = 20
pkg = _pkg.load()
R, M, A = 65536, bench.M, bench.A
THR = 200000.0  # about two steps of this workload's tokens per endpoint: the load term matters
SC_TL = bench.SCORERS + [("token_load", 2.0)]
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
del idx
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream


def make_engine(scorers):
    e = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                      max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19, token_load_threshold=THR))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    return e


def events_us(fn, iters):
    """CUDA-event time per call of fn() (an add followed by the matching release, captured into one CUDA graph) / 2"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    for _ in range(3):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(stream)
    for _ in range(iters):
        g.replay()
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3 / 2


rng = np.random.Generator(np.random.PCG64(1))
tokens = torch.from_numpy(rng.integers(100, 5000, R).astype(np.int64)).to(dev)
spread = torch.from_numpy(rng.integers(0, M, R).astype(np.int32)).to(dev)
one = torch.full((R,), 17, dtype=torch.int32, device=dev)
arms, checks = {}, {}
for name, scorers in (("update", bench.SCORERS), ("update_and_prepare", SC_TL)):
    e = make_engine(scorers)
    for dist, ep in (("spread", spread), ("one_endpoint", one)):
        def pair(ep=ep, e=e):
            e.inflight_add(ep, tokens, device=True, stream=sptr)
            e.inflight_release(ep, tokens, device=True, stream=sptr)
        arms[f"{name}_{dist}"] = events_us(pair, ITERS)
        req, tok = e.inflight_get(M)
        checks[f"{name}_{dist}_balanced"] = bool((req == 0).all() and (tok == 0).all())
    e.inflight_add(spread, tokens, device=True, stream=sptr)
    e.inflight_add(one, tokens, device=True, stream=sptr)
    t = I.Tracker()
    t.add(spread.cpu().numpy(), tokens.cpu().numpy())
    t.add(one.cpu().numpy(), tokens.cpu().numpy())
    got, want = e.inflight_get(M), t.get(M)
    checks[f"{name}_vs_oracle"] = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]))
    e.close()

# ---- closed-loop step ----
sets = []
for i in range(3):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100 + i, prefix_seed=7)
    sets.append(dict(prompt_bytes=torch.from_numpy(p).to(dev), prompt_off=torch.from_numpy(off).to(dev),
                     model_seed=torch.from_numpy(np.full(R, seed, np.uint64).view(np.int64)).to(dev),
                     adapter_id=torch.from_numpy(zipf_adapters(R, A=A, seed=100 + i)).to(dev),
                     chars=torch.from_numpy(np.diff(off).astype(np.int32)).to(dev)))


def closed_loop(producer):
    e = make_engine(SC_TL)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, bench.MAX_BLOCKS), dtype=torch.int64, device=dev))
    picks = [torch.empty(R, dtype=torch.int32, device=dev) for _ in range(STEPS + 3)]
    ests = [torch.empty(R, dtype=torch.int64, device=dev) for _ in range(STEPS + 3)]

    marks = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS + 3)]

    def step(k):
        d = sets[k % 3]
        e.schedule(R, prompt_bytes=d["prompt_bytes"], prompt_off=d["prompt_off"], model_seed=d["model_seed"],
                   adapter_id=d["adapter_id"], device=True, stream=sptr, out=out)
        e.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], touch_bound=R * 32, stream=sptr)
        picks[k].copy_(out["pick"])
        if producer:
            marks[k][0].record(stream)
            e.estimate_tokens(R, prompt_chars=d["chars"], device=True, stream=sptr, out=ests[k])
            e.inflight_add(picks[k], ests[k], device=True, stream=sptr)
            if k >= 2:
                e.inflight_release(picks[k - 2], ests[k - 2], device=True, stream=sptr)
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
    if producer:  # the producer's share of the step: estimate + add + release, between events on the same stream
        producer_us.append(sum(marks[k][0].elapsed_time(marks[k][1]) for k in range(3, STEPS + 3)) / STEPS * 1e3)
    ok, distinct = None, int(torch.unique(out["pick"]).numel())
    if producer:  # the counters against the oracle's tracker fed with the same picks and its own estimates
        t, est_prev = I.Tracker(), {}
        for k in range(STEPS + 3):
            est = I.estimate(None, None, sets[k % 3]["chars"].cpu().numpy())
            ok = bool(np.array_equal(ests[k].cpu().numpy(), est)) if ok is None else ok and bool(np.array_equal(ests[k].cpu().numpy(), est))
            t.add(picks[k].cpu().numpy(), est)
            if k >= 2:
                t.release(picks[k - 2].cpu().numpy(), est_prev[k - 2])
            est_prev[k] = est
        got, want = e.inflight_get(M), t.get(M)
        ok = ok and bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]))
    e.close()
    return us, ok, distinct


producer_us = []
step_base, _, distinct_base = closed_loop(False)
step_prod, ok_loop, distinct_prod = closed_loop(True)
step_base2, _, _ = closed_loop(False)
checks["closed_loop_vs_oracle"] = ok_loop
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inflight_load", "R": R, "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "inflight_add_us": arms,
                  "closed_loop_step_us": {"without_producer": [step_base, step_base2], "with_producer": step_prod,
                                          "of_which_estimate_add_release": producer_us[0]},
                  "distinct_endpoints_last_batch": {"without_producer": distinct_base, "with_producer": distinct_prod},
                  "checks": checks,
                  "note": "inflight_add_us: one eppscore_inflight_add of 64K device entries (a CUDA graph of add + release, halved); "
                          "update: profile without token-load (the update kernel alone); update_and_prepare: token-load profile, "
                          "so the snapshot terms are prepared again behind every update. closed_loop_step_us: schedule -> "
                          "commit_picks_device -> [estimate -> add -> release of step k-2], token-load profile, eager launches, "
                          "CUDA events over 20 steps; the run without the producer is timed before and after the one with it. The step is "
                          "dominated by the commit, whose cost depends on how the picks spread over the endpoints (one CTA per "
                          "endpoint), and the producer changes that spread"}))
