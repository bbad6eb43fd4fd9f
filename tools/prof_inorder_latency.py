"""The in-order batch with the latency scorer ordered against the running-request queues
(eppscore_schedule_batch_inorder_latency) at 1024 endpoints, a latency + token-load profile (plus the prefix scorer in the
index form), 2 KB prompts: device time per request of one graph-replayed call at R = 4K and 64K, against
  loop            the R-call loop it replaces: per request eppscore_schedule_batch (R = 1) + eppscore_running_add +
                  eppscore_inflight_add (+ eppscore_commit_picks_device in the index form); captured at R = 4K only
  no_latency      eppscore_schedule_batch_inorder(_index) on the same profile without the latency scorer
and, in an all-negative world (every TTFT SLO below every prediction, k endpoints idle), the distinct endpoints among the
first k picks and the busiest endpoint's picks, batch-wide against in order.  Prints one JSON line with the GPU's name and
power limit.
usage: prof_inorder_latency.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
pkg = _pkg.load()
M, NB, THR = 1024, 32, 200000.0
LAT = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5, ttft_prefix=-40.0,
           tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9, tpot_running=0.35, tpot_generated=0.01,
           streaming_mode=1)
snap = synth_snapshot(M, seed=0)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream


def scorers(index, latency):
    return ([("kv", 1.0)] + ([("prefix", 3.0)] if index else []) + ([("latency", 2.0)] if latency else []) +
            [("token_load", 1.0)])


def engine(R, index, latency):
    e = pkg.Engine(pkg.default_config(scorers(index, latency), max_endpoints=M, max_blocks=NB, prefix_capacity=1 << 19,
                                      token_load_threshold=THR))
    e.set_latency_params(pkg.latency_params(**LAT))
    e.set_snapshot(**snap)
    e.running_reserve(8 * R + 4096)  # every replay adds R fresh entries
    if index:
        e.prefix_reserve(live_hashes=1 << 22, touches_per_call=R * NB, overflow_rows=R * NB + (1 << 18))
    return e


def timed(fn):
    """CUDA-event time per replay of a graph holding fn(), after one call outside the capture and one warm-up replay"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(ITERS):
        g.replay()
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / ITERS * 1e3


def inputs(R, seed=100):
    rng = np.random.default_rng(seed)
    p, off, _ = synth_prompts(R, prompt_len=2048, groups=150, shared=1024, seed=seed, prefix_seed=7)
    return dict(prompt_bytes=torch.from_numpy(p).to(dev), prompt_off=torch.from_numpy(off).to(dev),
                model_seed=torch.from_numpy(np.full(R, 5, np.uint64)).to(dev),
                input_tokens=torch.from_numpy(np.full(R, 512, np.int32)).to(dev),
                ttft_slo=torch.from_numpy(rng.choice([200.0, 400.0, 1e6], R)).to(dev),
                tpot_slo=torch.from_numpy(rng.choice([14.0, 20.0, 40.0], R)).to(dev))


def outputs(R):
    return dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                hashes_out=torch.zeros((R, NB), dtype=torch.int64, device=dev), pick_match=torch.empty(R, dtype=torch.uint16, device=dev),
                added_out=torch.empty(R, dtype=torch.uint8, device=dev))


res = {}
for form in ("inflight", "index"):
    ix = form == "index"
    for R in (4096, 65536):
        d_in = inputs(R)
        tok = torch.full((R,), 600, dtype=torch.int64, device=dev)
        key = torch.arange(1, R + 1, dtype=torch.int64, device=dev)  # + R per replay
        out = outputs(R)
        row = {}
        e = engine(R, ix, True)
        def call():  # fresh keys every replay (the offset moves inside the graph): every Add creates its entry
            e.schedule_inorder_latency(R, tokens=tok, request_key=key, index=ix, device=True, stream=sptr, out=out, **d_in)
            key.add_(R)
        row["inorder_latency"] = timed(call)
        e.close()
        e = engine(R, ix, False)
        plain = {k: v for k, v in out.items() if k not in ("added_out",) and (ix or k != "pick_match")}
        nolat = {k: v for k, v in d_in.items() if k in ("prompt_bytes", "prompt_off", "model_seed")}
        if ix:
            row["no_latency"] = timed(lambda: e.schedule_inorder_index(R, tokens=tok, device=True, stream=sptr, out=plain, **nolat))
        else:
            row["no_latency"] = timed(lambda: e.schedule_inorder(R, tokens=tok, device=True, stream=sptr, out=plain, **nolat))
        e.close()
        if R == 4096:
            e = engine(R, ix, True)
            views = [{k: (v[r:r + 2] if k == "prompt_off" else v if k == "prompt_bytes" else v[r:r + 1]) for k, v in d_in.items()}
                     for r in range(R)]
            outs = [{k: v[r:r + 1] for k, v in out.items() if k not in ("pick_match", "added_out")} for r in range(R)]

            def loop():
                for r in range(R):
                    e.schedule(1, device=True, stream=sptr, out=outs[r], request_base=r, **views[r])
                    e.running_add(outs[r]["pick"], key[r:r + 1], d_in["tpot_slo"][r:r + 1], device=True, stream=sptr)
                    e.inflight_add(outs[r]["pick"], tok[r:r + 1], device=True, stream=sptr)
                    if ix:
                        e.commit_picks_device(outs[r]["pick"], outs[r]["hashes_out"], outs[r]["total_blocks"], stream=sptr)
                key.add_(R)
            row["loop"] = timed(loop)
            e.close()
        res[f"{form}_{R}"] = row

# spread in an all-negative world: k idle endpoints, the rest running one request each, every TTFT SLO below every prediction
R, k = 4096, 64
idle = np.arange(0, M, M // k)[:k]
busy = np.setdiff1d(np.arange(M), idle).astype(np.int32)
spread = {}
for route in ("batch_wide", "in_order"):
    e = engine(R, False, True)
    e.running_add(busy, np.arange(1, len(busy) + 1, dtype=np.uint64), np.full(len(busy), 30.0))
    e.set_snapshot(**snap)
    d_in = inputs(R, seed=5)
    d_in["ttft_slo"] = torch.full((R,), 1.0, dtype=torch.float64, device=dev)
    out = outputs(R)
    if route == "batch_wide":
        e.schedule(R, device=True, stream=sptr, out={k_: v for k_, v in out.items() if k_ not in ("pick_match", "added_out")}, **d_in)
    else:
        key = torch.arange(10**6, 10**6 + R, dtype=torch.int64, device=dev)
        e.schedule_inorder_latency(R, request_key=key, device=True, stream=sptr, out=out, **d_in)
    torch.cuda.synchronize()
    pick = out["pick"].cpu().numpy()
    spread[route] = dict(distinct_in_first_k=len(set(pick[:k].tolist())), busiest_endpoint_picks=int(np.bincount(pick[pick >= 0]).max()))
    e.close()

q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inorder_latency", "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "call_us": res, "per_request_us": {n: {k_: v / int(n.split("_")[1]) for k_, v in row.items()} for n, row in res.items()},
                  "all_negative_world": dict(k=k, **spread),
                  "note": "call_us: CUDA events over graph replays on one stream; each replay adds R fresh keys (a device-side "
                          "offset bumped inside the graph), so every Add creates its entry; the queues and counters keep growing"}))
