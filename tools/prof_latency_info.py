"""eppscore_predict_latency at the headline shape (R = 65 536 requests, M = 1024 endpoints, the bench's warm index after the
warm-up commit, the batch hashed once and its hashes kept), with a latency profile (latency scorer + queue + kv) on the GPU:
  - schedule + predict_latency at k = 1 (the pick), 4 and 16 (lists of endpoints) on those hashes,
  - schedule alone,
  - schedule with pred_out (the R x M x 2 diagnostics route that predict_latency replaces for the chosen endpoints).
Each is captured `--calls` times into one CUDA graph; time per call = CUDA events around a replay / calls, median of `--reps`
replays.  The card's name and power limit are read in the same run.  Prints one JSON line; --out writes it.

    python tools/prof_latency_info.py [--calls 10] [--reps 15] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot  # noqa: E402

LAT = dict(ttft_intercept=50.0, ttft_kv=30.0, ttft_input=0.05, ttft_waiting=8.0, ttft_running=4.0, ttft_prefix=-40.0,
           tpot_intercept=10.0, tpot_kv=5.0, tpot_input=0.001, tpot_waiting=1.0, tpot_running=1.0, tpot_generated=0.01,
           streaming_mode=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = _pkg.load()
    R, M = 65536, bench.M
    snap = synth_snapshot(M, seed=1)
    _, _, _, _, seed, warm = bench.oracle_setup(snap)
    eng = pkg.Engine(pkg.default_config([("latency", 2.0), ("queue", 1.0), ("kv", 1.0)], max_endpoints=M, block_chars=bench.BLOCK_CHARS,
                                        max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19))
    eng.set_latency_params(pkg.latency_params(**LAT))
    rng = np.random.Generator(np.random.PCG64(2))
    eng.set_snapshot(**snap, min_tpot_slo=rng.uniform(0, 80, M), dispatched=rng.integers(0, 4, M).astype(np.int32))
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    dev = torch.device("cuda:0")
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100, prefix_seed=7)
    h, n = eng.hash_prompts(p, off, np.full(R, seed, np.uint64), block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS)
    d_h, d_n = torch.from_numpy(h.view(np.int64)).to(dev), torch.from_numpy(n.view(np.int16)).to(dev)
    req = dict(input_tokens=torch.from_numpy(rng.integers(0, 3000, R).astype(np.int32)).to(dev),
               ttft_slo=torch.from_numpy(rng.uniform(50, 400, R)).to(dev), tpot_slo=torch.from_numpy(rng.uniform(5, 60, R)).to(dev))
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    diag = dict(out, pred_out=torch.empty((R, M, 2), dtype=torch.float64, device=dev))
    s = torch.cuda.Stream(device=dev)
    hs = dict(hashes_in=d_h, n_hashes_in=d_n, **req)

    def sched(o_):
        return lambda: eng.schedule(R, device=True, stream=s.cuda_stream, out=o_, **hs)
    sched(out)()
    torch.cuda.synchronize()
    pick = out["pick"].cpu().numpy()
    lists = {k: torch.from_numpy(((pick[:, None] + np.arange(k)[None, :] * 37) % M).astype(np.int32)).to(dev) for k in (1, 4, 16)}
    info = {k: torch.empty((R, k, 48), dtype=torch.uint8, device=dev) for k in lists}

    def predict(k):
        return lambda: eng.predict_latency(d_h, d_n, lists[k], device=True, stream=s.cuda_stream, out=info[k], **req)

    def sched_predict(k):
        a, b = sched(out), predict(k)
        return lambda: (a(), b())
    # bit-exact check at k = 4 against the R x M x 2 route's pred_out, gathered at the same entries
    sched(diag)()
    predict(4)()
    torch.cuda.synchronize()
    po = diag["pred_out"].cpu().numpy()
    got = info[4].cpu().numpy().reshape(-1).view(pkg.LATENCY_INFO_DTYPE).reshape(R, 4)
    e = lists[4].cpu().numpy()
    ok = bool(np.array_equal(np.take_along_axis(po[:, :, 0], e, axis=1).view(np.uint64), got["ttft"].view(np.uint64)) and
              np.array_equal(np.take_along_axis(po[:, :, 1], e, axis=1).view(np.uint64), got["tpot"].view(np.uint64)))

    def time_call(fn):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(args.calls):
                fn()
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            with torch.cuda.stream(s):
                g.replay()
            b.record(s)
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3 / args.calls)
        return float(np.median(ts))

    res = {"card": card(), "R": R, "M": M, "max_blocks": bench.MAX_BLOCKS, "mean_blocks": float(n.mean()), "calls_per_graph": args.calls,
           "ttft_tpot_equal_pred_out": ok}
    for k in (1, 4, 16):
        res[f"predict_latency_k{k}_us"] = time_call(predict(k))
        res[f"schedule_plus_predict_latency_k{k}_us"] = time_call(sched_predict(k))
    res["schedule_us"] = time_call(sched(out))
    res["schedule_with_pred_out_us"] = time_call(sched(diag))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
