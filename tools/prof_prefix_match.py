"""eppscore_prefix_match at the headline shape (R = 65 536 requests, M = 1024 endpoints, the bench's warm index after the
warm-up commit, the batch hashed once and its hashes kept, as a batch scheduled with hashes_out leaves them), on the GPU:
  - prefix_match at k = 1 (the pick), 8 and 16 (lists of endpoints) on those hashes,
  - pick_sparse alone on the same hashes (eppscore_schedule_batch with hashes_in: one kernel, the probe pass it makes),
  - the same batch with match_blocks set (the R x M diagnostics route that prefix_match replaces for a per-endpoint answer).
Each is captured `--calls` times into one CUDA graph; time per call = CUDA events around a replay / calls, median of `--reps`
replays.  The card's name and power limit are read in the same run.  Prints one JSON line; --out writes it.

    python tools/prof_prefix_match.py [--calls 20] [--reps 15] [--out FILE]"""
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
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = _pkg.load()
    R, M, A = 65536, bench.M, bench.A
    snap = synth_snapshot(M, A=A, seed=1)
    o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
    eng = pkg.Engine(pkg.default_config(bench.SCORERS, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                        max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19))
    eng.set_snapshot(**snap)
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    dev = torch.device("cuda:0")
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100, prefix_seed=7)
    h, n = eng.hash_prompts(p, off, np.full(R, seed, np.uint64), block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS)
    d_h, d_n = torch.from_numpy(h.view(np.int64)).to(dev), torch.from_numpy(n.view(np.int16)).to(dev)
    d_ad = torch.from_numpy(zipf_adapters(R, A=A, seed=100)).to(dev)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    diag = dict(out, match_blocks=torch.empty((R, M), dtype=torch.int16, device=dev))
    s = torch.cuda.Stream(device=dev)
    hs = dict(hashes_in=d_h, n_hashes_in=d_n, adapter_id=d_ad)

    def sched(o_):
        return lambda: eng.schedule(R, device=True, stream=s.cuda_stream, out=o_, **hs)
    sched(out)()
    torch.cuda.synchronize()
    pick = out["pick"].cpu().numpy()
    lists = {k: torch.from_numpy(((pick[:, None] + np.arange(k)[None, :] * 37) % M).astype(np.int32)).to(dev) for k in (1, 8, 16)}
    mout = {k: torch.empty((R, k), dtype=torch.int16, device=dev) for k in lists}

    def match(k):
        return lambda: eng.prefix_match(d_h, d_n, lists[k], device=True, stream=s.cuda_stream, out=mout[k])
    # bit-exact check at k = 8 against the R x M route's match_blocks, gathered at the same entries
    sched(diag)()
    match(8)()
    torch.cuda.synchronize()
    mb = diag["match_blocks"].cpu().numpy().view(np.uint16)
    ok = bool(np.array_equal(np.take_along_axis(mb, lists[8].cpu().numpy(), axis=1), mout[8].cpu().numpy().view(np.uint16)))

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
           "prefix_match_equals_match_blocks": ok}
    for k in (1, 8, 16):
        res[f"prefix_match_k{k}_us"] = time_call(match(k))
    res["pick_sparse_on_hashes_us"] = time_call(sched(out))
    res["batch_with_match_blocks_us"] = time_call(sched(diag))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
