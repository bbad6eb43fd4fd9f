"""Small device batches on reserved streams (eppscore_reserve_stream), on the GPU: the headline profile (queue / kv / prefix /
lora) at M = 1024 with 2 KiB prompts, R in {256, 1024, 4096, 16384}, each stream replaying a CUDA graph of `--per-graph`
back-to-back batches.  One stream against two and four reserved streams replaying their graphs at the same time: requests/s
over all streams, and the per-batch latency a stream sees (the window over the batches each stream ran).  Medians of
alternating rounds; every stream's picks are checked against the one-stream picks.  Prints one JSON line; --out writes it.

    python tools/prof_stream_scratch.py [--rounds 5] [--requests 4194304] [--per-graph 8] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
SIZES = (256, 1024, 4096, 16384)
STREAMS = (1, 2, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--requests", type=int, default=1 << 22, help="requests per timed window (all streams together)")
    ap.add_argument("--per-graph", type=int, default=8, help="batches captured back to back in each stream's graph")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_stream_scratch needs a CUDA device")
    pkg = _pkg.load()
    M = 1024
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, prefix_capacity=1 << 18))
    eng.set_snapshot(**synth_snapshot(M, seed=1))
    seed = eng.model_seed("prof")
    Rw = 4 * M  # one committed batch warms the index on the prompt pool the timed batches draw from
    wp, woff, _ = synth_prompts(Rw, prompt_len=2048, groups=150, shared=1024, seed=1)
    warm = eng.schedule(Rw, prompt_bytes=wp, prompt_off=woff, model_seed=np.full(Rw, seed, np.uint64), want_hashes=True)
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    streams = [torch.cuda.Stream() for _ in range(max(STREAMS))]
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    res = {}
    for R in SIZES:
        prompts, off, _ = synth_prompts(R, prompt_len=2048, groups=150, shared=1024, seed=2, prefix_seed=1)
        d = dict(prompt_bytes=cuda(prompts), prompt_off=cuda(off), model_seed=cuda(np.full(R, seed, np.uint64).view(np.int64)),
                 adapter_id=cuda(zipf_adapters(R, seed=2)))
        graphs, outs = [], []
        for s in streams:
            eng.reserve_stream(s, R)
            out = dict(pick=torch.empty(R, dtype=torch.int32, device="cuda"), pick_score=torch.empty(R, dtype=torch.float64, device="cuda"),
                       tie_count=torch.empty(R, dtype=torch.int32, device="cuda"))
            s.wait_stream(torch.cuda.current_stream())
            eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d)
            s.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                for _ in range(args.per_graph):
                    eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d)
            graphs.append(g)
            outs.append(out)
        times = {n: [] for n in STREAMS}
        for _ in range(args.rounds):
            for n in STREAMS:
                iters = max(4, args.requests // (R * n * args.per_graph))
                main_s = torch.cuda.current_stream()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                main_s.synchronize()
                e0.record(main_s)
                for s in streams[:n]:
                    s.wait_stream(main_s)
                for _ in range(iters):
                    for s, g in zip(streams[:n], graphs[:n]):
                        with torch.cuda.stream(s):
                            g.replay()
                for s in streams[:n]:
                    main_s.wait_stream(s)
                e1.record(main_s)
                e1.synchronize()
                ms = e0.elapsed_time(e1)
                batches = iters * args.per_graph
                times[n].append((ms, batches))
        torch.cuda.synchronize()
        same = all(torch.equal(o["pick"], outs[0]["pick"]) and torch.equal(o["pick_score"], outs[0]["pick_score"]) for o in outs)
        for s in streams:
            eng.release_stream(s)
        for n in STREAMS:
            ms = float(np.median([t for t, _ in times[n]]))
            batches = times[n][0][1]
            res[f"R{R}_streams{n}"] = {"requests_per_s": n * batches * R / (ms / 1e3), "batch_latency_us": ms * 1e3 / batches,
                                       "picks_equal": bool(same)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    line = json.dumps({"gpu": q, "M": M, "per_graph": args.per_graph, "rounds": args.rounds, **res})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
