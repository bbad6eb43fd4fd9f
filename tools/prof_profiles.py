"""Several scheduler profiles at the headline shape (64K requests x 1024 endpoints), on the GPU: one
eppscore_schedule_batch_profiles call with a decode profile (queue / kv / prefix / lora on the odd 512 endpoints) and a prefill
profile (kv / prefix on the even 512), against the route without profiles: two eppscore_schedule_batch calls with per-request
role masks, the first writing hashes_out, the second fed them as hashes_in.  Also the two-pick device commit
(eppscore_commit_picks_profiles) against two eppscore_commit_picks_device calls.  Schedule calls are CUDA-graph replays, commits
are timed with CUDA events around the calls; medians of alternating rounds.  Prints one JSON line; --out writes it to a file.

    python tools/prof_profiles.py [--rounds 7] [--reps 20] [--out FILE]"""
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

DECODE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
PREFILL = [("kv", 1), ("prefix", 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_profiles needs a CUDA device")
    pkg = _pkg.load()
    R, M, mb = 65536, 1024, 32
    eng = pkg.Engine(pkg.default_config(DECODE, max_endpoints=M, prefix_capacity=1 << 22))
    pid = eng.add_profile(PREFILL)
    mw = M // 32
    odd = np.full(mw, 0xAAAAAAAA, np.uint32)
    even = np.full(mw, 0x55555555, np.uint32)
    eng.set_profile_endpoints(0, odd)
    eng.set_profile_endpoints(pid, even)
    sd = synth_snapshot(M, seed=1)
    eng.set_snapshot(**sd)
    prompts, off, _ = synth_prompts(R, prompt_len=2048, groups=150, shared=1024, seed=1)
    seeds = np.full(R, eng.model_seed("prof"), np.uint64)
    ad = zipf_adapters(R, seed=1)
    warm, runs = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], prompt_bytes=prompts, prompt_off=off, model_seed=seeds,
                                       adapter_id=ad, max_blocks=mb, want_hashes=True)
    eng.commit_picks_profiles([runs[0]["pick"], runs[1]["pick"]], warm["hashes_out"], warm["total_blocks"])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d = dict(prompt_bytes=dev(prompts), prompt_off=dev(off), model_seed=dev(seeds), adapter_id=dev(ad))
    out32 = lambda: torch.empty(R, dtype=torch.int32, device="cuda")  # noqa: E731
    out64 = lambda: torch.empty(R, dtype=torch.float64, device="cuda")  # noqa: E731
    prun = [dict(profile=p, pick=out32(), pick_score=out64(), tie_count=out32()) for p in (0, pid)]
    mask_dec, mask_pre = dev(np.tile(odd, (R, 1))), dev(np.tile(even, (R, 1)))
    hashes = torch.zeros((R, mb), dtype=torch.int64, device="cuda")
    nh = torch.zeros(R, dtype=torch.int16, device="cuda")
    base = [dict(pick=out32(), pick_score=out64(), tie_count=out32()) for _ in range(2)]
    # without profiles an engine serves one scorer set: the prefill call goes to a second engine whose index got the same commits
    eng2 = pkg.Engine(pkg.default_config(PREFILL, max_endpoints=M, prefix_capacity=1 << 22))
    eng2.set_snapshot(**sd)
    eng2.commit_picks_profiles([runs[0]["pick"], runs[1]["pick"]], warm["hashes_out"], warm["total_blocks"])
    s = torch.cuda.Stream()

    def two_runs():
        eng.schedule_profiles(R, prun, device=True, stream=s.cuda_stream, max_blocks=mb, **d)

    def two_calls():
        eng.schedule(R, cand_mask=mask_dec, max_blocks=mb, device=True, stream=s.cuda_stream,
                     out=dict(base[0], hashes_out=hashes, total_blocks=nh), **d)
        eng2.schedule(R, cand_mask=mask_pre, hashes_in=hashes, n_hashes_in=nh, hash_stride=mb, adapter_id=d["adapter_id"],
                      device=True, stream=s.cuda_stream, out=base[1])

    graphs = {}
    for name, fn in (("two_run_call", two_runs), ("two_masked_calls", two_calls)):
        with torch.cuda.stream(s):
            fn()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fn()
        graphs[name] = g
    # both routes give the same picks (max-score with lowest-index ties draws nothing, so the profiles' seeds do not matter)
    graphs["two_run_call"].replay()
    graphs["two_masked_calls"].replay()
    torch.cuda.synchronize()
    same = all(bool(torch.equal(a["pick"], b["pick"]) and torch.equal(a["pick_score"], b["pick_score"])) for a, b in zip(prun, base))
    times = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for name, g in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            g.replay()
            e0.record()
            for _ in range(args.reps):
                g.replay()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1000.0 / args.reps)
    # launches of one call of each route
    l0 = eng.stats().kernel_launches
    two_runs()
    torch.cuda.synchronize()
    launches_two_run = eng.stats().kernel_launches - l0
    # commits: two picks in one commit against two single commits, device arrays, small repeated batches of the headline rows
    Rc = 4096
    pk = [prun[0]["pick"][:Rc].contiguous(), prun[1]["pick"][:Rc].contiguous()]
    hc = torch.from_numpy(warm["hashes_out"][:Rc].view(np.int64)).cuda()
    nc = torch.from_numpy(warm["total_blocks"][:Rc].astype(np.int16)).cuda()
    bound = int(warm["total_blocks"][:Rc].sum()) * 2
    ctimes = {"two_pick_commit": [], "two_single_commits": []}
    for _ in range(args.rounds):
        for name in ctimes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                if name == "two_pick_commit":
                    eng.commit_picks_profiles(pk, hc, nc, device=True, touch_bound=bound)
                else:
                    eng.commit_picks_device(pk[0], hc, nc, touch_bound=bound // 2)
                    eng.commit_picks_device(pk[1], hc, nc, touch_bound=bound // 2)
            e1.record()
            e1.synchronize()
            ctimes[name].append(e0.elapsed_time(e1) * 1000.0 / args.reps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res = {"gpu": q, "shape": f"{R} x {M}, 2 KiB prompts, {mb} blocks", "picks_equal": same,
           "launches_two_run_call": launches_two_run,
           **{f"{k}_us": float(np.median(v)) for k, v in times.items()},
           **{f"{k}_us": float(np.median(v)) for k, v in ctimes.items()}, "commit_requests": Rc}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
