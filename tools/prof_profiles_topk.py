"""maxNumOfEndpoints lists from several scheduler profiles at the headline shape (64K requests x 1024 endpoints), on the GPU, with
the decode / prefill split of tools/prof_profiles.py (decode queue / kv / prefix / lora on the odd 512 endpoints, prefill kv /
prefix on the even 512):
  (a) one eppscore_schedule_batch_profiles_topk call: decode max-score k = 4, prefill k = 1;
  (b) the same with the decode profile weighted-random, k = 16;
  (c) the route without profiles for each: an eppscore_schedule_batch_topk (a) or _topk_wide (b) call with the decode role mask
      writing hashes_out, then an eppscore_schedule_batch_topk call with the prefill role mask fed them as hashes_in (on a second
      engine with the prefill scorers whose index got the same commits).
Every form is a CUDA-graph replay; medians of alternating rounds.  Prints one JSON line; --out writes it to a file.

    python tools/prof_profiles_topk.py [--rounds 7] [--reps 20] [--out FILE]"""
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
GOLDEN = 0x9E3779B97F4A7C15


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_profiles_topk needs a CUDA device")
    pkg = _pkg.load()
    R, M, mb = 65536, 1024, 32
    mw = M // 32
    odd = np.full(mw, 0xAAAAAAAA, np.uint32)
    even = np.full(mw, 0x55555555, np.uint32)
    sd = synth_snapshot(M, seed=1)
    eng = pkg.Engine(pkg.default_config(DECODE, max_endpoints=M, prefix_capacity=1 << 22))
    pid = eng.add_profile(PREFILL)
    pwr = eng.add_profile(DECODE, pick_mode=pkg.PICK_WEIGHTED_RANDOM)  # (b)'s decode profile
    eng.set_profile_endpoints(0, odd)
    eng.set_profile_endpoints(pid, even)
    eng.set_profile_endpoints(pwr, odd)
    eng.set_snapshot(**sd)
    prompts, off, _ = synth_prompts(R, prompt_len=2048, groups=150, shared=1024, seed=1)
    seeds = np.full(R, eng.model_seed("prof"), np.uint64)
    ad = zipf_adapters(R, seed=1)
    warm, runs = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], prompt_bytes=prompts, prompt_off=off, model_seed=seeds,
                                       adapter_id=ad, max_blocks=mb, want_hashes=True)
    commits = ([runs[0]["pick"], runs[1]["pick"]], warm["hashes_out"], warm["total_blocks"])
    eng.commit_picks_profiles(*commits)
    # without profiles an engine serves one scorer set and one picker: one engine per (scorers, picker), same index
    eng_pre = pkg.Engine(pkg.default_config(PREFILL, max_endpoints=M, prefix_capacity=1 << 22))
    eng_wr = pkg.Engine(pkg.default_config(DECODE, max_endpoints=M, prefix_capacity=1 << 22, pick_mode=pkg.PICK_WEIGHTED_RANDOM,
                                           tie_seed=(pwr * GOLDEN) & (2 ** 64 - 1)))  # profile pwr's draws
    for e in (eng_pre, eng_wr):
        e.set_snapshot(**sd)
        e.commit_picks_profiles(*commits)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d = dict(prompt_bytes=dev(prompts), prompt_off=dev(off), model_seed=dev(seeds), adapter_id=dev(ad))

    def outs(k):
        o = dict(pick=torch.empty(R, dtype=torch.int32, device="cuda"), pick_score=torch.empty(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.empty(R, dtype=torch.int32, device="cuda"))
        if k:
            o["topk_pick"] = torch.empty((R, k), dtype=torch.int32, device="cuda")
            o["topk_score"] = torch.empty((R, k), dtype=torch.float64, device="cuda")
        return o

    run_a = [dict(profile=0, topk=4, **outs(4)), dict(profile=pid, topk=1, **outs(1))]
    run_b = [dict(profile=pwr, topk=16, **outs(16)), dict(profile=pid, topk=1, **outs(1))]
    base_a, base_b = [outs(4), outs(1)], [outs(16), outs(1)]
    mask_dec, mask_pre = dev(np.tile(odd, (R, 1))), dev(np.tile(even, (R, 1)))
    hashes = torch.zeros((R, mb), dtype=torch.int64, device="cuda")
    nh = torch.zeros(R, dtype=torch.int16, device="cuda")
    s = torch.cuda.Stream()

    def profiles(runs_):
        return lambda: eng.schedule_profiles(R, runs_, device=True, stream=s.cuda_stream, max_blocks=mb, **d)

    def two_calls(e_dec, call, base):
        def fn():
            e_dec.schedule(R, cand_mask=mask_dec, max_blocks=mb, device=True, stream=s.cuda_stream,
                           out=dict(base[0], hashes_out=hashes, total_blocks=nh), **call, **d)
            eng_pre.schedule(R, cand_mask=mask_pre, hashes_in=hashes, n_hashes_in=nh, hash_stride=mb, adapter_id=d["adapter_id"],
                             topk=1, device=True, stream=s.cuda_stream, out=base[1])
        return fn

    forms = {"a_profiles_topk": profiles(run_a), "c_two_topk_calls": two_calls(eng, dict(topk=4), base_a),
             "b_profiles_topk_wide": profiles(run_b), "c_two_topk_wide_calls": two_calls(eng_wr, dict(topk_wide=16), base_b)}
    graphs = {}
    for name, fn in forms.items():
        with torch.cuda.stream(s):
            fn()  # outside a capture first: sizes the scratch (the wide score rows among it)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fn()
        graphs[name] = g
    for g in graphs.values():
        g.replay()
    torch.cuda.synchronize()

    def same(xs, ys):
        return all(bool(torch.equal(x[k], y[k])) for x, y in zip(xs, ys) for k in ("pick", "pick_score", "tie_count", "topk_pick",
                                                                                   "topk_score"))
    lists_equal = {"a": same(run_a, base_a), "b": same(run_b, base_b)}
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res = {"gpu": q, "shape": f"{R} x {M}, 2 KiB prompts, {mb} blocks", "lists_equal": lists_equal,
           **{f"{k}_us": float(np.median(v)) for k, v in times.items()},
           **{f"{k}_us_minmax": [float(np.min(v)), float(np.max(v))] for k, v in times.items()}}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
