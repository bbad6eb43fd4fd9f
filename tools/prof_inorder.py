"""The in-order batch at the headline shape (1024 endpoints, the four-scorer profile plus token-load weight 1): the device time
of one graph-replayed eppscore_schedule_batch_inorder against eppscore_schedule_batch + eppscore_inflight_add (the batch route,
one load view) at R = 4K, 16K and 64K, and for both routes the largest number of picks any endpoint gets in one batch (the
dog-pile the in-order call removes).  The in-order picks of the first batch are checked against the sequential reference on
the first 256 requests.  Prints one JSON line with the GPU's name and power limit.  usage: prof_inorder.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from oracle import oracle_py as o  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402
from tests.inorder_reference import schedule_inorder  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
pkg = _pkg.load()
M, A = bench.M, bench.A
THR = 200000.0
SC = bench.SCORERS + [("token_load", 1.0)]
snap = synth_snapshot(M, A=A, seed=0)
_, _, _, _, _, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)  # graph replays run on the current stream: the events must be on the same one
sptr = stream.cuda_stream


def engine():
    e = pkg.Engine(pkg.default_config(SC, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS,
                                      prefix_capacity=1 << 19, token_load_threshold=THR))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    return e


def timed(fn):
    """CUDA-event time per replay of a graph holding fn(), after warm-up replays"""
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


res, pile, checks = {}, {}, {}
for R in (4096, 16384, 65536):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100, prefix_seed=7)
    seeds = np.full(R, 5, np.uint64)
    ad = zipf_adapters(R, A=A, seed=1)
    d_in = dict(prompt_bytes=torch.from_numpy(p).to(dev), prompt_off=torch.from_numpy(off).to(dev),
                model_seed=torch.from_numpy(seeds).to(dev), adapter_id=torch.from_numpy(ad).to(dev))
    chars = torch.from_numpy(np.diff(off).astype(np.int32)).to(dev)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    est = torch.empty(R, dtype=torch.int64, device=dev)
    row = {}
    for route in ("batch_plus_add", "inorder"):
        e = engine()
        e.estimate_tokens(R, prompt_chars=chars, device=True, stream=sptr, out=est)
        if route == "inorder":
            # the first batch from zero counters: its pile-up, and (at 4K) its picks against the sequential reference
            torch.cuda.synchronize()
            e.schedule_inorder(R, tokens=est, device=True, stream=sptr, out=out, **d_in)
            torch.cuda.synchronize()
            pile.setdefault(str(R), {})[route] = int(torch.bincount(out["pick"][out["pick"] >= 0].long(), minlength=M).max())
            if R == 4096:
                n = 256
                want, _ = schedule_inorder(snap, o.make_profile([(pkg.SCORER[k], w) for k, w in SC], token_load_threshold=THR),
                                           None, n, est.cpu().numpy()[:n], prompt_bytes=p, prompt_off=off, model_seed=seeds,
                                           adapter_id=ad, block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS)
                checks["first_256_vs_sequential_reference"] = bool(np.array_equal(out["pick"].cpu().numpy()[:n], want["pick"]))
            e.close()
            e = engine()
            fn = lambda: e.schedule_inorder(R, tokens=est, device=True, stream=sptr, out=out, **d_in)  # noqa: E731
        else:
            e.schedule(R, device=True, stream=sptr, out=out, **d_in)
            torch.cuda.synchronize()
            pile.setdefault(str(R), {})[route] = int(torch.bincount(out["pick"][out["pick"] >= 0].long(), minlength=M).max())

            def fn():
                e.schedule(R, device=True, stream=sptr, out=out, **d_in)
                e.inflight_add(out["pick"], est, device=True, stream=sptr)
        row[route] = timed(fn)
        e.close()
    res[str(R)] = row

q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inorder", "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "call_us": res, "max_picks_per_endpoint": pile, "checks": checks,
                  "per_request_us_inorder": {R: res[R]["inorder"] / int(R) for R in res},
                  "note": "call_us: CUDA events over graph replays on one stream; batch_plus_add = eppscore_schedule_batch + "
                          "eppscore_inflight_add; inorder = eppscore_schedule_batch_inorder (its batch kernels, the min/max pass "
                          "and the cluster's in-order walk). Counters keep growing across replays, as in a closed loop without "
                          "releases. max_picks_per_endpoint: the first batch of a fresh engine (all counters 0)"}))
