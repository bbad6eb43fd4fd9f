"""The in-order batch that commits as it schedules (eppscore_schedule_batch_inorder_index) at the headline shape (1024
endpoints, the four-scorer profile plus token-load weight 1, 2 KB prompts of 32 blocks): device time per request of one
graph-replayed call at R = 4K and 64K, against
  inorder_plus_commit  eppscore_schedule_batch_inorder + one eppscore_commit_picks_device of the whole batch (index batch-wide)
  loop                 the R-call loop it replaces: per request eppscore_schedule_batch (R = 1) + eppscore_commit_picks_device +
                       eppscore_inflight_add (captured at R = 4K only: a graph of 64K such calls is not practical)
and, on a fresh warmed engine, the distinct endpoints per shared-prefix group for prefixes new to the index, for the
batch-wide call and the index-ordered one.  Prints one JSON line with the GPU's name and power limit.
usage: prof_inorder_index.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
pkg = _pkg.load()
M, A = bench.M, bench.A
THR = 200000.0
SC = bench.SCORERS + [("token_load", 1.0)]
NB = bench.PROMPT_LEN // bench.BLOCK_CHARS
snap = synth_snapshot(M, A=A, seed=0)
_, _, _, _, _, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream


def engine(R):
    e = pkg.Engine(pkg.default_config(SC, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS, max_blocks=NB,
                                      prefix_capacity=1 << 19, token_load_threshold=THR))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"][:, :NB], np.minimum(warm["total_blocks"], NB))
    e.prefix_reserve(live_hashes=1 << 22, touches_per_call=R * NB, overflow_rows=R * NB + (1 << 18))  # a pool that never skips
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


def inputs(R, prefix_seed, groups):
    p, off, gid = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=groups, shared=1024, seed=100, prefix_seed=prefix_seed)
    d = dict(prompt_bytes=torch.from_numpy(p).to(dev), prompt_off=torch.from_numpy(off).to(dev),
             model_seed=torch.from_numpy(np.full(R, 5, np.uint64)).to(dev),
             adapter_id=torch.from_numpy(zipf_adapters(R, A=A, seed=1)).to(dev))
    return d, gid


def outputs(R):
    return dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                hashes_out=torch.zeros((R, NB), dtype=torch.int64, device=dev), pick_match=torch.empty(R, dtype=torch.uint16, device=dev))


res, skips = {}, {}
for R in (4096, 65536):
    d_in, _ = inputs(R, 7, 150)
    tok = torch.full((R,), 600, dtype=torch.int64, device=dev)
    out = outputs(R)
    row = {}
    e = engine(R)
    row["inorder_index"] = timed(lambda: e.schedule_inorder_index(R, tokens=tok, device=True, stream=sptr, out=out, **d_in))
    skips[f"{R}_inorder_index"] = int(e.stats().index_error)
    e.close()
    e = engine(R)

    def plus_commit():
        e.schedule_inorder(R, tokens=tok, device=True, stream=sptr, out=out, **d_in)
        e.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], stream=sptr)
    row["inorder_plus_commit"] = timed(plus_commit)
    skips[f"{R}_inorder_plus_commit"] = int(e.stats().index_error)
    e.close()
    if R == 4096:
        e = engine(R)
        views = [{k: (v[r:r + 2] if k == "prompt_off" else v if k == "prompt_bytes" else v[r:r + 1]) for k, v in d_in.items()}
                 for r in range(R)]
        outs = [{k: v[r:r + 1] for k, v in out.items() if k != "pick_match"} for r in range(R)]

        def loop():
            for r in range(R):
                e.schedule(1, device=True, stream=sptr, out=outs[r], request_base=r, **views[r])
                e.commit_picks_device(outs[r]["pick"], outs[r]["hashes_out"], outs[r]["total_blocks"], stream=sptr)
                e.inflight_add(outs[r]["pick"], tok[r:r + 1], device=True, stream=sptr)
        row["loop"] = timed(loop)
        skips[f"{R}_loop"] = int(e.stats().index_error)
        e.close()
    res[str(R)] = row

# routing effect: a warmed engine, 4096 requests over 64 shared prefixes none of which the index holds yet
R = 4096
d_in, gid = inputs(R, 12345, 64)
tok = torch.full((R,), 600, dtype=torch.int64, device=dev)
spread = {}
for route in ("inorder", "inorder_index"):
    e = engine(R)
    out = outputs(R)
    if route == "inorder":
        e.schedule_inorder(R, tokens=tok, device=True, stream=sptr, out=out, **d_in)
    else:
        e.schedule_inorder_index(R, tokens=tok, device=True, stream=sptr, out=out, **d_in)
    torch.cuda.synchronize()
    pick = out["pick"].cpu().numpy()
    spread[route] = float(np.mean([len(set(pick[gid == g].tolist())) for g in np.unique(gid)]))
    e.close()

q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inorder_index", "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "call_us": res, "per_request_us": {R: {k: v / int(R) for k, v in row.items()} for R, row in res.items()},
                  "index_error_after": skips, "distinct_endpoints_per_new_prefix_group": spread,
                  "note": "call_us: CUDA events over graph replays on one stream, reserved index; the counters and the index keep "
                          "growing across replays, as in a closed loop without releases. index_error_after: stats.index_error "
                          "(bit 4 = a mutation skipped for lack of room, which would make its commits free)"}))
