"""The prefill/decode batch in arrival order (eppscore_schedule_batch_inorder_profiles, index form) at 1024 endpoints in the
README's P/D shape: decode = queue/kv/prefix/lora + token-load on endpoints 0-511, prefill = kv/prefix + token-load on
512-1023, the "prefill" profile's pick getting the second Add.  Device time per request of one graph-replayed call at R = 4K
and 64K, against
  loop                 the R-call loop it replaces (per request: eppscore_schedule_batch_profiles (R = 1) +
                       eppscore_commit_picks_profiles + eppscore_inflight_add of both picks), at R = 4K only
  profiles_plus_commit eppscore_schedule_batch_profiles + eppscore_commit_picks_profiles + eppscore_inflight_add of the whole
                       batch (index and load batch-wide)
  inorder_index        the single-profile eppscore_schedule_batch_inorder_index (the decode profile alone) at the same R
and, on a fresh warmed engine, the distinct prefill endpoints per shared-prefix group for prefixes new to the index, batch-wide
against ordered, with a token-load threshold of 8192 so that the load moves.  Prints one JSON line with the GPU's name and power limit.
usage: prof_inorder_profiles.py [iters]"""
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
DECODE = bench.SCORERS + [("token_load", 1.0)]
PREFILL = [("kv", 2.0), ("prefix", 3.0), ("token_load", 1.0)]
NB = bench.PROMPT_LEN // bench.BLOCK_CHARS
snap = synth_snapshot(M, A=A, seed=0)
_, _, _, _, _, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream
half = np.zeros(M // 32, np.uint32)
half[: M // 64] = 0xFFFFFFFF


def engine(R, profiles=True, thr=THR):
    e = pkg.Engine(pkg.default_config(DECODE, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS, max_blocks=NB,
                                      prefix_capacity=1 << 19, token_load_threshold=thr))
    if profiles:
        e.add_profile(PREFILL)
        e.set_profile_endpoints(0, half)
        e.set_profile_endpoints(1, ~half)
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"][:, :NB], np.minimum(warm["total_blocks"], NB))
    e.prefix_reserve(live_hashes=1 << 22, touches_per_call=2 * R * NB, overflow_rows=2 * R * NB + (1 << 18))
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


def run_out(R, p):
    return dict(profile=p, pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                tie_count=torch.empty(R, dtype=torch.int32, device=dev), pick_match=torch.empty(R, dtype=torch.uint16, device=dev))


def batch_out(R):
    return dict(total_blocks=torch.empty(R, dtype=torch.uint16, device=dev), hashes_out=torch.zeros((R, NB), dtype=torch.int64, device=dev))


def batch_wide(e, R, runs, out, tok2, d_in, request_base=0):
    e.schedule_profiles(R, runs, device=True, stream=sptr, out=out, request_base=request_base, **d_in)
    e.commit_picks_profiles([runs[0]["pick"], runs[1]["pick"]], out["hashes_out"], out["total_blocks"], device=True, stream=sptr)
    e.inflight_add(torch.cat([runs[0]["pick"], runs[1]["pick"]]), tok2, device=True, stream=sptr)


res, skips = {}, {}
for R in (4096, 65536):
    d_in, _ = inputs(R, 7, 150)
    tok = torch.full((R,), 600, dtype=torch.int64, device=dev)
    tok2 = torch.full((2 * R,), 600, dtype=torch.int64, device=dev)
    row = {}
    e = engine(R)
    runs, out = [run_out(R, 0), run_out(R, 1)], batch_out(R)
    row["inorder_profiles"] = timed(lambda: e.schedule_inorder_profiles(R, runs, tokens=tok, index=True, prefill_run=1, device=True,
                                                                        stream=sptr, out=out, **d_in))
    skips[f"{R}_inorder_profiles"] = int(e.stats().index_error)
    e.close()
    e = engine(R)
    runs_b = [{k: v for k, v in r.items() if k != "pick_match"} for r in (run_out(R, 0), run_out(R, 1))]
    row["profiles_plus_commit"] = timed(lambda: batch_wide(e, R, runs_b, out, tok2, d_in))
    skips[f"{R}_profiles_plus_commit"] = int(e.stats().index_error)
    e.close()
    e = engine(R, profiles=False)
    o1 = dict(pick=runs[0]["pick"], pick_score=runs[0]["pick_score"], tie_count=runs[0]["tie_count"], pick_match=runs[0]["pick_match"],
              **out)
    row["inorder_index"] = timed(lambda: e.schedule_inorder_index(R, tokens=tok, device=True, stream=sptr, out=o1, **d_in))
    e.close()
    if R == 4096:
        e = engine(R)
        views = [{k: (v[r:r + 2] if k == "prompt_off" else v if k == "prompt_bytes" else v[r:r + 1]) for k, v in d_in.items()}
                 for r in range(R)]
        rr = [[{k: (v[r:r + 1] if torch.is_tensor(v) else v) for k, v in x.items()} for x in runs_b] for r in range(R)]
        oo = [{k: v[r:r + 1] for k, v in out.items()} for r in range(R)]

        def loop():
            for r in range(R):
                batch_wide(e, 1, rr[r], oo[r], tok2[:2], views[r], request_base=r)
        row["loop"] = timed(loop)
        skips[f"{R}_loop"] = int(e.stats().index_error)
        e.close()
    res[str(R)] = row

# routing effect: a warmed engine, 4096 requests over 64 shared prefixes none of which the index holds yet.  The token-load
# threshold is SPREAD_THR here: at 600 tokens a request against 200000 the load term never moves, and kv-cache utilization alone
# would send every prefill request to one endpoint on either route.
SPREAD_THR = 8192.0
R = 4096
d_in, gid = inputs(R, 12345, 64)
tok = torch.full((R,), 600, dtype=torch.int64, device=dev)
tok2 = torch.full((2 * R,), 600, dtype=torch.int64, device=dev)
spread = {}
for route in ("batch_wide", "inorder_profiles"):
    e = engine(R, thr=SPREAD_THR)
    runs, out = [run_out(R, 0), run_out(R, 1)], batch_out(R)
    if route == "batch_wide":
        batch_wide(e, R, [{k: v for k, v in r.items() if k != "pick_match"} for r in runs], out, tok2, d_in)
    else:
        e.schedule_inorder_profiles(R, runs, tokens=tok, index=True, prefill_run=1, device=True, stream=sptr, out=out, **d_in)
    torch.cuda.synchronize()
    pick = runs[1]["pick"].cpu().numpy()
    spread[route] = float(np.mean([len(set(pick[gid == g].tolist())) for g in np.unique(gid)]))
    e.close()

q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inorder_profiles", "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "call_us": res, "per_request_us": {R: {k: v / int(R) for k, v in row.items()} for R, row in res.items()},
                  "index_error_after": skips, "distinct_prefill_endpoints_per_new_prefix_group": spread,
                  "note": "call_us: CUDA events over graph replays on one stream, reserved index; the counters and the index keep "
                          "growing across replays, as in a closed loop without releases"}))
