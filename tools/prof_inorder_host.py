"""The host-array in-order batch at the headline shape (1024 endpoints, the four-scorer profile plus token-load weight 1): the
wall time of one synchronous eppscore_schedule_batch_inorder on host arrays (inputs staged, the call scheduled on the engine
stream, results copied back, then a synchronise) at R = 4K and 64K.  Reports the median and the spread over the timed calls.
Prints one JSON line with the GPU's name and power limit.  usage: prof_inorder_host.py [calls]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

CALLS = int(sys.argv[1]) if len(sys.argv) > 1 else 9
pkg = _pkg.load()
M, A = bench.M, bench.A
SC = bench.SCORERS + [("token_load", 1.0)]
snap = synth_snapshot(M, A=A, seed=0)
_, _, _, _, _, warm = bench.oracle_setup(snap)

res = {}
for R in (4096, 65536):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100, prefix_seed=7)
    kw = dict(prompt_bytes=p, prompt_off=off, model_seed=np.full(R, 5, np.uint64), adapter_id=zipf_adapters(R, A=A, seed=1))
    e = pkg.Engine(pkg.default_config(SC, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS,
                                      prefix_capacity=1 << 19, token_load_threshold=200000.0))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    tok = e.estimate_tokens(R, prompt_chars=np.diff(off).astype(np.int32))
    for _ in range(2):  # warm-up: module loads, scratch and staging allocations
        e.schedule_inorder(R, tokens=tok, **kw)
    ms = []
    for _ in range(CALLS):
        t0 = time.perf_counter()
        e.schedule_inorder(R, tokens=tok, **kw)  # returns after its results are on the host
        ms.append((time.perf_counter() - t0) * 1e3)
    e.close()
    res[str(R)] = dict(median_ms=float(np.median(ms)), min_ms=float(min(ms)), max_ms=float(max(ms)))

q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "inorder_host", "M": M, "gpu": torch.cuda.get_device_name(0),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None, "calls": CALLS,
                  "call_ms": res,
                  "note": "host clock around each synchronous host-array call; the in-flight counters keep growing across calls"}))
