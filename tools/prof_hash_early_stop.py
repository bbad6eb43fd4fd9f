"""Times the headline step's probing hash kernel (hash_warp_kernel<64, true>) at three states of the prefix index, on the
headline batch (64K requests x 1024 endpoints, 2 KB prompts of 32 blocks, 150 shared 1 KB prefixes, 4 rotating input sets):
  none      an empty index: every request misses at block 0, the kernel streams one chunk per request (the best case);
  headline  the bench's warm index (4 * M earlier requests committed): 16 blocks match, the first miss is at block 16;
  all       every block of every timed request committed to one endpoint per prefix group: all 32 blocks match and every
            request stays resolvable to its last block, so the kernel streams every byte and runs every chunk's chain and
            probe rounds (the worst case).
Kernel times from a torch.profiler trace of CUDA-graph replays, the step (hash + pick, snapshot not re-prepared) from CUDA
events over graph replays without the profiler, and the requests the hash kernel resolved.
usage: python tools/prof_hash_early_stop.py [none] [headline] [all]"""
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

states = sys.argv[1:] or ["none", "headline", "all"]
_pkg.load_build().build()
pkg = _pkg.load()
R, M, A, NS = 65536, bench.M, bench.A, 4
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sp = stream.cuda_stream
host, sets = [], []
for i in range(NS):
    p, off, g = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=i, prefix_seed=7)
    ad = zipf_adapters(R, A=A, seed=i)
    host.append((p, off, ad, g))
    sets.append(dict(p=torch.from_numpy(p).to(dev), off=torch.from_numpy(off).to(dev), ad=torch.from_numpy(ad).to(dev),
                     seeds=torch.from_numpy(np.full(R, seed, np.uint64).view(np.int64)).to(dev)))
out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
           tie_count=torch.empty(R, dtype=torch.int32, device=dev))
print(torch.cuda.get_device_name(0), os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader").read().strip())


def engine(state):
    eng = pkg.Engine(pkg.default_config(bench.SCORERS, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                        max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19))
    eng.set_snapshot(**snap)
    if state == "headline":
        eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    elif state == "all":
        for p, off, ad, g in host:  # one endpoint per prefix group: every block's set is that one endpoint
            h = eng.schedule(R, prompt_bytes=p, prompt_off=off, model_seed=np.full(R, seed, np.uint64), adapter_id=ad, want_hashes=True)
            eng.commit_picks((g % M).astype(np.int32), h["hashes_out"], h["total_blocks"])
    return eng


for state in states:
    eng = engine(state)

    def step(i, eng=eng):
        d = sets[i % NS]
        eng.schedule(R, prompt_bytes=d["p"], prompt_off=d["off"], model_seed=d["seeds"], adapter_id=d["ad"], device=True, stream=sp, out=out)

    resolved = []
    for i in range(NS):
        r0 = eng.stats().probe_resolved
        step(i)
        torch.cuda.synchronize()
        resolved.append((eng.stats().probe_resolved - r0) % (1 << 32))
    gs = []
    for i in range(NS):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            step(i)
        gs.append(g)
    for i in range(8):
        gs[i % NS].replay()
    torch.cuda.synchronize()
    iters = 40
    with profile(activities=[ProfilerActivity.CUDA]) as tr:
        for i in range(iters):
            gs[i % NS].replay()
        torch.cuda.synchronize()
    print(f"== {state}: resolved by the hash kernel {resolved} of {R} per set")
    for ev in sorted(tr.key_averages(), key=lambda e: -e.self_device_time_total):
        if ev.device_type.name == "CUDA" and ev.count > 0 and ev.self_device_time_total / iters >= 1.0:
            print(f"  {ev.key[:90]:90s}: {ev.self_device_time_total / iters:8.2f} us per step")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 400
    a.record(stream)
    for i in range(iters):
        gs[i % NS].replay()
    b.record(stream)
    torch.cuda.synchronize()
    print(f"  hash + pick (graph, no profiler): {a.elapsed_time(b) / iters * 1e3:8.2f} us")
    del gs
    eng.close()
