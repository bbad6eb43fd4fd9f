"""maxNumOfEndpoints past 8 at the headline shape (64K requests x 1024 endpoints, queue 2 / kv 2 / prefix 3 / lora 1, warmed
index, device-resident block hashes, every call inside a CUDA graph, CUDA events, median of rounds):

  - eppscore_schedule_batch_topk_wide at k = 8, 16, 64, 256 in all three pick modes;
  - eppscore_schedule_batch_topk at k = 8 (the register lists), for comparison;
  - step 1 (scoring into the slice's score rows) and step 2 (topk_select_kernel) apart, from torch.profiler kernel times;
  - max-score k = 16 from host buffers: the wide call against the score-map route (the R x M score map copied to the host;
    the host-side sort is not included);
  - a 512-request check of the lists against the CPU oracle.

Prints one JSON line with the GPU's name and power limit.  With --slice-mib N the library is first rebuilt into a temporary
directory with a slice budget of N MiB (-DEPP_WIDE_SLICE_BYTES) and only the wide device arms are timed, so two runs compare
the budgets.  usage: prof_topk_wide.py [--rounds N] [--slice-mib N]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests import topk_oracle as T  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--iters", type=int, default=6)
ap.add_argument("--slice-mib", type=int, default=0)
args = ap.parse_args()

tmp = None
if args.slice_mib:  # the same sources with another slice budget, built apart from the tree
    tmp = tempfile.mkdtemp(prefix="eppscore_slice_")
    pkg_dir = os.path.join(tmp, os.path.basename(_pkg.PKG_DIR))
    shutil.copytree(_pkg.PKG_DIR, pkg_dir, ignore=shutil.ignore_patterns("build", "*.so", "__pycache__", "host_test", "host_bench"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    os.environ["EPPSCORE_NVCC_EXTRA"] = f"-DEPP_WIDE_SLICE_BYTES={args.slice_mib << 20}ull"
    _pkg.PKG_DIR = pkg_dir
    _pkg.load_build().build()
pkg = _pkg.load()
R, M, A = 65536, bench.M, bench.A
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream
NSETS = 3


def make_engine(**kw):
    e = pkg.Engine(pkg.default_config(bench.SCORERS, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                      max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19, **kw))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    return e


eng0 = make_engine()
sets, host_sets = [], []
for i in range(NSETS):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100 + i, prefix_seed=7)
    ad = zipf_adapters(R, A=A, seed=100 + i)
    h, n = eng0.hash_prompts(p, off, np.full(R, seed, np.uint64), block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS)
    host_sets.append((h, n, ad))
    sets.append((torch.from_numpy(h.view(np.int64)).to(dev), torch.from_numpy(n.view(np.int16)).to(dev), torch.from_numpy(ad).to(dev)))
eng0.close()


def outputs(k=0):
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    if k:
        out["topk_pick"] = torch.empty((R, k), dtype=torch.int32, device=dev)
        out["topk_score"] = torch.empty((R, k), dtype=torch.float64, device=dev)
    return out


def call(e, i, out, **kw):
    hh, nn, ad = sets[i % NSETS]
    e.schedule(R, hashes_in=hh, n_hashes_in=nn, hash_stride=bench.MAX_BLOCKS, adapter_id=ad, device=True, stream=sptr, out=out, **kw)


def graphs_for(e, out, **kw):
    for i in range(NSETS):
        call(e, i, out, **kw)
    torch.cuda.synchronize()
    gs = []
    for i in range(NSETS):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            call(e, i, out, **kw)
        gs.append(g)
    return gs


def time_ms(e, out, **kw):
    """median over rounds of the CUDA-event time per replay, each input set captured into its own graph"""
    gs = graphs_for(e, out, **kw)
    for i in range(3):
        gs[i % NSETS].replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        a.record(stream)
        for i in range(args.iters):
            gs[i % NSETS].replay()
        b.record(stream)
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) / args.iters)
    return float(np.median(per))


def steps_ms(e, out, **kw):
    """kernel time per replay from torch.profiler: step 2 = topk_select_kernel, step 1 = every other kernel"""
    gs = graphs_for(e, out, **kw)
    n = 2 * NSETS
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as pr:
        for i in range(n):
            gs[i % NSETS].replay()
        torch.cuda.synchronize()
    sel = other = 0.0
    for ev in pr.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "topk_select_kernel" in ev.name:
            sel += t
        elif "kernel" in ev.name.lower():
            other += t
    return {"step1_ms": other / n / 1e3, "step2_ms": sel / n / 1e3}


def parity(e, pick_mode, tie_seed, k, out, nreq=512):
    call(e, 0, out, topk_wide=k)
    torch.cuda.synchronize()
    h, nh, ad = host_sets[0]
    p = o.make_profile([({"queue": 0, "kv": 1, "prefix": 2, "lora": 3}[s], w) for s, w in bench.SCORERS], pick_mode=pick_mode,
                       tie_seed=tie_seed)
    want = T.schedule_batch(osnap, p, idx, nreq, topk=k, hashes_in=h[:nreq], n_hashes_in=nh[:nreq], adapter_id=ad[:nreq],
                            max_blocks=bench.MAX_BLOCKS, n_threads=os.cpu_count() or 1)
    return bool(np.array_equal(out["topk_pick"][:nreq].cpu().numpy(), want["topk_pick"]) and
                np.array_equal(out["topk_score"][:nreq].cpu().numpy().view(np.uint64), want["topk_score"].view(np.uint64)) and
                np.array_equal(out["pick"][:nreq].cpu().numpy(), want["pick"]))


def host_ms(e, **kw):
    """wall time of a host-buffer call (copies in both directions included), median over rounds"""
    h, nh, ad = host_sets[0]
    per = []
    for _ in range(max(3, args.rounds // 2)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e.schedule(R, hashes_in=h, n_hashes_in=nh, hash_stride=bench.MAX_BLOCKS, adapter_id=ad, want_total=False, **kw)
        per.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(per))


arms, steps, ok = {}, {}, {}
modes = (("max_score", pkg.PICK_MAX_SCORE, 0), ("weighted_random", pkg.PICK_WEIGHTED_RANDOM, 3), ("random", pkg.PICK_RANDOM, 5))
for name, mode, tie_seed in modes:
    e = make_engine(pick_mode=mode, tie_seed=tie_seed)
    if not args.slice_mib:
        arms[f"topk8_registers_{name}"] = time_ms(e, outputs(8), topk=8)
    for k in (8, 16, 64, 256):
        out = outputs(k)
        arms[f"wide{k}_{name}"] = time_ms(e, out, topk_wide=k)
        if k == 16:
            steps[f"wide16_{name}"] = steps_ms(e, out, topk_wide=k)
            ok[f"wide16_{name}"] = parity(e, mode, tie_seed, k, out)
        del out
    if mode == pkg.PICK_MAX_SCORE and not args.slice_mib:
        arms["host_wide16_max_score"] = host_ms(e, topk_wide=16)
        arms["host_score_map_max_score"] = host_ms(e, want_scores=True)
    e.close()
del idx  # the oracle's index, freed while its library is still loaded
if tmp:
    shutil.rmtree(tmp, ignore_errors=True)
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "topk_wide", "R": R, "M": M, "slice_mib": args.slice_mib or "default", "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "arms_ms": arms, "steps": steps, "parity_vs_oracle": {"requests": 512, "bit_exact": ok},
                  "note": "device arms: median CUDA-event time per graph replay; wideK_*: eppscore_schedule_batch_topk_wide; "
                          "topk8_registers_*: eppscore_schedule_batch_topk, k = 8; host_*: wall time of a host-buffer call, "
                          "score map = R x M float64 copied to the host (the host sort not included)"}))
