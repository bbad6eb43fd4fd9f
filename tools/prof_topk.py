"""maxNumOfEndpoints at the headline shape (64K requests x 1024 endpoints, four scorers, warmed index, device-resident
block hashes): the device time of eppscore_schedule_batch_topk against the route the host layer takes for k > 8 (the
whole R x M float64 score map written to HBM), plus a 512-request parity check of the lists against the CPU oracle.
Prints one JSON line with the GPU's name and power limit.  usage: prof_topk.py [iters]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests import topk_oracle as T  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
NSETS = 3
pkg = _pkg.load()
R, M, A = 65536, bench.M, bench.A
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sptr = stream.cuda_stream


def make_engine(**kw):
    e = pkg.Engine(pkg.default_config(bench.SCORERS, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                      max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19, **kw))
    e.set_snapshot(**snap)
    e.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    return e


eng = make_engine()
sets, host_sets = [], []
for i in range(NSETS):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=100 + i, prefix_seed=7)
    ad = zipf_adapters(R, A=A, seed=100 + i)
    h, n = eng.hash_prompts(p, off, np.full(R, seed, np.uint64), block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS)
    host_sets.append((h, n, ad))
    sets.append((torch.from_numpy(h.view(np.int64)).to(dev), torch.from_numpy(n.view(np.int16)).to(dev), torch.from_numpy(ad).to(dev)))


def outputs(k=0, scores=False):
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    if k:
        out["topk_pick"] = torch.empty((R, k), dtype=torch.int32, device=dev)
        out["topk_score"] = torch.empty((R, k), dtype=torch.float64, device=dev)
    if scores:
        out["scores_out"] = torch.empty((R, M), dtype=torch.float64, device=dev)
    return out


def call(e, i, k, out):
    hh, nn, ad = sets[i % NSETS]
    e.schedule(R, hashes_in=hh, n_hashes_in=nn, hash_stride=bench.MAX_BLOCKS, adapter_id=ad, topk=k, device=True, stream=sptr,
               out=out)


def time_us(e, k, out):
    """CUDA-event time per call, each input set captured into its own CUDA graph"""
    for i in range(NSETS):
        call(e, i, k, out)
    torch.cuda.synchronize()
    graphs = []
    for i in range(NSETS):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            call(e, i, k, out)
        graphs.append(g)
    for i in range(3):
        graphs[i % NSETS].replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(stream)
    for i in range(ITERS):
        graphs[i % NSETS].replay()
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / ITERS * 1e3


def parity(e, pick_mode, tie_seed, k, out, n=512):
    call(e, 0, k, out)
    torch.cuda.synchronize()
    h, nh, ad = host_sets[0]
    p = o.make_profile([({"queue": 0, "kv": 1, "prefix": 2, "lora": 3}[s], w) for s, w in bench.SCORERS], pick_mode=pick_mode,
                       tie_seed=tie_seed)
    want = T.schedule_batch(osnap, p, idx, n, topk=k, hashes_in=h[:n], n_hashes_in=nh[:n], adapter_id=ad[:n],
                            max_blocks=bench.MAX_BLOCKS, n_threads=os.cpu_count() or 1)
    return bool(np.array_equal(out["topk_pick"][:n].cpu().numpy(), want["topk_pick"]) and
                np.array_equal(out["topk_score"][:n].cpu().numpy().view(np.uint64), want["topk_score"].view(np.uint64)) and
                np.array_equal(out["pick"][:n].cpu().numpy(), want["pick"]))


arms, ok = {}, {}
o1, o4 = outputs(1), outputs(4)
eng.set_debug(1, 1)  # the fully general kernels: without a list this is score_matrix_kernel<E,P,L>
arms["k0_generic_matrix"] = time_us(eng, 0, outputs())
arms["k1_generic_matrix"] = time_us(eng, 1, o1)
eng.set_debug(1, 0)
arms["k4_max_score"] = time_us(eng, 4, o4)
ok["k4_max_score"] = parity(eng, 0, 0, 4, o4)
os_ = outputs(scores=True)
arms["scores_out_max_score"] = time_us(eng, 0, os_)
del os_
eng.close()
eng_w = make_engine(pick_mode=pkg.PICK_WEIGHTED_RANDOM, tie_seed=3)
arms["k4_weighted_random"] = time_us(eng_w, 4, o4)
ok["k4_weighted_random"] = parity(eng_w, 1, 3, 4, o4)
eng_w.close()
del idx  # the oracle's index, freed while its library is still loaded
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True)
print(json.dumps({"leg": "topk_pickers", "R": R, "M": M, "gpu": torch.cuda.get_device_name(dev),
                  "power_limit_w": float(q.stdout.split()[0]) if q.returncode == 0 and q.stdout.strip() else None,
                  "arms": {k: {"us": t, "picks_per_s": R / (t * 1e-6)} for k, t in arms.items()},
                  "parity_vs_oracle": {"requests": 512, "bit_exact": ok},
                  "note": "k0/k1_generic_matrix: engine debug key 1 without / with a one-entry list; k4_*: "
                          "eppscore_schedule_batch_topk, k = 4; scores_out_max_score: the R x M float64 score map written to HBM "
                          "(device time only, no copy to the host)"}))
