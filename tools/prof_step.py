"""Times the kernels of the headline step one by one (device-resident inputs, rotating input sets > L2) and the host-buffer
call at several chunk sizes.  usage: python tools/prof_step.py [what ...]   what in {hash, hash2, pick, step, probe, split, e2e, commit}
probe: the step's kernels one by one as the step runs them (the probing hash kernel, pick_sparse fed by its records), from a
torch.profiler trace of CUDA-graph replays over the rotating input sets, and the shares of resolved / table-path / deferred
requests: resolved counted by the engine (eppscore_stats.probe_resolved), deferred from the oracle's match counts."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

what = sys.argv[1:] or ["hash", "hash2", "pick", "step", "e2e", "commit"]
_pkg.load_build().build()
pkg = _pkg.load()
R, M, A = 65536, bench.M, bench.A
snap = synth_snapshot(M, A=A, seed=0)
o, osnap, prof, idx, seed, warm = bench.oracle_setup(snap)
eng = pkg.Engine(pkg.default_config(bench.SCORERS, max_endpoints=M, max_adapters=A, block_chars=bench.BLOCK_CHARS,
                                    max_blocks=bench.MAX_BLOCKS, prefix_capacity=1 << 19))
eng.set_snapshot(**snap)
eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
dev = torch.device("cuda:0")
stream = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(stream)
sp = stream.cuda_stream
NS = 4
host, sets = [], []
for i in range(NS):
    p, off, _ = synth_prompts(R, prompt_len=bench.PROMPT_LEN, groups=150, shared=1024, seed=i, prefix_seed=7)
    ad = zipf_adapters(R, A=A, seed=i)
    host.append((p, off, ad))
    sets.append(dict(p=torch.from_numpy(p).to(dev), off=torch.from_numpy(off).to(dev), ad=torch.from_numpy(ad).to(dev),
                     seeds=torch.from_numpy(np.full(R, seed, np.uint64).view(np.int64)).to(dev),
                     h=torch.zeros((R, bench.MAX_BLOCKS), dtype=torch.uint64, device=dev), n=torch.zeros(R, dtype=torch.uint16, device=dev)))
out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
           tie_count=torch.empty(R, dtype=torch.int32, device=dev))
L = pkg.lib()


def hash_only(i):
    d = sets[i % NS]
    assert L.eppscore_hash_prompts(eng._h, R, 1, d["p"].data_ptr(), d["off"].data_ptr(), None, d["seeds"].data_ptr(), bench.BLOCK_CHARS,
                                   bench.MAX_BLOCKS, d["h"].data_ptr(), d["n"].data_ptr(), sp) == 0


def pick_only(i):
    d = sets[i % NS]
    eng.schedule(R, hashes_in=d["h"], n_hashes_in=d["n"], hash_stride=bench.MAX_BLOCKS, adapter_id=d["ad"], device=True, stream=sp, out=out)


def step(i):
    d = sets[i % NS]
    eng.schedule(R, prompt_bytes=d["p"], prompt_off=d["off"], model_seed=d["seeds"], adapter_id=d["ad"], device=True, stream=sp, out=out)


def timeit(fn, iters=40, graph=True):
    """CUDA-event time per call; fn is captured into one CUDA graph per input set so the host's launch rate is not what is measured"""
    for i in range(NS):
        fn(i)
    call = fn
    if graph and "NOGRAPH" not in os.environ:
        torch.cuda.synchronize()
        gs = []
        for i in range(NS):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                fn(i)
            gs.append(g)
        call = lambda i: gs[i % NS].replay()  # noqa: E731
    for i in range(4):
        call(i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(stream)
    for i in range(iters):
        call(4 + i)
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3


for i in range(NS):
    hash_only(i)
torch.cuda.synchronize()
want = o.schedule_batch(osnap, prof, idx, 4096, prompt_bytes=host[0][0][: host[0][1][4096]], prompt_off=host[0][1][:4097],
                        model_seed=np.full(4096, seed, np.uint64), adapter_id=host[0][2][:4096], block_chars=bench.BLOCK_CHARS,
                        max_blocks=bench.MAX_BLOCKS, n_threads=os.cpu_count(), want_hashes=True)
assert np.array_equal(sets[0]["h"][:4096, :32].cpu().numpy().view(np.uint64), want["hashes_out"][:, :32]), "fused hash kernel differs"
if "hash" in what:
    print(f"hash (default)  : {timeit(hash_only):8.2f} us")
if "hash2" in what:
    for mask, name in ((1, "bodies only"), (2, "chain (warp tiles) only"), (18, "chain (r1 CTA tiles) only"), (8, "warp-tile fused"), (19, "bodies + chain"), (4, "CTA-tile fused")):
        eng.set_debug(2, mask)
        print(f"  {name:26s}: {timeit(hash_only):8.2f} us")
    eng.set_debug(2, 0)
    for i in range(NS):
        hash_only(i)
if "pick" in what:
    print(f"pick_sparse     : {timeit(pick_only):8.2f} us")
    pick_only(0)
    torch.cuda.synchronize()
    assert np.array_equal(out["pick"][:4096].cpu().numpy(), want["pick"]) and np.array_equal(out["pick_score"][:4096].cpu().numpy(), want["pick_score"])
if "step" in what:
    print(f"hash + pick     : {timeit(step):8.2f} us (direct launches, snapshot not re-prepared)")
if "probe" in what:
    from torch.profiler import ProfilerActivity, profile
    from tests.score_constants import score_constants
    for i in range(NS):
        step(i)
    torch.cuda.synchronize()
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
    per = {}
    for ev in tr.key_averages():
        if ev.device_type.name == "CUDA" and ev.count > 0:
            per[ev.key] = (ev.self_device_time_total if hasattr(ev, "self_device_time_total") else ev.self_cuda_time_total, ev.count)
    for k, (tot, n) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print(f"  {k[:90]:90s}: {tot / iters:8.2f} us per step ({n // iters} per step)")
    print(f"hash + pick     : {timeit(step):8.2f} us (graph, no profiler)")
    resolved = []
    for i in range(NS):
        r0 = eng.stats().probe_resolved
        step(i)
        torch.cuda.synchronize()
        resolved.append((eng.stats().probe_resolved - r0) % (1 << 32))
    kx = score_constants().exc_max
    full = o.schedule_batch(osnap, prof, idx, R, prompt_bytes=host[0][0], prompt_off=host[0][1], model_seed=np.full(R, seed, np.uint64),
                            adapter_id=host[0][2], block_chars=bench.BLOCK_CHARS, max_blocks=bench.MAX_BLOCKS, n_threads=os.cpu_count(),
                            want_match=True)
    deferred = int(((full["match_blocks"] > 0).sum(axis=1) > kx).sum())
    step(0)
    torch.cuda.synchronize()
    assert np.array_equal(out["pick"].cpu().numpy(), full["pick"]) and np.array_equal(out["pick_score"].cpu().numpy(), full["pick_score"])
    print(f"resolved by the hash kernel: {resolved} of {R} per set; set 0: resolved {resolved[0] / R:.4f}, "
          f"deferred {deferred / R:.4f}, table path {(R - resolved[0] - deferred) / R:.4f}")
if "split" in what:
    # the body kernel's two forms, then the device-resident batch cut into slices over several streams (debug keys 5 / 6)
    for mask, name in ((1, "bodies, one-shot"), (33, "bodies, pipelined (exp.)")):
        eng.set_debug(2, mask)
        print(f"  {name:26s}: {timeit(hash_only):8.2f} us")
    eng.set_debug(2, 19)
    for i in range(NS):
        hash_only(i)
    for mask in (19,):
        eng.set_debug(2, mask)
        for split, streams in ((1, 1), (2, 2), (4, 2), (4, 3), (8, 2), (8, 3), (8, 4), (16, 4)):
            eng.set_debug(5, split)
            eng.set_debug(6, streams)
            t = timeit(step)
            out["pick"].zero_()
            step(0)
            torch.cuda.synchronize()
            ok = np.array_equal(out["pick"][:4096].cpu().numpy(), want["pick"]) and np.array_equal(out["pick_score"][:4096].cpu().numpy(), want["pick_score"])
            print(f"hash + pick, {split:2d} slices / {streams} streams: {t:8.2f} us  parity {'ok' if ok else 'FAILED'}")
    eng.set_debug(2, 0)
    eng.set_debug(5, 1)
if "e2e" in what:
    pin = []
    for p, off, ad in host:
        t = [torch.from_numpy(x).pin_memory() for x in (p, off, ad, np.full(R, seed, np.uint64).view(np.int64))]
        pin.append(t)
    for chunk in (0, 4096, 8192, 16384):
        eng.set_debug(3, chunk)
        ts = []
        for i in range(12):
            hp, ho, ha, hs = pin[i % NS]
            t0 = time.perf_counter()
            r = eng.schedule(R, prompt_bytes=hp.numpy(), prompt_off=ho.numpy(), model_seed=hs.numpy().view(np.uint64), adapter_id=ha.numpy(),
                             want_total=False)
            ts.append(time.perf_counter() - t0)
        assert np.array_equal(r["pick"][:4096], o.schedule_batch(osnap, prof, idx, 4096, prompt_bytes=host[11 % NS][0][: host[11 % NS][1][4096]],
                                                                 prompt_off=host[11 % NS][1][:4097], model_seed=np.full(4096, seed, np.uint64),
                                                                 adapter_id=host[11 % NS][2][:4096], block_chars=bench.BLOCK_CHARS,
                                                                 max_blocks=bench.MAX_BLOCKS, n_threads=os.cpu_count())["pick"])
        med = float(np.median(ts[2:]))
        print(f"e2e chunk {chunk:6d}: {med * 1e3:7.3f} ms  {R / med / 1e6:6.1f} M picks/s  ({135.6e6 / med / 1e9:.1f} GB/s H2D)")
    eng.set_debug(3, 8192)
if "commit" in what:
    # closed loop on the device: schedule -> commit, K batches
    outc = dict(out, total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                hashes_out=torch.zeros((R, bench.MAX_BLOCKS), dtype=torch.uint64, device=dev))

    def loop(i):
        d = sets[i % NS]
        eng.schedule(R, prompt_bytes=d["p"], prompt_off=d["off"], model_seed=d["seeds"], adapter_id=d["ad"], device=True, stream=sp, out=outc)
        eng.commit_picks_device(outc["pick"], outc["hashes_out"], outc["total_blocks"], touch_bound=R * 32, stream=sp)

    t = timeit(loop, iters=8, graph=False)
    st = eng.stats()
    print(f"schedule+commit : {t:8.2f} us per 64K batch = {R / t:.1f} M requests/s; live {st.prefix_live_hashes} used {st.prefix_hashes} "
          f"lru {st.lru_entries} rebuilds {st.prefix_rebuilds} err {st.index_error}")
