"""The device-resident closed loop with a reserved prefix index (eppscore_prefix_reserve), on the GPU.  One step is
schedule -> commit_picks_device -> estimate_tokens -> inflight_add -> inflight_release (the step before last), the headline
profile plus the token-load scorer, M = 256 endpoints, 1 KiB prompts (16 blocks), R in {1024, 4096, 16384, 65536}, a
snapshot with many tied endpoints and seeded-random tie-breaking:
  - eager on an unreserved engine (the commit passes touch_bound = R * 16, as a caller that knows its shapes does),
  - eager on a reserved engine (no host wait inside the commit),
  - one CUDA graph per step on a reserved engine.
Step time = host clock around `--steps` back-to-back steps ending in a device synchronise, median of `--rounds` alternating
rounds.  Then the cost of one same-size device rebuild at the reserved size: kernel times (torch.profiler, a run of its
own) of the room kernels over an eager reserved loop that churns the table, with and without a rebuild due.  Prints one
JSON line; --out writes it.

    python tools/prof_index_graph.py [--rounds 5] [--steps 20] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 2)]
SIZES = (1024, 4096, 16384, 65536)
M, MB, PLEN, LRU = 256, 16, 1024, 4096


def _engine(pkg, reserve_touches, lru=LRU):
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, token_load_threshold=1e9, max_blocks=MB, prefix_capacity=1 << 20,
                                        lru_capacity_default=lru, tie_mode=pkg.TIE_SEEDED_RANDOM))
    eng.set_snapshot(**synth_snapshot(M, seed=1, tie_heavy=True))
    if reserve_touches:
        eng.prefix_reserve(M * lru, reserve_touches, 0)
    return eng


class Step:
    def __init__(self, eng, R, reserved, seed):
        import torch
        self.eng, self.R, self.reserved = eng, R, reserved
        cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        p, off, _ = synth_prompts(R, prompt_len=PLEN, groups=64, shared=256, seed=seed, prefix_seed=1)
        self.d = dict(prompt_bytes=cuda(p), prompt_off=cuda(off), model_seed=cuda(np.full(R, 0x5EED, np.uint64).view(np.int64)),
                      adapter_id=cuda(zipf_adapters(R, seed=seed)))
        self.chars = cuda(np.full(R, PLEN, np.int32))
        dev = "cuda"
        self.out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                        tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                        hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
        self.est = torch.empty(R, dtype=torch.int64, device=dev)
        self.prev = torch.full((R,), -1, dtype=torch.int32, device=dev)
        self.s = torch.cuda.Stream()
        self.g = None

    def body(self):
        e, o, s = self.eng, self.out, self.s.cuda_stream
        e.schedule(self.R, device=True, stream=s, out=o, **self.d)
        e.commit_picks_device(o["pick"], o["hashes_out"], o["total_blocks"], touch_bound=0 if self.reserved else self.R * MB, stream=s)
        e.estimate_tokens(self.R, prompt_chars=self.chars, device=True, stream=s, out=self.est)
        e.inflight_add(o["pick"], self.est, device=True, stream=s)
        e.inflight_release(self.prev, self.est, device=True, stream=s)

    def capture(self):
        import torch
        self.body()
        torch.cuda.synchronize()
        self.g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g, stream=self.s):
            self.body()
        torch.cuda.synchronize()

    def run(self, n):
        import torch
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            if self.g is not None:
                self.g.replay()
            else:
                self.body()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n


ROOM_KERNELS = ("index_room_kernel", "table_clear_spare_kernel", "table_rebuild_kernel")


def rebuild_cost(pkg, R, steps):
    """Eager reserved steps with fresh prompts each time; LRUs of 128 blocks keep the live set small, so that the churn
    rebuilds a table sized for it every few steps.  Kernel times of the room kernels per commit (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng = _engine(pkg, R * MB, lru=128)
    st = Step(eng, R, True, seed=7)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(steps):
            p, _, _ = synth_prompts(R, prompt_len=PLEN, groups=64, shared=256, seed=1000 + k, prefix_seed=1)
            st.d["prompt_bytes"].copy_(torch.from_numpy(p))
            eng.schedule(R, device=True, stream=st.s.cuda_stream, out=st.out, **st.d)
            eng.commit_picks_device(st.out["pick"], st.out["hashes_out"], st.out["total_blocks"], stream=st.s.cuda_stream)
            torch.cuda.synchronize()
    t = {n: [] for n in ROOM_KERNELS + ("index_commit_kernel",)}
    for ev in prof.events():
        for n in t:
            if n in ev.name:
                t[n].append(ev.time_range.elapsed_us())
    s = eng.stats()
    reb = sorted(t["table_rebuild_kernel"])
    n_reb = int(s.prefix_rebuilds)
    res = dict(R=R, slots_per_table=2 * s.prefix_capacity, table_bytes=s.prefix_table_bytes, commits=steps, rebuilds=n_reb,
               room_kernel_us=float(np.median(t["index_room_kernel"])),
               clear_us_idle=float(np.median(sorted(t["table_clear_spare_kernel"])[: steps - n_reb])),
               rebuild_us_idle=float(np.median(reb[: steps - n_reb])),
               clear_us_due=float(np.median(sorted(t["table_clear_spare_kernel"])[steps - n_reb:])) if n_reb else None,
               rebuild_us_due=float(np.median(reb[steps - n_reb:])) if n_reb else None,
               commit_kernel_us=float(np.median(t["index_commit_kernel"])))
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_index_graph needs a CUDA device")
    pkg = _pkg.load()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, M=M, blocks=MB, lru=LRU, steps=args.steps, rounds=args.rounds, loop={})
    for R in SIZES:
        arms = {"eager_unreserved": Step(_engine(pkg, 0), R, False, 3), "eager_reserved": Step(_engine(pkg, R * MB), R, True, 3),
                "graph_reserved": Step(_engine(pkg, R * MB), R, True, 3)}
        arms["graph_reserved"].capture()
        for a in arms.values():
            a.run(3)  # warm
        t = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, a in arms.items():
                t[k].append(a.run(args.steps))
        res["loop"][R] = {k: round(float(np.median(v)) * 1e6, 1) for k, v in t.items()}
        res["loop"][R]["slots_reserved"] = 2 * arms["eager_reserved"].eng.stats().prefix_capacity
        for a in arms.values():
            a.eng.close()
    res["rebuild"] = [rebuild_cost(pkg, R, 30) for R in (4096, 16384)]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
