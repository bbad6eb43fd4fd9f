"""A fixed sequence of batches on the GPU, one for each way a batch is cut: a chunked host batch (debug key 3), a sliced device
batch (keys 5 / 6), a wide top-k batch and a profiles top-k batch with a wide run.  Prints one JSON line with the engine's
stats().kernel_launches after the sequence and a digest of every output, so that two builds can be compared: a change to
host code alone leaves both as they were.

    python tools/count_launches.py"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import _pkg  # noqa: E402
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters  # noqa: E402

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("count_launches needs a CUDA device")
    pkg = _pkg.load()
    M, R = 1024, 6400
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, prefix_capacity=1 << 16))
    eng.set_snapshot(**synth_snapshot(M, seed=5))
    pid = eng.add_profile([("kv", 1), ("prefix", 2)], pick_mode=1)
    seed = eng.model_seed("count-launches")
    wp, woff, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=5)
    warm = eng.schedule(R, prompt_bytes=wp, prompt_off=woff, model_seed=np.full(R, seed, np.uint64), want_hashes=True)
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=6, prefix_seed=5)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, seed, np.uint64), adapter_id=zipf_adapters(R, seed=6))
    digest = hashlib.sha256()

    def add(outputs):
        for key in sorted(outputs):
            digest.update(key.encode())
            digest.update(np.ascontiguousarray(outputs[key]).tobytes())

    eng.set_debug(3, 1000)  # host batch in chunks of 1000 requests
    add(eng.schedule(R, topk=4, want_hashes=True, **kw))
    eng.set_debug(3, 8192)

    eng.set_debug(5, 3)  # device batch in three slices over two streams
    eng.set_debug(6, 2)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}
    out = dict(pick=torch.empty(R, dtype=torch.int32, device="cuda"), pick_score=torch.empty(R, dtype=torch.float64, device="cuda"),
               tie_count=torch.empty(R, dtype=torch.int32, device="cuda"), total_blocks=torch.empty(R, dtype=torch.int16, device="cuda"),
               topk_pick=torch.empty((R, 4), dtype=torch.int32, device="cuda"),
               topk_score=torch.empty((R, 4), dtype=torch.float64, device="cuda"))
    eng.schedule(R, topk=4, device=True, out=out, **dev)
    torch.cuda.synchronize()
    add({k: v.cpu().numpy() for k, v in out.items()})
    eng.set_debug(5, 1)

    add(eng.schedule(R, topk_wide=40, **kw))
    res, runs = eng.schedule_profiles(R, [dict(profile=0, topk=4), dict(profile=pid, topk=24)], **kw)
    add(res)
    for i, r in enumerate(runs):
        add({f"{i}.{k}": v for k, v in r.items()})
    print(json.dumps(dict(kernel_launches=int(eng.stats().kernel_launches), outputs_sha256=digest.hexdigest())))
    eng.close()


if __name__ == "__main__":
    main()
