"""A fixed sequence of batches on the GPU, one for each way a batch is cut: a chunked host batch (debug key 3), a sliced device
batch (keys 5 / 6), a wide top-k batch and a profiles top-k batch with a wide run; then an in-order batch and the token
estimate, hash, field-count, prefix-match and latency-info calls, each on host and on device arrays (the latency info on a
second engine whose profile has the latency scorer).  Prints one JSON line with the engines' stats().kernel_launches after
the sequence and a digest of every output, so that two builds can be compared: a change to host code alone leaves both as
they were.

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

    # the in-order batch on host and on device arrays, then the calls that stage host arrays, in both locations
    lib = pkg.lib()
    tok = eng.estimate_tokens(R, prompt_chars=np.diff(off).astype(np.int32))
    d_tok = torch.empty(R, dtype=torch.int64, device="cuda")
    eng.estimate_tokens(R, prompt_chars=torch.from_numpy(np.diff(off).astype(np.int32)).cuda(), device=True, out=d_tok)
    add(dict(tokens=tok, d_tokens=d_tok.cpu().numpy()))
    add(eng.schedule_inorder(R, tokens=tok, want_hashes=True, **kw))
    io = {k: out[k] for k in ("pick", "pick_score", "tie_count", "total_blocks")}
    eng.schedule_inorder(R, tokens=d_tok, device=True, out=io, **dev)
    torch.cuda.synchronize()
    add({f"io.{k}": v.cpu().numpy() for k, v in io.items()})
    add(dict(zip(("inflight_req", "inflight_tok"), eng.inflight_get(M))))
    hashes, nh = eng.hash_prompts(prompts, off, kw["model_seed"])
    d_hashes = torch.zeros(hashes.shape, dtype=torch.int64, device="cuda")
    d_nh = torch.zeros(R, dtype=torch.int16, device="cuda")
    d_fields = torch.zeros(R, dtype=torch.int32, device="cuda")
    assert lib.eppscore_hash_prompts(eng._h, R, 1, dev["prompt_bytes"].data_ptr(), dev["prompt_off"].data_ptr(), None,
                                     dev["model_seed"].data_ptr(), 0, 0, d_hashes.data_ptr(), d_nh.data_ptr(), None) == 0
    assert lib.eppscore_count_fields(eng._h, R, 1, dev["prompt_bytes"].data_ptr(), dev["prompt_off"].data_ptr(), None,
                                     d_fields.data_ptr(), None) == 0
    torch.cuda.synchronize()
    add(dict(hashes=hashes, nh=nh, fields=eng.count_fields(prompts, off), d_hashes=d_hashes.cpu().numpy(),
             d_nh=d_nh.cpu().numpy(), d_fields=d_fields.cpu().numpy()))
    eps = np.stack([warm["pick"], (warm["pick"] + 1) % M], axis=1).astype(np.int32)
    d_eps, d_h, d_n = torch.from_numpy(eps).cuda(), torch.from_numpy(hashes.view(np.int64)).cuda(), torch.from_numpy(nh.view(np.int16)).cuda()
    d_match = torch.zeros(eps.shape, dtype=torch.int16, device="cuda")
    eng.prefix_match(d_h, d_n, d_eps, device=True, out=d_match)
    torch.cuda.synchronize()
    add(dict(match=eng.prefix_match(hashes, nh, eps), d_match=d_match.cpu().numpy()))

    # predict_latency on an engine whose profile has the latency scorer
    lat = pkg.Engine(pkg.default_config([("latency", 1), ("prefix", 1)], max_endpoints=M, prefix_capacity=1 << 16))
    lat.set_latency_params(pkg.latency_params())
    lat.set_snapshot(**synth_snapshot(M, seed=5))
    lat.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    in_tok = np.diff(off).astype(np.int32) // 4
    info, match = lat.predict_latency(hashes, nh, eps, input_tokens=in_tok, match_out=True)
    d_info = torch.zeros((R, 2, 48), dtype=torch.uint8, device="cuda")
    lat.predict_latency(d_h, d_n, d_eps, input_tokens=torch.from_numpy(in_tok).cuda(), device=True, out=d_info, match_out=d_match)
    torch.cuda.synchronize()
    add(dict(info=info, lat_match=match, d_info=d_info.cpu().numpy(), d_lat_match=d_match.cpu().numpy()))
    launches = int(eng.stats().kernel_launches) + int(lat.stats().kernel_launches)
    print(json.dumps(dict(kernel_launches=launches, outputs_sha256=digest.hexdigest())))
    lat.close()
    eng.close()


if __name__ == "__main__":
    main()
