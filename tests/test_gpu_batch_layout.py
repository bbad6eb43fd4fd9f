"""A batch's per-request arrays on every way of running it, on the GPU: one batch that sets every optional per-request array,
then a second one that brings its hashes as hashes_in.  The host call, chunks of a size that is not a multiple of 64 (debug
key 3) and device buffers with the slicing keys (5 / 6) set give the uncut device call's outputs bit for bit, so every array is
cut, staged and returned at the same rows on every route."""
import numpy as np
import pytest

import _pkg
from tests.helpers import zipf_adapters
from tests.test_gpu_profiles_topk import LAT_COEF, _dev_runs, random_masks, world

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def test_every_optional_array_on_every_route(pkg):
    """inputs prompt_len, input_tokens, ttft_slo / tpot_slo (a latency profile behind device filters), adapter_id, cand_mask
    and hashes_in / n_hashes_in; outputs total_blocks, hashes_out, filter_mask_out and two lists, k = 4 and a wide k = 24
    (the wide run's score scratch holds fewer rows than the batch, so that run is cut as well)"""
    import torch
    M, R = 1024, 4608
    make, _, _, sd, kw = world(pkg, M, 44, R=R)
    eng = make()
    eng.set_latency_params(pkg.latency_params(**LAT_COEF))
    lat = eng.add_profile([("latency", 1), ("kv", 0.5)], filters=[(1, (0.5, 0.0, 5000.0)), (2, (0.01, 0, 0))])
    eng.set_snapshot(**sd)
    rng = np.random.Generator(np.random.PCG64(46))
    per_request = dict(model_seed=kw["model_seed"], adapter_id=zipf_adapters(R, seed=46),
                       input_tokens=rng.integers(0, 6000, R).astype(np.int32), ttft_slo=rng.uniform(0, 2000, R),
                       tpot_slo=rng.uniform(0, 80, R))
    off = kw["prompt_off"]
    prompts = dict(per_request, prompt_bytes=kw["prompt_bytes"], prompt_off=off,
                   prompt_len=np.maximum(np.diff(off) - rng.integers(0, 200, R), 0).astype(np.int32))
    runs = [(0, random_masks(R, M, rng), 4), (lat, None, 24)]
    mw = (M + 31) // 32

    def signed(a):
        a = np.ascontiguousarray(a)
        return a.view(a.dtype.str.replace("u", "i"))

    def host(bkw, hashes):
        res, got = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m, topk=k, want_filter_mask=p == lat) for p, m, k in runs],
                                         want_hashes=hashes, **bkw)
        return dict(res, **{f"{i}.{x}": v for i, g in enumerate(got) for x, v in g.items()})

    def device(bkw, hashes):
        druns = _dev_runs(R, [(p, None, k) for p, _, k in runs])
        druns[0]["cand_mask"] = torch.from_numpy(signed(runs[0][1])).cuda()
        druns[1]["filter_mask_out"] = torch.zeros((R, mw), dtype=torch.int32, device="cuda")
        out = dict(total_blocks=torch.zeros(R, dtype=torch.int16, device="cuda"))
        if hashes:
            out["hashes_out"] = torch.zeros((R, eng.cfg.max_blocks), dtype=torch.int64, device="cuda")
        eng.schedule_profiles(R, druns, device=True, out=out, **{k: torch.from_numpy(signed(v)).cuda() for k, v in bkw.items()})
        torch.cuda.synchronize()
        got = {k: v.cpu().numpy() for k, v in out.items()}
        for i, d in enumerate(druns):
            got.update({f"{i}.{x}": d[x].cpu().numpy() for x in ("pick", "pick_score", "tie_count", "topk_pick", "topk_score",
                                                                  "filter_mask_out") if x in d})
        return got

    def same_bytes(got, want, what):
        assert sorted(got) == sorted(want), what
        for x in want:
            assert got[x].shape == want[x].shape and got[x].tobytes() == want[x].tobytes(), (what, x)

    first = host(prompts, True)
    from_hashes = dict(per_request, hashes_in=first["hashes_out"],
                       n_hashes_in=np.minimum(first["total_blocks"], eng.cfg.max_blocks).astype(np.uint16))
    for name, bkw, hashes in (("prompts", prompts, True), ("hashes_in", from_hashes, False)):
        ref = device(bkw, hashes)
        same_bytes(host(bkw, hashes), ref, (name, "host"))
        eng.set_debug(3, 1000)
        same_bytes(host(bkw, hashes), ref, (name, "chunked"))
        eng.set_debug(3, 8192)
        for split, streams in ((3, 2), (4, 3)):
            eng.set_debug(5, split)
            eng.set_debug(6, streams)
            same_bytes(device(bkw, hashes), ref, (name, "sliced", split, streams))
        eng.set_debug(5, 1)
        eng.set_debug(6, 2)
    eng.close()
