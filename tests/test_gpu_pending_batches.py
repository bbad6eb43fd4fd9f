"""Ordering of the engine's rewrites against device-location batches that are still running on caller streams: the index,
the snapshot terms and the shared scratch are rewritten only after every such batch has finished with them."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests.helpers import synth_prompts, synth_snapshot
from tests.test_gpu_parity import assert_same, make_engine, profile_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


@pytest.mark.parametrize("between", ["host_batch", "other_stream"])
def test_commit_waits_for_every_pending_device_batch(pkg, between):
    """A device-location batch still queued on caller stream S1 (behind a ~1 s spin) reads the index as it was when the batch
    was issued, although a host commit that changes its matches follows it.  In between runs either a host-location batch
    or a device-location batch on a second stream S2: neither may make the commit forget the batch on S1."""
    import torch
    M, R, mb = 256, 4096, 16
    scorers = [("queue", 2), ("kv", 2), ("prefix", 3)]
    eng = make_engine(pkg, scorers, M, max_blocks=mb, prefix_capacity=1 << 18)
    sd = synth_snapshot(M, seed=13)
    eng.set_snapshot(**sd)
    snap, prof, idx = o.SnapshotData(**sd), profile_of(pkg, scorers), o.Index()
    # an earlier, larger commit on both sides, so the calls below find every buffer they use already allocated
    wp, woff, _ = synth_prompts(2 * R, prompt_len=640, groups=16, shared=320, seed=14)
    wseeds = np.full(2 * R, eng.model_seed("warm"), np.uint64)
    warm = o.schedule_batch(snap, prof, idx, 2 * R, prompt_bytes=wp, prompt_off=woff, model_seed=wseeds, max_blocks=mb,
                            want_hashes=True, n_threads=8)
    idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    prompts, off, _ = synth_prompts(R, prompt_len=640, groups=16, shared=320, seed=15)
    seeds = np.full(R, eng.model_seed("pending"), np.uint64)
    want = o.schedule_batch(snap, prof, idx, R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, max_blocks=mb,
                            want_hashes=True, n_threads=8)
    # the commit moves every request's blocks to another endpoint: after it, the picks change
    moved = ((want["pick"] + 1) % M).astype(np.int32)
    idx.commit(moved, want["hashes_out"], want["total_blocks"])
    after = o.schedule_batch(snap, prof, idx, R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, max_blocks=mb, n_threads=8)
    assert (after["pick"] != want["pick"]).mean() > 0.5

    dev = torch.device("cuda", 0)
    s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    d_in = dict(prompt_bytes=torch.from_numpy(prompts).to(dev), prompt_off=torch.from_numpy(off).to(dev),
                model_seed=torch.from_numpy(seeds.view(np.int64)).to(dev))

    def outputs():
        return dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                    tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                    hashes_out=torch.zeros((R, mb), dtype=torch.uint64, device=dev))
    out1, out2 = outputs(), outputs()

    def batches(spin):
        with torch.cuda.stream(s1):
            if spin:
                torch.cuda._sleep(2_000_000_000)  # ~1 s of clock cycles: the batch below is still queued when the commit is issued
            eng.schedule(R, device=True, stream=s1.cuda_stream, out=out1, **d_in)
        if between == "host_batch":  # R / 2 < 2 x 8192 requests: one chunk, on the engine stream, in scratch set 0
            eng.schedule(R // 2, prompt_bytes=prompts, prompt_off=off[: R // 2 + 1], model_seed=seeds[: R // 2])
        else:  # the same requests: the shared scratch set 0 receives the same values
            with torch.cuda.stream(s2):
                eng.schedule(R, device=True, stream=s2.cuda_stream, out=out2, **d_in)

    torch.cuda.synchronize()
    batches(spin=False)  # sizes the scratch the calls below use
    torch.cuda.synchronize()
    batches(spin=True)
    eng.commit_picks(moved, want["hashes_out"], want["total_blocks"])
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out1.items()}
    assert_same(got, want, ("pick", "pick_score", "tie_count", "total_blocks"))
    eng.close()


