"""eppscore_schedule_batch_inorder on the GPU, bit-exact against the sequential reference (tests/inorder_reference.py: R
single-request oracle schedules, each followed by the in-flight add of its pick): picks, scores, tie counts, totals and the
counters eppscore_inflight_get returns afterwards — over endpoint counts from 1 to 8192, batches up to 64K, every pick and tie
mode, candidate masks, supplied hashes, a token-load-only profile and the four-scorer profile plus token-load; in host, device,
reserved-stream and CUDA-graph execution; and the refusals, which leave the counters untouched."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.helpers import synth_ragged_prompts, synth_snapshot, zipf_adapters
from tests.inorder_reference import schedule_inorder

pytestmark = pytest.mark.gpu

FOUR = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 1)]
TL = [("token_load", 1)]
THR = 20000.0
MB = 16


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


class World:
    """An engine and its oracle twin: the same snapshot, one committed warm-up batch in both indexes, the same counters."""

    def __init__(self, pkg, M, scorers, pick_mode=0, tie_mode=0, seed=0):
        self.pkg, self.M = pkg, M
        self.eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=max(M, 64), token_load_threshold=THR, max_blocks=MB,
                                                 prefix_capacity=1 << 16, pick_mode=pick_mode, tie_mode=tie_mode, tie_seed=77))
        self.sd = synth_snapshot(M, seed=seed)
        self.eng.set_snapshot(**self.sd)
        self.prof = o.make_profile([(pkg.SCORER[s], w) for s, w in scorers], tie_mode=tie_mode, tie_seed=77,
                                   token_load_threshold=THR, pick_mode=pick_mode)
        self.idx, self.tracker = o.Index(), I.Tracker()
        self.rng = np.random.Generator(np.random.PCG64(seed + 5))
        w = self.workload(256, seed + 1)
        warm = self.eng.schedule(256, want_hashes=True, max_blocks=MB, **w)
        self.eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
        self.idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])

    def workload(self, R, seed):
        pb, off = synth_ragged_prompts(R, max_len=MB * 64, seed=seed)
        return dict(prompt_bytes=pb, prompt_off=off, model_seed=np.full(R, 5, np.uint64), adapter_id=zipf_adapters(R, seed=seed))

    def masks(self, R):
        mw = (self.M + 31) // 32
        m = self.rng.integers(0, 2 ** 32, size=(R, mw), dtype=np.uint64).astype(np.uint32)
        m[::7] = 0  # requests without candidates
        return m

    def tokens(self, R):
        return self.rng.integers(0, 3000, size=R).astype(np.int64)

    def reference(self, R, tokens, request_base=0, **kw):
        want, _ = schedule_inorder(self.sd, self.prof, self.idx, R, tokens, tracker=self.tracker, request_base=request_base,
                                   max_blocks=MB, **kw)
        return want

    def check(self, got, want, what):
        for k in ("pick", "tie_count", "total_blocks"):
            assert np.array_equal(np.asarray(got[k]), want[k]), (what, k)
        assert np.array_equal(np.asarray(got["pick_score"]).view(np.uint64), want["pick_score"].view(np.uint64)), what
        req, tok = self.eng.inflight_get(self.M)
        wreq, wtok = self.tracker.get(self.M)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), what


CASES = [  # (M, R, scorers, pick_mode, tie_mode, masked)
    (1, 31, FOUR, 0, 0, False),
    (5, 31, FOUR, 1, 1, True),
    (33, 31, TL, 2, 1, False),
    (1024, 1, FOUR, 0, 1, False),
    (1024, 4096, FOUR, 0, 0, True),
    (1024, 4096, FOUR, 1, 0, False),
    (1024, 4096, TL, 0, 1, False),
    (4097, 31, FOUR, 2, 0, True),
    (8192, 31, FOUR, 0, 1, False),
    (8192, 31, TL, 1, 1, True),
    (8192, 2500, FOUR, 0, 1, True),  # two slices of 2048 rows: the counters carry from one slice to the next
]


@pytest.mark.parametrize("M,R,scorers,pick_mode,tie_mode,masked", CASES)
def test_host_batch_matches_sequential_reference(pkg, M, R, scorers, pick_mode, tie_mode, masked):
    w = World(pkg, M, scorers, pick_mode, tie_mode, seed=M + R)
    kw = w.workload(R, 3)
    mask = w.masks(R) if masked else None
    tok = w.tokens(R)
    for rnd in range(2):  # the second batch starts from the counters the first left
        got = w.eng.schedule_inorder(R, tokens=tok, cand_mask=mask, max_blocks=MB, request_base=rnd * R, **kw)
        want = w.reference(R, tok, request_base=rnd * R, cand_mask=mask, **kw)
        w.check(got, want, (M, R, rnd))
    w.eng.close()


def test_64k_batch_every_request(pkg):
    R = 65536
    w = World(pkg, 1024, FOUR, seed=64)
    kw = w.workload(R, 11)
    tok = w.tokens(R)
    got = w.eng.schedule_inorder(R, tokens=tok, max_blocks=MB, **kw)
    want = w.reference(R, tok, **kw)
    w.check(got, want, "64K")
    w.eng.close()


@pytest.mark.parametrize("M,R", [(1024, 512), (8192, 2500)])
def test_hashes_in_and_plain_schedule_after(pkg, M, R):
    """supplied hashes (at 8192 endpoints over two slices); and a plain eppscore_schedule_batch after the call sees what it sees
    after the sequential loop"""
    w = World(pkg, M, FOUR, seed=21)
    kw = w.workload(R, 12)
    hashes = w.eng.schedule(R, want_hashes=True, max_blocks=MB, **kw)
    hin = dict(hashes_in=hashes["hashes_out"], n_hashes_in=hashes["total_blocks"], adapter_id=kw["adapter_id"])
    tok = w.tokens(R)
    got = w.eng.schedule_inorder(R, tokens=tok, **hin)
    want = w.reference(R, tok, **hin)
    w.check(got, want, "hashes_in")
    after = w.eng.schedule(R, max_blocks=MB, **kw)
    snap = o.SnapshotData(**w.sd, inflight_tokens=w.tracker.get(w.M)[1])
    want2 = o.schedule_batch(snap, w.prof, w.idx, R, max_blocks=MB, **kw)
    for k in ("pick", "tie_count"):
        assert np.array_equal(after[k], want2[k]), k
    assert np.array_equal(after["pick_score"].view(np.uint64), want2["pick_score"].view(np.uint64))
    w.eng.close()


@pytest.mark.parametrize("mode", ["device", "reserved", "graph"])
def test_device_reserved_and_graph(pkg, mode):
    """device arrays on a caller stream (reserved or not); the graph estimate_tokens -> schedule_batch_inorder ->
    commit_picks_device replayed three rounds equals three rounds of the sequential loop with their commits"""
    import torch
    R, M = 1024, 1024
    w = World(pkg, M, FOUR, pick_mode=0, tie_mode=1, seed=31)
    kw = w.workload(R, 13)
    mask = w.masks(R)
    lens = (np.diff(kw["prompt_off"])).astype(np.int32)
    tok = I.estimate(chars=lens)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream()
    if mode == "reserved":
        w.eng.reserve_stream(s.cuda_stream, R, MB)
    d_in = {k: _dev(v) for k, v in kw.items()}
    d_in["cand_mask"] = _dev(mask)
    d_len = _dev(lens)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
    est = torch.empty(R, dtype=torch.int64, device=dev)

    def step():
        w.eng.estimate_tokens(R, prompt_chars=d_len, device=True, stream=s.cuda_stream, out=est)
        w.eng.schedule_inorder(R, tokens=est, device=True, stream=s.cuda_stream, out=out, max_blocks=MB, **d_in)

    def check_round(rnd):
        want = w.reference(R, tok, cand_mask=mask, want_hashes=True, **kw)
        got = {k: v.cpu().numpy() for k, v in out.items()}
        w.check(got, want, (mode, rnd))
        assert np.array_equal(got["hashes_out"].view(np.uint64), want["hashes_out"])
        return want

    torch.cuda.synchronize()
    if mode != "graph":
        with torch.cuda.stream(s):
            step()
        torch.cuda.synchronize()
        check_round(0)
    else:
        w.eng.prefix_reserve()
        step()  # outside a capture first: it allocates the stream's slice scratch
        torch.cuda.synchronize()
        want = check_round(0)
        w.eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], stream=s.cuda_stream)
        w.idx.commit(want["pick"], want["hashes_out"], want["total_blocks"])
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
            w.eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], stream=s.cuda_stream)
        for rnd in range(1, 4):
            g.replay()
            torch.cuda.synchronize()
            want = check_round(rnd)
            w.idx.commit(want["pick"], want["hashes_out"], want["total_blocks"])
    if mode == "reserved":
        w.eng.release_stream(s.cuda_stream)
    w.eng.close()


def test_refusals_leave_the_counters_untouched(pkg):
    R, M = 64, 128
    w = World(pkg, M, FOUR, seed=41)
    kw = w.workload(R, 14)
    tok = w.tokens(R)
    w.eng.schedule_inorder(R, tokens=tok, max_blocks=MB, **kw)
    w.reference(R, tok, **kw)
    before = w.eng.inflight_get(M)
    B = pkg.Batch
    for flag in ("want_match", "want_scores", "want_filter_mask", "want_pred"):
        with pytest.raises(ValueError):
            w.eng.schedule_inorder(R, tokens=tok, **{flag: True}, **kw)
    # the C entry point itself, with each R x M output / dense rows set
    import ctypes as C
    lib = pkg.lib()
    for field, dt, shape in (("match_blocks", np.uint16, (R, M)), ("scores_out", np.float64, (R, M)),
                             ("pred_out", np.float64, (R, M, 2)), ("filter_mask_out", np.uint32, (R, 4)),
                             ("dense_feat", np.float32, (R, M, 4))):
        b = B()
        b.struct_size = C.sizeof(B)
        b.R = R
        outs = [np.zeros(R, np.int32), np.zeros(R, np.float64), np.zeros(R, np.int32), np.zeros(shape, dt)]
        b.pick, b.pick_score, b.tie_count = (x.ctypes.data for x in outs[:3])
        setattr(b, field, outs[3].ctypes.data)
        assert lib.eppscore_schedule_batch_inorder(w.eng._h, C.byref(b), tok.ctypes.data) == -1, field
    after = w.eng.inflight_get(M)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    w.eng.close()
    # a snapshot that supplies inflight_tokens
    eng = pkg.Engine(pkg.default_config(TL, max_endpoints=M))
    eng.set_snapshot(**synth_snapshot(M, seed=1), inflight_tokens=np.arange(M, dtype=np.int64))
    with pytest.raises(pkg.EppscoreError) as e:
        eng.schedule_inorder(R, tokens=tok)
    assert e.value.code == -1
    assert not eng.inflight_get(M)[1].any()
    eng.close()
    # a profile with the latency scorer
    eng = pkg.Engine(pkg.default_config([("latency", 1), ("token_load", 1)], max_endpoints=M))
    eng.set_latency_params(pkg.latency_params())
    eng.set_snapshot(**synth_snapshot(M, seed=1))
    with pytest.raises(pkg.EppscoreError) as e:
        eng.schedule_inorder(R, tokens=tok)
    assert e.value.code == -1
    assert not eng.inflight_get(M)[1].any()
    eng.close()
