"""eppscore_schedule_batch_inorder_profiles on the GPU, bit-exact against the sequential reference
(tests/inorder_profiles_reference.py): every run's picks, scores (as uint64), tie counts and pick_match, the totals, the
in-flight counters afterwards and, in the index form, the WHOLE prefix index afterwards — in both forms, at every cluster shape,
with one to four runs, disjoint / overlapping / empty subsets, candidate masks and run masks, every picker mixed across runs in
both tie modes, supplied hashes, two slices, device arrays, the one-run equality with the single-profile in-order calls, and
the refusals."""
import numpy as np
import pytest

from tests.inorder_profiles_reference import schedule_inorder_profiles
from tests.test_gpu_inorder_index import MB, SLICE_BYTES, THR, World, _dev, _u64, pkg  # noqa: F401  (pkg: the module fixture)

pytestmark = pytest.mark.gpu

DECODE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 1)]
PREFILL = [("kv", 2), ("prefix", 3), ("token_load", 1)]


def _bits(M, members):
    out = np.zeros(max((M + 31) // 32, 1), np.uint32)
    for m in members:
        out[m >> 5] |= np.uint32(1 << (m & 31))
    return out


class PWorld(World):
    """World (tests/test_gpu_inorder_index.py) with profiles: run i = (scorers, pick_mode, subset members or None)."""

    def __init__(self, pkg, M, runs, tie_mode=1, seed=0, warm=128, **kw):
        super().__init__(pkg, M, scorers=runs[0][0], pick_mode=runs[0][1], tie_mode=tie_mode, seed=seed, warm=warm, **kw)
        self.tie_mode = tie_mode
        self.runs = []
        for i, (scorers, pick_mode, members) in enumerate(runs):
            pid = 0 if i == 0 else self.eng.add_profile(scorers, pick_mode=pick_mode)
            sub = None if members is None else _bits(M, members)
            if sub is not None:
                self.eng.set_profile_endpoints(pid, sub)
            self.runs.append(dict(profile=pid, scorers=[(pkg.SCORER[s], w) for s, w in scorers], pick_mode=pick_mode, subset=sub))
        self.eng.set_snapshot(**self.sd)

    def run(self, R, tok, index, prefill_run=-1, run_mask=None, cand=None, request_base=0, **kw):
        eng_runs = [dict(profile=u["profile"], cand_mask=None if cand is None else cand[i]) for i, u in enumerate(self.runs)]
        got = self.eng.schedule_inorder_profiles(R, eng_runs, tokens=tok, index=index, prefill_run=prefill_run,
                                                 run_mask=run_mask, max_blocks=MB, request_base=request_base,
                                                 want_hashes="prompt_bytes" in kw, **kw)
        ref_runs = [dict(u, cand_mask=None if cand is None else cand[i]) for i, u in enumerate(self.runs)]
        want = schedule_inorder_profiles(self.sd, ref_runs, self.idx, R, tok, self.tracker, self.M, ordered_index=index,
                                         prefill_run=prefill_run, run_mask=run_mask, tie_mode=self.tie_mode, tie_seed=77,
                                         token_load_threshold=THR, max_blocks=MB, request_base=request_base, **kw)
        if index:
            for j in (0, prefill_run):
                if j >= 0:
                    self.note_keys(want[1][j]["pick"], want[0]["hashes"], want[0]["total_blocks"])
        return got, want

    def run_reference(self, R, tok, index, prefill_run=-1, **kw):
        want = schedule_inorder_profiles(self.sd, [dict(u) for u in self.runs], self.idx, R, tok, self.tracker, self.M,
                                         ordered_index=index, prefill_run=prefill_run, tie_mode=self.tie_mode, tie_seed=77,
                                         token_load_threshold=THR, max_blocks=MB, **kw)
        if index:
            for j in (0, prefill_run):
                if j >= 0:
                    self.note_keys(want[1][j]["pick"], want[0]["hashes"], want[0]["total_blocks"])
        return want

    def check(self, got, want, index, what):
        (gb, gr), (wb, wr, _) = got, want
        assert np.array_equal(gb["total_blocks"], wb["total_blocks"]), what
        if "hashes_out" in gb:
            assert np.array_equal(_u64(gb["hashes_out"]), wb["hashes"]), what
        for i, (g, w) in enumerate(zip(gr, wr)):
            for k in ("pick", "tie_count", "pick_match"):
                bad = np.flatnonzero(np.asarray(g[k]) != w[k])
                assert len(bad) == 0, (what, i, k, bad[:5], np.asarray(g[k])[bad[:5]], w[k][bad[:5]])
            assert np.array_equal(_u64(g["pick_score"]), _u64(w["pick_score"])), (what, i)
        req, tok = self.eng.inflight_get(self.M)
        wreq, wtok = self.tracker.get(self.M)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), what
        if index:
            self.check_index(what)


def _pd(M, prefill_mode=1):
    half = M // 2
    return [(DECODE, 0, range(half)), (PREFILL, prefill_mode, range(half, M))]


@pytest.mark.parametrize("index", [False, True])
@pytest.mark.parametrize("M", [64, 256, 1024, 2048, 4096, 8192])
def test_pd_every_cluster_shape(pkg, M, index):
    """decode max-score on one half, prefill weighted-random on the other, half the prefixes new to the index"""
    R = 80
    w = PWorld(pkg, M, _pd(M), seed=M)
    kw = w.workload(R, 12, groups=4, new_groups=4)
    got, want = w.run(R, w.tokens(R), index, prefill_run=1, **kw)
    w.check(got, want, index, (M, index))
    w.close()


RUN_SETS = {
    "one": [(DECODE, 0, None)],
    "two_overlap": [(DECODE, 0, range(0, 400)), (PREFILL, 2, range(200, 512))],
    "three": [(PREFILL, 1, range(0, 300)), (DECODE, 0, None), ([("kv", 1), ("prefix", 1)], 0, range(100, 200))],
    "four_empty": [(DECODE, 1, range(256)), (PREFILL, 0, range(256, 512)), ([("queue", 1), ("kv", 1)], 2, []),
                   ([("prefix", 2), ("token_load", 2)], 0, None)],
}


@pytest.mark.parametrize("index", [False, True])
@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("name", list(RUN_SETS))
def test_runs_pickers_and_masks(pkg, name, tie_mode, index):
    M, R = 512, 120
    runs = RUN_SETS[name]
    w = PWorld(pkg, M, runs, tie_mode=tie_mode, seed=3)
    kw = w.workload(R, 21, groups=6, new_groups=6)
    rng = np.random.default_rng(len(runs) * 10 + tie_mode)
    mw = (M + 31) // 32
    cand = [rng.integers(0, 2 ** 32, size=(R, mw), dtype=np.uint32) | rng.integers(0, 2 ** 32, size=(R, mw), dtype=np.uint32)
            for _ in runs]
    run_mask = rng.integers(0, 16, R).astype(np.uint8) | 1
    prefill = 1 if len(runs) > 1 else -1
    got, want = w.run(R, w.tokens(R), index, prefill_run=prefill, run_mask=run_mask, cand=cand, **kw)
    w.check(got, want, index, (name, tie_mode, index))
    # a second batch continues from the counters and the index the first left
    kw = w.workload(R, 22, groups=6, new_groups=6)
    got, want = w.run(R, w.tokens(R), index, prefill_run=prefill, request_base=R, **kw)
    w.check(got, want, index, (name, tie_mode, index, "second"))
    w.close()


@pytest.mark.parametrize("index", [False, True])
def test_hashes_in_evictions_and_bitset_rows(pkg, index):
    """supplied hashes with empty rows, small LRUs that evict inside the batch, and sets past 10 endpoints"""
    M, R = 256, 200
    w = PWorld(pkg, M, [([("kv", 1), ("prefix", 1), ("token_load", 3)], 0, range(128)),
                        ([("kv", 1), ("prefix", 1), ("token_load", 3)], 2, range(128, 256))], seed=9, lru_default=24, warm=0)
    rng = np.random.default_rng(4)
    base = rng.integers(1, 2 ** 63, size=(4, MB), dtype=np.uint64)
    h = base[rng.integers(0, 4, R)].copy()
    n = rng.integers(0, MB + 1, R).astype(np.uint16)
    n[::17] = 0
    got, want = w.run(R, w.tokens(R), index, prefill_run=1, hashes_in=h, n_hashes_in=n)
    w.check(got, want, index, ("hashes_in", index))
    w.close()


@pytest.mark.parametrize("index", [False, True])
def test_two_slices(pkg, index):
    M = 8192
    R = SLICE_BYTES // (M * 2) + 40
    w = PWorld(pkg, M, _pd(M, prefill_mode=0), seed=5, warm=64)
    kw = w.workload(R, 31, groups=4, new_groups=4, prompt_len=MB * 16)
    got, want = w.run(R, w.tokens(R), index, prefill_run=1, **kw)
    w.check(got, want, index, ("two slices", index))
    w.close()


@pytest.mark.parametrize("index", [False, True])
def test_one_run_equals_single_profile_call(pkg, index):
    M, R = 1024, 200
    a, b = World(pkg, M, seed=2), World(pkg, M, seed=2)
    kw = a.workload(R, 41, groups=8, new_groups=8)
    tok = a.tokens(R)
    single = (a.eng.schedule_inorder_index if index else a.eng.schedule_inorder)(R, tokens=tok, max_blocks=MB, **kw)
    _, runs = b.eng.schedule_inorder_profiles(R, [dict(profile=0)], tokens=tok, index=index, max_blocks=MB, **kw)
    for k in ("pick", "tie_count"):
        assert np.array_equal(single[k], runs[0][k]), k
    assert np.array_equal(_u64(single["pick_score"]), _u64(runs[0]["pick_score"]))
    if index:
        assert np.array_equal(single["pick_match"], runs[0]["pick_match"])
    ra, ta = a.eng.inflight_get(M)
    rb, tb = b.eng.inflight_get(M)
    assert np.array_equal(ra, rb) and np.array_equal(ta, tb)
    for m in range(0, M, 37):
        assert a.eng.prefix_lru_keys(m) == b.eng.prefix_lru_keys(m)
    a.close()
    b.close()


def test_device_arrays(pkg):
    import torch
    M, R = 1024, 150
    w = PWorld(pkg, M, _pd(M), seed=6)
    kw = w.workload(R, 51, groups=6, new_groups=6)
    tok = w.tokens(R)
    want = PWorld(pkg, M, _pd(M), seed=6)
    wg, wr = want.eng.schedule_inorder_profiles(R, [dict(profile=0), dict(profile=1)], tokens=tok, index=True, prefill_run=1,
                                                max_blocks=MB, **kw)
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    runs = [dict(profile=p, pick=torch.empty(R, dtype=torch.int32, device="cuda"),
                 pick_score=torch.empty(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.empty(R, dtype=torch.int32, device="cuda"),
                 pick_match=torch.empty(R, dtype=torch.uint16, device="cuda")) for p in (0, 1)]
    dkw = {k: d(v) for k, v in kw.items()}
    out = dict(total_blocks=torch.empty(R, dtype=torch.uint16, device="cuda"))
    w.eng.schedule_inorder_profiles(R, runs, tokens=d(tok), index=True, prefill_run=1, max_blocks=MB, device=True, out=out, **dkw)
    torch.cuda.synchronize()
    for i in range(2):
        assert np.array_equal(runs[i]["pick"].cpu().numpy(), wr[i]["pick"])
        assert np.array_equal(runs[i]["pick_match"].cpu().numpy(), wr[i]["pick_match"])
        assert np.array_equal(_u64(runs[i]["pick_score"].cpu().numpy()), _u64(wr[i]["pick_score"]))
    assert np.array_equal(out["total_blocks"].cpu().numpy(), wg["total_blocks"])
    w.close()
    want.close()


def _dev_runs(R, n):
    import torch
    return [dict(profile=p, pick=torch.empty(R, dtype=torch.int32, device="cuda"),
                 pick_score=torch.empty(R, dtype=torch.float64, device="cuda"), tie_count=torch.empty(R, dtype=torch.int32, device="cuda"),
                 pick_match=torch.empty(R, dtype=torch.uint16, device="cuda")) for p in range(n)]


def test_reserved_stream_and_graph(pkg):
    """device arrays on a reserved stream and a reserved index: one call outside a capture, then a CUDA graph of the call
    replayed twice, each equal to one more round of the sequential loop (the index form, both Adds per request)"""
    import torch
    M, R = 512, 256
    w = PWorld(pkg, M, _pd(M), seed=19)
    w.eng.prefix_reserve()
    kw = w.workload(R, 20, groups=4, new_groups=4)
    tok = w.tokens(R)
    s = torch.cuda.Stream()
    w.eng.reserve_stream(s.cuda_stream, R, MB)
    d_in = {k: _dev(v) for k, v in kw.items()}
    d_tok = _dev(tok)
    runs = _dev_runs(R, 2)
    out = dict(total_blocks=torch.empty(R, dtype=torch.uint16, device="cuda"),
               hashes_out=torch.zeros((R, MB), dtype=torch.int64, device="cuda"))

    def step():
        w.eng.schedule_inorder_profiles(R, runs, tokens=d_tok, index=True, prefill_run=1, max_blocks=MB, device=True,
                                        stream=s.cuda_stream, out=out, **d_in)

    def check(rnd):
        want = w.run_reference(R, tok, True, prefill_run=1, **kw)
        got = ({k: v.cpu().numpy() for k, v in out.items()},
               [{k: v.cpu().numpy() for k, v in r.items() if k != "profile"} for r in runs])
        w.check(got, want, True, ("graph", rnd))

    torch.cuda.synchronize()
    step()
    torch.cuda.synchronize()
    check(0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step()
    for rnd in (1, 2):
        g.replay()
        torch.cuda.synchronize()
        check(rnd)
    assert w.eng.stats().index_error == 0
    w.eng.release_stream(s.cuda_stream)
    w.close()


def test_reserved_index_without_room(pkg):
    """a slice without room for its primary and prefill Adds is walked without commits: the outputs equal the in-flight form's
    on the frozen index, the index is unchanged, stats.index_error has bit 4, and the next index call reports the skip"""
    M, R = 256, 200
    w = PWorld(pkg, M, _pd(M), seed=23, warm=0)
    w.eng.prefix_reserve(live_hashes=16, touches_per_call=16, overflow_rows=16)
    kw = w.workload(R, 24, groups=2, new_groups=2)
    tok = w.tokens(R)
    got = w.eng.schedule_inorder_profiles(R, [dict(profile=0), dict(profile=1)], tokens=tok, index=True, prefill_run=1,
                                          max_blocks=MB, want_hashes=True, **kw)
    want = w.run_reference(R, tok, False, prefill_run=1, **kw)
    w.check(got, want, False, "no room")
    assert w.eng.stats().prefix_live_hashes == 0
    assert all(w.eng.prefix_lru_len(m) == -1 for m in range(M))
    assert w.eng.stats().index_error & 4
    with pytest.raises(pkg.EppscoreError) as e:
        w.eng.schedule_inorder_profiles(R, [dict(profile=0), dict(profile=1)], tokens=tok, index=True, prefill_run=1,
                                        max_blocks=MB, **kw)
    assert e.value.code == -3
    w.close()


def test_refusals(pkg):
    M = 256
    w = PWorld(pkg, M, _pd(M), seed=8, warm=0)
    lat = w.eng.add_profile([("latency", 1)])
    filt = w.eng.add_profile([("latency", 1), ("kv", 0.5)], filters=[(1, (0.5, 0.0, 5000.0))])
    kw = w.workload(4, 1)
    two = [dict(profile=0), dict(profile=1)]
    bad = [
        dict(runs=two, primary_run=2),
        dict(runs=two, prefill_run=0),
        dict(runs=two, prefill_run=2),
        dict(runs=[dict(profile=0), dict(profile=0)]),
        dict(runs=[dict(profile=0), dict(profile=lat)]),
        dict(runs=[dict(profile=0), dict(profile=filt)]),
    ]
    for b in bad:
        runs = b.pop("runs")
        with pytest.raises(w.pkg.EppscoreError) as e:
            w.eng.schedule_inorder_profiles(4, runs, max_blocks=MB, **b, **kw)
        assert e.value.code == -1, b
    # a run's scores_out (device arrays, so the library's own check sees it)
    import torch
    runs = _dev_runs(4, 2)
    runs[1]["scores_out"] = torch.empty((4, M), dtype=torch.float64, device="cuda")
    with pytest.raises(w.pkg.EppscoreError) as e:
        w.eng.schedule_inorder_profiles(4, runs, prefill_run=1, max_blocks=MB, device=True, out={},
                                        **{k: _dev(v) for k, v in kw.items()})
    assert e.value.code == -1 and "scores_out" in str(e.value)
    # the struct itself: a wrong struct_size and an index outside {0, 1}
    import ctypes as C
    for size, index in ((C.sizeof(w.pkg._capi.InOrderProfiles) - 8, 0), (C.sizeof(w.pkg._capi.InOrderProfiles), 2)):
        x = w.pkg._capi.InOrderProfiles()
        x.struct_size = size
        x.index = index
        x.prefill_run = -1
        with pytest.raises(w.pkg.EppscoreError) as e:
            w.eng.schedule_profiles(4, [dict(profile=0)], max_blocks=MB, _inorder=(None, x, None), **kw)
        assert e.value.code == -1
    # a snapshot that supplies inflight_tokens
    w.eng.set_snapshot(**w.sd, inflight_tokens=np.zeros(M, np.int64))
    with pytest.raises(w.pkg.EppscoreError) as e:
        w.eng.schedule_inorder_profiles(4, two, prefill_run=1, max_blocks=MB, **kw)
    assert e.value.code == -1 and "inflight_tokens" in str(e.value)
    req, _ = w.eng.inflight_get(M)
    assert req.sum() == 0
    w.close()
