"""eppscore_schedule_batch_inorder_latency on the GPU, bit-exact against the sequential reference
(tests/inorder_latency_reference.py: R single-request oracle schedules whose snapshot takes min_tpot_slo / dispatched from the
running-request queue oracle and inflight_tokens from the in-flight oracle, each followed by the queue add, the in-flight add
and, in the index form, the prefix match and the Add of its blocks): picks, scores (as uint64), tie counts, totals, added_out,
pick_match, the in-flight counters, the running-request view and, in the index form, the whole prefix index afterwards.  Both
forms at every cluster shape, every picker, predictions on and off, streaming and prefill roles, an overloaded fleet, refused adds
(key 0, negative tpot, a key repeated on one pick, a pair live before the call), masks, supplied and device-counted input
tokens, NULL SLO arrays, two slices, device arrays on a reserved stream and in a CUDA graph, a compaction followed by
removes, NULL keys, and the refusals."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q
from tests.helpers import synth_ragged_prompts, synth_snapshot
from tests.inorder_latency_reference import schedule_inorder_latency

pytestmark = pytest.mark.gpu

LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01)
BASE = [("kv", 1), ("latency", 2), ("token_load", 1)]
WIDE = [("queue", 1), ("kv", 1), ("prefix", 1), ("latency", 2), ("running", 1), ("token_load", 1)]
THR = 20000.0
MB = 16


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _u64(x):
    return np.ascontiguousarray(x).view(np.uint64)


class World:
    """An engine and its oracle twin: the same snapshot, latency parameters and pre-populated running queues."""

    def __init__(self, pkg, M, scorers=BASE, pick_mode=0, tie_mode=1, seed=0, predictions=1, streaming=1, prefill=False,
                 max_endpoints=None, live=200):
        self.pkg, self.M = pkg, M
        self.E = max_endpoints or max(M, 64)
        lat = dict(LAT_COEF, has_predictions=predictions, streaming_mode=streaming)
        self.eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=self.E, token_load_threshold=THR, max_blocks=MB,
                                                 prefix_capacity=1 << 16, pick_mode=pick_mode, tie_mode=tie_mode, tie_seed=31))
        self.eng.set_latency_params(pkg.latency_params(**lat))
        self.sd = synth_snapshot(M, seed=seed)
        rng = np.random.Generator(np.random.PCG64(seed + 3))
        if prefill:
            self.sd["prefill_role"] = (rng.random(M) < 0.3).astype(np.uint8)
        self.eng.set_snapshot(**self.sd)
        self.prof = o.make_profile([(pkg.SCORER[s], w) for s, w in scorers], tie_mode=tie_mode, tie_seed=31,
                                   token_load_threshold=THR, pick_mode=pick_mode, latency=o.make_latency_params(**lat))
        self.q, self.tracker, self.idx = Q.Queues(self.E), I.Tracker(), o.Index()
        self.rng = rng
        self.next_key = 1
        if live:  # pairs live before the call: about half the endpoints hold a request, some of them idle again
            ep = rng.integers(0, M, live).astype(np.int32)
            key = self.keys(live)
            tp = rng.choice([0.0, 12.0, 20.0, 35.0], live)
            self.live = (ep, key)
            assert np.array_equal(self.eng.running_add(ep, key, tp), self.q.add(ep, key, tp))
        self.eng.set_snapshot(**self.sd)

    def keys(self, R):
        k = np.arange(self.next_key, self.next_key + R, dtype=np.uint64)
        self.next_key += R
        return k

    def batch(self, R, seed, refused=True, masks=False, supply_tokens=True, slos=True):
        rng = np.random.Generator(np.random.PCG64(seed))
        pb, off = synth_ragged_prompts(R, max_len=MB * 64, seed=seed, groups=8, shared=256)
        kw = dict(prompt_bytes=pb, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64))
        if supply_tokens:
            kw["input_tokens"] = rng.integers(0, 6000, R).astype(np.int32)
        if slos:
            kw["ttft_slo"] = rng.choice([0.0, 60.0, 140.0, 400.0, 1e6], R)
            kw["tpot_slo"] = rng.choice([0.0, 14.0, 18.0, 24.0, 30.0, 80.0], R)
        key = self.keys(R)
        if refused:
            key[::37] = 0                                   # no x-request-id
            if slos:
                kw["tpot_slo"][5::41] = -1.0                # negative tpot
            key[7::53] = key[6::53][: len(key[7::53])]      # the previous request's key: refused when both land on one pick
            key[3] = self.live[1][0]                        # a key live before the call (refused only at its endpoint)
        if masks:
            bits = rng.random((R, self.M)) < 0.7
            bits[::29] = False                              # empty candidate sets
            pad = np.zeros((R, ((self.M + 31) // 32) * 32), bool)
            pad[:, :self.M] = bits
            kw["cand_mask"] = (pad.reshape(R, -1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)
        return kw, key, rng.integers(0, 3000, R).astype(np.int64)

    def reference(self, R, kw, key, tok, index_form, request_base=0):
        want, _ = schedule_inorder_latency(self.sd, self.prof, self.idx if index_form else None, R, self.q, tokens=tok,
                                           request_key=key, tracker=self.tracker, M=self.M, index_form=index_form,
                                           max_blocks=MB, request_base=request_base, **kw)
        return want

    def check(self, got, want, what, index_form):
        for k in ("pick", "tie_count", "total_blocks"):
            assert np.array_equal(np.asarray(got[k]), want[k]), (what, k, np.flatnonzero(np.asarray(got[k]) != want[k])[:5])
        assert np.array_equal(np.asarray(got["added"]).astype(bool), want["added"]), (what, "added")
        if index_form:
            assert np.array_equal(np.asarray(got["pick_match"]), want["pick_match"]), (what, "pick_match")
        assert np.array_equal(_u64(got["pick_score"]), _u64(want["pick_score"])), what
        self.check_state(what, index_form)

    def check_state(self, what, index_form):
        req, tok = self.eng.inflight_get(self.M)
        wreq, wtok = self.tracker.get(self.M)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), what
        gm, gc = self.eng.running_get(self.E)
        wm, wc = self.q.get(self.E)
        assert np.array_equal(gc, wc), (what, "count")
        assert np.array_equal(_u64(gm), _u64(Q.canonical(wm))), (what, "min")
        if index_form:
            for m in range(self.M):
                assert self.eng.prefix_lru_keys(m) == self.idx.lru_keys(m), (what, "lru", m)
            assert self.eng.stats().prefix_live_hashes == self.idx.num_hashes(), what

    def run(self, R, seed, index_form, request_base=0, **bk):
        kw, key, tok = self.batch(R, seed, **bk)
        got = self.eng.schedule_inorder_latency(R, tokens=tok, request_key=key, index=index_form, max_blocks=MB,
                                                request_base=request_base, **kw)
        want = self.reference(R, kw, key, tok, index_form, request_base)
        self.check(got, want, (seed, index_form), index_form)
        return got, want

    def close(self):
        self.eng.close()


@pytest.mark.parametrize("index_form", [False, True])
@pytest.mark.parametrize("M", [1, 40, 256, 257, 512, 513, 1024, 2048, 4096, 8192])
def test_every_cluster_shape(pkg, index_form, M):
    w = World(pkg, M, scorers=WIDE, seed=M)
    for k in range(2):
        w.run(160, 100 + k, index_form, request_base=160 * k, masks=k == 1)
    assert w.q.get(w.E)[1].sum() > 200
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
@pytest.mark.parametrize("pick_mode,tie_mode", [(0, 0), (0, 1), (1, 1), (2, 1)])
def test_pickers(pkg, index_form, pick_mode, tie_mode):
    w = World(pkg, 300, pick_mode=pick_mode, tie_mode=tie_mode, seed=7)
    w.run(400, 11, index_form, masks=True)
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
@pytest.mark.parametrize("predictions,streaming,prefill", [(1, 1, False), (1, 0, False), (1, 1, True), (0, 1, False)])
def test_prediction_modes(pkg, index_form, predictions, streaming, prefill):
    w = World(pkg, 200, scorers=WIDE, seed=3, predictions=predictions, streaming=streaming, prefill=prefill)
    w.run(300, 21, index_form, supply_tokens=False)  # input tokens counted from the prompt bytes on the device
    w.run(200, 22, index_form, request_base=300, slos=False)  # NULL SLO arrays
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_overloaded_fleet_and_idle_endpoints_leaving(pkg, index_form):
    """64 endpoints, 11 of them idle, SLOs from tight to loose: the idle endpoints leave the idle tier one pick at a time."""
    M, R = 64, 600
    w = World(pkg, M, seed=9, live=0)
    busy = np.setdiff1d(np.arange(M), np.arange(0, M, 6)).astype(np.int32)
    k = w.keys(len(busy))
    tp = np.full(len(busy), 30.0)
    assert np.array_equal(w.eng.running_add(busy, k, tp), w.q.add(busy, k, tp))
    w.eng.set_snapshot(**w.sd)
    rng = np.random.Generator(np.random.PCG64(5))
    kw, key, tok = w.batch(R, 31, refused=False)
    kw["ttft_slo"] = rng.choice([1.0, 60.0, 1e6], R)
    kw["tpot_slo"] = rng.choice([1e-3, 12.0, 1e3], R)
    got = w.eng.schedule_inorder_latency(R, tokens=tok, request_key=key, index=index_form, max_blocks=MB, **kw)
    want = w.reference(R, kw, key, tok, index_form)
    w.check(got, want, "overloaded", index_form)
    assert set(np.arange(0, M, 6).tolist()) <= set(want["pick"].tolist())
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_two_slices_and_compaction_then_removes(pkg, index_form):
    """M = 8192 puts 2048 rows in a slice: R = 5000 is three slices; the running table compacts inside the call; then half of
    the batch's keys are removed and the view compared with the oracle again."""
    w = World(pkg, 8192, seed=13)
    w.eng.running_reserve(16384)  # 32768 slots: room for the batch without growing (a growth would drop the tombstones)
    cap = _churn(w, 4096, 3)
    got, want = w.run(5000, 41, index_form)
    assert w.eng.running_reserve(0) == cap  # the table did not grow: the call's pre-add compaction cleared the tombstones
    half = np.flatnonzero(want["added"])[::2]
    ep = want["pick"][half].astype(np.int32)
    kw, key, _ = w.batch(5000, 41)
    w.next_key -= 5000
    removed = w.eng.running_remove(ep, key[half])
    assert np.array_equal(removed, w.q.remove(ep, key[half]))
    w.check_state("removed", index_form)
    w.close()


def _churn(w, L, cycles):
    """`cycles` add / remove rounds of L entries on the engine and the oracle: L * cycles tombstones, no compaction of their
    own (each add stays within half the slots).  Returns running_reserve(0), half the capacity, which must not change."""
    cap = w.eng.running_reserve(0)
    live = w.q.get(w.E)[1].sum()
    for c in range(cycles):
        assert 2 * (live + L * (c + 1)) <= 2 * cap, "the churn itself would compact"
        ep = w.rng.integers(0, w.M, L).astype(np.int32)
        key = w.keys(L)
        tp = w.rng.choice([10.0, 20.0], L)
        assert np.array_equal(w.eng.running_add(ep, key, tp), w.q.add(ep, key, tp))
        assert np.array_equal(w.eng.running_remove(ep, key), w.q.remove(ep, key))
    assert w.eng.running_reserve(0) == cap
    w.eng.set_snapshot(**w.sd)
    return cap


@pytest.mark.parametrize("index_form", [False, True])
def test_compaction_inside_the_call_then_removes(pkg, index_form):
    """1536 tombstones in a table of 4096 slots, then a batch of 1024: live + tombstones + R passes half the slots while
    live + R stays within a quarter, so the call compacts (on the device, before its walk) without growing; its Adds land in
    the compacted table, and removing half of them afterwards matches the oracle."""
    w = World(pkg, 256, seed=29, live=0)
    cap = _churn(w, 512, 3)
    assert cap == 2048
    R = 1024
    kw, key, tok = w.batch(R, 81, refused=False)
    got = w.eng.schedule_inorder_latency(R, tokens=tok, request_key=key, index=index_form, max_blocks=MB, **kw)
    want = w.reference(R, kw, key, tok, index_form)
    w.check(got, want, "compaction", index_form)
    assert want["added"].sum() > R // 2 and w.eng.running_reserve(0) == cap
    half = np.flatnonzero(want["added"])[::2]
    ep = want["pick"][half].astype(np.int32)
    assert np.array_equal(w.eng.running_remove(ep, key[half]), w.q.remove(ep, key[half]))
    w.check_state("removed", index_form)
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_refused_adds_happen(pkg, index_form):
    """Masks force the refused cases: request 3 onto the endpoint where its key is live before the call, requests 6 and 7 (one
    key) onto one endpoint, request 9 with key 0 and request 11 with a negative tpot."""
    M, R = 64, 32
    w = World(pkg, M, seed=31)
    kw, key, tok = w.batch(R, 91, refused=False)
    bits = np.ones((R, M), bool)
    live_ep = int(w.live[0][0])
    bits[3] = False
    bits[3, live_ep] = True
    key[3] = w.live[1][0]
    bits[6] = bits[7] = False
    bits[6, 5] = bits[7, 5] = True
    key[7] = key[6]
    key[9] = 0
    kw["tpot_slo"][11] = -1.0
    kw["cand_mask"] = (bits.reshape(R, -1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)
    got = w.eng.schedule_inorder_latency(R, tokens=tok, request_key=key, index=index_form, max_blocks=MB, **kw)
    want = w.reference(R, kw, key, tok, index_form)
    w.check(got, want, "refused", index_form)
    assert want["pick"][3] == live_ep and want["pick"][6] == want["pick"][7] == 5
    assert want["pick"][9] >= 0 and want["pick"][11] >= 0
    assert not want["added"][[3, 7, 9, 11]].any() and want["added"][6]
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_profile_subset(pkg, index_form):
    """profile 0 limited to a subset of the endpoints (its member bits): the reference sees the subset as every request's mask"""
    M, R = 200, 300
    w = World(pkg, M, scorers=WIDE, seed=37)
    member = np.zeros(M, bool)
    member[::3] = True
    member[7] = True
    pad = np.zeros(((M + 31) // 32) * 32, bool)
    pad[:M] = member
    words = (pad.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    w.eng.set_profile_endpoints(0, words)
    w.eng.set_snapshot(**w.sd)
    kw, key, tok = w.batch(R, 97)
    got = w.eng.schedule_inorder_latency(R, tokens=tok, request_key=key, index=index_form, max_blocks=MB, **kw)
    kw_ref = dict(kw, cand_mask=np.tile(words, (R, 1)))
    want = w.reference(R, kw_ref, key, tok, index_form)
    w.check(got, want, "subset", index_form)
    assert member[want["pick"][want["pick"] >= 0]].all()
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_null_keys_leave_the_queues(pkg, index_form):
    w = World(pkg, 256, seed=17)
    before = w.eng.running_get(w.E)
    kw, key, tok = w.batch(300, 51)
    got = w.eng.schedule_inorder_latency(300, tokens=tok, request_key=None, index=index_form, max_blocks=MB, **kw)
    want = w.reference(300, kw, None, tok, index_form)
    w.check(got, want, "null keys", index_form)
    after = w.eng.running_get(w.E)
    assert np.array_equal(before[1], after[1]) and np.array_equal(_u64(before[0]), _u64(after[0]))
    assert not np.asarray(got["added"]).any()
    w.close()


@pytest.mark.parametrize("index_form", [False, True])
def test_device_reserved_stream_and_graph(pkg, index_form):
    import torch
    M, R = 512, 256
    w = World(pkg, M, seed=19)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream()
    w.eng.reserve_stream(s.cuda_stream, R, MB)
    w.eng.running_reserve(8 * R + 1000)
    if index_form:
        w.eng.prefix_reserve(1 << 16, R * MB * 4)

    def out():
        return dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                    tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                    pick_match=torch.zeros(R, dtype=torch.uint16, device=dev), added_out=torch.zeros(R, dtype=torch.uint8, device=dev))

    def host(o_):
        torch.cuda.synchronize()
        h = {k: v.cpu().numpy() for k, v in o_.items()}
        h["added"] = h.pop("added_out")
        return h

    for rnd in range(3):  # a plain device call, then twice through a captured graph
        kw, key, tok = w.batch(R, 61 + rnd)
        d_in = {k: _dev(v) for k, v in kw.items()}
        d_key, d_tok = _dev(key), _dev(tok)
        o_ = out()
        torch.cuda.synchronize()
        call = lambda: w.eng.schedule_inorder_latency(R, tokens=d_tok, request_key=d_key, index=index_form, device=True,
                                                      stream=s.cuda_stream, out=o_, max_blocks=MB, request_base=R * rnd, **d_in)
        if rnd == 0:
            call()
        else:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                call()
            g.replay()
        want = w.reference(R, kw, key, tok, index_form, request_base=R * rnd)
        w.check(host(o_), want, ("device", rnd), index_form)
    w.eng.release_stream(s.cuda_stream)
    w.close()


def test_refusals_leave_everything_untouched(pkg):
    w = World(pkg, 128, seed=23)
    kw, key, tok = w.batch(64, 71)
    E = pkg.EppscoreError

    def unchanged():
        w.check_state("refused", True)

    with pytest.raises(E):  # NaN tpot in host arrays
        bad = dict(kw, tpot_slo=np.where(np.arange(64) == 9, np.nan, kw["tpot_slo"]))
        w.eng.schedule_inorder_latency(64, tokens=tok, request_key=key, max_blocks=MB, **bad)
    unchanged()
    for extra in (dict(min_tpot_slo=np.zeros(128)), dict(dispatched=np.zeros(128, np.int32))):  # the snapshot supplies the view
        w.eng.set_snapshot(**w.sd, **extra)
        for index_form in (False, True):
            with pytest.raises(E):
                w.eng.schedule_inorder_latency(64, tokens=tok, request_key=key, index=index_form, max_blocks=MB, **kw)
    w.eng.set_snapshot(**w.sd)
    unchanged()
    import ctypes as C
    capi = pkg._capi
    for index_form in (False, True):  # a wrong struct_size
        q = capi.InOrderRunning()
        q.struct_size = C.sizeof(capi.InOrderRunning) + 8
        x = None
        if index_form:
            x = capi.InOrderIndex()
            x.struct_size = C.sizeof(capi.InOrderIndex)
        with pytest.raises(E):
            w.eng.schedule(64, _inorder=(tok, x, q, key), max_blocks=MB, **kw)
    unchanged()
    with pytest.raises(E):  # the existing in-order calls keep refusing the latency scorer
        w.eng.schedule_inorder(64, tokens=tok, max_blocks=MB, **kw)
    with pytest.raises(E):
        w.eng.schedule_inorder_index(64, tokens=tok, max_blocks=MB, **kw)
    unchanged()
    w.close()
    # no latency scorer; device filters
    e2 = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=64))
    e2.set_snapshot(**synth_snapshot(64, seed=1))
    with pytest.raises(E):
        e2.schedule_inorder_latency(4, request_key=np.arange(1, 5, dtype=np.uint64))
    e2.close()
    e3 = pkg.Engine(pkg.default_config(BASE, filters=[(pkg.FILTER_SLO_HEADROOM_TIER, (0.3,))], max_endpoints=64))
    e3.set_latency_params(pkg.latency_params(**LAT_COEF))
    e3.set_snapshot(**synth_snapshot(64, seed=1))
    for index_form in (False, True):
        with pytest.raises(E):
            e3.schedule_inorder_latency(4, request_key=np.arange(1, 5, dtype=np.uint64), index=index_form)
        with pytest.raises(E):  # with NULL keys too
            e3.schedule_inorder_latency(4, request_key=None, index=index_form)
    e3.close()


def test_host_program_on_the_engine(pkg):
    """SchedulerConfig::InOrderRunningRequests of the C++ host layer (tests/cpp/host_inorder_latency_test.cpp) on the engine
    itself: the batch equals a Scheduler fed one request at a time, one queue Add per request, ResponseComplete, refusals."""
    import os
    import subprocess
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cpp, pkgdir = os.path.join(root, "tests", "cpp"), os.path.join(root, "gateway-api-inference-extension_b200")
    exe = os.path.join(tempfile.mkdtemp(), "host_inorder_latency_engine")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread",
                           os.path.join(cpp, "host_inorder_latency_test.cpp"), os.path.join(cpp, "engine_inorder_latency_shim.cpp"),
                           "-I" + os.path.join(root, "include"), "-L" + pkgdir, "-leppscore", "-Wl,-rpath," + pkgdir,
                           "-Wl,--wrap=eppscore_schedule_batch_inorder_latency", "-Wl,--wrap=eppscore_running_add", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host inorder latency: all checks passed" in r.stdout
