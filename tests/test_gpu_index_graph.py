"""A reserved prefix index on the GPU (eppscore_prefix_reserve): commits that decide their room on the device run inside CUDA
graphs.  One graph per round holds schedule -> commit -> estimate_tokens -> inflight_add -> inflight_release (round k-2) on
two streams; it is replayed with new prompts written into its captured inputs, and every round's picks, scores and tie counts
are bit-exact to the CPU oracle while small LRUs churn the table through several same-size device rebuilds.  Also: the
eager path of a reserved engine against an unreserved one, host-side index calls after replays, an undersized reservation
(the replayed commit is skipped whole and reported), a refused capture on an unreserved engine, and two replicas."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

pytestmark = pytest.mark.gpu

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 2)]
M, R, MB, PLEN, LRU, THR, ROUNDS = 64, 512, 16, 1024, 48, 6000.0, 24
ERR_CAPACITY = -3


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _engine(pkg, reserve_touches=0, live=M * LRU + 1024):
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, token_load_threshold=THR, max_blocks=MB, prefix_capacity=1 << 10,
                                        lru_capacity_default=LRU))
    sd = synth_snapshot(M, seed=9)
    eng.set_snapshot(**sd)
    if reserve_touches:
        eng.prefix_reserve(live, reserve_touches, 0)
    return eng, sd


def _inputs(k):
    prompts, off, _ = synth_prompts(R, prompt_len=PLEN, groups=16, shared=256, seed=300 + k, prefix_seed=7)
    return dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64),
                adapter_id=zipf_adapters(R, seed=k))


def _calls(pick, hashes, nh, n_picks):
    """The (request, slot) calls of a commit with n_picks picks in request order: the second pick is (pick + 7) % M."""
    if n_picks == 1:
        return pick, hashes, nh
    p2 = np.stack([pick, (pick + 7) % M], axis=1).reshape(-1).astype(np.int32)
    return p2, np.repeat(hashes, 2, axis=0), np.repeat(nh, 2)


def _same_index(eng, idx, keys):
    for e in range(M):
        assert eng.prefix_lru_keys(e) == idx.lru_keys(e), e
    for key in keys:
        assert eng.prefix_get(int(key)) == idx.get(int(key)), int(key)
    assert eng.stats().prefix_live_hashes == idx.num_hashes()


class Loop:
    """One round: schedule on s_batch -> commit (n_picks picks) on s_batch -> estimate, add, release round k-2 on s_upd."""

    def __init__(self, eng, n_picks, shadow=None):
        import torch
        dev = torch.device("cuda:0")
        self.eng, self.n_picks, self.shadow = eng, n_picks, shadow
        kw = _inputs(0)
        self.d_in = {key: _dev(v) for key, v in kw.items()}
        self.chars = _dev(np.full(R, PLEN, np.int32))
        self.out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                        tie_count=torch.empty(R, dtype=torch.int32, device=dev),
                        total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                        hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
        self.pick2 = torch.empty(R, dtype=torch.int32, device=dev)
        self.est = torch.empty(R, dtype=torch.int64, device=dev)
        self.prev = [(torch.full((R,), -1, dtype=torch.int32, device=dev), torch.zeros(R, dtype=torch.int64, device=dev)) for _ in range(2)]
        self.s_batch, self.s_upd = torch.cuda.Stream(), torch.cuda.Stream()

    def body(self):
        import torch
        e, o_, sb, su = self.eng, self.out, self.s_batch, self.s_upd
        e.schedule(R, device=True, stream=sb.cuda_stream, out=o_, **self.d_in)
        if self.n_picks == 1:
            e.commit_picks_device(o_["pick"], o_["hashes_out"], o_["total_blocks"], stream=sb.cuda_stream)
        else:
            with torch.cuda.stream(sb):
                self.pick2.copy_(torch.remainder(o_["pick"] + 7, M))
            e.commit_picks_profiles([o_["pick"], self.pick2], o_["hashes_out"], o_["total_blocks"], device=True, stream=sb.cuda_stream)
        if self.shadow is not None:  # an unreserved engine committing the same calls
            self.shadow.commit_picks_device(o_["pick"], o_["hashes_out"], o_["total_blocks"], stream=sb.cuda_stream)
        su.wait_stream(sb)
        e.estimate_tokens(R, prompt_chars=self.chars, device=True, stream=su.cuda_stream, out=self.est)
        e.inflight_add(o_["pick"], self.est, device=True, stream=su.cuda_stream)
        e.inflight_release(self.prev[0][0], self.prev[0][1], device=True, stream=su.cuda_stream)

    def capture(self):
        import torch
        self.eng.schedule(R, device=True, stream=self.s_batch.cuda_stream, out=self.out, **self.d_in)  # warm the scratch
        torch.cuda.synchronize()
        self.g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g, stream=self.s_upd):
            self.s_batch.wait_stream(self.s_upd)
            self.body()
        torch.cuda.synchronize()

    def round(self, k, graph):
        import torch
        kw = _inputs(k)
        for key in ("prompt_bytes", "adapter_id"):  # (offsets and model seeds are the same every round)
            self.d_in[key].copy_(torch.from_numpy(kw[key]))
        torch.cuda.synchronize()
        if graph:
            self.g.replay()
        else:
            self.body()
        torch.cuda.synchronize()
        # round k-2's picks leave with the next round
        self.prev[0][0].copy_(self.prev[1][0])
        self.prev[0][1].copy_(self.prev[1][1])
        self.prev[1][0].copy_(self.out["pick"])
        self.prev[1][1].copy_(self.est)
        torch.cuda.synchronize()


def _run_loop(pkg, n_picks, graph, shadow=False):
    eng, sd = _engine(pkg, reserve_touches=R * MB * n_picks)
    sh = _engine(pkg)[0] if shadow else None
    cap0, rebuilds0 = eng.stats().prefix_capacity, eng.stats().prefix_rebuilds
    prof = o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], token_load_threshold=THR)
    idx, tracker = o.Index(LRU), I.Tracker()
    loop = Loop(eng, n_picks, sh)
    if graph:
        loop.capture()
    picks, ests, keys = [], [], []
    w_est = I.estimate(None, None, np.full(R, PLEN, np.int32))
    for k in range(ROUNDS):
        loop.round(k, graph)
        kw = _inputs(k)
        snap = o.SnapshotData(**sd, inflight_tokens=tracker.get(M)[1])
        want = o.schedule_batch(snap, prof, idx, R, max_blocks=MB, want_hashes=True, n_threads=8, **kw)
        what = (n_picks, graph, k)
        assert np.array_equal(loop.out["pick"].cpu().numpy(), want["pick"]), what
        assert np.array_equal(loop.out["pick_score"].cpu().numpy().view(np.uint64), want["pick_score"].view(np.uint64)), what
        assert np.array_equal(loop.out["tie_count"].cpu().numpy(), want["tie_count"]), what
        assert np.array_equal(loop.est.cpu().numpy(), w_est), what
        idx.commit(*_calls(want["pick"], want["hashes_out"], want["total_blocks"], n_picks))
        keys.append(want["hashes_out"][:, :4].ravel())
        tracker.add(want["pick"], w_est)
        if k >= 2:
            tracker.release(picks[k - 2], ests[k - 2])
        picks.append(want["pick"])
        ests.append(w_est)
        got_r, got_t = eng.inflight_get(M)
        want_r, want_t = tracker.get(M)
        assert np.array_equal(got_r, want_r) and np.array_equal(got_t, want_t), what
    sample = np.unique(np.concatenate(keys[-3:]))[:1500]
    _same_index(eng, idx, sample)
    st = eng.stats()
    assert st.prefix_capacity == cap0 and st.prefix_rebuilds >= rebuilds0 + 2 and st.index_error == 0
    return eng, sh, idx, sample


@pytest.mark.parametrize("n_picks", [1, 2], ids=["one-pick", "two-picks"])
def test_one_graph_per_round_matches_oracle(pkg, n_picks):
    """>= 20 replays of one graph; then host-side index calls see the exact state the replays left."""
    eng, _, idx, sample = _run_loop(pkg, n_picks, graph=True)
    rng = np.random.Generator(np.random.PCG64(5))
    extra = rng.integers(1, 2 ** 63, size=20, dtype=np.uint64)
    eng.prefix_add(extra, 3)
    idx.add(extra, 3)
    for e in (5, 17, 40):
        eng.prefix_remove_endpoint(e)
        idx.remove_pod(e)
    eng.prefix_add(np.zeros(0, np.uint64), 40)  # creates the LRU (indexer.go:57-68), as the reserve documents
    idx.add(np.zeros(0, np.uint64), 40)
    _same_index(eng, idx, np.concatenate([sample[:500], extra]))
    assert eng.prefix_lru_len(40) == 0
    eng.close()


def test_reserved_eager_matches_unreserved(pkg):
    """The same loop without a graph: the reserved engine and an unreserved one fed the same commits end with the same index."""
    eng, sh, idx, sample = _run_loop(pkg, 1, graph=False, shadow=True)
    _same_index(sh, idx, sample)
    assert sh.stats().prefix_live_hashes == eng.stats().prefix_live_hashes
    eng.close()
    sh.close()


def _commit_graph(eng, pick, hashes, nh, s):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.commit_picks_device(pick, hashes, nh, stream=s.cuda_stream)
    torch.cuda.synchronize()
    return g


def test_undersized_reservation_skips_the_replayed_commit(pkg):
    """A replay that needs more room than the reservation skips the commit whole: the index is unchanged, the sticky bit is
    set, and the next index call outside a capture fails with ERR_CAPACITY (once); nothing hangs or aborts."""
    import torch
    eng, _ = _engine(pkg, reserve_touches=16, live=16)  # 128 slots: room for 16 touches per call
    rng = np.random.Generator(np.random.PCG64(3))
    small = rng.integers(1, 2 ** 63, size=8, dtype=np.uint64)
    eng.prefix_add(small, 2)
    before = eng.stats()
    n = 64
    pick = _dev(np.arange(n, dtype=np.int32) % M)
    hashes = _dev(rng.integers(1, 2 ** 63, size=(n, MB), dtype=np.uint64).view(np.int64))
    nh = _dev(np.full(n, MB, np.uint16))
    s = torch.cuda.Stream()
    g = _commit_graph(eng, pick, hashes, nh, s)
    g.replay()
    torch.cuda.synchronize()
    st = eng.stats()
    assert st.index_error & 4
    assert st.prefix_live_hashes == before.prefix_live_hashes == 8 and st.prefix_hashes == before.prefix_hashes
    assert all(eng.prefix_lru_len(e) == -1 for e in range(M) if e != 2) and eng.prefix_lru_keys(2) == [int(x) for x in small]
    with pytest.raises(pkg.EppscoreError) as ei:
        eng.prefix_add(small[:1], 9)
    assert ei.value.code == ERR_CAPACITY and "skipped" in str(ei.value)
    eng.prefix_add(small[:1], 9)  # reported once: the index works on
    assert eng.prefix_lru_len(9) == 1
    eng.close()


def test_unreserved_capture_is_refused_and_the_capture_completes(pkg):
    import torch
    eng, _ = _engine(pkg)
    pick = _dev(np.zeros(4, np.int32))
    hashes = _dev(np.arange(1, 9, dtype=np.int64).reshape(4, 2))
    nh = _dev(np.full(4, 2, np.uint16))
    x = torch.zeros(4, device="cuda:0")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        with pytest.raises(pkg.EppscoreError) as ei:
            eng.commit_picks_device(pick, hashes, nh, stream=s.cuda_stream)
        x += 1
    assert ei.value.code == ERR_CAPACITY and "reserve" in str(ei.value)
    g.replay()
    torch.cuda.synchronize()
    assert float(x.sum()) == 4.0
    assert eng.prefix_lru_len(0) == -1
    eng.commit_picks_device(pick, hashes, nh)  # eager commits are unaffected
    assert eng.prefix_lru_len(0) == 8
    eng.close()


def test_replicas_replaying_one_commit_stream_stay_identical(pkg):
    """Two reserved engines, each with a graph of the same commit, replayed over the same 30 rounds of random commits on a
    small table (several device rebuilds): the two indexes and the oracle's agree."""
    import torch
    n, nmax = 256, 16
    engs = [_engine(pkg, reserve_touches=n * nmax, live=M * LRU)[0] for _ in range(2)]
    caps = [e.stats().prefix_capacity for e in engs]
    rng = np.random.Generator(np.random.PCG64(21))
    pick = _dev(np.zeros(n, np.int32))
    hashes = torch.zeros((n, nmax), dtype=torch.int64, device="cuda:0")
    nh = _dev(np.zeros(n, np.uint16))
    s = torch.cuda.Stream()
    graphs = [_commit_graph(e, pick, hashes, nh, s) for e in engs]
    idx = o.Index(LRU)
    pool = rng.integers(1, 2 ** 63, size=n, dtype=np.uint64)  # re-touched keys; the rest are new every round
    keys = []
    for k in range(30):
        p = rng.integers(-1, M, size=n).astype(np.int32)
        h = rng.integers(1, 2 ** 63, size=(n, nmax), dtype=np.uint64)
        h[:, :4] = pool[rng.integers(0, n, size=(n, 4))]
        c = rng.integers(0, nmax + 1, size=n).astype(np.uint16)
        pick.copy_(torch.from_numpy(p))
        hashes.copy_(torch.from_numpy(h.view(np.int64)))
        nh.copy_(torch.from_numpy(c))
        torch.cuda.synchronize()
        for g in graphs:
            g.replay()
        torch.cuda.synchronize()
        idx.commit(p, h, c)
        keys.append(h[:, :6].ravel())
    sample = np.unique(np.concatenate(keys[-4:]))[:2000]
    for e, cap in zip(engs, caps):
        _same_index(e, idx, sample)
        st = e.stats()
        assert st.prefix_capacity == cap and st.prefix_rebuilds >= 2 and st.index_error == 0
    assert engs[0].stats().prefix_hashes == engs[1].stats().prefix_hashes
    for e in engs:
        e.close()
