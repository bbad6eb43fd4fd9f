"""eppscore_schedule_batch_inorder_index at the edges of its walk (inorder_index_kernel, and inorder_index_lat_kernel through
schedule_inorder_latency(index=True) with a latency profile), bit-exact against the sequential references
(tests/inorder_index_reference.py, tests/inorder_latency_reference.py) on the cases of tests/inorder_walk_scenarios.py: supplied
rows probed over four rounds with the first miss at each round edge, a set emptied by eviction, a bitset row and the last inline
member word; calls of one to three commit chunks at the default capacity and at capacities around the chunk (chunked and
sequential), probed from a pick in the last CTA of a 16-CTA cluster with pick_match past 255 and 512; bitset rows that form and
empty over 16 CTAs; every picker and both tie modes at C = 4 and 16; and the index's room: a same-size rebuild on the device, a
second slice skipped whole, an unreserved table growing between slices and a captured graph replayed across rebuilds.  Picks,
scores (as uint64), tie counts, totals, pick_match, added_out, the in-flight counters, the running-request view (bitwise) and the
whole prefix index afterwards are compared.  The index walk's C (its CTAs of kCommitThreads threads) names each case."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inorder_walk_scenarios as S
from tests import running_oracle as Q
from tests.inorder_reference import schedule_inorder

pytestmark = pytest.mark.gpu

MB = S.MB


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _u64(x):
    return np.ascontiguousarray(x).view(np.uint64)


class CaseWorld:
    """An engine built from a scenario case and its oracle twin (S.Ref): the same snapshot, seeded index, latency parameters
    and running entries."""

    def __init__(self, pkg, case, prefix_capacity=1 << 16):
        c = self.case = case
        self.pkg, self.M, self.E = pkg, c.M, c.E
        self.eng = pkg.Engine(pkg.default_config(c.scorers, max_endpoints=c.E, token_load_threshold=c.threshold, max_blocks=MB,
                                                 prefix_capacity=prefix_capacity, pick_mode=c.pick_mode, tie_mode=c.tie_mode,
                                                 tie_seed=S.SEED, lru_capacity_default=c.lru_default, lru_capacity_max=c.lru_max))
        if c.lat is not None:
            self.eng.set_latency_params(pkg.latency_params(**c.lat))
        self.eng.set_snapshot(**c.sd)
        for keys, ep, cap in c.seeds:
            self.eng.prefix_add(keys, ep, cap)
        self.ref = S.Ref(c)
        if c.live is not None:
            assert np.array_equal(self.eng.running_add(*c.live), self.ref.live_added)
            self.eng.set_snapshot(**c.sd)
        self.keys = [np.asarray(k, np.uint64) for k, _, _ in c.seeds]

    def note(self, b):
        if "hashes_in" in b.kw:
            H, n = b.kw["hashes_in"], b.kw["n_hashes_in"]
            self.keys += [H[r, :n[r]] for r in range(b.R)]
        else:
            pb, off = b.kw["prompt_bytes"], b.kw["prompt_off"]
            self.keys += [o.hash_prompt(bytes(pb[off[r]:off[r + 1]]), int(b.kw["model_seed"][r]), 64, MB) for r in range(b.R)]

    def call(self, b, index_form=True, request_base=0, **extra):
        c = self.case
        if c.lat is not None:
            return self.eng.schedule_inorder_latency(b.R, tokens=b.tokens, request_key=b.key, index=index_form,
                                                     lru_capacity=b.caps, max_blocks=MB, request_base=request_base, **b.kw, **extra)
        return self.eng.schedule_inorder_index(b.R, tokens=b.tokens, lru_capacity=b.caps, max_blocks=MB,
                                               request_base=request_base, **b.kw, **extra)

    def run(self, b, index_form=True, request_base=0, what=""):
        got = self.call(b, index_form, request_base)
        want = self.ref.run(b, index_form, request_base)
        if index_form:
            self.note(b)
        self.check_outputs(got, want, (self.case.name, what), index_form)
        return got, want

    def check_outputs(self, got, want, what, index_form=True, counters=True):
        keys = ["pick", "tie_count", "total_blocks"] + (["pick_match"] if index_form else [])
        for k in keys:
            assert np.array_equal(np.asarray(got[k]), want[k]), (what, k, np.flatnonzero(np.asarray(got[k]) != want[k])[:5])
        assert np.array_equal(_u64(got["pick_score"]), _u64(want["pick_score"])), (what, "score")
        if self.case.lat is not None:
            assert np.array_equal(np.asarray(got["added"]).astype(bool), want["added"]), (what, "added")
        if counters:
            self.check_counters(what)

    def check_counters(self, what):
        req, tok = self.eng.inflight_get(self.E)
        wreq, wtok = self.ref.tracker.get(self.E)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), (what, "inflight")
        if self.case.lat is not None:
            gm, gc = self.eng.running_get(self.E)
            wm, wc = self.ref.q.get(self.E)
            assert np.array_equal(gc, wc), (what, "running count")
            assert np.array_equal(_u64(gm), _u64(Q.canonical(wm))), (what, "running min")

    def check_index(self, what, chunk=1024):
        """every endpoint's LRU oldest -> newest, the set of every key ever seeded or committed, and len(hashToPods)"""
        for m in range(self.M):
            assert self.eng.prefix_lru_keys(m) == self.ref.idx.lru_keys(m), (what, "lru", m)
        keys = np.unique(np.concatenate(self.keys)) if self.keys else np.zeros(0, np.uint64)
        eps = np.arange(self.M, dtype=np.int32)
        for c0 in range(0, len(keys), chunk):
            k = np.ascontiguousarray(keys[c0:c0 + chunk])
            got = self.eng.prefix_match(k[:, None], np.ones(len(k), np.uint16), np.broadcast_to(eps, (len(k), self.M))) > 0
            want = np.zeros_like(got)
            for i, key in enumerate(k):
                want[i, sorted(self.ref.idx.get(int(key)))] = True
            bad = np.flatnonzero((got != want).any(axis=1))
            assert len(bad) == 0, (what, f"{len(bad)} of {len(k)} sets differ", hex(int(k[bad[0]])))
        s = self.eng.stats()
        assert s.prefix_live_hashes == self.ref.idx.num_hashes(), what
        return s

    def close(self):
        self.eng.close()


FORMS = ["index", "latency"]


def _case(make, form, seed):
    c = make()
    if form == "latency":
        S.add_latency(c, seed)
    return c


# ---------------------------------------------------------------------------------------------------------------------------
# probe rounds

@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("M", [512, 1024, 8192], ids=lambda M: f"C{S.index_cluster(M)[0]}")
def test_probe_rounds(pkg, M, form):
    w = CaseWorld(pkg, _case(lambda: S.probe_case(M, seed=M), form, M))
    b = w.case.batches[0]
    w.run(b)
    w.check_index("probe")
    w.close()


# ---------------------------------------------------------------------------------------------------------------------------
# commits past one chunk

@pytest.mark.parametrize("form", FORMS)
def test_commit_past_one_chunk_C16(pkg, form):
    w = CaseWorld(pkg, _case(S.chunk_case, form, 3))
    got, want = w.run(w.case.batches[0])
    assert want["pick_match"].max() > 512
    w.check_index("chunks")
    w.close()


# ---------------------------------------------------------------------------------------------------------------------------
# bitset rows over the whole cluster

@pytest.mark.parametrize("form", FORMS)
def test_bitset_rows_C16(pkg, form):
    w = CaseWorld(pkg, _case(S.bitset_case, form, 5))
    w.run(w.case.batches[0])
    w.check_index("bitset")
    w.close()


# ---------------------------------------------------------------------------------------------------------------------------
# pickers and ties over several CTAs

@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("M", [2048, 8192], ids=lambda M: f"C{S.index_cluster(M)[0]}")
@pytest.mark.parametrize("name", list(S.PICKERS))
def test_pickers_and_ties(pkg, name, M, form):
    w = CaseWorld(pkg, S.picker_case(name, M, seed=M + len(name), lat=form == "latency"))
    got, want = w.run(w.case.batches[0])
    C, T = S.index_cluster(M)
    picked = want["pick"][want["pick"] >= 0]
    assert len(set((picked // T).tolist())) > 1
    if w.case.pick_mode == 0:
        assert (want["tie_count"] > 1).sum() >= 10
    w.check_index(name)
    w.close()


# ---------------------------------------------------------------------------------------------------------------------------
# room

def _fresh_batches(M, n_calls, R, seed, blocks=8):
    """calls of R rows of `blocks` new keys each (no longer than the LRUs: a longer call keeps every key in hashToPods)"""
    kg, rng = S.KeyGen(seed), np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n_calls):
        H, n = S.rows_array([kg(blocks) for _ in range(R)], stride=MB)
        out.append(S.Batch(R, dict(hashes_in=H, n_hashes_in=n), rng.integers(0, 3000, R).astype(np.int64)))
    return out


def _room_case(M, batches, form, seed, lru=8):
    c = S.Case("room", M, M, [("kv", 1), ("prefix", 2), ("token_load", 1)], S.synth_snapshot(M, seed=seed), lru_default=lru,
               batches=batches)
    if form == "latency":
        S.add_latency(c, seed)
    return c


@pytest.mark.parametrize("form", FORMS)
def test_reserved_rebuild_same_size(pkg, form):
    """LRUs of 8 blocks: fresh keys leave dead slots behind; live + touches stays within a quarter of the reserved table, so
    once used + touches pass half of it the call rebuilds it in place (on the device, before the walk) and proceeds"""
    M = 256
    w = CaseWorld(pkg, _room_case(M, _fresh_batches(M, 7, 256, 41), form, 41), prefix_capacity=16)
    w.eng.prefix_reserve(live_hashes=M * 8, touches_per_call=256 * 8)
    r0 = w.eng.stats().prefix_rebuilds
    cap0 = w.eng.stats().prefix_capacity
    for i, b in enumerate(w.case.batches):
        w.run(b, request_base=i * b.R, what=i)
    s = w.check_index("rebuild")
    assert s.prefix_rebuilds > r0 and s.index_error == 0 and s.prefix_capacity == cap0
    w.close()


def test_reserved_second_slice_skipped(pkg):
    """8192 endpoints: one slice per 2048 rows.  Slice 1 fits the reserved table and commits; slice 2's touches fit neither
    half the table nor a quarter after a rebuild, so it is walked without commits: its outputs are schedule_inorder's on the
    index slice 1 left, the index stays as slice 1 left it, and the next index call is refused with -3."""
    M = 8192
    rows = S.slice_rows(M)
    kg, rng = S.KeyGen(43), np.random.Generator(np.random.PCG64(43))
    R = rows + 40
    H, n = S.rows_array([kg(4) for _ in range(rows)] + [kg(300) for _ in range(40)])
    tok = rng.integers(0, 3000, R).astype(np.int64)
    c = S.Case("skip", M, M, [("kv", 1), ("prefix", 2), ("token_load", 1)], S.synth_snapshot(M, seed=43))
    w = CaseWorld(pkg, c, prefix_capacity=16)
    w.eng.prefix_reserve(live_hashes=2 * rows, touches_per_call=2 * rows, overflow_rows=8 * rows)
    slots = 2 * w.eng.stats().prefix_capacity  # (the stat is half the table: the most it holds before a rebuild)
    assert (4 * rows) * 2 <= slots < (4 * rows + 300 * 40) * 2
    got = w.eng.schedule_inorder_index(R, tokens=tok, hashes_in=H, n_hashes_in=n, max_blocks=MB)
    first = S.Batch(rows, dict(hashes_in=H[:rows], n_hashes_in=n[:rows]), tok[:rows])
    want1 = w.ref.run(first)
    w.note(first)
    w.check_outputs({k: v[:rows] for k, v in got.items()}, want1, "slice 1", counters=False)  # (they hold both slices)
    want2, _ = schedule_inorder(c.sd, w.ref.prof, w.ref.idx, 40, tok[rows:], tracker=w.ref.tracker, M=M, request_base=rows,
                                max_blocks=MB, hashes_in=H[rows:], n_hashes_in=n[rows:])
    want2["pick_match"] = np.array([w.ref.idx.match(H[rows + r, :n[rows + r]], M)[p] if p >= 0 else 0
                                    for r, p in enumerate(want2["pick"])], np.uint16)
    w.check_outputs({k: v[rows:] for k, v in got.items()}, want2, "slice 2")
    s = w.check_index("skip")
    assert s.index_error & 4
    with pytest.raises(pkg.EppscoreError) as e:
        w.eng.schedule_inorder_index(4, tokens=tok[:4], hashes_in=H[:4], n_hashes_in=n[:4])
    assert e.value.code == -3
    w.close()


@pytest.mark.parametrize("form", FORMS)
def test_unreserved_growth_between_slices(pkg, form):
    """an unreserved table of 32 slots: slice 1 (2048 rows of 2 blocks) grows it once, slice 2 (40 rows of 600 blocks) must grow
    it again before its walk"""
    M = 8192
    rows = S.slice_rows(M)
    kg, rng = S.KeyGen(47), np.random.Generator(np.random.PCG64(47))
    R = rows + 40
    H, n = S.rows_array([kg(2) for _ in range(rows)] + [kg(600) for _ in range(40)])
    b = S.Batch(R, dict(hashes_in=H, n_hashes_in=n), rng.integers(0, 3000, R).astype(np.int64))
    w = CaseWorld(pkg, _room_case(M, [b], form, 47, lru=31250), prefix_capacity=16)
    w.run(b)
    s = w.check_index("grow")
    assert s.prefix_capacity >= 2 * (2 * rows + 600 * 40) and s.index_error == 0
    w.close()


def test_graph_replayed_across_rebuilds(pkg):
    """a CUDA graph of one index call on a reserved stream and a reserved index, replayed with new keys in its input tensors:
    the replays rebuild the table on the device, and each equals the next call of the sequential loop"""
    import torch
    M, R = 256, 256
    batches = _fresh_batches(M, 8, R, 53)
    w = CaseWorld(pkg, _room_case(M, batches, "index", 53), prefix_capacity=16)
    w.eng.prefix_reserve(live_hashes=M * 8, touches_per_call=R * 8)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream()
    w.eng.reserve_stream(s.cuda_stream, R, MB)
    d_h = torch.zeros((R, MB), dtype=torch.int64, device=dev)
    d_n = torch.zeros(R, dtype=torch.int16, device=dev)
    d_t = torch.zeros(R, dtype=torch.int64, device=dev)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.int16, device=dev),
               pick_match=torch.empty(R, dtype=torch.int16, device=dev))

    def stage(b):
        d_h.copy_(torch.from_numpy(b.kw["hashes_in"].view(np.int64)))
        d_n.copy_(torch.from_numpy(b.kw["n_hashes_in"].view(np.int16)))
        d_t.copy_(torch.from_numpy(b.tokens))
        torch.cuda.synchronize()

    def step(i):
        w.eng.schedule_inorder_index(R, tokens=d_t, hashes_in=d_h, n_hashes_in=d_n, device=True, stream=s.cuda_stream, out=out,
                                     max_blocks=MB, request_base=0)

    def check(i, b):
        torch.cuda.synchronize()
        got = {k: v.cpu().numpy() for k, v in out.items()}
        got["total_blocks"] = got["total_blocks"].view(np.uint16)
        got["pick_match"] = got["pick_match"].view(np.uint16)
        want = w.ref.run(b)
        w.note(b)
        w.check_outputs(got, want, ("graph", i))

    stage(batches[0])
    step(0)
    check(0, batches[0])
    r0 = w.eng.stats().prefix_rebuilds
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step(1)
    for i, b in enumerate(batches[1:], 1):
        stage(b)
        g.replay()
        check(i, b)
    w.eng.release_stream(s.cuda_stream)
    st = w.check_index("graph")
    assert st.prefix_rebuilds > r0 and st.index_error == 0
    w.close()
