"""The edge cases of tests/inorder_walk_scenarios.py reach the edges they name, checked through the CPU oracle and the sequential
references alone (no GPU): the first miss of every probe row against the seeded index, the call lengths against the LRU
capacities and the chunk size, bitset rows that form and empty inside a batch, pick_match past 255 and 512, which ranks occur
as a request's lowest latency tier (from the oracle's predictions and the queue view each request sees), the one-side-degenerate
headroom ranges, tie sets over several CTAs and the weighted-random picker's fall into its uniform draw."""
import numpy as np
import pytest

from oracle import oracle_py as o
from tests import inorder_walk_scenarios as S


def test_constants_parsed():
    assert S.T == 512 and S.CHUNK == 4 * S.T and S.INLINE_EPS == 10 and S.SLICE_BYTES == 32 << 20
    assert S.index_cluster(512) == (1, S.T) and S.index_cluster(1024) == (2, S.T) and S.index_cluster(8192) == (16, S.T)


@pytest.mark.parametrize("M", [512, 1024, 8192])
def test_probe_rows_first_miss(M):
    c = S.probe_case(M, seed=M)
    b = c.batches[0]
    idx = o.Index(c.lru_default)
    S.seed_oracle(c, idx)
    H, n = b.kw["hashes_in"], b.kw["n_hashes_in"]
    for r in range(b.R):
        assert S.first_miss(idx, H[r, :n[r]]) == b.meta["first_miss"][r], (r, b.meta["kinds"][r])
        # every block after the miss hits at the owner, so a walk that probes past it counts more
        assert n[r] // S.T >= 3
    kinds = b.meta["kinds"]
    at = {k: [r for r in range(b.R) if kinds[r] == k] for k in set(kinds)}
    r = at["emptied"][0]
    assert idx.get(int(H[r, S.T + 5])) == set()                      # a set emptied by eviction, in round 2
    r = at["bitset"][0]
    assert len(idx.get(int(H[r, S.T + 9]))) > S.INLINE_EPS            # a bitset row, in round 2
    for members in (S.INLINE_EPS, S.INLINE_EPS - 1):
        r = at[f"inline{members}"][0]
        s = sorted(idx.get(int(H[r, S.T + 3])))
        assert len(s) == members and s[-1] == b.meta["owner"][r]      # the owner is the last staged member
    # consecutive requests end in rounds of both parities
    rounds = [(min(f, int(n[r]) - 1) // S.T) for r, f in enumerate(b.meta["first_miss"])]
    assert {x % 2 for x in rounds} == {0, 1}
    # through the reference: the counts at the owners are the probe depths
    want = S.Ref(c).run(b)
    owner_hits = (want["pick"] == np.array(b.meta["owner"]))
    assert owner_hits[np.array(b.meta["first_miss"]) > 0].all()
    assert (want["pick_match"][owner_hits] >= np.array(b.meta["first_miss"])[owner_hits]).all()


def test_chunk_case():
    c = S.chunk_case()
    b = c.batches[0]
    n = b.kw["n_hashes_in"].astype(int)
    assert {S.CHUNK - 1, S.CHUNK, S.CHUNK + 1, 2 * S.CHUNK + 1} <= set(n.tolist())
    ref = S.Ref(c)
    want = ref.run(b)
    C, T = S.index_cluster(c.E)
    assert C == 16 and b.meta["last"] // T == C - 1
    assert want["pick"][3] == b.meta["last"] and n[3] == 2 * S.CHUNK + 1
    assert want["pick_match"].max() > 512 and ((want["pick_match"] > 255) & (want["pick_match"] <= 512)).any()
    caps = b.caps
    paths = set()
    for r in range(b.R):
        p = int(want["pick"][r])
        cap = caps[p] if caps[p] > 0 else c.lru_default
        paths.add(("sequential" if n[r] > cap else "chunked", int(cap) if caps[p] > 0 else 0, n[r] > S.CHUNK))
    assert ("sequential", S.CHUNK - 1, False) in paths and ("sequential", S.CHUNK, True) in paths
    assert ("chunked", S.CHUNK, False) in paths and ("chunked", S.CHUNK + 1, True) in paths and ("chunked", 0, True) in paths
    for p, cap in zip(b.meta["caps_at"], (S.CHUNK - 1, S.CHUNK, S.CHUNK + 1)):
        assert 0 < ref.idx.lru_len(p) <= cap


def test_bitset_rows_form_and_empty():
    c = S.bitset_case()
    b = c.batches[0]
    ref = S.Ref(c)
    want = ref.run(b)
    eps = b.meta["eps"]
    C, T = S.index_cluster(c.E)
    assert len({e // T for e in eps}) == C == 16
    assert (want["pick"][:len(eps)] == eps).all()
    # after the first 24 requests every shared block is held by 24 endpoints; the second 24 requests probe those rows
    assert (want["pick_match"][len(eps):2 * len(eps)] >= len(b.meta["shared"])).all()
    # the last 24 requests evict the shared blocks everywhere: the rows are emptied again
    assert all(ref.idx.get(int(k)) == set() for k in b.meta["shared"])


@pytest.mark.parametrize("M", [2048, 8192])
@pytest.mark.parametrize("name", list(S.PICKERS))
def test_pickers_span_ctas(name, M):
    c = S.picker_case(name, M, seed=M + len(name))
    b = c.batches[0]
    ref = S.Ref(c)
    want = ref.run(b)
    C, T = S.index_cluster(M)
    picked = want["pick"][want["pick"] >= 0]
    assert len(set((picked // T).tolist())) > 1
    if name == "weighted":
        assert (want["pick_score"] > 0).any() and ((want["pick"] >= 0) & (want["pick_score"] <= 0)).any()
    if c.pick_mode == 0:
        assert (want["tie_count"] > 1).sum() >= 10
        crossing = _crossing_ties(c, b, want, T)
        assert crossing >= 5, crossing


def _crossing_ties(c, b, want, T):
    """requests whose tie set spans CTAs, from single-request oracle schedules against the index and loads requests 0..r-1
    left (replayed from the reference's picks)"""
    idx = o.Index(c.lru_default)
    S.seed_oracle(c, idx)
    from tests import inflight_oracle as I
    tracker = I.Tracker()
    prof = c.profile()
    crossing = 0
    for r in range(b.R):
        a, z = int(b.kw["prompt_off"][r]), int(b.kw["prompt_off"][r + 1])
        x = o.schedule_batch(o.SnapshotData(**c.sd, inflight_tokens=tracker.get(c.M)[1]), prof, idx, 1, request_base=r,
                             max_blocks=S.MB, want_tie_set=True, want_hashes=True,
                             prompt_bytes=np.ascontiguousarray(b.kw["prompt_bytes"][a:z]), prompt_off=np.array([0, z - a], np.int64),
                             model_seed=b.kw["model_seed"][r:r + 1], adapter_id=b.kw["adapter_id"][r:r + 1])
        assert x["pick"][0] == want["pick"][r]
        if want["tie_count"][r] > 1:
            members = np.nonzero(np.unpackbits(x["tie_set"][0].view(np.uint8), bitorder="little")[:c.M])[0]
            crossing += len(set((members // T).tolist())) > 1
        if x["pick"][0] >= 0:
            tracker.add(x["pick"][:1], b.tokens[r:r + 1])
            idx.commit(x["pick"][:1], x["hashes_out"][:1], x["total_blocks"][:1])
    return crossing


def test_latency_tiers_and_ranges():
    """every rank 0-4 occurs as a request's lowest tier, with single-candidate rows and each one-side-degenerate range"""
    seen, tdeg, pdeg, both, single = set(), 0, 0, 0, 0
    for M, E in ((200, 256), (3000, 4096)):
        c = S.tier_case(M, E, seed=M)
        b = c.batches[0]
        want = S.Ref(c).run(b, index_form=False)
        for t in S.tiers(c, b, want):
            seen.add(t["rank"])
            tdeg += t["tdeg"] and not t["pdeg"]
            pdeg += t["pdeg"] and not t["tdeg"]
            both += t["tdeg"] and t["pdeg"] and len(t["members"]) > 1
            single += len(t["members"]) == 1
    assert seen >= {0, 1, 2, 3, 4}, seen
    assert tdeg and pdeg and both and single, (tdeg, pdeg, both, single)


def test_latency_tier_in_one_cta():
    M = E = 4096
    C, T = S.flight_cluster(E)
    lo, hi = 9 * T, 10 * T
    c = S.tier_case(M, E, seed=5, one_cta=(lo, hi))
    b = c.batches[0]
    want = S.Ref(c).run(b, index_form=False)
    ts = S.tiers(c, b, want)
    inside = [t for t in ts if len(t["members"]) and t["members"].min() >= lo and t["members"].max() < hi]
    assert len(inside) >= b.R // 4 and C == 16


@pytest.mark.parametrize("name", list(S.PARAMS))
def test_latency_params(name):
    c = S.param_case(name, 300, 512)
    b = c.batches[0]
    want = S.Ref(c).run(b, index_form=False)
    assert (want["pick"] >= 0).all()
    if name == "most":
        ranks = {t["rank"] for t in S.tiers(c, b, want)}
        assert 0 in ranks and len(ranks) > 1, ranks
    if name == "composite-nonpos":
        q = c.sd["queue"]
        assert int(q.max()) - int(q.min()) > 2 ** 53 and (q < 0).any()
    if name == "composite":
        assert (c.sd["queue"] < 0).any()


def test_queue_values():
    c = S.queue_case(300, 512)
    b = c.batches[0]
    ref = S.Ref(c)
    want = ref.run(b, index_form=False)
    tp = b.kw["tpot_slo"]
    for v in S.SPECIAL_TPOT:
        sel = (tp == v) & (np.signbit(tp) == np.signbit(v)) & want["added"]
        assert sel.any(), v
    down = b.meta["down"]
    assert (want["pick"][0:40:2] == down).all() and want["added"][0:40:2].all()
    assert (want["pick"][1:40:2] == b.meta["flat"]).all() and want["added"][1:40:2].all()
    mn, cnt = ref.q.get(c.E)
    assert mn[b.meta["flat"]] == 7.0 and cnt[b.meta["flat"]] >= 20
    assert all(cnt[m] > 0 for m in b.meta["far"])


def test_repeat_keys_across_slices():
    c = S.repeat_keys_case(300, 8192)
    b = c.batches[0]
    rows = b.meta["rows"]
    assert b.R > rows
    want = S.Ref(c).run(b, index_form=False)
    assert want["added"][:40].all()
    assert not want["added"][rows:rows + 20].any() and want["added"][rows + 20:rows + 40].all()
