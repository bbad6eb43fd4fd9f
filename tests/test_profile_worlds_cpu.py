"""The worlds of tests/test_gpu_profile_edges.py reach the edges their GPU tests are about, checked with the CPU oracle alone:
a subset that drops the zero-match arg-max, deferred requests on a subset profile, member min/max ranges that decide the
value-bucket table, device batches large enough to be sliced, and producer state that changes the picks."""
import numpy as np
import pytest

from oracle import oracle_py as o
from tests import profile_worlds as W


@pytest.fixture(scope="module")
def argmax_world():
    return W.world_argmax()


def _prof(scorers, tie_mode=0):
    return o.make_profile([(W.SCORER[k], wt) for k, wt in scorers], tie_mode=tie_mode, token_load_threshold=W.TOKEN_THR)


def test_argmax_world_drops_the_zero_match_argmax(argmax_world):
    w = argmax_world
    snap, prof, mem = w.snap(), _prof(W.ARGMAX_SCORERS), set(w.members)
    member_mask = W.bits(w.M, w.members)
    member_ties = {}
    for a in W.ARGMAX_ADAPTERS:
        g = o.schedule_one(snap, prof, adapter_id=a)
        sub = o.schedule_one(snap, prof, adapter_id=a, mask=member_mask)
        member_ties[a] = sub["tie_count"]
        assert sub["pick"] in mem and g["pick"] not in mem, a
        if a == 4:  # the member maximum ties with a non-member
            assert g["score"] == sub["score"] and set(g["tie_set"]) - mem and set(g["tie_set"]) & mem
        else:       # the whole all-endpoint tie set lies outside the subset
            assert g["score"] > sub["score"] and not set(g["tie_set"]) & mem, a
    assert member_ties[5] == 3 and member_ties[3] == 1 and member_ties[4] == 1
    assert all(member_ties[a] == len(mem) - 1 for a in (0, 1, 2, 6, -1))  # every member but 14 (kv 0.75)
    # member exceptions that land exactly on the member maximum (pick_sparse's exc_ties case): rows 4 and 5 on the F and W
    # prompts (fully cached on members 30 and 20, zero-match score below the maximum... or, for 20 in row 5, in the tie set)
    want = W.oracle_run(w, W.ARGMAX_SCORERS, 0, 0, subset=member_mask)
    ad = w.kw["adapter_id"]
    tied = (w.kind == "F") & np.isin(ad, [4, 5])
    assert tied.sum() >= 10
    assert np.all(want["pick_score"][tied] == 4.0)
    assert np.all(want["tie_count"][tied] == np.where(ad[tied] == 5, 4, 2))
    assert np.all(want["pick"][tied] == np.where(ad[tied] == 5, 20, 16))
    # W in row 4: member 20 (zero-match 3.0, in no tie set) reaches 4.0 = the member maximum
    w4 = (w.kind == "W") & (ad == 4)
    assert w4.any() and np.all(want["tie_count"][w4] == 2)
    # N prompts: every exception is a non-member, so the subset's result is the zero-match one
    n = w.kind == "N"
    nomatch = W.oracle_run(w, W.ARGMAX_SCORERS, 0, 0, subset=member_mask, idx=o.Index())
    assert np.array_equal(want["pick"][n], nomatch["pick"][n]) and np.array_equal(want["tie_count"][n], nomatch["tie_count"][n])


def test_deferral_world_classes():
    w = W.world_deferral()
    idx = w.index()
    h, n = w.batch_hashes()
    mem = set(w.members)
    seen = set()
    for r in range(w.R):
        c = w.cls[r]
        eps = set(np.nonzero(idx.match(h[r, :n[r]], w.M))[0].tolist())
        inm = eps & mem
        if c == "a":
            assert len(eps) > W.EXC_MAX and 0 < len(inm)
        elif c == "b":
            assert len(eps) > W.EXC_MAX and not inm
        elif c == "c":
            assert len(eps) > W.EXC_MAX and 0 < len(inm) <= W.EXC_MAX
        elif c == "d":
            sizes = [len(idx.get(int(x))) for x in h[r, :12]]
            assert max(sizes) > W.INLINE_EPS and 0 < min(sizes) <= W.INLINE_EPS and len(eps) <= W.EXC_MAX
            assert idx.get(int(h[r, 12])) == set()  # the tail is new: 12 matched blocks
        elif c == "e":
            sets = [idx.get(int(x)) for x in h[r, :12]]
            assert all(s == sets[0] for s in sets) and len(sets[0]) <= W.INLINE_EPS and sets[0] & mem
            assert len(eps) == len(sets[0])
        else:
            assert not eps
        seen.add(c)
    assert seen == set(W.DEFER_CLASSES)
    # on the deferred classes the all-endpoint pick is a non-member for some requests: scoring them on all-member rows
    # would be caught
    allp = W.oracle_run(w, W.PREFILL, 0, 0)
    sub = W.oracle_run(w, W.PREFILL, 0, 0, subset=W.bits(w.M, w.members))
    for c in "abc":
        rows = w.cls == c
        assert np.isin(allp["pick"][rows], w.members, invert=True).any(), c
        assert np.isin(sub["pick"][rows], w.members).all(), c


@pytest.mark.parametrize("variant", W.MINMAX_VARIANTS)
def test_minmax_world_ranges(variant):
    w = W.world_minmax(variant)
    M, mem = w.M, w.members
    assert M % 32 and M < w.max_endpoints
    for which in ("queue", "running"):
        v = w.sd[which]
        full, sub = W.value_range(v, range(M)), W.value_range(v, mem)
        if variant == "bucket_by_subset":
            assert full >= 256 > sub
        elif variant == "scan":
            assert sub >= 256
        else:
            assert sub < 256 and np.asarray(v)[mem].min() >= 2 ** 40
        # the member min / max is not the all-endpoint one, so a term folded over every endpoint differs
        vv = np.asarray(v)
        assert (vv[mem].min(), vv[mem].max()) != (vv.min(), vv.max())
    encs = W.minmax_encodings(w)
    for name, words, eff in encs:
        assert W.members_of(words, M) == list(eff), name
    names = {n: wd for n, wd, _ in encs}
    assert names["above_M"].size * 32 == w.max_endpoints and W.members_of(names["above_M"], 256) != list(mem)
    assert names["past_max"].size * 32 > w.max_endpoints and names["short"].size * 32 < w.max_endpoints
    # the no-mask run of the subset profile differs from the run over every endpoint
    sub = W.oracle_run(w, W.QUEUE_RUNNING, 0, 0, subset=W.bits(M, mem))
    allp = W.oracle_run(w, W.QUEUE_RUNNING, 0, 0)
    assert not np.array_equal(sub["pick_score"], allp["pick_score"])


def test_sliced_world_is_sliced_and_defers():
    w = W.world_sliced()
    for K in (3, 4, 6):
        assert w.R // K >= W.SLICE_MIN
    idx = w.index()
    h, n = w.batch_hashes()
    rows_b = np.nonzero(w.pool == "b")[0]
    per = ((w.R + 5) // 6 + 63) // 64 * 64
    assert len(set(rows_b // per)) == 6  # every slice of six has pool-b requests
    odd = set(range(1, w.M, 2))
    many = [len(set(np.nonzero(idx.match(h[r, :n[r]], w.M))[0].tolist())) for r in rows_b[:40]]
    assert min(many) > W.EXC_MAX  # deferred on profile 1 (odd endpoints) ...
    assert any(set(np.nonzero(idx.match(h[r, :n[r]], w.M))[0].tolist()) & odd for r in rows_b[:40])  # ... with members


def test_producer_world_state_changes_picks():
    w = W.world_producers()
    rng = np.random.Generator(np.random.PCG64(5))
    tokens = rng.integers(0, 60000, w.M).astype(np.int64)
    a = W.oracle_run(w, W.TOKEN_PROFILE, 0, 0, subset=w.token_subset)
    b = W.oracle_run(w, W.TOKEN_PROFILE, 0, 0, subset=w.token_subset, snap=w.snap(inflight_tokens=tokens))
    assert (a["pick"] != b["pick"]).sum() > w.R // 10
    lat = o.make_latency_params(**W.LAT_COEF)
    c = W.oracle_run(w, W.LATENCY_PROFILE, 0, 0, subset=w.latency_subset, latency=lat)
    d = W.oracle_run(w, W.LATENCY_PROFILE, 0, 0, subset=w.latency_subset, latency=lat,
                     snap=w.snap(min_tpot_slo=rng.choice([0.0, 20.0, 26.0], w.M), dispatched=rng.integers(0, 3, w.M).astype(np.int32)))
    assert not np.array_equal(c["pick_score"].view(np.uint64), d["pick_score"].view(np.uint64))
