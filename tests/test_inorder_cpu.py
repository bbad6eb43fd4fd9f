"""The sequential reference of eppscore_schedule_batch_inorder (tests/inorder_reference.py) against a hand restatement of the
token-load scorer (token_load.go:83-111) and PreRequest's add (inflightload/producer.go:101-120) on small worlds: a batch route
that piles every request onto one endpoint where the sequential one spreads them, the threshold clamp, counters made negative
by releases, and a request without candidates."""
import numpy as np
import pytest

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.inorder_reference import schedule_inorder

TOKEN_LOAD, KV = 6, 1


@pytest.fixture(scope="module", autouse=True)
def built():
    o.build()
    I.build()


def hand(loads, tokens, threshold, weight=1.0, kv=None, kv_weight=0.0, cand=None):
    """max-score picks (lowest index on ties) with the counters moving after every pick"""
    loads = list(loads)
    picks, scores = [], []
    for r, t in enumerate(tokens):
        best, arg = None, -1
        for m, load in enumerate(loads):
            if cand is not None and not cand[r][m]:
                continue
            tl = 1.0 if load <= 0 else 1.0 - min(load, threshold) / threshold
            s = 0.0
            if kv is not None:
                s += (1.0 - kv[m]) * kv_weight
            s += min(max(tl, 0.0), 1.0) * weight
            if best is None or s > best:
                best, arg = s, m
        picks.append(arg)
        scores.append(best if arg >= 0 else 0.0)
        if arg >= 0:
            loads[arg] += t
    return picks, scores, loads


def snapshot(M, kv=None):
    return dict(kv_usage=np.zeros(M) if kv is None else np.asarray(kv, np.float64), queue=np.zeros(M, np.int64))


def test_sequential_spreads_where_the_batch_piles_up():
    M, R = 4, 12
    prof = o.make_profile([(TOKEN_LOAD, 1.0)], token_load_threshold=1000.0)
    tokens = np.full(R, 100, np.int64)
    batch = o.schedule_batch(o.SnapshotData(**snapshot(M)), prof, None, R)
    assert set(batch["pick"].tolist()) == {0}  # one load view: every request on the arg-max endpoint
    got, tr = schedule_inorder(snapshot(M), prof, None, R, tokens)
    picks, scores, loads = hand([0] * M, tokens, 1000.0)
    assert got["pick"].tolist() == picks == [0, 1, 2, 3] * 3
    assert got["pick_score"].tolist() == scores
    req, tok = tr.get(M)
    assert tok.tolist() == loads and req.tolist() == [3] * M


def test_threshold_clamp_and_kv_order():
    M = 3
    kv = [0.5, 0.25, 0.0]
    prof = o.make_profile([(KV, 2.0), (TOKEN_LOAD, 1.0)], token_load_threshold=50.0)
    tokens = np.array([80, 10, 60, 5, 5, 200, 1], np.int64)
    got, tr = schedule_inorder(snapshot(M, kv), prof, None, len(tokens), tokens)
    picks, scores, loads = hand([0] * M, tokens, 50.0, 1.0, kv, 2.0)
    assert got["pick"].tolist() == picks
    assert got["pick_score"].tolist() == scores
    assert tr.get(M)[1].tolist() == loads
    assert max(loads) > 50  # past the threshold the term stays at 0


def test_negative_counters_after_releases():
    M = 3
    prof = o.make_profile([(TOKEN_LOAD, 1.0)], token_load_threshold=100.0)
    tr = I.Tracker()
    tr.add([1, 2], [30, 5])
    tr.remove(1)
    tr.release([1], [30])  # endpoint 1 now holds -30 tokens: a load <= 0 scores 1.0
    tokens = np.array([20, 20, 20, 20], np.int64)
    got, tr = schedule_inorder(snapshot(M), prof, None, 4, tokens, tracker=tr)
    picks, scores, loads = hand([0, -30, 5], tokens, 100.0)
    assert got["pick"].tolist() == picks
    assert got["pick_score"].tolist() == scores
    assert tr.get(M)[1].tolist() == loads


def test_request_without_candidates_adds_nothing():
    M, R = 2, 4
    prof = o.make_profile([(TOKEN_LOAD, 1.0)], token_load_threshold=100.0)
    cand = np.array([[3], [0], [2], [3]], np.uint32)
    rows = [[bool((w[0] >> m) & 1) for m in range(M)] for w in cand]
    tokens = np.array([10, 99, 10, 10], np.int64)
    got, tr = schedule_inorder(snapshot(M), prof, None, R, tokens, cand_mask=cand)
    picks, scores, loads = hand([0] * M, tokens, 100.0, cand=rows)
    assert got["pick"].tolist() == picks and picks[1] == -1
    assert got["tie_count"][1] == 0
    req, tok = tr.get(M)
    assert tok.tolist() == loads and int(req.sum()) == 3
