"""maxNumOfEndpoints (picker/common.go:39-42) on the CPU oracle: tests/cpp/topk_oracle.c against the reference's own picker tests
(maxscore/picker_test.go:43-110, random/picker_test.go:40-119), the exact successive-sampling law of the weighted-random
picker (weightedrandom/picker.go:121-152), and entry 0 against orc_schedule_one's pick in every mode."""
import itertools
import json
import os

import numpy as np
import pytest

from oracle import oracle_py as o
from tests import topk_oracle as T
from tests.helpers import mask_from_list, synth_snapshot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _scores_snapshot(scores):
    # scores arrive through a custom per-endpoint column scorer with weight 100: score = clamp(col) * 100
    M = len(scores)
    return o.SnapshotData([0.0] * M, [0] * M, endpoint_cols=[np.array(scores, np.float64) / 100.0])


def _weighted(scores, **prof):
    res = o.schedule_one(_scores_snapshot(scores), o.make_profile([(o.SCORER_ENDPOINT_COL0, 100.0)], **prof))
    return res["weighted"]


@pytest.mark.parametrize("tie_mode", [o.TIE_LOWEST_INDEX, o.TIE_SEEDED_RANDOM])
def test_max_score_vectors(golden, tie_mode):
    for c in golden["picker"]["cases"]:
        n, k, t = len(c["scores"]), c["max_num"], c["tie_break_candidates"]
        prof = o.make_profile([(o.SCORER_ENDPOINT_COL0, 100.0)], tie_mode=tie_mode, tie_seed=11)
        for r in range(16):
            got, sc = T.pick_topk(_weighted(c["scores"]), prof, r, k)
            want = c["want_order"]
            assert len(want) == min(k, n)
            assert (got[len(want):] == -1).all() and (sc[len(want):] == 0.0).all(), c["name"]
            got = [int(x) for x in got[: len(want)]]
            if tie_mode == o.TIE_LOWEST_INDEX:
                assert got == want, c["name"]
            else:  # a uniformly random order inside the tie class
                assert sorted(got[:t]) == sorted(want[:t]) and got[t:] == want[t:], c["name"]
            assert list(sc[: len(want)]) == [float(c["scores"][m]) for m in got]


def test_max_score_seeded_ties_are_shuffled():
    # five equal scores: every order of the tie class shows up, each first position about equally often
    prof = o.make_profile([(o.SCORER_ENDPOINT_COL0, 100.0)], tie_mode=o.TIE_SEEDED_RANDOM, tie_seed=5)
    w = _weighted([40] * 5)
    firsts = np.zeros(5)
    orders = set()
    for r in range(4000):
        got, _ = T.pick_topk(w, prof, r, 5)
        assert sorted(got) == [0, 1, 2, 3, 4]
        firsts[got[0]] += 1
        orders.add(tuple(got))
    assert np.abs(firsts / 4000 - 0.2).max() <= 0.05
    assert len(orders) == 120


def test_random_picker_vectors():
    with open(os.path.join(ROOT, "tests", "golden", "random_picker_vectors.json")) as f:
        g = json.load(f)
    n_it, tol = g["iterations"], g["tolerance"]
    prof = o.make_profile([(o.SCORER_ENDPOINT_COL0, 100.0)], tie_seed=99, pick_mode=o.PICK_RANDOM)
    for c in g["cases"]:
        n, k = len(c["scores"]), c["max_num"]
        w = _weighted(c["scores"])
        counts = np.zeros(n)
        for r in range(n_it):
            got, sc = T.pick_topk(w, prof, r, k)
            real = got[got >= 0]
            assert len(real) == c["num_pods"] and len(set(real.tolist())) == len(real), c["name"]
            assert list(sc[: len(real)]) == [float(c["scores"][m]) for m in real]
            counts[real] += 1
        want = min(c["num_pods"] / n, 1.0)
        assert np.abs(counts / n_it - want).max() <= tol, (c["name"], counts / n_it)


def _successive_sampling_inclusion(w, k):
    """P(m among the first k draws without replacement, each draw proportional to w): enumerate the ordered draws,
    P(sequence) = prod w_i / (W - sum of the earlier draws).  Zero weights are never drawn while a positive one is left;
    they fill the remaining places uniformly."""
    w = np.asarray(w, np.float64)
    pos = [m for m in range(len(w)) if w[m] > 0]
    zero = [m for m in range(len(w)) if w[m] <= 0]
    p = np.zeros(len(w))
    kp = min(k, len(pos))
    W = w[pos].sum()
    for seq in itertools.permutations(pos, kp):
        pr, rest = 1.0, W
        for m in seq:
            pr *= w[m] / rest
            rest -= w[m]
        p[list(seq)] += pr
    if k > len(pos) and zero:
        p[zero] = min(k - len(pos), len(zero)) / len(zero)
    return p


@pytest.mark.parametrize("k", [2, 3])
def test_weighted_random_inclusion_law(golden, k):
    n_it, tol = 10000, 0.05
    cases = [c["scores"] for c in golden["stochastic_pickers"]["weighted"]] + [[5, 0, 0, 20], [0, 0, 0]]
    for scores in cases:
        prof = o.make_profile([(o.SCORER_ENDPOINT_COL0, 100.0)], tie_seed=1234, pick_mode=o.PICK_WEIGHTED_RANDOM)
        w = _weighted(scores)
        counts = np.zeros(len(scores))
        for r in range(n_it):
            got, _ = T.pick_topk(w, prof, r, k)
            real = got[got >= 0]
            assert len(real) == min(k, len(scores)) and len(set(real.tolist())) == len(real)
            # the candidates with score > 0 come first
            npos = int((np.asarray(scores)[real] > 0).sum())
            assert (np.asarray(scores)[real[:npos]] > 0).all()
            counts[real] += 1
        want = _successive_sampling_inclusion(scores, k)
        assert np.abs(counts / n_it - want).max() <= tol, (scores, counts / n_it, want)


@pytest.mark.parametrize("pick_mode", [o.PICK_MAX_SCORE, o.PICK_WEIGHTED_RANDOM, o.PICK_RANDOM])
@pytest.mark.parametrize("tie_mode", [o.TIE_LOWEST_INDEX, o.TIE_SEEDED_RANDOM])
def test_entry0_is_the_pick(pick_mode, tie_mode):
    rng = np.random.default_rng(3 + pick_mode * 2 + tie_mode)
    for trial in range(40):
        M = int(rng.integers(1, 70))
        sd = synth_snapshot(M, seed=trial, tie_heavy=True)
        snap = o.SnapshotData(**sd)
        prof = o.make_profile([(o.SCORER_QUEUE, 1.0), (o.SCORER_KV_CACHE, 1.0), (o.SCORER_LORA, 1.0)], tie_mode=tie_mode,
                              tie_seed=int(rng.integers(0, 2**63)), pick_mode=pick_mode)
        keep = [m for m in range(M) if rng.random() < 0.7]
        mask = mask_from_list(M, keep)
        k = int(rng.integers(1, 9))
        r = int(rng.integers(0, 1 << 40))
        one = o.schedule_one(snap, prof, request_index=r, adapter_id=int(rng.integers(-1, 64)), mask=mask)
        got, sc = T.pick_topk(one["weighted"], prof, r, k)
        n = min(k, len(keep))
        assert (got[n:] == -1).all() and (sc[n:] == 0.0).all()
        assert len(set(got[:n].tolist())) == n and set(got[:n].tolist()) <= set(keep)
        if not keep:
            assert one["pick"] == -1
            continue
        assert got[0] == one["pick"] and sc[0] == one["score"]
        assert np.array_equal(sc[:n], one["weighted"][got[:n]])
        if pick_mode == o.PICK_MAX_SCORE:
            assert (np.diff(sc[:n]) <= 0).all()


def test_schedule_batch_topk_rows():
    M, R = 40, 64
    snap = o.SnapshotData(**synth_snapshot(M, seed=4, tie_heavy=True))
    prof = o.make_profile([(o.SCORER_QUEUE, 2.0), (o.SCORER_KV_CACHE, 1.0)], tie_mode=o.TIE_SEEDED_RANDOM, tie_seed=9)
    res = T.schedule_batch(snap, prof, None, R, request_base=1000, topk=4)
    assert res["topk_pick"].shape == (R, 4) and res["topk_score"].shape == (R, 4)
    assert np.array_equal(res["topk_pick"][:, 0], res["pick"]) and np.array_equal(res["topk_score"][:, 0], res["pick_score"])
    for r in range(R):
        got, sc = T.pick_topk(res["weighted_out"][r], prof, 1000 + r, 4)
        assert np.array_equal(got, res["topk_pick"][r]) and np.array_equal(sc, res["topk_score"][r])
