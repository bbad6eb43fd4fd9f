"""eppscore_schedule_batch_inorder_latency at the edges of its walk, in both forms (inorder_pick_lat_kernel and
inorder_index_lat_kernel) at C = 1 and at the widest cluster each has, bit-exact against the sequential reference
(tests/inorder_latency_reference.py) on the cases of tests/inorder_walk_scenarios.py: strategy "most" over batches whose lowest
tier is 0 for some requests and not for others, slo_buffer_factor 0.5 and 1.3, TTFT / TPOT weights (1, 0), (0, 1), (0, 0) and
(1, -0.99999999), composite weights (non-default, summing to <= 0) over negative queue values and ranges past 2^53; every rank
0-4 as a lowest tier, a lowest tier held by one non-zero CTA only, one-side-degenerate headroom ranges and single candidates;
queue values -0.0, +0.0, +Inf, 5e-324 and 1e308, a falling minimum, equal minima removed one at a time afterwards, live entries
past M and keys repeated across slices; and every picker over several CTAs.  Picks, scores (as uint64), tie counts, totals,
added_out, pick_match, the in-flight counters, running_get (bitwise) and, in the index form, the whole prefix index are
compared."""
import numpy as np
import pytest

from tests import inorder_walk_scenarios as S
from tests.helpers import synth_ragged_prompts
from tests.test_gpu_inorder_index_edges import CaseWorld, _u64, pkg  # noqa: F401  (pkg: the module fixture)

pytestmark = pytest.mark.gpu

# (index form, max_endpoints): C = 1 and the widest cluster of each walk
SHAPES = [(False, 256), (False, 4096), (True, 512), (True, 8192)]


def _shape_id(s):
    index_form, E = s
    C = (S.index_cluster(E) if index_form else S.flight_cluster(E))[0]
    return f"{'index' if index_form else 'inflight'}-C{C}"


def _prompts(c, seed):
    """the index form walks the index too: prompts whose blocks it probes and commits"""
    for b in c.batches:
        pb, off = synth_ragged_prompts(b.R, max_len=S.MB * 64, seed=seed, groups=6, shared=512)
        b.kw.update(prompt_bytes=pb, prompt_off=off, model_seed=np.full(b.R, 5, np.uint64))


def _run(pkg, c, index_form, seed):
    if index_form:
        _prompts(c, seed)
    w = CaseWorld(pkg, c)
    b = c.batches[0]
    got, want = w.run(b, index_form=index_form)
    if index_form:
        w.check_index(c.name)
    return w, got, want


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
@pytest.mark.parametrize("name", list(S.PARAMS))
def test_params(pkg, name, shape):
    index_form, E = shape
    c = S.param_case(name, min(E, 300) if E <= 512 else E - 5, E)
    w, got, want = _run(pkg, c, index_form, 7)
    w.close()


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_tiers(pkg, shape):
    index_form, E = shape
    c = S.tier_case(min(E, 200) if E <= 512 else E - 96, E, seed=E)
    w, got, want = _run(pkg, c, index_form, 11)
    w.close()


@pytest.mark.parametrize("index_form", [False, True], ids=["inflight-C16", "index-C16"])
def test_lowest_tier_in_one_cta(pkg, index_form):
    E = 4096 if not index_form else 8192
    C, T = (S.index_cluster(E) if index_form else S.flight_cluster(E))
    c = S.tier_case(E, E, seed=5, one_cta=(9 * T, 10 * T))
    w, got, want = _run(pkg, c, index_form, 13)
    assert C == 16
    w.close()


@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
def test_queue_values_then_removes(pkg, shape):
    """after the batch, the view compared after each remove call: `down`'s entries one call at a time, the minimum first (a
    count at the minimum the walk left too high keeps a minimum that is gone), then all of `flat`'s equal minima in one call
    (a count left too low never reaches 0 there, so the minimum is not recomputed); the entries live on endpoints in [M, E)
    come back unchanged"""
    index_form, E = shape
    M = min(E, 300) if E <= 512 else E - 40
    c = S.queue_case(M, E)
    b = c.batches[0]
    far = b.meta["far"]
    w, got, want = _run(pkg, c, index_form, 17)
    gm, gc = w.eng.running_get(E)
    for e in far:
        assert gc[e] == 1
    tp = b.kw["tpot_slo"]
    down = np.flatnonzero((want["pick"] == b.meta["down"]) & want["added"])
    for r in down[np.argsort(tp[down], kind="stable")]:
        e, k = want["pick"][r:r + 1], b.key[r:r + 1]
        assert np.array_equal(w.eng.running_remove(e, k), w.ref.q.remove(e, k))
        w.check_counters(("remove", r))
    flat = np.flatnonzero((want["pick"] == b.meta["flat"]) & want["added"] & (tp == 7.0))
    assert len(flat) >= 20
    e, k = want["pick"][flat], b.key[flat]
    assert np.array_equal(w.eng.running_remove(e, k), w.ref.q.remove(e, k))
    w.check_counters("remove the equal minima")
    gm2, gc2 = w.eng.running_get(E)
    assert np.array_equal(_u64(gm2[far]), _u64(gm[far])) and np.array_equal(gc2[far], gc[far])
    w.close()


@pytest.mark.parametrize("index_form", [False, True], ids=["inflight-C16", "index-C16"])
def test_keys_repeated_across_slices(pkg, index_form):
    c = S.repeat_keys_case(300, 8192)
    w, got, want = _run(pkg, c, index_form, 19)
    rows = c.batches[0].meta["rows"]
    assert not want["added"][rows:rows + 20].any() and want["added"][rows + 20:rows + 40].all()
    w.close()


@pytest.mark.parametrize("E", [2048, 4096], ids=lambda E: f"C{S.flight_cluster(E)[0]}")
@pytest.mark.parametrize("name", list(S.PICKERS))
def test_pickers_and_ties(pkg, name, E):
    """the in-flight latency walk (the index form's pickers run in tests/test_gpu_inorder_index_edges.py)"""
    c = S.picker_case(name, E, seed=E + len(name), lat=True)
    w = CaseWorld(pkg, c)
    got, want = w.run(c.batches[0], index_form=False)
    C, T = S.flight_cluster(E)
    picked = want["pick"][want["pick"] >= 0]
    assert len(set((picked // T).tolist())) > 1
    w.close()


@pytest.mark.parametrize("E", [256, 4096])
def test_infinite_slos_plain_batch(pkg, E):
    """score_matrix_kernel's scoreBucket on the same edge as the walk's: TPOT SLO +Inf makes every idle endpoint's TPOT headroom
    +Inf, so the idle tier's range is infinite and those weights NaN (math.MinInt64 through int(), then 0); TTFT SLO +Inf the
    same for the TTFT headroom.  A plain batch against the oracle with the queue view in the snapshot."""
    from oracle import oracle_py as o
    M, R = E - 3, 300
    c = S.lat_base(M, E, R, seed=E)
    rng = np.random.Generator(np.random.PCG64(E))
    b = c.batches[0]
    b.kw["ttft_slo"] = rng.choice([0.0, 140.0, np.inf], R)
    b.kw["tpot_slo"] = rng.choice([0.0, 24.0, np.inf], R)
    mn = np.where(rng.random(M) < 0.5, 0.0, rng.choice([12.0, 30.0, np.inf, 5e-324], M))
    cnt = np.where(mn > 0, rng.integers(1, 4, M), 0).astype(np.int32)
    eng = pkg.Engine(pkg.default_config(c.scorers, max_endpoints=E, token_load_threshold=c.threshold, tie_seed=S.SEED, tie_mode=1))
    eng.set_latency_params(pkg.latency_params(**c.lat))
    eng.set_snapshot(**c.sd, min_tpot_slo=mn, dispatched=cnt)
    got = eng.schedule(R, **b.kw)
    want = o.schedule_batch(o.SnapshotData(**c.sd, min_tpot_slo=mn, dispatched=cnt), c.profile(), None, R, **b.kw)
    for k in ("pick", "tie_count"):
        assert np.array_equal(got[k], want[k]), (k, np.flatnonzero(got[k] != want[k])[:5])
    assert np.array_equal(_u64(got["pick_score"]), _u64(want["pick_score"]))
    assert (np.isinf(b.kw["tpot_slo"]) & (b.kw["ttft_slo"] == 0)).any()
    eng.close()
