"""The sequential reference of eppscore_schedule_batch_inorder_latency (tests/inorder_latency_reference.py) on the CPU oracle:
in an overloaded fleet the first k requests of a batch spread over the k idle endpoints where a batch-wide view sends them all
to one, and a request with a tight TPOT SLO takes its target out of the positive tier for the requests after it."""
import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q
from tests.inorder_latency_reference import schedule_inorder_latency

KV, LATENCY = 1, 5
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01, streaming_mode=1)


def setup_module():
    o.build()
    I.build()
    Q.build()


def _world(M, seed):
    rng = np.random.default_rng(seed)
    return dict(kv_usage=rng.random(M), queue=rng.integers(0, 8, M).astype(np.int64), running=rng.integers(0, 8, M).astype(np.int64))


def _mask(rows, M):
    out = np.zeros((len(rows), (M + 31) // 32), np.uint32)
    for r, eps in enumerate(rows):
        for m in eps:
            out[r, m >> 5] |= np.uint32(1 << (m & 31))
    return out


def test_overloaded_fleet_spreads_over_the_idle_endpoints():
    M, k, R = 16, 5, 12
    snap = _world(M, 1)
    prof = o.make_profile([(KV, 1.0), (LATENCY, 2.0)], latency=o.make_latency_params(**LAT_COEF))
    idle = [2, 5, 9, 11, 14]
    q = Q.Queues(M)
    busy = [m for m in range(M) if m not in idle]
    q.add(np.array(busy, np.int32), np.arange(1, len(busy) + 1, dtype=np.uint64), np.full(len(busy), 50.0))
    ttft = np.full(R, 1.0)  # below every prediction: every candidate's TTFT headroom is negative
    tpot = np.full(R, 50.0)
    key = np.arange(1000, 1000 + R, dtype=np.uint64)
    # batch-wide: every request sees the same idle set, and the least-deficit rule sends all of them to one endpoint
    mn, cnt = q.get(M)
    wide = o.schedule_batch(o.SnapshotData(**snap, min_tpot_slo=Q.canonical(mn), dispatched=cnt), prof, None, R,
                            ttft_slo=ttft, tpot_slo=tpot)
    assert len(set(wide["pick"][:k].tolist())) == 1 and wide["pick"][0] in idle
    # in order: each pick leaves the idle tier, so the first k requests take the k idle endpoints
    got, _ = schedule_inorder_latency(snap, prof, None, R, q, request_key=key, ttft_slo=ttft, tpot_slo=tpot)
    assert sorted(got["pick"][:k].tolist()) == idle
    assert got["added"].all()
    assert np.array_equal(q.get(M)[1], np.ones(M, np.int32) + np.bincount(got["pick"][k:], minlength=M))


def test_tight_tpot_slo_tightens_its_target_for_later_requests():
    M = 8
    snap = _world(M, 2)
    prof = o.make_profile([(KV, 1.0), (LATENCY, 2.0)], latency=o.make_latency_params(**LAT_COEF))
    ttft, tpot = np.array([1e6, 1e6]), np.array([1e-3, 1e3])  # request 0 tight, request 1 loose
    # where the loose request goes when nothing tightened any endpoint
    mn, cnt = Q.Queues(M).get(M)
    alone = o.schedule_batch(o.SnapshotData(**snap, min_tpot_slo=Q.canonical(mn), dispatched=cnt), prof, None, 1,
                             ttft_slo=ttft[1:], tpot_slo=tpot[1:])
    P = int(alone["pick"][0])
    mask = _mask([[P], range(M)], M)  # the tight request is sent there
    q = Q.Queues(M)
    got, _ = schedule_inorder_latency(snap, prof, None, 2, q, request_key=np.array([1, 2], np.uint64), cand_mask=mask,
                                      ttft_slo=ttft, tpot_slo=tpot)
    assert got["pick"][0] == P and got["added"].all()
    assert got["pick"][1] != P  # P's TPOT bound is now the tight request's: negative headroom, out of the positive tier
    # its latency score for request 1: 0 at P (outside the selected positive tier), positive at every other endpoint
    q1 = Q.Queues(M)
    q1.add([P], [1], tpot[:1])
    mn, cnt = q1.get(M)
    scores, _ = o.score_latency(prof.latency.contents, o.SnapshotData(**snap, min_tpot_slo=Q.canonical(mn), dispatched=cnt),
                             ttft_slo=ttft[1], tpot_slo=tpot[1])
    assert scores[P] == 0.0 and (np.delete(scores, P) > 0).all()
