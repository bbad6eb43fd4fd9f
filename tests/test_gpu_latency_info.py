"""eppscore_predict_latency on the GPU: the predicted-latency producer's LatencyPredictionInfo and prefix cache score at the
endpoints a request was sent to, bit-exact to the oracle's orc_latency_predict + orc_latency_validate fed the oracle's
matchLongestPrefix count (and, for `dispatched` / podMinTPOTSLO from the running-request queues, the queue oracle).  Covered:
picks and lists of the sparse, full-matrix, masked, latency-behind-both-filters, top-k, wide top-k and two-profile routes;
ttft / tpot against a diagnostic batch's pred_out; TTFT == SLO, TPOT == buffered, SLO 0, podMinTPOTSLO 0 / below / above,
streaming and not, prefill-role endpoints, has_predictions = 0; total 0 and partial matches; dispatched from the snapshot and
from the queues before and after running_add; entries -1 and >= M; k 1 / 32 / 33 / max_endpoints; n_hashes 0 / 256 / 1000;
M 5 / 1024 / 4097; host and device location; a reserved stream next to batches on other streams; ordering against running_add
on another stream; 24 replays of a schedule -> predict_latency -> commit -> running_add graph; invalid arguments; and the host
layer's test program (tests/cpp/host_latency_info_test.cpp) on the engine."""
import ctypes as C

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests.helpers import synth_prompts, synth_snapshot
from tests.prefix_match_scenarios import Query, endpoint_lists, expected
from tests.running_oracle import Queues

pytestmark = pytest.mark.gpu
ERR_INVALID = -1
SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3)]
LAT = dict(ttft_intercept=50.0, ttft_kv=30.0, ttft_input=0.05, ttft_waiting=8.0, ttft_running=4.0, ttft_prefix=-40.0,
           tpot_intercept=10.0, tpot_kv=5.0, tpot_input=0.001, tpot_waiting=1.0, tpot_running=1.0, tpot_generated=0.01)
FIELDS = ("ttft", "tpot", "ttft_headroom", "tpot_headroom", "prefix_cache_score", "dispatched", "present", "ttft_valid",
          "tpot_valid", "reserved")


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _olp(pkg, p):
    """the oracle's LatencyParams from the engine's"""
    return o.LatencyParams(**{f: getattr(p, f) for f in o.LATENCY_FIELDS if hasattr(p, f)})


class View:
    """What the engine's current snapshot gives the producer: kv, queue, running, podMinTPOTSLO, dispatched, prefill role."""

    def __init__(self, snap, M, min_tpot=None, dispatched=None, prefill=None):
        self.M = M
        self.kv, self.queue = snap["kv_usage"], snap["queue"]
        self.running = snap.get("running")
        self.min_tpot = np.zeros(M) if min_tpot is None else np.asarray(min_tpot, np.float64)
        self.disp = np.zeros(M, np.int32) if dispatched is None else np.asarray(dispatched, np.int32)
        self.prefill = np.zeros(M, np.uint8) if prefill is None else np.asarray(prefill, np.uint8)


def oracle_info(lp, view, match, n_hashes, endpoints, input_tokens=None, ttft_slo=None, tpot_slo=None):
    """[R, k] records: orc_latency_predict + orc_latency_validate per entry, `match` the oracle's matchLongestPrefix at the entries."""
    R, k = endpoints.shape
    out = np.zeros((R, k), _pkg.load().LATENCY_INFO_DTYPE)
    if not lp.has_predictions:
        return out
    for r in range(R):
        n = int(n_hashes[r])
        it = int(input_tokens[r]) if input_tokens is not None else 0
        ts = float(ttft_slo[r]) if ttft_slo is not None else 0.0
        ps = float(tpot_slo[r]) if tpot_slo is not None else 0.0
        for j in range(k):
            m = int(endpoints[r, j])
            if m < 0 or m >= view.M:
                continue
            prefix = int(match[r, j]) / n if n else 0.0
            run = int(view.running[m]) if view.running is not None else 0
            t, p = o.latency_predict(lp, float(view.kv[m]), it, int(view.queue[m]), run, prefix)
            neutral = not lp.streaming_mode or bool(view.prefill[m])
            v = o.latency_validate(lp, t, p, ts, ps, float(view.min_tpot[m]), neutral)
            out[r, j] = (t, p, v["ttft_headroom"], v["headroom"], prefix, view.disp[m], 1, v["ttft_ok"], v["tpot_ok"], 0)
    return out


def assert_same(got, want):
    for f in FIELDS:
        g, w = got[f], want[f]
        if g.dtype.kind == "f":  # bit-exact, the sign of zero included
            assert np.array_equal(g.view(np.uint64), w.view(np.uint64)), (f, np.argwhere(g.view(np.uint64) != w.view(np.uint64))[:5])
        else:
            assert np.array_equal(g, w), (f, np.argwhere(g != w)[:5])


def device_info(eng, hashes, nh, eps, stream=None, match=False, **kw):
    import torch
    R, k = eps.shape
    out = torch.full((R, k, 48), 0x5A, dtype=torch.uint8, device="cuda:0")
    m_out = torch.full((R, k), 0x7777, dtype=torch.int16, device="cuda:0") if match else None
    dkw = {key: (None if v is None else _dev(v)) for key, v in kw.items()}
    eng.predict_latency(_dev(hashes.view(np.int64)), _dev(nh.view(np.int16)), _dev(eps), device=True, stream=stream, out=out,
                        match_out=m_out, **dkw)
    torch.cuda.synchronize()
    info = out.cpu().numpy().reshape(-1).view(eng_dtype()).reshape(R, k)
    return (info, m_out.cpu().numpy().view(np.uint16)) if match else info


def eng_dtype():
    return _pkg.load().LATENCY_INFO_DTYPE


def check_both(eng, lp, view, idx, limit, hashes, nh, eps, **kw):
    """host and device location against the oracle; match_out against prefix_match and the oracle's match"""
    q = Query(hashes, nh, np.ascontiguousarray(eps, np.int32))
    match = expected(idx, q, limit)
    want = oracle_info(lp, view, match, nh, q.endpoints, **kw)
    info, m = eng.predict_latency(hashes, nh, q.endpoints, match_out=True, **kw)
    assert_same(info, want)
    assert np.array_equal(m, match)
    assert np.array_equal(eng.predict_latency(hashes, nh, q.endpoints, **kw), info)
    dinfo, dm = device_info(eng, hashes, nh, q.endpoints, match=True, **kw)
    assert_same(dinfo, want)
    assert np.array_equal(dm, match)
    assert_same(device_info(eng, hashes, nh, q.endpoints, **kw), want)
    return info


def _world(pkg, M, R, seed=3, scorers=SCORERS, lat=None, snap_extra=None, lat_profile=True, max_blocks=32, **cfg):
    """An engine with a latency profile (the default one, or an added one), a snapshot and an index warmed by three committed
    batches; returns (eng, oracle params, view, oracle index, the next batch's inputs)."""
    eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, max_blocks=max_blocks, prefix_capacity=1 << 16, **cfg))
    p = pkg.latency_params(**dict(LAT, **(lat or {})))
    eng.set_latency_params(p)
    if lat_profile and not any(s[0] == "latency" for s in scorers):
        eng.add_profile([(pkg.SCORER["latency"], 1.0)])
    snap = synth_snapshot(M, seed=seed)
    extra = snap_extra or {}
    eng.set_snapshot(**snap, **extra)
    view = View(snap, M, extra.get("min_tpot_slo"), extra.get("dispatched"), extra.get("prefill_role"))
    idx = o.Index(31250)
    for k in range(3):
        prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=50 + k, prefix_seed=9)
        kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64), max_blocks=max_blocks)
        res = eng.schedule(R, want_hashes=True, **kw)
        eng.commit_picks(res["pick"], res["hashes_out"], res["total_blocks"])
        idx.commit(res["pick"], res["hashes_out"], res["total_blocks"])
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=99, prefix_seed=9)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64), max_blocks=max_blocks)
    return eng, _olp(pkg, p), view, idx, kw


def _req(R, seed=1):
    rng = np.random.Generator(np.random.PCG64(seed))
    return dict(input_tokens=rng.integers(0, 3000, R).astype(np.int32), ttft_slo=rng.uniform(0, 400, R),
                tpot_slo=rng.uniform(0, 60, R))


def _snap_lat(M, seed=4):
    rng = np.random.Generator(np.random.PCG64(seed))
    return dict(min_tpot_slo=np.where(rng.random(M) < 0.5, rng.uniform(0, 80, M), 0.0),
                dispatched=rng.integers(0, 3, M).astype(np.int32), prefill_role=(rng.random(M) < 0.25).astype(np.uint8))


@pytest.mark.parametrize("route", ["sparse", "full-matrix", "masked", "latency-filters", "topk4", "wide16", "wide-max", "profiles"])
def test_routes(pkg, route):
    M, R = 64, 2048
    lat = dict(streaming_mode=1)
    extra = _snap_lat(M)
    if route == "full-matrix":
        w = _world(pkg, M, R, pick_mode=pkg.PICK_WEIGHTED_RANDOM, lat=lat, snap_extra=extra)
    elif route == "latency-filters":
        w = _world(pkg, M, R, scorers=[("latency", 1.0)], lat=lat, snap_extra=extra, pick_mode=pkg.PICK_WEIGHTED_RANDOM,
                   filters=[(pkg.FILTER_PREFIX_AFFINITY, (0.8, 0.1, 5000.0)), (pkg.FILTER_SLO_HEADROOM_TIER, (0.1,))])
    else:
        w = _world(pkg, M, R, lat=lat, snap_extra=extra)
    eng, lp, view, idx, kw = w
    req = _req(R)
    rng = np.random.Generator(np.random.PCG64(11))
    if route in ("sparse", "full-matrix", "latency-filters"):
        res = eng.schedule(R, want_hashes=True, **req, **kw)
        lists = [res["pick"][:, None]]
    elif route == "masked":
        mask = rng.integers(0, 2 ** 32, size=(R, (M + 31) // 32), dtype=np.uint64).astype(np.uint32)
        res = eng.schedule(R, want_hashes=True, cand_mask=mask, **req, **kw)
        lists = [res["pick"][:, None]]
    elif route in ("topk4", "wide16", "wide-max"):
        lk = {"topk4": {"topk": 4}, "wide16": {"topk_wide": 16}, "wide-max": {"topk_wide": M}}[route]
        res = eng.schedule(R, want_hashes=True, **lk, **req, **kw)
        lists = [res["topk_pick"]]
    else:  # profile 1 is the latency profile _world added
        res, runs = eng.schedule_profiles(R, [{"profile": 0}, {"profile": 1, "topk": 3}], want_hashes=True, **req, **kw)
        lists = [runs[0]["pick"][:, None], runs[1]["topk_pick"], np.stack([runs[0]["pick"], runs[1]["pick"]], axis=1)]
    for ls in lists:
        check_both(eng, lp, view, idx, M, res["hashes_out"], res["total_blocks"], ls, **req)


@pytest.mark.parametrize("streaming", [0, 1])
def test_pred_out_cross_check(pkg, streaming):
    """ttft / tpot equal a diagnostic batch's pred_out at every candidate entry (the batch's own hashes and match)."""
    M, R = 64, 512
    eng, lp, view, idx, kw = _world(pkg, M, R, scorers=[("latency", 1.0)], lat=dict(streaming_mode=streaming),
                                    snap_extra=_snap_lat(M))
    req = _req(R, seed=3)
    res = eng.schedule(R, want_hashes=True, want_pred=True, **req, **kw)
    eps = np.tile(np.arange(M, dtype=np.int32), (R, 1))
    info = check_both(eng, lp, view, idx, M, res["hashes_out"], res["total_blocks"], eps, **req)
    assert np.array_equal(info["ttft"].view(np.uint64), res["pred_out"][:, :, 0].view(np.uint64))
    assert np.array_equal(info["tpot"].view(np.uint64), res["pred_out"][:, :, 1].view(np.uint64))


def test_validity_edges(pkg):
    """TTFT == SLO and TPOT == buffered (strict: not valid, headroom +0.0), SLO 0, podMinTPOTSLO 0 / below / above the request's
    buffered TPOT, streaming with prefill-role endpoints and not streaming."""
    M, R = 8, 64
    rng = np.random.Generator(np.random.PCG64(7))
    hs = rng.integers(1, 2 ** 63, size=(R, 16), dtype=np.uint64)
    nh = rng.integers(0, 17, R).astype(np.uint16)
    eps = rng.integers(0, M, size=(R, 4)).astype(np.int32)
    for streaming in (1, 0):
        for factor in (1.0, 0.9):
            eng = pkg.Engine(pkg.default_config([("latency", 1.0)], max_endpoints=M, max_blocks=16))
            p = pkg.latency_params(**dict(LAT, streaming_mode=streaming, slo_buffer_factor=factor))
            eng.set_latency_params(p)
            lp = _olp(pkg, p)
            snap = synth_snapshot(M, seed=5)
            base = eng.predict_latency  # first: the predictions with every SLO 0
            for pod in ("zero", "below", "above"):
                prefill = (np.arange(M) % 3 == 0).astype(np.uint8)
                eng.set_snapshot(**snap, prefill_role=prefill, dispatched=np.arange(M, dtype=np.int32))
                it = rng.integers(0, 500, R).astype(np.int32)
                z = base(hs, nh, eps, input_tokens=it)
                ttft_slo = z["ttft"][:, 0].copy()                        # TTFT == SLO at entry 0
                ttft_slo[::4] = 0.0                                      # SLO 0
                tpot_slo = z["tpot"][:, 1] / factor                      # (approximately) TPOT == buffered at entry 1
                tpot_slo[1::4] = 0.0
                if pod == "zero":
                    mn = np.zeros(M)
                else:  # podMinTPOTSLO*factor below / above every request's bufferedTPOT
                    mn = np.full(M, 0.5 if pod == "below" else 1e6)
                eng.set_snapshot(**snap, prefill_role=prefill, dispatched=np.arange(M, dtype=np.int32), min_tpot_slo=mn)
                view = View(snap, M, mn, np.arange(M, dtype=np.int32), prefill)
                idx = o.Index(31250)
                req = dict(input_tokens=it, ttft_slo=ttft_slo, tpot_slo=tpot_slo)
                info = check_both(eng, lp, view, idx, M, hs, nh, eps, **req)
                eq = info["ttft"][:, 0] == ttft_slo
                assert eq[1::4].all() and not info["ttft_valid"][eq, 0].any()
                assert not np.signbit(info["ttft_headroom"][eq, 0]).any() and (info["ttft_headroom"][eq, 0] == 0).all()
                if streaming and factor == 1.0 and pod != "below":
                    live = prefill[eps[:, 1]] == 0
                    eqp = (info["tpot"][:, 1] == tpot_slo) & live
                    assert eqp.sum() > R // 4 and not info["tpot_valid"][eqp, 1].any()
                neutral = (prefill[eps] == 1) | (not streaming)
                assert info["tpot_valid"][neutral].all() and (info["tpot_headroom"][neutral] == 0).all()


def test_has_predictions_off(pkg):
    M, R = 32, 256
    eng, lp, view, idx, kw = _world(pkg, M, R, lat=dict(has_predictions=0))
    res = eng.schedule(R, want_hashes=True, **kw)
    eps = endpoint_lists(np.random.Generator(np.random.PCG64(2)), R, 4, M, M)
    info = check_both(eng, lp, view, idx, M, res["hashes_out"], res["total_blocks"], eps, **_req(R))
    assert not info["present"].any() and not info["ttft"].any()


def test_totals_and_partial_matches(pkg):
    """total 0, partial matches (a shared prefix with fresh tails) and fresh prompts."""
    M, R = 16, 64
    eng = pkg.Engine(pkg.default_config([("latency", 1.0), ("prefix", 1.0)], max_endpoints=M, max_blocks=64, prefix_capacity=1 << 12))
    p = pkg.latency_params(**LAT)
    eng.set_latency_params(p)
    snap = synth_snapshot(M, seed=2)
    eng.set_snapshot(**snap)
    idx = o.Index(31250)
    rng = np.random.Generator(np.random.PCG64(3))
    base = rng.integers(1, 2 ** 63, size=(R, 64), dtype=np.uint64)
    nh = np.full(R, 64, np.uint16)
    pick = (np.arange(R) % M).astype(np.int32)
    eng.commit_picks(pick, base, nh)
    idx.commit(pick, base, nh)
    hs = base.copy()
    cut = rng.integers(0, 64, R)
    for r in range(R):
        hs[r, cut[r]:] = rng.integers(1, 2 ** 63, size=64 - cut[r], dtype=np.uint64)
    n2 = rng.integers(0, 65, R).astype(np.uint16)
    n2[::5] = 0
    eps = endpoint_lists(rng, R, 8, M, M)
    eps[:, 0] = pick
    check_both(eng, _olp(pkg, p), View(snap, M), idx, M, hs, n2, eps, **_req(R))


def test_dispatched_from_queues(pkg):
    """Without the snapshot arrays, dispatched and podMinTPOTSLO come from the running-request queues: before and after running_add
    (host and device location), and a call issued before a running_add on another stream does not see it."""
    import torch
    M, R = 32, 512
    eng, lp, _, idx, kw = _world(pkg, M, R, lat=dict(streaming_mode=1))
    snap = synth_snapshot(M, seed=3)
    q = Queues(M)
    res = eng.schedule(R, want_hashes=True, **kw)
    eps = endpoint_lists(np.random.Generator(np.random.PCG64(5)), R, 4, M, M)
    req = _req(R, seed=8)
    rng = np.random.Generator(np.random.PCG64(6))
    key = 1
    for rnd in range(3):
        mn, cnt = q.get(M)
        check_both(eng, lp, View(snap, M, mn, cnt), idx, M, res["hashes_out"], res["total_blocks"], eps, **req)
        n = 40
        ep = rng.integers(0, M, n).astype(np.int32)
        tp = rng.uniform(1, 60, n)
        keys = np.arange(key, key + n, dtype=np.uint64)
        key += n
        if rnd % 2:
            eng.running_add(_dev(ep), _dev(keys), _dev(tp), device=True)
        else:
            eng.running_add(ep, keys, tp)
        q.add(ep, keys, tp)
    # ordering: predict_latency on s1, then running_add on s2 -> the result is the view before the add; then the reverse
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    mn0, cnt0 = q.get(M)
    want0 = oracle_info(lp, View(snap, M, mn0, cnt0), expected(idx, Query(res["hashes_out"], res["total_blocks"], eps), M),
                        res["total_blocks"], eps, **req)
    ep = rng.integers(0, M, 64).astype(np.int32)
    keys = np.arange(key, key + 64, dtype=np.uint64)
    tp = rng.uniform(0.5, 3, 64)
    q.add(ep, keys, tp)
    mn1, cnt1 = q.get(M)
    want1 = oracle_info(lp, View(snap, M, mn1, cnt1), expected(idx, Query(res["hashes_out"], res["total_blocks"], eps), M),
                        res["total_blocks"], eps, **req)
    d = dict(hashes=_dev(res["hashes_out"].view(np.int64)), nh=_dev(res["total_blocks"].view(np.int16)), ep=_dev(eps))
    dreq = {k_: _dev(v) for k_, v in req.items()}
    outs = [torch.zeros((R, 4, 48), dtype=torch.uint8, device="cuda:0") for _ in range(2)]
    d_ep, d_keys, d_tp = _dev(ep), _dev(keys), _dev(tp)
    torch.cuda.synchronize()
    eng.predict_latency(d["hashes"], d["nh"], d["ep"], device=True, stream=s1.cuda_stream, out=outs[0], **dreq)
    eng.running_add(d_ep, d_keys, d_tp, device=True, stream=s2.cuda_stream)
    eng.predict_latency(d["hashes"], d["nh"], d["ep"], device=True, stream=s1.cuda_stream, out=outs[1], **dreq)
    torch.cuda.synchronize()
    got = [x.cpu().numpy().reshape(-1).view(eng_dtype()).reshape(R, 4) for x in outs]
    assert_same(got[0], want0)
    assert_same(got[1], want1)


@pytest.mark.parametrize("M", [5, 1024, 4097])
def test_geometries(pkg, M):
    R = 256
    eng, lp, view, idx, kw = _world(pkg, M, R, lat=dict(streaming_mode=1), snap_extra=_snap_lat(M))
    res = eng.schedule(R, want_hashes=True, **kw)
    rng = np.random.Generator(np.random.PCG64(M))
    for k in sorted({1, min(32, M), min(33, M), M}):
        R2 = R if k <= 33 else 16
        check_both(eng, lp, view, idx, M, res["hashes_out"][:R2], res["total_blocks"][:R2], endpoint_lists(rng, R2, k, M, M),
                   **{k_: v[:R2] for k_, v in _req(R).items()})


def test_hash_counts(pkg):
    """n_hashes 0, 256 and 1000 (one long shared prefix committed on a few endpoints)."""
    M, R = 16, 48
    eng = pkg.Engine(pkg.default_config([("latency", 1.0), ("prefix", 1.0)], max_endpoints=M, max_blocks=1000,
                                        prefix_capacity=1 << 14, lru_capacity_default=4000))
    p = pkg.latency_params(**LAT)
    eng.set_latency_params(p)
    snap = synth_snapshot(M, seed=6)
    eng.set_snapshot(**snap)
    idx = o.Index(4000)
    rng = np.random.Generator(np.random.PCG64(9))
    pre = rng.integers(1, 2 ** 63, size=1000, dtype=np.uint64)
    hs = np.tile(pre, (R, 1))
    nh = np.array([0, 256, 1000] * (R // 3), np.uint16)
    pick = np.array([1, 2, 3] * (R // 3), np.int32)
    eng.commit_picks(pick[:3], hs[:3], np.array([1000, 700, 256], np.uint16))
    idx.commit(pick[:3], hs[:3], np.array([1000, 700, 256], np.uint16))
    eps = endpoint_lists(rng, R, 6, 5, M)
    check_both(eng, _olp(pkg, p), View(snap, M), idx, M, hs, nh, eps, **_req(R, seed=4))


def test_reserved_streams_concurrent(pkg):
    import torch
    M, R = 64, 1024
    eng, lp, view, idx, kw = _world(pkg, M, R, lat=dict(streaming_mode=1), snap_extra=_snap_lat(M))
    res = eng.schedule(R, want_hashes=True, **kw)
    streams = [torch.cuda.Stream() for _ in range(3)]
    for s in streams:
        eng.reserve_stream(s.cuda_stream, R, 32)
    eps = endpoint_lists(np.random.Generator(np.random.PCG64(4)), R, 8, M, M)
    req = _req(R)
    want = oracle_info(lp, view, expected(idx, Query(res["hashes_out"], res["total_blocks"], eps), M), res["total_blocks"], eps, **req)
    d_in = {key: _dev(v) for key, v in kw.items() if key != "max_blocks"}
    dev = torch.device("cuda:0")
    outs = [dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                 tie_count=torch.empty(R, dtype=torch.int32, device=dev)) for _ in range(2)]
    info = torch.zeros((R, 8, 48), dtype=torch.uint8, device=dev)
    d_h, d_nh, d_ep = _dev(res["hashes_out"].view(np.int64)), _dev(res["total_blocks"].view(np.int16)), _dev(eps)
    dreq = {k_: _dev(v) for k_, v in req.items()}
    torch.cuda.synchronize()
    for _ in range(3):
        for i in range(2):
            eng.schedule(R, device=True, stream=streams[i].cuda_stream, out=outs[i], max_blocks=32, **d_in)
        eng.predict_latency(d_h, d_nh, d_ep, device=True, stream=streams[2].cuda_stream, out=info, **dreq)
    torch.cuda.synchronize()
    assert_same(info.cpu().numpy().reshape(-1).view(eng_dtype()).reshape(R, 8), want)
    for i in range(2):
        assert np.array_equal(outs[i]["pick"].cpu().numpy(), res["pick"])
    for s in streams:
        eng.release_stream(s.cuda_stream)


def test_graph_replays(pkg):
    """24 replays of one schedule -> predict_latency -> commit -> running_add graph (the queues feed dispatched and
    podMinTPOTSLO): every round bit-exact to the oracle fed by the queue oracle, read before the round's commit and add."""
    import torch
    M, R, MB, LRU = 64, 256, 16, 48
    eng = pkg.Engine(pkg.default_config([("latency", 1.0), ("prefix", 1.0)], max_endpoints=M, max_blocks=MB, prefix_capacity=1 << 10,
                                        lru_capacity_default=LRU))
    p = pkg.latency_params(**dict(LAT, streaming_mode=1))
    eng.set_latency_params(p)
    lp = _olp(pkg, p)
    snap = synth_snapshot(M, seed=9)
    eng.set_snapshot(**snap)
    eng.prefix_reserve(M * LRU + 1024, R * MB, 0)
    eng.running_reserve(24 * R + 64)
    idx = o.Index(LRU)
    q = Queues(M)
    dev = torch.device("cuda:0")
    req = _req(R, seed=12)

    def inputs(k):
        prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=16, shared=256, seed=300 + k, prefix_seed=7)
        return dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64))
    d_in = {key: _dev(v) for key, v in inputs(0).items()}
    d_req = {key: _dev(v) for key, v in req.items()}
    keys = torch.zeros(R, dtype=torch.int64, device=dev)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
    info = torch.zeros((R, 1, 48), dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream()

    def body():
        eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d_in, **d_req)
        eng.predict_latency(out["hashes_out"], out["total_blocks"], out["pick"].view(R, 1), device=True, stream=s.cuda_stream,
                            out=info, **d_req)
        eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], stream=s.cuda_stream)
        eng.running_add(out["pick"], keys, d_req["tpot_slo"], device=True, stream=s.cuda_stream)
    eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d_in, **d_req)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        body()
    torch.cuda.synchronize()
    for k in range(24):
        d_in["prompt_bytes"].copy_(torch.from_numpy(inputs(k)["prompt_bytes"]))
        kk = np.arange(1 + k * R, 1 + (k + 1) * R, dtype=np.uint64)
        keys.copy_(torch.from_numpy(kk.view(np.int64)))
        torch.cuda.synchronize()
        mn, cnt = q.get(M)
        g.replay()
        torch.cuda.synchronize()
        pick = out["pick"].cpu().numpy()
        hs = out["hashes_out"].cpu().numpy().view(np.uint64)
        nh = out["total_blocks"].cpu().numpy()
        eps = pick[:, None].copy()
        want = oracle_info(lp, View(snap, M, mn, cnt), expected(idx, Query(hs, nh, eps), M), nh, eps, **req)
        assert_same(info.cpu().numpy().reshape(-1).view(eng_dtype()).reshape(R, 1), want)
        idx.commit(pick, hs, nh)
        q.add(pick, kk, req["tpot_slo"])
    mn, cnt = q.get(M)
    assert np.array_equal(eng.running_get(M)[1], cnt)


def test_invalid_arguments(pkg):
    M = 8
    eng = pkg.Engine(pkg.default_config([("latency", 1.0)], max_endpoints=M))
    lib, h = eng._lib, eng._h
    hs = np.zeros((2, 4), np.uint64)
    nh = np.array([1, 4], np.uint16)
    ep = np.zeros((2, 1), np.int32)
    out = np.zeros((2, 9), eng_dtype())
    p = lambda a: a.ctypes.data  # noqa: E731

    def call(R=2, k=1, loc=0, hs_=hs, nh_=nh, stride=4, ep_=ep, out_=out):
        return lib.eppscore_predict_latency(h, R, k, loc, None if hs_ is None else p(hs_), None if nh_ is None else p(nh_), stride,
                                            None, None, None, None if ep_ is None else p(ep_), None if out_ is None else p(out_),
                                            None, None)
    assert call() == ERR_INVALID  # no snapshot yet
    eng.set_snapshot(**synth_snapshot(M, seed=1))
    assert call() == 0
    nh[1] = 5
    assert call() == ERR_INVALID  # n_hashes > hash_stride
    nh[1] = 4
    for k in (0, M + 1, -3):
        assert call(k=k) == ERR_INVALID
    assert call(hs_=None) == ERR_INVALID
    assert call(nh_=None) == ERR_INVALID
    assert call(ep_=None, loc=1) == ERR_INVALID
    assert call(out_=None) == ERR_INVALID
    assert call(loc=2) == ERR_INVALID
    assert call(R=-1) == ERR_INVALID
    for stride in (0, -4):
        assert call(stride=stride) == ERR_INVALID
    launches = eng.stats().kernel_launches
    eng.predict_latency(hs, nh, ep)
    assert eng.stats().kernel_launches == launches + 1
    plain = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M))  # no latency scorer: no latency tile
    plain.set_snapshot(**synth_snapshot(M, seed=1))
    assert plain._lib.eppscore_predict_latency(plain._h, 2, 1, 0, p(hs), p(nh), 4, None, None, None, p(ep), p(out), None,
                                               None) == ERR_INVALID
    assert C.sizeof(pkg.LatencyInfo) == 48


def test_host_program_on_the_engine(pkg):
    """tests/cpp/host_latency_info_test.cpp (the host layer's SchedulingResult::TargetLatency and dispatch record) linked against the engine."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = os.path.join(root, "tests", "cpp", "_build")
    os.makedirs(build, exist_ok=True)
    lib_dir = os.path.dirname(pkg.lib()._name)
    oracle_dir = os.path.dirname(o.build())
    exe = os.path.join(build, "host_latency_info_test_engine")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread",
                           os.path.join(root, "tests", "cpp", "host_latency_info_test.cpp"), "-L" + lib_dir, "-leppscore",
                           "-L" + oracle_dir, "-loracle", "-Wl,-rpath," + lib_dir + ":" + oracle_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    assert not any(line.startswith(("FAIL", "refused")) for line in r.stdout.splitlines())
