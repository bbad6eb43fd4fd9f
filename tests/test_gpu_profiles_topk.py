"""maxNumOfEndpoints per scheduler profile on the GPU (eppscore_schedule_batch_profiles_topk): every run's list equals, bit for
bit, the CPU oracle's top-k (tests/cpp/topk_oracle.c) over oracle_py.schedule_batch with that profile's scorers and picker, the
derived tie seed tie_seed ^ p * 0x9E3779B97F4A7C15 and the candidates subset ∧ cand_mask; pick / pick_score / tie_count equal
eppscore_schedule_batch_profiles without lists; and every way of running a batch (host, chunked, device, sliced, graph) gives the
same lists."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import topk_oracle as T
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

pytestmark = pytest.mark.gpu

GOLDEN = 0x9E3779B97F4A7C15
HEADLINE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
PREFILL = [("kv", 1), ("prefix", 2)]
QUEUE_RUNNING = [("queue", 1), ("running", 1.5), ("prefix", 2)]
KV_LORA = [("kv", 1), ("lora", 2)]
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01)
ERR_INVALID, ERR_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def seed_of(seed, p):
    return (seed ^ (p * GOLDEN)) & (2 ** 64 - 1)


def bits(M, members):
    """uint32 natural-order bitmask of the endpoints in `members`"""
    out = np.zeros(max((M + 31) // 32, 1), np.uint32)
    for m in members:
        out[m >> 5] |= np.uint32(1 << (m & 31))
    return out


def random_masks(R, M, rng, density=0.6):
    mw = (M + 31) // 32
    b = np.zeros((R, mw * 32), bool)
    b[:, :M] = rng.random((R, M)) < density
    return (b.reshape(R, mw, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


def oracle_run(pkg, snap, idx, R, scorers, tie_mode, seed, pick_mode, subset, run_mask, M, kw, k, latency=None, filters=(),
               request_base=0):
    """oracle_py.schedule_batch of one profile on subset ∧ run_mask, plus its first k entries (k 0: no list)"""
    prof = o.make_profile([(pkg.SCORER[n], w) for n, w in scorers], tie_mode=tie_mode, tie_seed=seed, pick_mode=pick_mode,
                          latency=latency, filters=filters)
    mask = None
    if subset is not None or run_mask is not None:
        mw = (M + 31) // 32
        mask = np.full((R, mw), 0xFFFFFFFF, np.uint32)
        if subset is not None:
            mask &= subset[None, :mw]
        if run_mask is not None:
            mask &= run_mask
    out = o.schedule_batch(snap, prof, idx, R, cand_mask=mask, want_scores=True, n_threads=8, request_base=request_base, **kw)
    if k:
        out["topk_pick"], out["topk_score"] = T.lists(out["weighted_out"], prof, k, request_base)
    return out


def assert_run(got, want, what):
    assert np.array_equal(got["pick"], want["pick"]), what
    assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what
    assert np.array_equal(got["tie_count"], want["tie_count"]), what


def assert_lists(got, want, what):
    assert np.array_equal(got["topk_pick"], want["topk_pick"]), what
    assert np.array_equal(got["topk_score"].view(np.uint64), want["topk_score"].view(np.uint64)), what


def world(pkg, M, seed, R=320, grouped=False, **cfg):
    """snapshot + a warm prefix index (committed picks replayed on every engine `make` builds) + the test batch.  grouped: each
    shared prefix is committed on one endpoint, so the probing hash kernel resolves the test batch's requests (new tails)"""
    sd = synth_snapshot(M, seed=seed)
    snap, idx = o.SnapshotData(**sd), o.Index()
    ms = o.model_seed("profiles-topk")
    pw, offw, gw = synth_prompts(R, prompt_len=1024, groups=12, shared=768, seed=seed, prefix_seed=100)
    seeds = np.full(R, ms, np.uint64)
    warm_prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], pick_mode=o.PICK_RANDOM, tie_seed=3)
    w = o.schedule_batch(snap, warm_prof, idx if not grouped else None, R, prompt_bytes=pw, prompt_off=offw, model_seed=seeds,
                         want_hashes=True, n_threads=8)
    if grouped:
        w["pick"] = ((np.asarray(gw) * 7 + 1) % M).astype(np.int32)
    idx.commit(w["pick"], w["hashes_out"], w["total_blocks"])
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=12, shared=768, seed=seed + 1, prefix_seed=100)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=seeds, adapter_id=zipf_adapters(R, seed=seed))

    def make(scorers=HEADLINE, **over):
        c = dict(cfg)
        c.update(over)
        c.setdefault("max_endpoints", M)
        eng = pkg.Engine(pkg.default_config(scorers, prefix_capacity=1 << 16, **c))
        eng.commit_picks(w["pick"], w["hashes_out"], w["total_blocks"])
        eng.set_snapshot(**sd)
        return eng

    return make, snap, idx, sd, kw


def ks_for(M, max_endpoints):
    return [k for k in (0, 1, 2, 8, 9, 16, M - 1, M, max_endpoints) if 0 <= k <= max_endpoints]


def check_call(pkg, eng, snap, idx, R, M, kw, profiles, runs, tie_mode, seed, what, oracle_cache=None, kmax=1, **call):
    """runs: [(profile, run_mask, k)]; profiles[p] = (scorers, pick_mode, subset).  Checks every run against the oracle and
    against eppscore_schedule_batch_profiles without lists; returns the per-run outputs."""
    spec = [dict(profile=p, cand_mask=m, topk=k) for p, m, k in runs]
    _, got = eng.schedule_profiles(R, spec, **kw, **call)
    _, plain = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m) for p, m, _ in runs], **kw, **call)
    for (p, m, k), g, pl in zip(runs, got, plain):
        w = (what, p, k, m is not None)
        sc, pm, sub = profiles[p]
        key = (p, id(m))
        want = oracle_cache.get(key) if oracle_cache is not None else None
        if want is None or want.get("k", 0) < k:
            want = oracle_run(pkg, snap, idx, R, sc, tie_mode, seed_of(seed, p), pm, sub, m, M, kw, max(k, kmax))
            want["k"] = max(k, kmax)
            if oracle_cache is not None:
                oracle_cache[key] = want
        assert_run(g, pl, w)
        assert_run(g, want, w)
        if k:
            assert g["topk_pick"].shape == (R, k)
            assert_lists(g, dict(topk_pick=want["topk_pick"][:, :k], topk_score=want["topk_score"][:, :k]), w)
            assert np.array_equal(g["topk_pick"][:, 0], g["pick"]), w
        else:
            assert "topk_pick" not in g
    return got


@pytest.mark.parametrize("M", [5, 600, 1024, 4096])
@pytest.mark.parametrize("tie_mode", [0, 1])
def test_lists_match_oracle(pkg, M, tie_mode):
    """one to four runs with mixed k per run, the three pick modes over the profiles, subsets with and without run masks,
    and a subset with fewer members than k (padded lists)"""
    R = 256 if M < 4096 else 160
    max_endpoints = M + 37 if M > 5 else 8
    seed = 0x70CC0000 + M * 5 + tie_mode
    make, snap, idx, sd, kw = world(pkg, M, M + tie_mode, R=R, tie_mode=tie_mode, tie_seed=seed, max_endpoints=max_endpoints)
    eng = make()
    rng = np.random.Generator(np.random.PCG64(M * 11 + tie_mode))
    few = sorted(rng.choice(M, size=min(3, M), replace=False).tolist())
    profiles = [  # (scorers, pick_mode, subset)
        (HEADLINE, 0, bits(M, range(0, M, 2))),
        (PREFILL, 1, bits(M, range(1, M, 2)) if M > 1 else None),
        (QUEUE_RUNNING, 2, bits(M, few)),  # fewer candidates than most k: padded
        (KV_LORA, 0, None),
    ]
    for p in range(1, 4):
        assert eng.add_profile(profiles[p][0], pick_mode=profiles[p][1]) == p
    for p, (_, _, sub) in enumerate(profiles):
        eng.set_profile_endpoints(p, sub)
    eng.set_snapshot(**sd)
    masks = random_masks(R, M, rng)
    ks = ks_for(M, max_endpoints)
    cache = {}
    calls = [
        [(1, None, ks[-1])],
        [(0, None, 4), (1, None, 0)],
        [(0, None, 0), (1, masks, min(9, max_endpoints)), (2, None, 16 if M > 5 else 2)],
        [(0, masks, 8), (1, None, 2), (2, masks, 1), (3, None, M)],
    ]
    for i, k in enumerate(ks):  # every k on some run, next to the others
        calls.append([(i % 4, masks if i % 2 else None, k), ((i + 1) % 4, None, ks[(i + 3) % len(ks)]),
                      ((i + 2) % 4, masks, ks[(i + 5) % len(ks)])])
    for c in calls:
        check_call(pkg, eng, snap, idx, R, M, kw, profiles, c, tie_mode, seed, (M, tie_mode, c), oracle_cache=cache,
                   kmax=max_endpoints)
    eng.close()


def test_lists_equal_single_profile_calls_on_a_fresh_engine(pkg):
    """run i's list equals eppscore_schedule_batch_topk (k <= 8) and _topk_wide on an engine whose profile 0 is that profile
    (scorers, picker, subset, derived seed)"""
    M, tie_mode, seed = 600, 1, 0xABCDEF12345
    make, snap, idx, sd, kw = world(pkg, M, 31, R=300, tie_mode=tie_mode, tie_seed=seed)
    eng = make()
    profiles = [(HEADLINE, 0, bits(M, range(0, M, 3))), (PREFILL, 1, bits(M, range(1, M, 3))), (QUEUE_RUNNING, 2, None)]
    for p in (1, 2):
        eng.add_profile(profiles[p][0], pick_mode=profiles[p][1])
    for p, (_, _, sub) in enumerate(profiles):
        eng.set_profile_endpoints(p, sub)
    eng.set_snapshot(**sd)
    rm = random_masks(300, M, np.random.Generator(np.random.PCG64(2)))
    runs = [(0, None, 5), (1, rm, 40), (2, None, 8)]
    _, got = eng.schedule_profiles(300, [dict(profile=p, cand_mask=m, topk=k) for p, m, k in runs], **kw)
    for (p, m, k), g in zip(runs, got):
        sc, pm, sub = profiles[p]
        one = make(sc, pick_mode=pm, tie_seed=seed_of(seed, p))
        one.set_profile_endpoints(0, sub)
        one.set_snapshot(**sd)
        calls = [dict(topk_wide=k)] + ([dict(topk=k)] if k <= 8 else [])
        for call in calls:
            alone = one.schedule(300, cand_mask=m, **call, **kw)
            assert_run(g, alone, (p, call))
            assert_lists(g, alone, (p, call))
        one.close()
    eng.close()


def test_latency_profile_behind_device_filters_and_dense_rows(pkg):
    M, R = 256, 288
    make, snap, idx, sd, kw = world(pkg, M, 9, R=R)
    eng = make()
    eng.set_latency_params(pkg.latency_params(**LAT_COEF))
    filters = [(1, (0.5, 0.0, 5000.0)), (2, (0.01, 0, 0))]
    lat = [("latency", 1), ("kv", 0.5)]
    pid = eng.add_profile(lat, filters=filters)
    sub = bits(M, range(M // 2, M))
    eng.set_profile_endpoints(pid, sub)
    eng.set_snapshot(**sd)
    slo = dict(ttft_slo=np.full(R, 900.0), tpot_slo=np.full(R, 40.0),
               input_tokens=np.random.Generator(np.random.PCG64(4)).integers(0, 6000, R).astype(np.int32))
    olp = o.make_latency_params(**LAT_COEF)
    for k0, k1 in ((0, 3), (4, 24), (12, M)):
        _, got = eng.schedule_profiles(R, [dict(profile=0, topk=k0), dict(profile=pid, topk=k1)], **kw, **slo)
        want = oracle_run(pkg, snap, idx, R, lat, 0, seed_of(0, pid), 0, sub, None, M, dict(kw, **slo), k1, latency=olp,
                          filters=filters)
        assert_run(got[1], want, ("latency", k1))
        assert_lists(got[1], want, ("latency", k1))
        w0 = oracle_run(pkg, snap, idx, R, HEADLINE, 0, 0, 0, None, None, M, dict(kw, **slo), k0)
        assert_run(got[0], w0, ("headline", k0))
        if k0:
            assert_lists(got[0], w0, ("headline", k0))
    # dense rows: max-score on both profiles
    eng2 = make()
    p2 = eng2.add_profile(PREFILL)
    eng2.set_profile_endpoints(p2, bits(M, range(0, M, 5)))
    eng2.set_snapshot(**sd)
    rng = np.random.Generator(np.random.PCG64(12))
    total = rng.integers(0, 40, R).astype(np.uint16)
    feat = np.zeros((R, M, 4), np.float32)
    feat[..., 0] = np.floor(rng.random((R, M)) * (total[:, None] + 1))
    feat[..., 1] = rng.integers(0, 4, (R, M))
    dkw = dict(dense_feat=feat, dense_total=total, adapter_id=kw["adapter_id"])
    for k0, k1 in ((2, 9), (8, 0), (0, 64)):
        _, got = eng2.schedule_profiles(R, [dict(profile=0, topk=k0), dict(profile=p2, topk=k1)], **dkw)
        for g, (sc, p, sub, k) in zip(got, ((HEADLINE, 0, None, k0), (PREFILL, p2, bits(M, range(0, M, 5)), k1))):
            want = oracle_run(pkg, snap, None, R, sc, 0, seed_of(0, p), 0, sub, None, M, dkw, k)
            assert_run(g, want, ("dense", p, k))
            if k:
                assert_lists(g, want, ("dense", p, k))
    eng.close()
    eng2.close()


def _dev(kw):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}


def _dev_runs(R, runs):
    import torch
    out = []
    for p, m, k in runs:
        d = dict(profile=p, topk=k, cand_mask=None if m is None else torch.from_numpy(m).cuda(),
                 pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"),
                 pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.zeros(R, dtype=torch.int32, device="cuda"))
        if k:
            d["topk_pick"] = torch.full((R, k), -7, dtype=torch.int32, device="cuda")
            d["topk_score"] = torch.zeros((R, k), dtype=torch.float64, device="cuda")
        out.append(d)
    return out


def _host(d):
    return {k: d[k].cpu().numpy() for k in ("pick", "pick_score", "tie_count", "topk_pick", "topk_score") if k in d}


def _same(got, want, what):
    assert_run(got, want, what)
    if "topk_pick" in want:
        assert_lists(got, want, what)


def test_execution_forms(pkg):
    """host, chunked host (key 3), device buffers, sliced device batches (keys 5 / 6) and a CUDA graph give the host call's
    lists; a graph replays after a larger wide call; a wide run captured before any wide call is ERR_CAPACITY"""
    import torch
    M, R = 1024, 4608
    make, snap, idx, sd, kw = world(pkg, M, 44, R=R)
    eng = make()
    pid = eng.add_profile(PREFILL, pick_mode=1)
    eng.set_profile_endpoints(0, bits(M, range(0, M, 2)))
    eng.set_profile_endpoints(pid, bits(M, range(1, M, 2)))
    eng.set_snapshot(**sd)
    kw = {k: v for k, v in kw.items() if k != "adapter_id"}  # sliceable device batches carry no per-request scorer inputs
    narrow = [(0, None, 4), (pid, None, 1)]
    wide = [(0, None, 4), (pid, None, 16)]
    for runs in (narrow, wide):
        _, ref = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m, topk=k) for p, m, k in runs], **kw)
        sample = slice(0, 256)
        for (p, m, k), g in zip(runs, ref):  # the reference itself, on a sample
            sc, pm, sub = (HEADLINE, 0, bits(M, range(0, M, 2))) if p == 0 else (PREFILL, 1, bits(M, range(1, M, 2)))
            skw = dict(prompt_bytes=kw["prompt_bytes"], prompt_off=kw["prompt_off"][:257], model_seed=kw["model_seed"][:256])
            want = oracle_run(pkg, snap, idx, 256, sc, 0, seed_of(0, p), pm, sub, None, M, skw, k)
            _same({x: g[x][sample] for x in g}, want, ("oracle", runs, p))
        eng.set_debug(3, 1000)
        _, chunked = eng.schedule_profiles(R, [dict(profile=p, topk=k) for p, _, k in runs], **kw)
        eng.set_debug(3, 8192)
        for c, g in zip(chunked, ref):
            _same(c, g, ("chunked", runs))
        dev = _dev(kw)
        for split, streams in ((1, 2), (2, 2), (2, 3)):
            eng.set_debug(5, split)
            eng.set_debug(6, streams)
            druns = _dev_runs(R, runs)
            eng.schedule_profiles(R, druns, device=True, **dev)
            torch.cuda.synchronize()
            for d, g in zip(druns, ref):
                _same(_host(d), g, ("device", runs, split, streams))
        eng.set_debug(5, 1)
        eng.set_debug(6, 2)
    eng.close()

    # graphs: a wide run captured before any wide call fails with ERR_CAPACITY; after one, a graph survives a larger call
    Rg = 600
    eng = make()
    pid = eng.add_profile(PREFILL, pick_mode=1)
    eng.set_profile_endpoints(pid, bits(M, range(1, M, 2)))
    eng.set_snapshot(**sd)
    gkw = dict(prompt_bytes=kw["prompt_bytes"], prompt_off=kw["prompt_off"][:Rg + 1], model_seed=kw["model_seed"][:Rg])
    dev = _dev(gkw)
    s = torch.cuda.Stream()
    runs = [(0, None, 3), (pid, None, 20)]
    druns = _dev_runs(Rg, runs)
    torch.cuda.synchronize()
    g0 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g0, stream=s):  # no wide call has allocated the score scratch yet
        with pytest.raises(pkg.EppscoreError) as ex:
            eng.schedule_profiles(Rg, druns, device=True, stream=s.cuda_stream, **dev)
    assert ex.value.code == ERR_CAPACITY and "outside" in str(ex.value)
    del g0
    torch.cuda.synchronize()
    _, ref = eng.schedule_profiles(Rg, [dict(profile=p, topk=k) for p, _, k in runs], **gkw)
    with torch.cuda.stream(s):
        eng.schedule_profiles(Rg, druns, device=True, stream=s.cuda_stream, **dev)  # the first wide call, outside a capture
    s.synchronize()
    for d in druns:
        d["pick"].fill_(-7)
        d["topk_pick"].fill_(-7)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.schedule_profiles(Rg, druns, device=True, stream=s.cuda_stream, **dev)
    big = eng.schedule_profiles(R, [dict(profile=0, topk=300), dict(profile=pid, topk=40)], **kw)  # larger, wider
    assert big[1][0]["topk_pick"].shape == (R, 300)
    g.replay()
    torch.cuda.synchronize()
    for d, w in zip(druns, ref):
        _same(_host(d), w, "graph")
    eng.close()


def test_routing_edges(pkg):
    """a sparse run next to a listed run: the hash kernel gives no records to a run that reads hashes without taking them, and
    probe_resolved counts only real resolutions; three wide runs whose slice division leaves a remainder"""
    M, R = 1024, 3000
    make, snap, idx, sd, kw = world(pkg, M, 61, R=R, grouped=True)
    eng = make()
    p_pre = eng.add_profile(PREFILL)       # reads the hashes
    p_kv = eng.add_profile([("kv", 1)])    # reads no hash
    p_rnd = eng.add_profile(QUEUE_RUNNING, pick_mode=2)
    eng.set_snapshot(**sd)
    before = eng.stats().probe_resolved
    _, alone = eng.schedule_profiles(R, [dict(profile=0)], **kw)
    resolved = eng.stats().probe_resolved - before
    assert resolved > 0  # the batch exercises the probing hash kernel
    # a listed run that reads the hashes: no probe at all
    before = eng.stats().probe_resolved
    _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=p_pre, topk=4)], **kw)
    assert eng.stats().probe_resolved - before == 0
    assert_run(got[0], alone[0], "sparse next to a hash-reading list")
    want = oracle_run(pkg, snap, idx, R, PREFILL, 0, seed_of(0, p_pre), 0, None, None, M, kw, 4)
    _same(got[1], want, "hash-reading list")
    # a listed run that reads no hash: the sparse run still takes the records
    for k in (4, 20):
        before = eng.stats().probe_resolved
        _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=p_kv, topk=k)], **kw)
        assert eng.stats().probe_resolved - before == resolved, k
        assert_run(got[0], alone[0], ("sparse next to a kv list", k))
        _same(got[1], oracle_run(pkg, snap, idx, R, [("kv", 1)], 0, seed_of(0, p_kv), 0, None, None, M, kw, k), ("kv", k))
    # three wide runs: 4096 scratch rows / 3 leaves a remainder, and R leaves a short last slice
    runs = [(0, 33), (p_pre, 9), (p_rnd, 17), (p_kv, 0)]
    _, got = eng.schedule_profiles(R, [dict(profile=p, topk=k) for p, k in runs], **kw)
    specs = {0: (HEADLINE, 0), p_pre: (PREFILL, 0), p_rnd: (QUEUE_RUNNING, 2), p_kv: ([("kv", 1)], 0)}
    for (p, k), g in zip(runs, got):
        sc, pm = specs[p]
        _same(g, oracle_run(pkg, snap, idx, R, sc, 0, seed_of(0, p), pm, None, None, M, kw, k), ("three wide", p, k))
    eng.close()


def test_invalid_arguments(pkg):
    M = 64
    eng = pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=M))
    eng.set_snapshot(np.zeros(M), np.zeros(M, np.int64))
    pid = eng.add_profile(PREFILL)
    R = 4
    for runs in ([dict(profile=0, topk=-1)], [dict(profile=0, topk=M + 1)], [dict(profile=0, topk=2), dict(profile=pid, topk=-3)],
                 [dict(profile=0, topk=1), dict(profile=0, topk=1)], [dict(profile=7, topk=1)]):
        with pytest.raises(pkg.EppscoreError) as ex:
            eng.schedule_profiles(R, runs)
        assert ex.value.code == ERR_INVALID, runs
    # NULL arrays with k > 0, a wrong struct_size, and topk NULL, through the raw call
    import ctypes as C
    L = eng._lib
    b = pkg.Batch()
    b.struct_size = C.sizeof(pkg.Batch)
    b.R = R
    picks = [np.zeros(R, np.int32), np.zeros(R, np.float64), np.zeros(R, np.int32)]
    arr = (pkg._capi.ProfileRun * 1)()
    arr[0].struct_size = C.sizeof(pkg._capi.ProfileRun)
    arr[0].pick, arr[0].pick_score, arr[0].tie_count = (x.ctypes.data for x in picks)
    t = (pkg.TopK * 1)()
    t[0].struct_size = C.sizeof(pkg.TopK)
    t[0].k = 2
    assert L.eppscore_schedule_batch_profiles_topk(eng._h, C.byref(b), 1, arr, t) == ERR_INVALID
    lm, ls = np.zeros(R * 2, np.int32), np.zeros(R * 2, np.float64)
    t[0].endpoints, t[0].scores = lm.ctypes.data, ls.ctypes.data
    t[0].struct_size = 3
    assert L.eppscore_schedule_batch_profiles_topk(eng._h, C.byref(b), 1, arr, t) == ERR_INVALID
    assert L.eppscore_schedule_batch_profiles_topk(eng._h, C.byref(b), 1, arr, None) == ERR_INVALID
    t[0].struct_size = C.sizeof(pkg.TopK)
    assert L.eppscore_schedule_batch_profiles_topk(eng._h, C.byref(b), 1, arr, t) == 0
    # k == 0 on every run is schedule_batch_profiles; NULL arrays are fine there
    t[0].k, t[0].endpoints, t[0].scores = 0, None, None
    assert L.eppscore_schedule_batch_profiles_topk(eng._h, C.byref(b), 1, arr, t) == 0
    eng.close()


def test_headline_shape_sampled(pkg):
    """64K requests x 1024 endpoints, decode (max-score, k = 4) and prefill (weighted-random, k = 16) profiles on the two halves;
    512 requests checked against the oracle"""
    M, R = 1024, 65536
    sd = synth_snapshot(M, seed=1)
    snap, idx = o.SnapshotData(**sd), o.Index()
    eng = pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=M))
    ms = o.model_seed("headline")
    pw, offw, _ = synth_prompts(2048, prompt_len=1024, groups=150, shared=768, seed=3, prefix_seed=7)
    warm = o.schedule_batch(snap, o.make_profile([(o.SCORER_KV_CACHE, 1.0)], pick_mode=o.PICK_RANDOM, tie_seed=1), idx, 2048,
                            prompt_bytes=pw, prompt_off=offw, model_seed=np.full(2048, ms, np.uint64), want_hashes=True,
                            n_threads=8)
    idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    pid = eng.add_profile(PREFILL, pick_mode=1)
    dec, pre = bits(M, range(0, M // 2)), bits(M, range(M // 2, M))
    eng.set_profile_endpoints(0, dec)
    eng.set_profile_endpoints(pid, pre)
    eng.set_snapshot(**sd)
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=150, shared=768, seed=4, prefix_seed=7)
    seeds = np.full(R, ms, np.uint64)
    ad = zipf_adapters(R, seed=4)
    _, got = eng.schedule_profiles(R, [dict(profile=0, topk=4), dict(profile=pid, topk=16)], prompt_bytes=prompts, prompt_off=off,
                                   model_seed=seeds, adapter_id=ad)
    for base in (0, 40000):
        n = 256
        skw = dict(prompt_bytes=prompts, prompt_off=off[base:base + n + 1], model_seed=seeds[base:base + n],
                   adapter_id=ad[base:base + n])
        for g, (sc, p, pm, sub, k) in zip(got, ((HEADLINE, 0, 0, dec, 4), (PREFILL, pid, 1, pre, 16))):
            want = oracle_run(pkg, snap, idx, n, sc, 0, seed_of(0, p), pm, sub, None, M, skw, k, request_base=base)
            _same({x: v[base:base + n] for x, v in g.items()}, want, ("headline", base, p))
    eng.close()
