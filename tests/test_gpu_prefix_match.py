"""eppscore_prefix_match on the GPU: matchLongestPrefix read at the endpoints a request was sent to, bit-exact to the oracle's
matchLongestPrefix and to the batch's own match_blocks gathered at the same entries.  Covered: the CPU scenarios (churn at LRU
capacities 3..31 250, inline -> row sets, a universal prefix, emptied sets mid-prompt, partial holders, 0 / 256 / 1000 hashes,
-1 and >= max_endpoints entries) in host and device location; picks and lists of the sparse, full-matrix, masked, latency
(behind both device filters), top-k, wide top-k (16 and k = max_endpoints) and two-profile routes; geometries M 5 / 1024 / 4097 at k = 1, 8, max_endpoints; R = 0, 1, 65 536; a call on a reserved stream
next to batches on other reserved streams; ordering against commits on other streams; 24 replays of one
schedule -> prefix_match -> commit graph on a reserved index with device rebuilds; invalid arguments; and the host layer's
test program (tests/cpp/host_prefix_match_test.cpp) on the engine."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests.helpers import synth_prompts, synth_snapshot
from tests.prefix_match_scenarios import CHURN, Query, churn_scenario, crafted_scenarios, endpoint_lists, expected

pytestmark = pytest.mark.gpu
ERR_INVALID = -1
SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3)]


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _device_match(eng, q, stream=None):
    import torch
    R, k = q.endpoints.shape
    out = torch.full((R, k), 0x7777, dtype=torch.int16, device="cuda:0")
    eng.prefix_match(_dev(q.hashes.view(np.int64)), _dev(q.n_hashes.view(np.int16)), _dev(q.endpoints), device=True, stream=stream, out=out)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint16)


def _both(eng, q, want):
    assert np.array_equal(eng.prefix_match(q.hashes, q.n_hashes, q.endpoints), want)
    assert np.array_equal(_device_match(eng, q), want)


def _run_scenario(pkg, sc, limit):
    """limit = the engine's max_endpoints (>= sc.M and >= every query's k)."""
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=limit, prefix_capacity=1 << 10, lru_capacity_default=sc.lru,
                                        lru_capacity_max=sc.lru_max))
    eng.set_snapshot(**synth_snapshot(limit, seed=1))  # a commit's lru_capacity is read for the snapshot's M endpoints
    idx = o.Index(sc.lru)
    caps = None if sc.caps is None else np.concatenate([sc.caps, np.zeros(limit - sc.M, np.int32)])
    for b, queries in sc.steps:
        eng.commit_picks(b.pick, b.hashes, b.n_hashes, lru_capacity=caps)
        idx.commit(b.pick, b.hashes, b.n_hashes, sc.caps)
        for q in queries:
            _both(eng, q, expected(idx, q, limit))


@pytest.mark.parametrize("M,lru,R,nmax,seed", CHURN, ids=[f"lru{c[1]}" for c in CHURN])
def test_churn_scenarios(pkg, M, lru, R, nmax, seed):
    _run_scenario(pkg, churn_scenario(M, lru, R, nmax, seed, k=8, limit=M + 1), M + 1)


def test_crafted_scenarios(pkg):
    for sc in crafted_scenarios(limit=10 ** 6):
        limit = sc.M + 3  # k = M + 3 columns: every endpoint, -1, max_endpoints and past it
        for _, queries in sc.steps:
            for q in queries:
                q.endpoints[:, -2:] = [limit, limit + 7]
        _run_scenario(pkg, sc, limit)


def test_one_prefix_on_1024_endpoints(pkg):
    """1024 endpoints holding one prefix: every set is an overflow row of 32 words."""
    M = 1024
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, prefix_capacity=1 << 12))
    idx = o.Index(31250)
    rng = np.random.Generator(np.random.PCG64(5))
    p = rng.integers(1, 2 ** 63, size=40, dtype=np.uint64)
    pick = np.arange(M, dtype=np.int32)
    hs = np.tile(p, (M, 1))
    nh = np.full(M, 40, np.uint16)
    nh[::3] = 17
    eng.commit_picks(pick, hs, nh)
    idx.commit(pick, hs, nh)
    q = Query(hs[:64].copy(), np.full(64, 40, np.uint16), endpoint_lists(rng, 64, M, M, M))
    _both(eng, q, expected(idx, q, M))


# ---- the routes: a batch's picks and lists, against the oracle and the batch's own match_blocks ----
LAT = dict(ttft_intercept=50.0, ttft_kv=30.0, ttft_input=0.05, ttft_waiting=8.0, ttft_running=4.0, ttft_prefix=-40.0,
           tpot_intercept=10.0, tpot_kv=5.0, tpot_input=0.001, tpot_waiting=1.0, tpot_running=1.0, tpot_generated=0.01)


def _world(pkg, M, R, seed=3, scorers=SCORERS, lat=False, **cfg):
    eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, max_blocks=32, prefix_capacity=1 << 16, **cfg))
    if lat:
        eng.set_latency_params(pkg.latency_params(**LAT))
    eng.set_snapshot(**synth_snapshot(M, seed=seed))
    idx = o.Index(31250)
    kw = None
    for k in range(3):  # warm the index with three committed batches
        prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=50 + k, prefix_seed=9)
        kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64), max_blocks=32)
        res = eng.schedule(R, want_hashes=True, **kw)
        eng.commit_picks(res["pick"], res["hashes_out"], res["total_blocks"])
        idx.commit(res["pick"], res["hashes_out"], res["total_blocks"])
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=24, shared=512, seed=99, prefix_seed=9)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64), max_blocks=32)
    return eng, idx, kw


def _check_lists(eng, idx, limit, hashes, nh, lists, match_blocks):
    q = Query(hashes, nh, np.ascontiguousarray(lists, np.int32))
    want = expected(idx, q, limit)
    _both(eng, q, want)
    e = q.endpoints
    gathered = np.where((e >= 0) & (e < limit), np.take_along_axis(match_blocks, np.clip(e, 0, match_blocks.shape[1] - 1), axis=1), 0)
    assert np.array_equal(gathered, want)


@pytest.mark.parametrize("route", ["sparse", "full-matrix", "masked", "latency-filters", "topk4", "wide16", "wide-max", "profiles"])
def test_routes(pkg, route):
    M, R = 64, 2048
    if route == "full-matrix":  # unmasked, but the weighted-random picker keeps the batch off the sparse path
        eng, idx, kw = _world(pkg, M, R, pick_mode=pkg.PICK_WEIGHTED_RANDOM)
    elif route == "latency-filters":  # the latency profile behind both device filters
        eng, idx, kw = _world(pkg, M, R, scorers=[("latency", 1.0)], lat=True, pick_mode=pkg.PICK_WEIGHTED_RANDOM,
                              filters=[(pkg.FILTER_PREFIX_AFFINITY, (0.8, 0.1, 5000.0)), (pkg.FILTER_SLO_HEADROOM_TIER, (0.1,))])
    else:
        eng, idx, kw = _world(pkg, M, R)
    diag = eng.schedule(R, want_match=True, **kw)["match_blocks"]
    rng = np.random.Generator(np.random.PCG64(11))
    if route in ("sparse", "full-matrix", "latency-filters"):
        res = eng.schedule(R, want_hashes=True, **kw)
        lists = [res["pick"][:, None]]
    elif route == "masked":
        mask = rng.integers(0, 2 ** 32, size=(R, (M + 31) // 32), dtype=np.uint64).astype(np.uint32)
        res = eng.schedule(R, want_hashes=True, cand_mask=mask, **kw)
        lists = [res["pick"][:, None]]
    elif route in ("topk4", "wide16", "wide-max"):
        lk = {"topk4": {"topk": 4}, "wide16": {"topk_wide": 16}, "wide-max": {"topk_wide": M}}[route]  # wide-max: k = max_endpoints
        res = eng.schedule(R, want_hashes=True, **lk, **kw)
        lists = [res["topk_pick"]]
    else:
        pid = eng.add_profile([(pkg.SCORER["kv"], 1), (pkg.SCORER["prefix"], 2)])
        eng.set_snapshot(**synth_snapshot(M, seed=3))
        res, runs = eng.schedule_profiles(R, [{"profile": 0}, {"profile": pid, "topk": 3}], want_hashes=True, **kw)
        lists = [runs[0]["pick"][:, None], runs[1]["topk_pick"], np.stack([runs[0]["pick"], runs[1]["pick"]], axis=1)]
    for ls in lists:
        _check_lists(eng, idx, M, res["hashes_out"], res["total_blocks"], ls, diag)


@pytest.mark.parametrize("M", [5, 1024, 4097])
def test_geometries(pkg, M):
    R = 512
    eng, idx, kw = _world(pkg, M, R)
    res = eng.schedule(R, want_hashes=True, want_match=True, **kw)
    rng = np.random.Generator(np.random.PCG64(M))
    for k in sorted({1, min(8, M), M}):  # (k <= max_endpoints)
        _check_lists(eng, idx, M, res["hashes_out"], res["total_blocks"], endpoint_lists(rng, R, k, M, M), res["match_blocks"])


def test_request_counts(pkg):
    """R = 0, 1 and 65 536 (k = 1 and 8)."""
    import torch
    M = 256
    eng, idx, kw = _world(pkg, M, 1024)
    res = eng.schedule(1024, want_hashes=True, want_match=True, **kw)
    z = np.zeros((0, 1), np.int32)
    assert eng.prefix_match(np.zeros((0, 32), np.uint64), np.zeros(0, np.uint16), z).shape == (0, 1)
    eng.prefix_match(_dev(np.zeros((1, 32), np.int64)), _dev(np.zeros(1, np.int16)), _dev(z), device=True,
                     out=torch.zeros((0, 1), dtype=torch.int16, device="cuda:0"))
    _check_lists(eng, idx, M, res["hashes_out"][:1], res["total_blocks"][:1], res["pick"][:1, None], res["match_blocks"][:1])
    rep = 64  # 65 536 requests: the 1024 prompts 64 times
    h, nh, mb = np.tile(res["hashes_out"], (rep, 1)), np.tile(res["total_blocks"], rep), np.tile(res["match_blocks"], (rep, 1))
    rng = np.random.Generator(np.random.PCG64(2))
    for k in (1, 8):
        _check_lists(eng, idx, M, h, nh, endpoint_lists(rng, 1024 * rep, k, M, M), mb)


def test_invalid_arguments(pkg):
    M = 8
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M))
    lib, h = eng._lib, eng._h
    hs = np.zeros((2, 4), np.uint64)
    nh = np.array([1, 5], np.uint16)  # 5 > hash_stride
    ep = np.zeros((2, 1), np.int32)
    out = np.zeros((2, 9), np.uint16)
    p = lambda a: a.ctypes.data  # noqa: E731
    assert lib.eppscore_prefix_match(h, 2, 1, 0, p(hs), p(nh), 4, p(ep), p(out), None) == ERR_INVALID
    nh[1] = 4
    assert lib.eppscore_prefix_match(h, 2, 1, 0, p(hs), p(nh), 4, p(ep), p(out), None) == 0
    for k in (0, M + 1, -3):
        assert lib.eppscore_prefix_match(h, 2, k, 0, p(hs), p(nh), 4, p(ep), p(out), None) == ERR_INVALID
    assert lib.eppscore_prefix_match(h, 2, 1, 0, None, p(nh), 4, p(ep), p(out), None) == ERR_INVALID
    assert lib.eppscore_prefix_match(h, 2, 1, 1, p(hs), p(nh), 4, None, p(out), None) == ERR_INVALID
    assert lib.eppscore_prefix_match(h, 2, 1, 0, p(hs), p(nh), 4, p(ep), None, None) == ERR_INVALID
    assert lib.eppscore_prefix_match(h, 2, 1, 2, p(hs), p(nh), 4, p(ep), p(out), None) == ERR_INVALID
    assert lib.eppscore_prefix_match(h, -1, 1, 0, p(hs), p(nh), 4, p(ep), p(out), None) == ERR_INVALID
    for stride in (0, -4):
        assert lib.eppscore_prefix_match(h, 2, 1, 0, p(hs), p(nh), stride, p(ep), p(out), None) == ERR_INVALID
    launches = eng.stats().kernel_launches
    eng.prefix_match(hs, nh, ep)
    assert eng.stats().kernel_launches == launches + 1


def test_ordering_across_streams(pkg):
    """A call after a device commit on another stream sees that commit; a commit issued after the call (one that evicts every
    block the call reads) does not change its result.  Nothing synchronises between the three calls of a round."""
    import torch
    M = R = 32
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, max_blocks=64, prefix_capacity=1 << 12, lru_capacity_default=64))
    rng = np.random.Generator(np.random.PCG64(8))
    hs = rng.integers(1, 2 ** 63, size=(R, 64), dtype=np.uint64)
    other = rng.integers(1, 2 ** 63, size=(R, 64), dtype=np.uint64)
    nh = np.full(R, 64, np.uint16)
    pick = rng.permutation(M).astype(np.int32)  # one request per endpoint: its 64 blocks fill the endpoint's LRU
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    d_h, d_other, d_nh, d_pick = _dev(hs.view(np.int64)), _dev(other.view(np.int64)), _dev(nh.view(np.int16)), _dev(pick)
    d_ep = _dev(pick[:, None])
    torch.cuda.synchronize()
    for rnd in range(4):
        out = torch.zeros((R, 1), dtype=torch.int16, device="cuda:0")
        eng.commit_picks_device(d_pick, d_h, d_nh, stream=s1.cuda_stream)              # commit on s1 ...
        eng.prefix_match(d_h, d_nh, d_ep, device=True, stream=s2.cuda_stream, out=out)   # ... seen by the match on s2,
        eng.commit_picks_device(d_pick, d_other, d_nh, stream=s1.cuda_stream)          # which this eviction waits for
        torch.cuda.synchronize()
        assert (out.cpu().numpy().view(np.uint16)[:, 0] == 64).all(), rnd
        assert eng.prefix_match(hs, nh, pick[:, None]).sum() == 0  # the second commit did evict them


def test_reserved_streams_concurrent(pkg):
    """A call on a reserved stream while batches run on two other reserved streams: every result bit-exact."""
    import torch
    M, R = 64, 1024
    eng, idx, kw = _world(pkg, M, R)
    res = eng.schedule(R, want_hashes=True, want_match=True, **kw)
    streams = [torch.cuda.Stream() for _ in range(3)]
    for s in streams:
        eng.reserve_stream(s.cuda_stream, R, 32)
    q = Query(res["hashes_out"], res["total_blocks"], endpoint_lists(np.random.Generator(np.random.PCG64(4)), R, 8, M, M))
    want = expected(idx, q, M)
    d_in = {key: _dev(v) for key, v in kw.items() if key != "max_blocks"}
    dev = torch.device("cuda:0")
    outs = [dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                 tie_count=torch.empty(R, dtype=torch.int32, device=dev)) for _ in range(2)]
    m_out = torch.zeros((R, 8), dtype=torch.int16, device=dev)
    d_h, d_nh, d_ep = _dev(q.hashes.view(np.int64)), _dev(q.n_hashes.view(np.int16)), _dev(q.endpoints)
    torch.cuda.synchronize()
    for _ in range(3):
        for i in range(2):
            eng.schedule(R, device=True, stream=streams[i].cuda_stream, out=outs[i], max_blocks=32, **d_in)
        eng.prefix_match(d_h, d_nh, d_ep, device=True, stream=streams[2].cuda_stream, out=m_out)
    torch.cuda.synchronize()
    assert np.array_equal(m_out.cpu().numpy().view(np.uint16), want)
    for i in range(2):
        assert np.array_equal(outs[i]["pick"].cpu().numpy(), res["pick"])
    for s in streams:
        eng.release_stream(s.cuda_stream)


def test_graph_replays_with_rebuilds(pkg):
    """24 replays of one schedule -> prefix_match -> commit graph on a reserved index with small LRUs: the table is rebuilt on the
    device several times and every round's match at the picks is bit-exact to the oracle's, read before the round's commit."""
    import torch
    M, R, MB, LRU = 64, 512, 16, 48
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, max_blocks=MB, prefix_capacity=1 << 10, lru_capacity_default=LRU))
    eng.set_snapshot(**synth_snapshot(M, seed=9))
    eng.prefix_reserve(M * LRU + 1024, R * MB, 0)
    idx = o.Index(LRU)
    dev = torch.device("cuda:0")

    def inputs(k):
        prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=16, shared=256, seed=300 + k, prefix_seed=7)
        return dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64))
    d_in = {key: _dev(v) for key, v in inputs(0).items()}
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
    m_out = torch.zeros((R, 1), dtype=torch.int16, device=dev)
    s = torch.cuda.Stream()

    def body():
        eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d_in)
        eng.prefix_match(out["hashes_out"], out["total_blocks"], out["pick"].view(R, 1), device=True, stream=s.cuda_stream, out=m_out)
        eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], stream=s.cuda_stream)
    eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **d_in)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        body()
    torch.cuda.synchronize()
    rebuilds0 = eng.stats().prefix_rebuilds
    for k in range(24):
        kw = inputs(k)
        for key in ("prompt_bytes",):
            d_in[key].copy_(torch.from_numpy(kw[key]))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        pick = out["pick"].cpu().numpy()
        hs = out["hashes_out"].cpu().numpy().view(np.uint64)
        nh = out["total_blocks"].cpu().numpy()
        q = Query(hs, nh, pick[:, None].copy())
        assert np.array_equal(m_out.cpu().numpy().view(np.uint16), expected(idx, q, M)), k
        idx.commit(pick, hs, nh)
    assert eng.stats().prefix_rebuilds - rebuilds0 >= 2


def test_host_program_on_the_engine(pkg):
    """tests/cpp/host_prefix_match_test.cpp (the host layer's PrefixCacheMatchInfo and prefix-indexer histograms against an oracle
    mirror of the index) linked against the engine library."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build = os.path.join(root, "tests", "cpp", "_build")
    os.makedirs(build, exist_ok=True)
    lib_dir = os.path.dirname(pkg.lib()._name)
    oracle_dir = os.path.dirname(o.build())
    exe = os.path.join(build, "host_prefix_match_test_engine")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread",
                           os.path.join(root, "tests", "cpp", "host_prefix_match_test.cpp"), "-L" + lib_dir, "-leppscore",
                           "-L" + oracle_dir, "-loracle", "-Wl,-rpath," + lib_dir + ":" + oracle_dir, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    assert not any(line.startswith(("FAIL", "refused")) for line in r.stdout.splitlines())
