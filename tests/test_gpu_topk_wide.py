"""maxNumOfEndpoints past 8 on the GPU (eppscore_schedule_batch_topk_wide): the first k endpoints of every request's pick order
for any k up to max_endpoints, bit-exact against the CPU oracle's top-k (tests/cpp/topk_oracle.c) in all three pick modes and
both tie modes; equal to eppscore_schedule_batch_topk's lists for k <= 8; pick / pick_score / tie_count unchanged; the radix
select's tie and threshold edges; every way of running a batch gives the same lists; and the reference's picker tests at k > 8."""
import ctypes as C
import itertools

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import topk_oracle as T
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

pytestmark = pytest.mark.gpu

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01)
ERR_INVALID, ERR_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def wide_ks(M, max_endpoints):
    return sorted({k for k in (1, 3, 8, 9, 16, 33, 255, 256, 257, M - 1, M, max_endpoints) if 1 <= k <= max_endpoints})


def assert_lists(got, want_m, want_s, what=""):
    assert np.array_equal(got["topk_pick"], want_m), what
    assert np.array_equal(got["topk_score"].view(np.uint64), want_s.view(np.uint64)), what


def assert_same_picks(got, want, what=""):
    assert np.array_equal(got["pick"], want["pick"]), what
    assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what
    assert np.array_equal(got["tie_count"], want["tie_count"]), what


def assert_entry0_is_pick(got, what=""):
    assert np.array_equal(got["topk_pick"][:, 0], got["pick"]), what
    s0 = np.where(got["pick"] >= 0, got["topk_score"][:, 0], 0.0)
    assert np.array_equal(s0.view(np.uint64), got["pick_score"].view(np.uint64)), what


def check_wide(eng, prof, weighted, R, ks, plain, what, request_base=0, **kw):
    """every k in ks against the oracle's order (the first k entries of one list of length max(ks)); k <= 8 also against
    eppscore_schedule_batch_topk"""
    km = max(ks)
    wm, ws = T.lists(weighted, prof, km, request_base)
    for k in ks:
        got = eng.schedule(R, topk_wide=k, request_base=request_base, **kw)
        w = (what, k)
        assert_same_picks(got, plain, w)
        assert_lists(got, wm[:, :k], ws[:, :k], w)
        assert_entry0_is_pick(got, w)
        if k <= 8:
            assert_lists(got, *(lambda t: (t["topk_pick"], t["topk_score"]))(eng.schedule(R, topk=k, request_base=request_base, **kw)), w)


def random_masks(R, M, rng):
    """per-row densities from empty to full; rows 0..2: no candidate, one, two"""
    dens = rng.choice([0.0, 0.002, 0.01, 0.1, 0.5, 0.9, 1.0], R)
    bits = rng.random((R, M)) < dens[:, None]
    bits[0] = False
    bits[1] = False
    bits[1, M // 2] = True
    bits[2] = False
    bits[2, [0, M - 1]] = True
    mw = (M + 31) // 32
    pad = np.zeros((R, mw * 32), bool)
    pad[:, :M] = bits
    return (pad.reshape(R, mw, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


def warmed(pkg, M, R, seed, **cfg):
    """engine + oracle with the same snapshot and a prefix index warmed by one committed batch"""
    cfg.setdefault("max_endpoints", M)
    eng = pkg.Engine(pkg.default_config(SCORERS, prefix_capacity=1 << 16, **cfg))
    sd = synth_snapshot(M, seed=seed)
    eng.set_snapshot(**sd)
    snap, idx = o.SnapshotData(**sd), o.Index()
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=12, shared=768, seed=seed)
    seeds = np.full(R, eng.model_seed("topk"), np.uint64)
    ad = zipf_adapters(R, seed=seed)
    warm_prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], pick_mode=o.PICK_RANDOM, tie_seed=3)
    w = o.schedule_batch(snap, warm_prof, idx, R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, want_hashes=True,
                         n_threads=8)
    idx.commit(w["pick"], w["hashes_out"], w["total_blocks"])
    eng.commit_picks(w["pick"], w["hashes_out"], w["total_blocks"])
    return eng, snap, idx, dict(prompt_bytes=prompts, prompt_off=off, model_seed=seeds, adapter_id=ad)


@pytest.mark.parametrize("M", [5, 600, 1024, 4096])
def test_wide_lists_match_oracle(pkg, M):
    R = 384
    rng = np.random.Generator(np.random.PCG64(M + 77))
    masks = random_masks(R, M, rng)
    for pick_mode, tie_mode in itertools.product((0, 1, 2), (0, 1)):
        seed = int(rng.integers(0, 2 ** 63))
        eng, snap, idx, kw = warmed(pkg, M, R, M + pick_mode, pick_mode=pick_mode, tie_mode=tie_mode, tie_seed=seed)
        prof = o.make_profile([(pkg.SCORER[k], w) for k, w in SCORERS], tie_mode=tie_mode, tie_seed=seed, pick_mode=pick_mode)
        for mask in (masks, None):
            want = o.schedule_batch(snap, prof, idx, R, cand_mask=mask, want_scores=True, n_threads=8, **kw)
            plain = eng.schedule(R, cand_mask=mask, **kw)
            assert_same_picks(plain, want, (M, pick_mode, tie_mode))
            check_wide(eng, prof, want["weighted_out"], R, wide_ks(M, M), plain, (M, pick_mode, tie_mode, mask is not None),
                       cand_mask=mask, **kw)
        eng.close()


def _col_engine(pkg, col, weight, pick_mode, tie_mode, seed, max_endpoints=None):
    M = len(col)
    eng = pkg.Engine(pkg.default_config([("col0", weight)], max_endpoints=max_endpoints or M, pick_mode=pick_mode,
                                        tie_mode=tie_mode, tie_seed=seed))
    eng.set_snapshot(np.zeros(M), np.zeros(M, np.int64), endpoint_cols=[np.asarray(col, np.float64)])
    return eng


def _bits(hi_mask, base, rng, M):
    """positive doubles below 1 that share the bits of `base` under hi_mask and differ below"""
    lo = rng.integers(0, 2 ** 52, M, dtype=np.uint64) & np.uint64(~hi_mask & (2 ** 64 - 1))
    return ((np.uint64(base) & np.uint64(hi_mask)) | lo).view(np.float64)


def test_ties_and_radix_threshold_edges(pkg):
    """one endpoint column scored with weight 1 (or -1): the score rows are exactly the column, so the rows are chosen bit by bit"""
    M, R = 1024, 96
    rng = np.random.Generator(np.random.PCG64(5))
    base = np.float64(0.75).view(np.uint64)
    cases = {
        "all equal": (np.full(M, 0.5), 1.0),
        "many equal to the k-th": (np.where(rng.random(M) < 0.7, 0.25, rng.choice([0.5, 0.125, 0.0625], M)), 1.0),
        "high 8 bits equal": (_bits(0xFF00000000000000, base, rng, M), 1.0),
        "high 16 bits equal": (_bits(0xFFFF000000000000, base, rng, M), 1.0),
        "high 32 bits equal": (_bits(0xFFFFFFFF00000000, base, rng, M), 1.0),
        "all scores <= 0": (rng.choice([0.0, 0.25, 0.5], M), -1.0),
        "mixed signs": (np.where(rng.random(M) < 0.5, 0.0, rng.random(M)), 1.0),
        "two values": (rng.choice([0.25, 0.5], M), 1.0),
    }
    for (name, (col, weight)), pick_mode, tie_mode in itertools.product(cases.items(), (0, 1, 2), (0, 1)):
        eng = _col_engine(pkg, col, weight, pick_mode, tie_mode, 1000 + pick_mode)
        prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], tie_mode=tie_mode, tie_seed=1000 + pick_mode, pick_mode=pick_mode)
        plain = eng.schedule(R, want_scores=True)
        check_wide(eng, prof, plain["scores_out"], R, (1, 8, 9, 100, 511, 512, 700, M), plain, (name, pick_mode, tie_mode))
        eng.close()
    # a snapshot smaller than max_endpoints: k up to max_endpoints, the lists padded past M
    eng = _col_engine(pkg, rng.random(600), 1.0, 1, 0, 3, max_endpoints=1024)
    prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], tie_seed=3, pick_mode=1)
    plain = eng.schedule(R, want_scores=True)
    check_wide(eng, prof, plain["scores_out"], R, (599, 600, 601, 1024), plain, "M < max_endpoints")
    eng.close()


def test_largest_geometry_every_endpoint(pkg):
    """M = max_endpoints = 8192 with k = 8192: the selection's shared-memory limit"""
    M, R = 8192, 24
    rng = np.random.Generator(np.random.PCG64(8192))
    col = rng.choice([0.0, 0.25, 0.5, 0.75], M) + rng.random(M) * (rng.random(M) < 0.5) * 0.01
    mask = random_masks(R, M, rng)
    for pick_mode in (0, 1, 2):
        eng = _col_engine(pkg, col, 1.0, pick_mode, 1, 42)
        prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], tie_mode=1, tie_seed=42, pick_mode=pick_mode)
        for m in (None, mask):
            plain = eng.schedule(R, cand_mask=m, want_scores=True)
            check_wide(eng, prof, plain["scores_out"], R, (8, 4096, 8191, 8192), plain, (pick_mode, m is not None), cand_mask=m)
        eng.close()


def test_latency_chart_profile_and_dense_rows(pkg):
    """three device filters + latency scorer + weighted-random picker; dense rows with the max-score picker"""
    M, R = 300, 768
    lkw = dict(LAT_COEF, streaming_mode=1)
    filt = [(pkg.FILTER_PREFIX_AFFINITY, (0.95, 0.2, 40.0)), (pkg.FILTER_SLO_HEADROOM_TIER, (0.3,)),
            (pkg.FILTER_PREFIX_AFFINITY, (0.50, 0.1, 5000.0))]
    eng = pkg.Engine(pkg.default_config([("latency", 1.0)], filters=filt, max_endpoints=M, max_blocks=16,
                                        pick_mode=pkg.PICK_WEIGHTED_RANDOM, tie_seed=21, prefix_capacity=1 << 15))
    eng.set_latency_params(pkg.latency_params(**lkw))
    rng = np.random.Generator(np.random.PCG64(31))
    sd = synth_snapshot(M, seed=6)
    sd["min_tpot_slo"] = rng.choice([0.0, 22.0, 60.0], M)
    sd["dispatched"] = rng.integers(0, 3, M).astype(np.int32)
    sd["prefill_role"] = (rng.random(M) < 0.1).astype(np.uint8)
    eng.set_snapshot(**sd)
    snap = o.SnapshotData(**sd)
    prof = o.make_profile([(o.SCORER_LATENCY, 1.0)], latency=o.make_latency_params(**lkw), pick_mode=o.PICK_WEIGHTED_RANDOM,
                          tie_seed=21, filters=[(k, par) for k, par in filt])
    prompts, off, _ = synth_prompts(R, prompt_len=1024, groups=6, shared=1024 - 64, seed=8)
    seeds = np.full(R, eng.model_seed("m"), np.uint64)
    idx = o.Index()
    warm_prof = o.make_profile([(o.SCORER_KV_CACHE, 1.0)], pick_mode=o.PICK_RANDOM, tie_seed=2)
    warm = o.schedule_batch(snap, warm_prof, idx, R, prompt_bytes=prompts, prompt_off=off, max_blocks=16, model_seed=seeds,
                            want_hashes=True, n_threads=8)
    nblk = np.where(np.arange(R) % 2 == 0, warm["total_blocks"], np.minimum(warm["total_blocks"], 8)).astype(np.uint16)
    idx.commit(warm["pick"], warm["hashes_out"], nblk)
    eng.commit_picks(warm["pick"], warm["hashes_out"], nblk)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=seeds, input_tokens=rng.integers(0, 3000, R).astype(np.int32),
              ttft_slo=rng.choice([0.0, 120.0, 180.0, 400.0], R), tpot_slo=rng.choice([0.0, 22.0, 30.0], R))
    for mask in (None, random_masks(R, M, rng)):
        want = o.schedule_batch(snap, prof, idx, R, max_blocks=16, cand_mask=mask, want_scores=True, n_threads=8, **kw)
        plain = eng.schedule(R, cand_mask=mask, **kw)
        assert_same_picks(plain, want)
        check_wide(eng, prof, want["weighted_out"], R, (1, 8, 9, 40, M), plain, ("latency", mask is not None), cand_mask=mask, **kw)
        got = eng.schedule(R, cand_mask=mask, topk_wide=40, **kw)
        assert (got["topk_pick"][:, -1] == -1).any() and (got["topk_pick"][:, 9] >= 0).any()  # the filters leave short lists
    eng.close()

    for M, R, masked, tie_mode in ((1024, 1024, False, 0), (333, 1024, True, 1)):
        scorers = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("pair0", 1.5), ("pair1", 0.5)]
        eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, prefix_capacity=1 << 14, tie_mode=tie_mode, tie_seed=5))
        sd = synth_snapshot(M, seed=M)
        eng.set_snapshot(**sd)
        rng = np.random.Generator(np.random.PCG64(M))
        feat = np.zeros((R, M, 4), np.float32)
        total = rng.integers(0, 40, R).astype(np.uint16)
        feat[:, :, 0] = np.minimum(rng.integers(0, 48, (R, M)) * (rng.random((R, M)) < 0.05), total[:, None] + 2)
        feat[:, :, 1] = rng.integers(0, 4, (R, M))
        feat[:, :, 2] = np.round(rng.random((R, M)), 1)  # coarse: many ties
        feat[:, :, 3] = np.round(rng.random((R, M)), 1)
        kw = dict(dense_feat=feat, dense_total=total)
        if masked:
            kw["cand_mask"] = random_masks(R, M, rng)
        prof = o.make_profile([(pkg.SCORER[k], w) for k, w in scorers], tie_mode=tie_mode, tie_seed=5)
        want = o.schedule_batch(o.SnapshotData(**sd), prof, None, R, want_scores=True, n_threads=8, **kw)
        plain = eng.schedule(R, **kw)
        assert_same_picks(plain, want, M)
        check_wide(eng, prof, want["weighted_out"], R, (1, 8, 9, 64, M), plain, ("dense", M), **kw)
        eng.close()
    # the stochastic pickers refuse dense rows here as eppscore_schedule_batch_topk does
    eng = pkg.Engine(pkg.default_config([("kv", 1), ("pair0", 1)], max_endpoints=64, pick_mode=pkg.PICK_RANDOM))
    eng.set_snapshot(np.linspace(0, 1, 64), np.zeros(64, np.int64))
    kw = dict(dense_feat=np.zeros((4, 64, 4), np.float32), dense_total=np.zeros(4, np.uint16))
    for call in (dict(topk=4), dict(topk_wide=12)):
        with pytest.raises(pkg.EppscoreError) as ex:
            eng.schedule(4, **call, **kw)
        assert ex.value.code == ERR_INVALID
    eng.close()


def test_every_way_of_running_a_batch_gives_the_same_lists(pkg):
    """host vs device buffers, chunked host batch (debug key 3), sliced device batch (keys 5 / 6), two shards with request_base,
    CUDA-graph replay (also after a larger wide call outside the capture), and a capture before the first wide call"""
    import torch
    M, R, k = 1024, 8192, 40
    eng, snap, idx, kw = warmed(pkg, M, R + 4096, 17, pick_mode=pkg.PICK_WEIGHTED_RANDOM, tie_seed=99)
    kw_big = kw
    kw = dict(kw, prompt_bytes=kw["prompt_bytes"][: kw["prompt_off"][R]], prompt_off=kw["prompt_off"][: R + 1],
              model_seed=kw["model_seed"][:R], adapter_id=kw["adapter_id"][:R])
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream()

    def outputs(R_, k_):
        return dict(pick=torch.empty(R_, dtype=torch.int32, device=dev), pick_score=torch.empty(R_, dtype=torch.float64, device=dev),
                    tie_count=torch.empty(R_, dtype=torch.int32, device=dev),
                    topk_pick=torch.empty((R_, k_), dtype=torch.int32, device=dev),
                    topk_score=torch.empty((R_, k_), dtype=torch.float64, device=dev))

    d_in = {key: torch.from_numpy(v).to(dev) for key, v in kw.items()}
    out = outputs(R, k)
    torch.cuda.synchronize()
    g0 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g0, stream=stream):  # no wide call has allocated the score scratch yet
        with pytest.raises(pkg.EppscoreError) as ex:
            eng.schedule(R, topk_wide=k, device=True, stream=stream.cuda_stream, out=out, **d_in)
    assert ex.value.code == ERR_CAPACITY and "outside" in str(ex.value)
    del g0

    ref = eng.schedule(R, topk_wide=k, **kw)
    prof = o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], tie_seed=99, pick_mode=o.PICK_WEIGHTED_RANDOM)
    want = o.schedule_batch(snap, prof, idx, 512, want_scores=True, n_threads=8,
                            **dict(kw, prompt_bytes=kw["prompt_bytes"][: kw["prompt_off"][512]], prompt_off=kw["prompt_off"][:513],
                                   model_seed=kw["model_seed"][:512], adapter_id=kw["adapter_id"][:512]))
    wm, ws = T.lists(want["weighted_out"], prof, k)
    assert np.array_equal(ref["topk_pick"][:512], wm) and np.array_equal(ref["topk_score"][:512].view(np.uint64), ws.view(np.uint64))

    def same(got, what):
        assert np.array_equal(got["topk_pick"], ref["topk_pick"]), what
        assert np.array_equal(got["topk_score"].view(np.uint64), ref["topk_score"].view(np.uint64)), what
        assert np.array_equal(got["pick"], ref["pick"]), what
        assert np.array_equal(got["tie_count"], ref["tie_count"]), what

    eng.set_debug(3, 1000)  # chunks of 1000 requests alternating over two streams
    same(eng.schedule(R, topk_wide=k, **kw), "chunked")
    eng.set_debug(3, 8192)
    h = 3000
    off = kw["prompt_off"]
    lo = eng.schedule(h, topk_wide=k, prompt_bytes=kw["prompt_bytes"][: off[h]], prompt_off=off[: h + 1],
                      model_seed=kw["model_seed"][:h], adapter_id=kw["adapter_id"][:h])
    hi = eng.schedule(R - h, topk_wide=k, prompt_bytes=kw["prompt_bytes"][off[h]:], prompt_off=off[h:] - off[h],
                      model_seed=kw["model_seed"][h:], adapter_id=kw["adapter_id"][h:], request_base=h)
    same({key: np.concatenate([lo[key], hi[key]]) for key in ("topk_pick", "topk_score", "pick", "tie_count")}, "two shards")

    def run_device(what, o_=out):
        with torch.cuda.stream(stream):
            for v in o_.values():
                v.zero_()
            eng.schedule(R, topk_wide=k, device=True, stream=stream.cuda_stream, out=o_, **d_in)
        stream.synchronize()
        same({key: v.cpu().numpy() for key, v in o_.items()}, what)

    run_device("device")
    with_scores = dict(out, scores_out=torch.empty((R, M), dtype=torch.float64, device=dev))
    run_device("device, caller's scores_out", with_scores)
    for split, streams in ((3, 2), (4, 3)):
        eng.set_debug(5, split)
        eng.set_debug(6, streams)
        run_device(("sliced", split, streams))
    eng.set_debug(5, 1)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        for v in out.values():
            v.zero_()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=stream):
        eng.schedule(R, topk_wide=k, device=True, stream=stream.cuda_stream, out=out, **d_in)
    g.replay()
    torch.cuda.synchronize()
    same({key: v.cpu().numpy() for key, v in out.items()}, "graph")
    # a larger wide call outside the capture (more requests, larger k) leaves the graph's scratch where it was
    Rb, kb = R + 4096, 300
    big_in = {key: torch.from_numpy(v).to(dev) for key, v in kw_big.items()}
    big = outputs(Rb, kb)
    with torch.cuda.stream(stream):
        eng.schedule(Rb, topk_wide=kb, device=True, stream=stream.cuda_stream, out=big, **big_in)
    stream.synchronize()
    assert np.array_equal(big["topk_pick"][:R, :k].cpu().numpy(), ref["topk_pick"])
    with torch.cuda.stream(stream):
        for v in out.values():
            v.zero_()
    stream.synchronize()
    g.replay()
    torch.cuda.synchronize()
    same({key: v.cpu().numpy() for key, v in out.items()}, "graph after a larger call")
    eng.close()


def test_headline_shape_lists(pkg):
    """64K requests x 1024 endpoints, four scorers, warmed index, k = 16 and 64: the lists of sampled rows against the oracle"""
    M, R = 1024, 65536
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, prefix_capacity=1 << 18))
    sd = synth_snapshot(M, seed=0)
    eng.set_snapshot(**sd)
    snap, prof, idx = o.SnapshotData(**sd), o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS]), o.Index()
    seed = eng.model_seed("headline")
    wp, woff, _ = synth_prompts(4 * M, seed=0)
    warm = o.schedule_batch(snap, prof, idx, 4 * M, prompt_bytes=wp, prompt_off=woff, model_seed=np.full(4 * M, seed, np.uint64),
                            want_hashes=True, n_threads=8)
    idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    prompts, off, _ = synth_prompts(R, seed=0)
    seeds = np.full(R, seed, np.uint64)
    ad = zipf_adapters(R, seed=0)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=seeds, adapter_id=ad)
    plain = eng.schedule(R, **kw)
    got = {k: eng.schedule(R, topk_wide=k, **kw) for k in (16, 64)}
    for r0 in (0, 40000, R - 512):
        n = 512
        want = o.schedule_batch(snap, prof, idx, n, prompt_bytes=prompts[off[r0]:off[r0 + n]], prompt_off=off[r0:r0 + n + 1] - off[r0],
                                model_seed=seeds[r0:r0 + n], adapter_id=ad[r0:r0 + n], request_base=r0, want_scores=True, n_threads=8)
        wm, ws = T.lists(want["weighted_out"], prof, 64, r0)
        for k, g in got.items():
            assert_same_picks(g, plain, k)
            assert np.array_equal(g["topk_pick"][r0:r0 + n], wm[:, :k]), (r0, k)
            assert np.array_equal(g["topk_score"][r0:r0 + n].view(np.uint64), ws[:, :k].view(np.uint64)), (r0, k)
    eng.close()


def test_reference_picker_tests_past_eight(pkg):
    n = 10000
    # random/picker_test.go:40-119 at k > 8: list length min(k, n) and inclusion min(k/n, 1) +- 0.05, n > 8 candidates
    for n_ep, k in ((20, 12), (20, 30), (50, 9), (12, 12)):
        eng = _col_engine(pkg, np.full(n_ep, 0.5), 1.0, pkg.PICK_RANDOM, 0, 99, max_endpoints=64)
        got = eng.schedule(n, topk_wide=k)
        real = got["topk_pick"] >= 0
        assert (real.sum(axis=1) == min(k, n_ep)).all(), (n_ep, k)
        freq = np.bincount(got["topk_pick"][real], minlength=n_ep) / n
        assert np.abs(freq - min(k / n_ep, 1.0)).max() <= 0.05, (n_ep, k, freq)
        eng.close()
    # weighted-random at k = 12: sampling without replacement, the zero scores filling the places the positive ones leave
    from tests.test_topk_cpu import _successive_sampling_inclusion
    for scores in ([5, 20, 1, 8, 3, 12] + [0] * 10, [1, 1, 2, 0, 0, 7, 30] + [0] * 9, [10, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]):
        eng = _col_engine(pkg, np.asarray(scores, np.float64) / 100.0, 100.0, pkg.PICK_WEIGHTED_RANDOM, 0, 1234)
        got = eng.schedule(n, topk_wide=12)
        real = got["topk_pick"] >= 0
        freq = np.bincount(got["topk_pick"][real], minlength=len(scores)) / n
        assert np.abs(freq - _successive_sampling_inclusion(scores, 12)).max() <= 0.05, (scores, freq)
        eng.close()


def test_invalid_arguments(pkg):
    import torch
    M, R = 64, 4
    eng = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=M))
    eng.set_snapshot(np.linspace(0, 1, M), np.zeros(M, np.int64))
    L = eng._lib
    pick, score, ties = np.zeros(R, np.int32), np.zeros(R), np.zeros(R, np.int32)
    tm, ts = np.zeros(R * M, np.int32), np.zeros(R * M)

    def call(k, m_ptr, s_ptr, size=None, location=0, arrays=(pick, score, ties)):
        b = pkg.Batch()
        b.struct_size = C.sizeof(pkg.Batch)
        b.R = R
        b.location = location
        b.pick, b.pick_score, b.tie_count = (a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr() for a in arrays)
        t = pkg.TopK()
        t.struct_size = C.sizeof(pkg.TopK) if size is None else size
        t.k = k
        t.endpoints = m_ptr
        t.scores = s_ptr
        return L.eppscore_schedule_batch_topk_wide(eng._h, C.byref(b), C.byref(t))

    ok = (tm.ctypes.data, ts.ctypes.data)
    assert call(M, *ok) == 0
    assert sorted(tm[:M].tolist()) == list(range(M)) and tm[0] == pick[0]  # every endpoint, the pick first
    for k in (0, -1, M + 1, 10000):
        assert call(k, *ok) == ERR_INVALID, k
    assert call(3, None, ts.ctypes.data) == ERR_INVALID
    assert call(3, tm.ctypes.data, None) == ERR_INVALID
    assert call(3, *ok, size=8) == ERR_INVALID
    assert L.eppscore_schedule_batch_topk_wide(eng._h, None, None) == ERR_INVALID
    dev = torch.device("cuda:0")
    d = [torch.zeros(R, dtype=torch.int32, device=dev), torch.zeros(R, dtype=torch.float64, device=dev),
         torch.zeros(R, dtype=torch.int32, device=dev)]
    dm, ds = torch.zeros(R * M, dtype=torch.int32, device=dev), torch.zeros(R * M, dtype=torch.float64, device=dev)
    assert call(M + 1, dm.data_ptr(), ds.data_ptr(), location=1, arrays=d) == ERR_INVALID
    assert call(0, dm.data_ptr(), ds.data_ptr(), location=1, arrays=d) == ERR_INVALID
    assert call(20, None, ds.data_ptr(), location=1, arrays=d) == ERR_INVALID
    assert call(20, dm.data_ptr(), None, location=1, arrays=d) == ERR_INVALID
    assert call(20, dm.data_ptr(), ds.data_ptr(), size=8, location=1, arrays=d) == ERR_INVALID
    assert call(20, dm.data_ptr(), ds.data_ptr(), location=1, arrays=d) == 0
    torch.cuda.synchronize()
    assert dm.cpu().numpy()[:R * 20].reshape(R, 20)[:, 0].tolist() == d[0].cpu().numpy().tolist()
    # eppscore_schedule_batch_topk keeps its limit
    b = pkg.Batch()
    b.struct_size = C.sizeof(pkg.Batch)
    b.R = R
    b.pick, b.pick_score, b.tie_count = pick.ctypes.data, score.ctypes.data, ties.ctypes.data
    t = pkg.TopK()
    t.struct_size = C.sizeof(pkg.TopK)
    t.k, t.endpoints, t.scores = 9, tm.ctypes.data, ts.ctypes.data
    assert L.eppscore_schedule_batch_topk(eng._h, C.byref(b), C.byref(t)) == ERR_INVALID
    with pytest.raises(pkg.EppscoreError):
        eng.schedule(R, topk=9)
    eng.close()
