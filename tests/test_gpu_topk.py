"""maxNumOfEndpoints on the GPU (eppscore_schedule_batch_topk): the first k endpoints of every request's pick order, from
the full-matrix and dense-row kernels, bit-exact against the CPU oracle's top-k (tests/cpp/topk_oracle.c) in all three pick modes and both
tie modes; pick / pick_score / tie_count unchanged by asking for the lists; every way of running a batch (host or device
buffers, chunked, sliced over streams, CUDA-graph replay, split into shards) gives the same lists; and the reference's own
picker tests hold on the engine's lists."""
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


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def oracle_topk(weighted, prof, k, request_base=0):
    return T.lists(weighted, prof, k, request_base)


def assert_lists(got, want_m, want_s, what=""):
    assert np.array_equal(got["topk_pick"], want_m), what
    assert np.array_equal(got["topk_score"].view(np.uint64), want_s.view(np.uint64)), what


def assert_same_picks(got, want, what=""):
    assert np.array_equal(got["pick"], want["pick"]), what
    assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what
    assert np.array_equal(got["tie_count"], want["tie_count"]), what


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
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, prefix_capacity=1 << 16, **cfg))
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
def test_matrix_lists_match_oracle(pkg, M):
    R = 384
    rng = np.random.Generator(np.random.PCG64(M))
    masks = random_masks(R, M, rng)
    for pick_mode, tie_mode in itertools.product((0, 1, 2), (0, 1)):
        seed = int(rng.integers(0, 2 ** 63))
        eng, snap, idx, kw = warmed(pkg, M, R, M + pick_mode, pick_mode=pick_mode, tie_mode=tie_mode, tie_seed=seed)
        prof = o.make_profile([(pkg.SCORER[k], w) for k, w in SCORERS], tie_mode=tie_mode, tie_seed=seed, pick_mode=pick_mode)
        for mask in (masks, None):
            want = o.schedule_batch(snap, prof, idx, R, cand_mask=mask, want_scores=True, n_threads=8, **kw)
            plain = eng.schedule(R, cand_mask=mask, **kw)
            assert_same_picks(plain, want, (M, pick_mode, tie_mode))
            for k in ((1, 2, 3, 8) if mask is not None else (3, 8)):
                what = (M, pick_mode, tie_mode, mask is not None, k)
                got = eng.schedule(R, cand_mask=mask, topk=k, want_scores=(k == 3), **kw)
                assert_same_picks(got, plain, what)
                wm, ws = oracle_topk(want["weighted_out"], prof, k)
                assert_lists(got, wm, ws, what)
                assert np.array_equal(got["topk_pick"][:, 0], got["pick"]), what
                assert np.array_equal(got["topk_score"][:, 0].view(np.uint64), got["pick_score"].view(np.uint64)), what
                if k == 3:
                    s, w = got["scores_out"], want["weighted_out"]
                    assert np.array_equal(np.isnan(s), np.isnan(w)) and np.array_equal(s[~np.isnan(s)], w[~np.isnan(w)]), what
        eng.close()


def test_latency_chart_profile_lists(pkg):
    """three device filters + latency scorer + weighted-random picker (config/charts/epplib/templates/_config.yaml:66-75)"""
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
    warm = o.schedule_batch(snap, warm_prof, idx, R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, max_blocks=16,
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
        for k in (1, 3, 8):
            got = eng.schedule(R, cand_mask=mask, topk=k, **kw)
            assert_same_picks(got, plain, k)
            wm, ws = oracle_topk(want["weighted_out"], prof, k)
            assert_lists(got, wm, ws, (mask is not None, k))
        # the filters leave short lists: some rows have fewer than 8 entries
        assert (got["topk_pick"][:, -1] == -1).any() and (got["topk_pick"][:, 1] >= 0).any()
    eng.close()


def test_dense_row_lists(pkg):
    for M, R, masked, tie_mode in ((1024, 1024, False, 0), (333, 1024, True, 1), (4096, 256, True, 0)):
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
        for k in (1, 2, 8):
            got = eng.schedule(R, topk=k, **kw)
            assert_same_picks(got, plain, (M, k))
            assert_same_picks(got, want, (M, k))
            wm, ws = oracle_topk(want["weighted_out"], prof, k)
            assert_lists(got, wm, ws, (M, masked, k))
        eng.close()


def test_every_way_of_running_a_batch_gives_the_same_lists(pkg):
    """host vs device buffers, chunked host batch (debug key 3), sliced device batch (keys 5 / 6), CUDA-graph replay, and two
    half batches with request_base == one batch"""
    import torch
    M, R, k = 1024, 8192, 4
    eng, snap, idx, kw = warmed(pkg, M, R, 17, pick_mode=pkg.PICK_WEIGHTED_RANDOM, tie_seed=99)
    ref = eng.schedule(R, topk=k, **kw)
    prof = o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], tie_seed=99, pick_mode=o.PICK_WEIGHTED_RANDOM)
    sample = slice(0, 512)
    want = o.schedule_batch(snap, prof, idx, 512, want_scores=True, n_threads=8,
                            **dict(kw, prompt_bytes=kw["prompt_bytes"][: kw["prompt_off"][512]], prompt_off=kw["prompt_off"][:513],
                                   model_seed=kw["model_seed"][:512], adapter_id=kw["adapter_id"][:512]))
    wm, ws = oracle_topk(want["weighted_out"], prof, k)
    assert np.array_equal(ref["topk_pick"][sample], wm) and np.array_equal(ref["topk_score"][sample], ws)

    def same(got, what):
        assert np.array_equal(got["topk_pick"], ref["topk_pick"]), what
        assert np.array_equal(got["topk_score"].view(np.uint64), ref["topk_score"].view(np.uint64)), what
        assert np.array_equal(got["pick"], ref["pick"]), what

    eng.set_debug(3, 1000)  # chunks of 1000 requests alternating over two streams
    same(eng.schedule(R, topk=k, **kw), "chunked")
    eng.set_debug(3, 8192)
    h = 3000
    off = kw["prompt_off"]
    lo = eng.schedule(h, topk=k, prompt_bytes=kw["prompt_bytes"][: off[h]], prompt_off=off[: h + 1], model_seed=kw["model_seed"][:h],
                      adapter_id=kw["adapter_id"][:h])
    hi = eng.schedule(R - h, topk=k, prompt_bytes=kw["prompt_bytes"][off[h]:], prompt_off=off[h:] - off[h],
                      model_seed=kw["model_seed"][h:], adapter_id=kw["adapter_id"][h:], request_base=h)
    same({key: np.concatenate([lo[key], hi[key]]) for key in ("topk_pick", "topk_score", "pick")}, "two shards")

    dev = torch.device("cuda:0")
    d_in = {key: torch.from_numpy(v).to(dev) for key, v in kw.items()}
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), topk_pick=torch.empty((R, k), dtype=torch.int32, device=dev),
               topk_score=torch.empty((R, k), dtype=torch.float64, device=dev))
    stream = torch.cuda.Stream()

    def run_device(what):
        with torch.cuda.stream(stream):
            for v in out.values():
                v.zero_()
            eng.schedule(R, topk=k, device=True, stream=stream.cuda_stream, out=out, **d_in)
        stream.synchronize()
        same({key: v.cpu().numpy() for key, v in out.items()}, what)

    run_device("device")
    for split, streams in ((3, 2), (4, 3)):
        eng.set_debug(5, split)
        eng.set_debug(6, streams)
        run_device(("sliced", split, streams))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        for v in out.values():
            v.zero_()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=stream):
        eng.schedule(R, topk=k, device=True, stream=stream.cuda_stream, out=out, **d_in)
    g.replay()
    torch.cuda.synchronize()
    same({key: v.cpu().numpy() for key, v in out.items()}, "graph")
    eng.close()


def test_headline_shape_lists(pkg):
    """64K requests x 1024 endpoints, four scorers, warmed index: the lists of sampled rows against the oracle"""
    M, R, k = 1024, 65536, 4
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
    got = eng.schedule(R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, adapter_id=ad, topk=k)
    plain = eng.schedule(R, prompt_bytes=prompts, prompt_off=off, model_seed=seeds, adapter_id=ad)
    assert_same_picks(got, plain)
    for r0 in (0, 40000, R - 512):
        n = 512
        want = o.schedule_batch(snap, prof, idx, n, prompt_bytes=prompts[off[r0]:off[r0 + n]], prompt_off=off[r0:r0 + n + 1] - off[r0],
                                model_seed=seeds[r0:r0 + n], adapter_id=ad[r0:r0 + n], request_base=r0, want_scores=True, n_threads=8)
        wm, ws = oracle_topk(want["weighted_out"], prof, k, r0)
        assert np.array_equal(got["topk_pick"][r0:r0 + n], wm), r0
        assert np.array_equal(got["topk_score"][r0:r0 + n].view(np.uint64), ws.view(np.uint64)), r0
    eng.close()


def _col_engine(pkg, scores, pick_mode, seed):
    M = len(scores)
    eng = pkg.Engine(pkg.default_config([("col0", 100.0)], max_endpoints=8, pick_mode=pick_mode, tie_seed=seed))
    eng.set_snapshot(np.zeros(M), np.zeros(M, np.int64), endpoint_cols=[np.array(scores, np.float64) / 100.0])
    return eng


def test_reference_picker_distributions_on_the_engine(pkg, golden):
    import json
    import os
    n = 10000
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "random_picker_vectors.json")) as f:
        g = json.load(f)
    for c in g["cases"]:  # random/picker_test.go:40-119: length, inclusion min(k/n, 1) +- 0.05
        eng = _col_engine(pkg, c["scores"], pkg.PICK_RANDOM, 99)
        got = eng.schedule(n, topk=c["max_num"])
        real = got["topk_pick"] >= 0
        assert (real.sum(axis=1) == c["num_pods"]).all(), c["name"]
        freq = np.bincount(got["topk_pick"][real], minlength=len(c["scores"])) / n
        assert np.abs(freq - min(c["num_pods"] / len(c["scores"]), 1.0)).max() <= g["tolerance"], (c["name"], freq)
        eng.close()
    from tests.test_topk_cpu import _successive_sampling_inclusion
    for c in golden["stochastic_pickers"]["weighted"]:  # weighted-random, k = 2: sampling without replacement
        eng = _col_engine(pkg, c["scores"], pkg.PICK_WEIGHTED_RANDOM, 1234)
        got = eng.schedule(n, topk=2)
        real = got["topk_pick"] >= 0
        freq = np.bincount(got["topk_pick"][real], minlength=len(c["scores"])) / n
        assert np.abs(freq - _successive_sampling_inclusion(c["scores"], 2)).max() <= 0.05, (c["name"], freq)
        eng.close()
    for c in golden["picker"]["cases"]:  # maxscore/picker_test.go:43-110, lowest-index ties
        eng = _col_engine(pkg, c["scores"], pkg.PICK_MAX_SCORE, 0)
        got = eng.schedule(1, topk=c["max_num"])
        want = c["want_order"] + [-1] * (c["max_num"] - len(c["want_order"]))
        assert got["topk_pick"][0].tolist() == want, c["name"]
        eng.close()


def test_invalid_arguments(pkg):
    import torch
    M, R = 64, 4
    eng = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=M))
    eng.set_snapshot(np.linspace(0, 1, M), np.zeros(M, np.int64))
    L = eng._lib
    pick, score, ties = np.zeros(R, np.int32), np.zeros(R), np.zeros(R, np.int32)
    tm, ts = np.zeros(R * 8, np.int32), np.zeros(R * 8)

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
        return L.eppscore_schedule_batch_topk(eng._h, C.byref(b), C.byref(t))

    ok = (tm.ctypes.data, ts.ctypes.data)
    assert call(3, *ok) == 0
    for k in (0, -1, 9, 100):
        assert call(k, *ok) == -1, k
    assert call(3, None, ts.ctypes.data) == -1
    assert call(3, tm.ctypes.data, None) == -1
    assert call(3, *ok, size=8) == -1
    assert L.eppscore_schedule_batch_topk(eng._h, None, None) == -1
    dev = torch.device("cuda:0")
    d = [torch.zeros(R, dtype=torch.int32, device=dev), torch.zeros(R, dtype=torch.float64, device=dev),
         torch.zeros(R, dtype=torch.int32, device=dev)]
    dm, ds = torch.zeros(R * 8, dtype=torch.int32, device=dev), torch.zeros(R * 8, dtype=torch.float64, device=dev)
    assert call(9, dm.data_ptr(), ds.data_ptr(), location=1, arrays=d) == -1
    assert call(8, None, ds.data_ptr(), location=1, arrays=d) == -1
    assert call(8, dm.data_ptr(), ds.data_ptr(), location=1, arrays=d) == 0
    torch.cuda.synchronize()
    assert dm.cpu().numpy()[:R * 8].reshape(R, 8)[:, 0].tolist() == d[0].cpu().numpy().tolist()
    eng.close()
