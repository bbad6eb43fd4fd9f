"""The sequential reference of eppscore_schedule_batch_inorder_profiles (tests/inorder_profiles_reference.py) on the CPU oracle:
a prefill run follows the fresh prefix an earlier request left on the prefill pool, a failed primary records nothing, two runs
on one endpoint count and Add twice, a run_mask skips a run, and a P/D window of requests sharing new prefixes stays on a few
prefill endpoints per prefix where the batch-wide call spreads it."""
import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.inorder_profiles_reference import schedule_inorder_profiles

QUEUE, KV, PREFIX, LORA, TOKEN_LOAD = 0, 1, 2, 3, 6


def setup_module():
    o.build()
    I.build()


def _pack(prompts):
    off = np.concatenate([[0], np.cumsum([len(p) for p in prompts])]).astype(np.int64)
    return np.concatenate(prompts), off


def _bits(M, members):
    out = np.zeros(max((M + 31) // 32, 1), np.uint32)
    for m in members:
        out[m >> 5] |= np.uint32(1 << (m & 31))
    return out


def _pd(M, decode_scorers=None, prefill_scorers=None):
    half = M // 2
    return [dict(profile=0, scorers=decode_scorers or [(KV, 1.0), (PREFIX, 3.0)], subset=_bits(M, range(half))),
            dict(profile=1, scorers=prefill_scorers or [(KV, 1.0), (PREFIX, 3.0)], subset=_bits(M, range(half, M)))]


def test_prefill_pick_follows_earlier_requests_fresh_prefix():
    rng = np.random.default_rng(3)
    M = 8
    snap = dict(kv_usage=np.linspace(0.9, 0.1, M), queue=np.zeros(M, np.int64))  # endpoints 3 and 7 are the least loaded
    shared = rng.integers(97, 123, 512, dtype=np.uint8)
    pb, off = _pack([np.concatenate([shared, rng.integers(97, 123, 128, dtype=np.uint8)]) for _ in range(2)])
    kw = dict(prompt_bytes=pb, prompt_off=off, model_seed=np.zeros(2, np.uint64))
    idx = o.Index()
    b, runs, _ = schedule_inorder_profiles(snap, _pd(M), idx, 2, ordered_index=True, prefill_run=1, **kw)
    assert runs[0]["pick"].tolist() == [3, 3] and runs[1]["pick"].tolist() == [7, 7]
    assert runs[1]["pick_match"].tolist() == [0, 8] and runs[0]["pick_match"].tolist() == [0, 8]
    assert idx.lru_len(3) == 12 and idx.lru_len(7) == 12  # both picks got both requests' blocks
    # batch-wide: request 1 does not see request 0's blocks
    frozen, fr, _ = schedule_inorder_profiles(snap, _pd(M), o.Index(), 2, prefill_run=1, **kw)
    assert fr[1]["pick_score"][1] == fr[1]["pick_score"][0]
    assert runs[1]["pick_score"][1] > runs[1]["pick_score"][0]


def test_primary_without_candidate_changes_nothing():
    M = 8
    snap = dict(kv_usage=np.linspace(0.9, 0.1, M), queue=np.zeros(M, np.int64))
    hashes = np.arange(1, 5, dtype=np.uint64)[None, :].repeat(2, 0)
    n = np.full(2, 4, np.uint16)
    runs = _pd(M)
    runs[0]["cand_mask"] = np.zeros((2, 1), np.uint32)  # the decode run has no candidate
    idx, tr = o.Index(), I.Tracker()
    _, out, tr = schedule_inorder_profiles(snap, runs, idx, 2, np.array([100, 100]), tr, ordered_index=True, prefill_run=1,
                                           hashes_in=hashes, n_hashes_in=n)
    assert out[0]["pick"].tolist() == [-1, -1] and out[1]["pick"].tolist() == [7, 7]
    assert out[1]["pick_match"].tolist() == [0, 0]
    req, tok = tr.get(M)
    assert req.sum() == 0 and tok.sum() == 0 and idx.num_hashes() == 0


def test_both_runs_on_one_endpoint_count_and_add_twice():
    M = 4
    snap = dict(kv_usage=np.array([0.9, 0.1, 0.8, 0.7]), queue=np.zeros(M, np.int64))
    runs = [dict(profile=0, scorers=[(KV, 1.0)]), dict(profile=1, scorers=[(KV, 2.0), (PREFIX, 1.0)])]
    hashes = np.array([[11, 12, 13]], np.uint64)
    idx, tr = o.Index(), I.Tracker()
    _, out, tr = schedule_inorder_profiles(snap, runs, idx, 1, np.array([50]), tr, ordered_index=True, prefill_run=1,
                                           hashes_in=hashes, n_hashes_in=np.array([3], np.uint16))
    assert out[0]["pick"][0] == 1 and out[1]["pick"][0] == 1
    req, tok = tr.get(M)
    assert req[1] == 2 and tok[1] == 100
    assert idx.lru_len(1) == 3 and idx.get(11) == {1}


def test_run_mask_skips_prefill():
    M = 8
    snap = dict(kv_usage=np.linspace(0.9, 0.1, M), queue=np.zeros(M, np.int64))
    hashes = np.arange(1, 4, dtype=np.uint64)[None, :].repeat(3, 0)
    idx, tr = o.Index(), I.Tracker()
    _, out, tr = schedule_inorder_profiles(snap, _pd(M), idx, 3, np.array([7, 7, 7]), tr, ordered_index=True, prefill_run=1,
                                           run_mask=np.array([3, 1, 3], np.uint8), hashes_in=hashes,
                                           n_hashes_in=np.full(3, 3, np.uint16))
    assert out[1]["pick"].tolist() == [7, -1, 7] and out[1]["tie_count"][1] == 0
    assert out[1]["pick_match"].tolist() == [0, 0, 3]
    req, _ = tr.get(M)
    assert req[3] == 3 and req[7] == 2


def test_pd_shared_prefix_window_stays_on_few_prefill_endpoints():
    """64 endpoints (decode 0-31: queue 2, kv 2, prefix 3, token-load 3; prefill 32-63: kv 2, prefix 3, token-load 3), 512
    requests of 2 KB: one of 8 fresh 1 KB shared prefixes plus a unique tail, 600 tokens each."""
    rng = np.random.default_rng(0)
    M, R, G = 64, 512, 8
    snap = dict(kv_usage=rng.random(M), queue=rng.poisson(8, M).astype(np.int64))
    runs = _pd(M, [(QUEUE, 2.0), (KV, 2.0), (PREFIX, 3.0), (TOKEN_LOAD, 3.0)], [(KV, 2.0), (PREFIX, 3.0), (TOKEN_LOAD, 3.0)])
    groups = [rng.integers(97, 123, 1024, dtype=np.uint8) for _ in range(G)]
    gid = rng.integers(0, G, R)
    pb, off = _pack([np.concatenate([groups[g], rng.integers(97, 123, 1024, dtype=np.uint8)]) for g in gid])
    kw = dict(prompt_bytes=pb, prompt_off=off, model_seed=np.zeros(R, np.uint64), prefill_run=1, token_load_threshold=8192.0)
    tokens = np.full(R, 600, np.int64)
    _, wide, _ = schedule_inorder_profiles(snap, runs, o.Index(), R, tokens, **kw)
    _, ordered, _ = schedule_inorder_profiles(snap, runs, o.Index(), R, tokens, ordered_index=True, **kw)

    def spread(pick):
        return np.mean([len(set(pick[gid == g].tolist())) for g in range(G)])

    assert spread(ordered[1]["pick"]) < spread(wide[1]["pick"]) / 2
    assert spread(ordered[1]["pick"]) <= 8
