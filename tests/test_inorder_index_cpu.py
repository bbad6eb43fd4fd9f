"""The sequential reference of eppscore_schedule_batch_inorder_index (tests/inorder_index_reference.py) on the CPU oracle: a
request follows the fresh prefix an earlier request of the same batch was sent with, and a window of requests sharing new
prefixes stays on a few endpoints per prefix where the batch-wide index spreads it over most of the fleet."""
import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.inorder_index_reference import schedule_inorder_index
from tests.inorder_reference import schedule_inorder

QUEUE, KV, PREFIX, TOKEN_LOAD = 0, 1, 2, 6


def setup_module():
    o.build()
    I.build()


def _pack(prompts):
    off = np.concatenate([[0], np.cumsum([len(p) for p in prompts])]).astype(np.int64)
    return np.concatenate(prompts), off


def test_second_request_follows_first_requests_fresh_prefix():
    rng = np.random.default_rng(3)
    M = 8
    snap = dict(kv_usage=np.linspace(0.9, 0.1, M), queue=np.zeros(M, np.int64))  # endpoint 7 is the least loaded
    prof = o.make_profile([(KV, 1.0), (PREFIX, 3.0)])
    shared = rng.integers(97, 123, 512, dtype=np.uint8)
    prompts = [np.concatenate([shared, rng.integers(97, 123, 128, dtype=np.uint8)]) for _ in range(2)]
    pb, off = _pack(prompts)
    seed = np.zeros(2, np.uint64)
    idx = o.Index()
    got, _ = schedule_inorder_index(snap, prof, idx, 2, prompt_bytes=pb, prompt_off=off, model_seed=seed)
    # request 0 sees no match anywhere and goes to the least loaded endpoint; request 1 sees its 8 shared blocks there
    assert got["pick"][0] == 7 and got["pick_match"][0] == 0
    assert got["pick"][1] == 7 and got["pick_match"][1] == 8
    assert got["total_blocks"].tolist() == [10, 10]
    assert idx.lru_len(7) == 12 and idx.lru_len(6) == -1  # 8 shared + 2 + 2 unique blocks, all on endpoint 7
    # the batch-wide index: request 1 does not see request 0's blocks, so it is scored as request 0 was
    frozen, _ = schedule_inorder(snap, prof, o.Index(), 2, prompt_bytes=pb, prompt_off=off, model_seed=seed)
    assert frozen["pick_score"][1] == frozen["pick_score"][0]
    assert got["pick_score"][1] > got["pick_score"][0]


def test_shared_prefix_window_stays_on_few_endpoints():
    """64 endpoints, 512 requests of 2 KB: one of 8 fresh 1 KB shared prefixes plus a unique tail; queue 2, kv 2, prefix 3,
    token-load 3 (threshold 8192) with 600 tokens per request."""
    rng = np.random.default_rng(0)
    M, R, G = 64, 512, 8
    prof = o.make_profile([(QUEUE, 2.0), (KV, 2.0), (PREFIX, 3.0), (TOKEN_LOAD, 3.0)], token_load_threshold=8192.0)
    snap = dict(kv_usage=rng.random(M), queue=rng.poisson(8, M).astype(np.int64))
    groups = [rng.integers(97, 123, 1024, dtype=np.uint8) for _ in range(G)]
    gid = rng.integers(0, G, R)
    pb, off = _pack([np.concatenate([groups[g], rng.integers(97, 123, 1024, dtype=np.uint8)]) for g in gid])
    kw = dict(prompt_bytes=pb, prompt_off=off, model_seed=np.zeros(R, np.uint64))
    tokens = np.full(R, 600, np.int64)
    wide, _ = schedule_inorder(snap, prof, o.Index(), R, tokens, **kw)
    ordered, _ = schedule_inorder_index(snap, prof, o.Index(), R, tokens, **kw)

    def spread(pick):
        return np.mean([len(set(pick[gid == g].tolist())) for g in range(G)])

    assert spread(wide["pick"]) == 40.375
    assert spread(ordered["pick"]) == 6.25
    assert np.bincount(wide["pick"], minlength=M).max() == 13
    assert np.bincount(ordered["pick"], minlength=M).max() == 29
    assert int((wide["pick"] != ordered["pick"]).sum()) == 494
