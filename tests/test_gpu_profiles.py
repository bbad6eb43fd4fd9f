"""Several scheduler profiles on one engine (eppscore_add_profile, eppscore_set_profile_endpoints,
eppscore_schedule_batch_profiles, eppscore_commit_picks_profiles) on the GPU, bit-exact against the CPU oracle: every run equals
oracle_py.schedule_batch with that profile (tie seed tie_seed ^ p * 0x9E3779B97F4A7C15) and mask = subset ∧ run mask, and
multi-pick commits equal Index.add calls in reference order (per request: primary pick, then the prefill pick)."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

pytestmark = pytest.mark.gpu

GOLDEN = 0x9E3779B97F4A7C15
HEADLINE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
PREFILL = [("kv", 1), ("prefix", 2)]
QUEUE_RUNNING = [("queue", 1), ("running", 1.5), ("prefix", 2)]
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
    mw = max((M + 31) // 32, 1)
    out = np.zeros(mw, np.uint32)
    for m in members:
        out[m >> 5] |= np.uint32(1 << (m & 31))
    return out


def random_masks(R, M, rng, density=0.6):
    mw = (M + 31) // 32
    b = np.zeros((R, mw * 32), bool)
    b[:, :M] = rng.random((R, M)) < density
    return (b.reshape(R, mw, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


def oracle_run(pkg, snap, idx, R, scorers, tie_mode, seed, pick_mode, subset, run_mask, M, kw, latency=None, filters=()):
    prof = o.make_profile([(pkg.SCORER[k], w) for k, w in scorers], tie_mode=tie_mode, tie_seed=seed, pick_mode=pick_mode,
                          latency=latency, filters=filters)
    mask = None
    if subset is not None or run_mask is not None:
        mw = (M + 31) // 32
        mask = np.full((R, mw), 0xFFFFFFFF, np.uint32)
        if subset is not None:
            mask &= subset[None, :mw]
        if run_mask is not None:
            mask &= run_mask
    return o.schedule_batch(snap, prof, idx, R, cand_mask=mask, n_threads=8, **kw)


def assert_run(got, want, what):
    assert np.array_equal(got["pick"], want["pick"]), what
    assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what
    assert np.array_equal(got["tie_count"], want["tie_count"]), what


def build_world(pkg, M, seed, lru=31250, **cfg):
    """engine + oracle sharing a snapshot and an index warmed so that the test batch has: requests whose prefix is cached on a
    few endpoints, all odd (ProbeRec-resolved: new tails), requests whose prefix is cached on more endpoints than the sparse
    kernel's exception table holds (deferred), and requests without any match"""
    cfg.setdefault("max_endpoints", M)
    eng = pkg.Engine(pkg.default_config(HEADLINE, prefix_capacity=1 << 16, lru_capacity_default=lru, **cfg))
    sd = synth_snapshot(M, seed=seed)
    snap, idx = o.SnapshotData(**sd), o.Index(lru)
    rng = np.random.Generator(np.random.PCG64(seed))
    pa, offa, ga = synth_prompts(240, prompt_len=1024, groups=40, shared=768, seed=seed, prefix_seed=100)
    pb, offb, _ = synth_prompts(120, prompt_len=1024, groups=2, shared=768, seed=seed + 1, prefix_seed=200)
    pick_a = np.where(ga < 20, 2 * ((ga * 7 + np.arange(240)) % (M // 2)) + 1, rng.integers(0, M, 240)).astype(np.int32)
    pick_b = rng.permutation(M)[:120].astype(np.int32) if M >= 120 else rng.integers(0, M, 120).astype(np.int32)
    ms = eng.model_seed("profiles")
    for prompts, off, pick in ((pa, offa, pick_a), (pb, offb, pick_b)):
        R = len(off) - 1
        seeds = np.full(R, ms, np.uint64)
        h, n = eng.hash_prompts(prompts, off, seeds)
        idx.commit(pick, h, n)
        eng.commit_picks(pick, h, n)
    # the test batch: new tails on both prefix pools, and unmatched prompts
    qa, _, _ = synth_prompts(240, prompt_len=1024, groups=40, shared=768, seed=seed + 7, prefix_seed=100)
    qb, _, _ = synth_prompts(120, prompt_len=1024, groups=2, shared=768, seed=seed + 8, prefix_seed=200)
    qc, _, _ = synth_prompts(64, prompt_len=1024, groups=4, shared=768, seed=seed + 9, prefix_seed=300)
    prompts = np.concatenate([qa, qb, qc])
    R = 424
    kw = dict(prompt_bytes=prompts, prompt_off=np.arange(R + 1, dtype=np.int64) * 1024, model_seed=np.full(R, ms, np.uint64),
              adapter_id=zipf_adapters(R, seed=seed))
    eng.set_snapshot(**sd)
    return eng, snap, idx, sd, kw, R


@pytest.mark.parametrize("M", [600, 1024])
@pytest.mark.parametrize("tie_mode", [0, 1])
def test_profiles_match_oracle(pkg, M, tie_mode):
    seed = 0x5EED0000 + M * 3 + tie_mode
    eng, snap, idx, sd, kw, R = build_world(pkg, M, M + tie_mode, tie_mode=tie_mode, tie_seed=seed)
    rng = np.random.Generator(np.random.PCG64(M))
    evens, odds = bits(M, range(0, M, 2)), bits(M, range(1, M, 2))
    q = sd["queue"]
    low_q = [m for m in range(M) if q[m] <= np.median(q)]  # member min/max differs from the all-endpoint one
    profiles = [  # (scorers, pick_mode, subset)
        (HEADLINE, 0, None),
        (PREFILL, 0, odds),
        (QUEUE_RUNNING, 1, bits(M, low_q)),
        ([("kv", 1), ("lora", 2)], 2, bits(M, [M // 3])),
    ]
    for p in range(1, len(profiles)):
        assert eng.add_profile(profiles[p][0], pick_mode=profiles[p][1]) == p
    # profile 0 with the decode half: subset through every profile
    profiles[0] = (HEADLINE, 0, evens)
    for p, (_, _, sub) in enumerate(profiles):
        eng.set_profile_endpoints(p, sub)
    eng.set_snapshot(**sd)
    run_mask = random_masks(R, M, rng)
    runs_spec = [(0, None), (1, None), (2, run_mask), (3, None)]
    batch, got = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m) for p, m in runs_spec], **kw)
    for (p, m), g in zip(runs_spec, got):
        sc_, pm, sub = profiles[p]
        want = oracle_run(pkg, snap, idx, R, sc_, tie_mode, seed_of(seed, p), pm, sub, m, M, kw)
        assert_run(g, want, (M, tie_mode, p))
        assert np.array_equal(batch["total_blocks"], want["total_blocks"])
    # each run alone gives the same outputs; one profile-0 run equals eppscore_schedule_batch
    single = eng.schedule(R, **kw)
    assert_run(single, got[0], "profile 0 alone")
    for (p, m), g in zip(runs_spec, got):
        _, alone = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m)], **kw)
        assert_run(alone[0], g, ("alone", p))
    # the same through the chunked host path and the device path
    eng.set_debug(3, 96)
    _, chunked = eng.schedule_profiles(R, [dict(profile=p, cand_mask=m) for p, m in runs_spec], **kw)
    eng.set_debug(3, 8192)
    for g, c in zip(got, chunked):
        assert_run(c, g, "chunked")
    import torch
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}
    druns = []
    for p, m in runs_spec:
        druns.append(dict(profile=p, cand_mask=None if m is None else torch.from_numpy(m).cuda(),
                          pick=torch.empty(R, dtype=torch.int32, device="cuda"),
                          pick_score=torch.empty(R, dtype=torch.float64, device="cuda"),
                          tie_count=torch.empty(R, dtype=torch.int32, device="cuda")))
    eng.schedule_profiles(R, druns, device=True, out=dict(total_blocks=torch.empty(R, dtype=torch.int16, device="cuda")), **dev)
    torch.cuda.synchronize()
    for g, d in zip(got, druns):
        assert_run({k: d[k].cpu().numpy() for k in ("pick", "pick_score", "tie_count")}, g, "device")
    eng.close()


def test_edges_empty_subset_nonmember_exceptions_and_deferral(pkg):
    M = 1024
    eng, snap, idx, sd, kw, R = build_world(pkg, M, 77)
    pid = eng.add_profile(PREFILL)
    evens = bits(M, range(0, M, 2))
    eng.set_profile_endpoints(pid, evens)
    eng.set_snapshot(**sd)
    before = eng.stats().probe_resolved
    single = eng.schedule(R, **kw)
    resolved_single = eng.stats().probe_resolved - before
    assert resolved_single > 0  # the ProbeRec path is exercised
    before = eng.stats().probe_resolved
    l0 = eng.stats().kernel_launches
    _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], **kw)
    l1 = eng.stats().kernel_launches
    assert eng.stats().probe_resolved - before == resolved_single  # one hash stage, the same probe
    assert_run(got[0], single, "profile 0")
    want = oracle_run(pkg, snap, idx, R, PREFILL, 0, seed_of(0, pid), 0, evens, None, M, kw)
    assert_run(got[1], want, "evens")
    # the first 240 requests with a group < 20 prefix are cached on odd endpoints only: all their exceptions are non-members
    _, alone = eng.schedule_profiles(R, [dict(profile=pid)], **kw)
    l2 = eng.stats().kernel_launches
    s0 = eng.stats().kernel_launches
    eng.schedule(R, **kw)
    s1 = eng.stats().kernel_launches
    assert l1 - l0 < (l2 - l1) + (s1 - s0)  # the hash stage ran once for both runs
    # empty subset: pick -1 everywhere; one endpoint: that endpoint everywhere
    for members, expect in (([], -1), ([5], 5)):
        eng.set_profile_endpoints(pid, bits(M, members))
        eng.set_snapshot(**sd)
        _, got = eng.schedule_profiles(R, [dict(profile=pid)], **kw)
        assert np.all(got[0]["pick"] == expect), members
        want = oracle_run(pkg, snap, idx, R, PREFILL, 0, seed_of(0, pid), 0, bits(M, members), None, M, kw)
        assert_run(got[0], want, members)
    # back to every endpoint
    eng.set_profile_endpoints(pid, None)
    eng.set_snapshot(**sd)
    _, got = eng.schedule_profiles(R, [dict(profile=pid)], **kw)
    assert_run(got[0], oracle_run(pkg, snap, idx, R, PREFILL, 0, seed_of(0, pid), 0, None, None, M, kw), "all")
    eng.close()


def test_profile0_subset_through_schedule_batch_and_topk(pkg):
    M = 600
    eng, snap, idx, sd, kw, R = build_world(pkg, M, 5)
    sub = bits(M, range(0, M, 3))
    eng.set_profile_endpoints(0, sub)
    eng.set_snapshot(**sd)
    want = oracle_run(pkg, snap, idx, R, HEADLINE, 0, 0, 0, sub, None, M, kw)
    assert_run(eng.schedule(R, **kw), want, "schedule_batch")
    for kk in ("topk", "topk_wide"):
        got = eng.schedule(R, **{kk: 4}, **kw)
        assert_run(got, want, kk)
        assert np.array_equal(got["topk_pick"][:, 0], want["pick"])
        cand = got["topk_pick"][got["topk_pick"] >= 0]
        assert np.all(cand % 3 == 0), kk  # only members in the lists
    rm = random_masks(R, M, np.random.Generator(np.random.PCG64(1)))
    want = oracle_run(pkg, snap, idx, R, HEADLINE, 0, 0, 0, sub, rm, M, kw)
    assert_run(eng.schedule(R, cand_mask=rm, **kw), want, "masked")
    eng.close()


def test_latency_profile_behind_device_filters(pkg):
    M = 256
    eng, snap, idx, sd, kw, R = build_world(pkg, M, 9)
    lp = pkg.latency_params(**LAT_COEF)
    eng.set_latency_params(lp)
    filters = [(1, (0.5, 0.0, 5000.0)), (2, (0.01, 0, 0))]
    pid = eng.add_profile([("latency", 1), ("kv", 0.5)], filters=filters)
    sub = bits(M, range(M // 2, M))
    eng.set_profile_endpoints(pid, sub)
    eng.set_snapshot(**sd)
    slo = dict(ttft_slo=np.full(R, 900.0), tpot_slo=np.full(R, 40.0),
               input_tokens=np.random.Generator(np.random.PCG64(4)).integers(0, 6000, R).astype(np.int32))
    _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], **kw, **slo)
    olp = o.make_latency_params(**LAT_COEF)
    want = oracle_run(pkg, snap, idx, R, [("latency", 1), ("kv", 0.5)], 0, seed_of(0, pid), 0, sub, None, M, dict(kw, **slo),
                      latency=olp, filters=filters)
    assert_run(got[1], want, "latency")
    assert np.all(got[1]["pick"][got[1]["pick"] >= 0] >= M // 2)
    eng.close()


def test_graph_replay(pkg):
    import torch
    M = 1024
    eng, snap, idx, sd, kw, R = build_world(pkg, M, 21)
    pid = eng.add_profile(PREFILL)
    eng.set_profile_endpoints(0, bits(M, range(0, M, 2)))
    eng.set_profile_endpoints(pid, bits(M, range(1, M, 2)))
    eng.set_snapshot(**sd)
    _, ref = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], **kw)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}
    runs = [dict(profile=p, pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"),
                 pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.zeros(R, dtype=torch.int32, device="cuda")) for p in (0, pid)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)  # sizes the scratch outside the capture
    s.synchronize()
    for r in runs:
        r["pick"].fill_(-7)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)
    g.replay()
    torch.cuda.synchronize()
    for r, w in zip(runs, ref):
        assert_run({k: r[k].cpu().numpy() for k in ("pick", "pick_score", "tie_count")}, w, "graph")
    eng.close()


def test_commit_picks_profiles_closed_loop(pkg):
    """Five rounds of schedule (decode, prefill) -> one two-pick device commit with small LRUs: every LRU and
    len(hashToPods) equal the oracle's Index.add calls in reference order, which differ from primary-first-for-all order."""
    import torch
    M, R, lru = 64, 256, 48
    eng = pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=M, prefix_capacity=1 << 14, lru_capacity_default=lru))
    sd = synth_snapshot(M, seed=3)
    eng.set_snapshot(**sd)
    pid = eng.add_profile(PREFILL)
    eng.set_profile_endpoints(0, bits(M, range(0, M, 2)))
    eng.set_profile_endpoints(pid, bits(M, range(1, M, 2)))
    eng.set_snapshot(**sd)
    idx, other = o.Index(lru), o.Index(lru)
    ms = eng.model_seed("loop")
    differs = False
    for rnd in range(5):
        prompts, off, _ = synth_prompts(R, prompt_len=512, groups=6, shared=256, seed=40 + rnd, prefix_seed=9)
        kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, ms, np.uint64))
        batch, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], want_hashes=True, **kw)
        dec, pre = got[0]["pick"].copy(), got[1]["pick"].copy()
        # prefill picks repeat later decode picks: the same endpoint appears in both lists across requests
        pre[1::4] = np.roll(dec, -1)[1::4]
        h, n = batch["hashes_out"], batch["total_blocks"]
        for r in range(R):  # reference order: per request, primary then prefill
            for p in (dec[r], pre[r]):
                if p >= 0:
                    idx.add(h[r, :n[r]], int(p))
        other.commit(dec, h, n)  # primary-first for all requests
        other.commit(pre, h, n)
        differs = differs or any(idx.lru_keys(m) != other.lru_keys(m) for m in range(M))
        eng.commit_picks_profiles([torch.from_numpy(dec).cuda(), torch.from_numpy(pre).cuda()], torch.from_numpy(h).cuda(),
                                  torch.from_numpy(n.astype(np.int16)).cuda(), device=True, touch_bound=int(n.sum()) * 2)
        torch.cuda.synchronize()
        for m in range(M):
            assert eng.prefix_lru_keys(m) == idx.lru_keys(m), (rnd, m)
        assert eng.stats().prefix_live_hashes == idx.num_hashes(), rnd
    assert differs  # the order is really exercised


def test_commit_picks_profiles_one_pick_equals_commit_picks(pkg):
    M, R = 128, 300
    rng = np.random.Generator(np.random.PCG64(8))
    engs = [pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=M, lru_capacity_default=40)) for _ in range(2)]
    for rnd in range(3):
        pick = rng.integers(-1, M, R).astype(np.int32)
        n = rng.integers(0, 30, R).astype(np.uint16)
        h = rng.integers(1, 2 ** 63, (R, 32), dtype=np.uint64) % np.uint64(500 + rnd)
        engs[0].commit_picks(pick, h, n)
        engs[1].commit_picks_profiles([pick], h, n)
    for m in range(M):
        assert engs[0].prefix_lru_keys(m) == engs[1].prefix_lru_keys(m)
    assert engs[0].stats().prefix_live_hashes == engs[1].stats().prefix_live_hashes
    for e in engs:
        e.close()


def test_invalid_arguments(pkg):
    M = 64
    eng = pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=M))
    eng.set_snapshot(np.zeros(M), np.zeros(M, np.int64))
    with pytest.raises(pkg.EppscoreError) as ex:
        eng.add_profile([(7, 1.0)])
    assert ex.value.code == ERR_INVALID
    with pytest.raises(pkg.EppscoreError):
        eng.add_profile([("queue", 1)], filters=[(1, (0.5, 0.0, 1.0))])  # filters need the latency scorer
    ids = [eng.add_profile(PREFILL) for _ in range(3)]
    assert ids == [1, 2, 3]
    with pytest.raises(pkg.EppscoreError) as ex:
        eng.add_profile(PREFILL)
    assert ex.value.code == ERR_CAPACITY
    with pytest.raises(pkg.EppscoreError):
        eng.set_profile_endpoints(4, None)
    with pytest.raises(pkg.EppscoreError):  # a profile in two runs
        eng.schedule_profiles(4, [dict(profile=1), dict(profile=1)])
    with pytest.raises(pkg.EppscoreError):  # unknown profile
        eng.schedule_profiles(4, [dict(profile=5)])
    with pytest.raises(pkg.EppscoreError):  # no runs
        eng.schedule_profiles(4, [])
    with pytest.raises(pkg.EppscoreError):  # n_picks out of range
        eng.commit_picks_profiles([np.zeros(4, np.int32)] * 5, np.zeros((4, 2), np.uint64), np.zeros(4, np.uint16))
    eng.close()
