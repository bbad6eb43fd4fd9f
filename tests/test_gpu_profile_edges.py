"""Scheduler profiles at the edges where per-profile state is kept apart from shared state, bit-exact against the CPU oracle
(oracle_py.schedule_batch with the profile's scorers and picker, tie seed tie_seed ^ p * 0x9E3779B97F4A7C15 and mask =
subset ∧ run mask): a subset that drops the zero-match arg-max, deferred requests on a subset profile, the member min/max of the
masked kernels, sliced device batches, producer mutations feeding profiles >= 1, and the subset across a captured
set_snapshot.  The worlds come from tests/profile_worlds.py; tests/test_profile_worlds_cpu.py checks that they reach these
edges.  Every case runs in both tie modes; cases on the sparse path also run on the generic kernels (set_debug(1, 1))."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import profile_worlds as W
from tests import running_oracle as Q

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
TIE_MODES = [0, 1]


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _world(build, *args):
    w = build(*args)
    return w, w.index()


@pytest.fixture(scope="module")
def argmax_world():
    return _world(W.world_argmax)


@pytest.fixture(scope="module")
def deferral_world():
    return _world(W.world_deferral)


@pytest.fixture(scope="module")
def minmax_worlds():
    return {v: _world(W.world_minmax, v) for v in W.MINMAX_VARIANTS}


@pytest.fixture(scope="module")
def sliced_world():
    return _world(W.world_sliced)


@pytest.fixture(scope="module")
def producer_world():
    return _world(W.world_producers)


def engine(pkg, w, scorers, tie_mode, tie_seed, **cfg):
    """an engine with the world's index history and snapshot; profile 0 = `scorers`"""
    eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=w.max_endpoints, prefix_capacity=1 << 16, tie_mode=tie_mode,
                                        tie_seed=tie_seed, token_load_threshold=W.TOKEN_THR, **cfg))
    for pick, h, n in w.warm:
        eng.commit_picks(pick, h, n)
    eng.set_snapshot(**w.sd)
    return eng


def assert_run(got, want, what):
    assert np.array_equal(got["pick"], want["pick"]), what
    assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what
    assert np.array_equal(got["tie_count"], want["tie_count"]), what


def host(x):
    return {k: x[k].cpu().numpy() for k in ("pick", "pick_score", "tie_count")}


def device_runs(R, profiles):
    import torch
    return [dict(profile=p, pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"),
                 pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.zeros(R, dtype=torch.int32, device="cuda")) for p in profiles]


def to_device(kw):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_mode", TIE_MODES)
def test_subset_drops_the_zero_match_argmax(pkg, argmax_world, tie_mode):
    """rows whose all-endpoint arg-max (and its whole tie set) are non-members, a member maximum tied with a non-member, a
    member maximum attained by three members, and member exceptions landing exactly on the member maximum"""
    w, idx = argmax_world
    seed = 0xA5A5 + tie_mode
    eng = engine(pkg, w, W.ARGMAX_SCORERS, tie_mode, seed)
    pid = eng.add_profile(W.ARGMAX_SCORERS)
    sub = W.bits(w.M, w.members)
    eng.set_profile_endpoints(pid, sub)
    eng.set_snapshot(**w.sd)
    want0 = W.oracle_run(w, W.ARGMAX_SCORERS, tie_mode, seed, idx=idx)
    want1 = W.oracle_run(w, W.ARGMAX_SCORERS, tie_mode, W.seed_of(seed, pid), subset=sub, idx=idx)
    for generic in (0, 1):
        eng.set_debug(1, generic)
        _, got = eng.schedule_profiles(w.R, [dict(profile=0), dict(profile=pid)], **w.kw)
        assert_run(got[0], want0, ("all endpoints", generic))
        assert_run(got[1], want1, ("members", generic))
        assert np.isin(got[1]["pick"], w.members).all()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_mode", TIE_MODES)
def test_deferral_on_a_subset_profile(pkg, deferral_world, tie_mode):
    """one batch with requests deferred with and without members among their endpoints, deferred with few members, matched
    through bitset-row slots and inline sets, and resolved by the hash kernel; profile 0 without a subset shares the hash
    stage and its probe records with the subset profile"""
    w, idx = deferral_world
    seed = 0xDEF0 + tie_mode
    eng = engine(pkg, w, W.HEADLINE, tie_mode, seed)
    pid = eng.add_profile(W.PREFILL)
    sub = W.bits(w.M, w.members)
    eng.set_profile_endpoints(pid, sub)
    eng.set_snapshot(**w.sd)
    want0 = W.oracle_run(w, W.HEADLINE, tie_mode, seed, idx=idx)
    want1 = W.oracle_run(w, W.PREFILL, tie_mode, W.seed_of(seed, pid), subset=sub, idx=idx)
    for generic in (0, 1):
        eng.set_debug(1, generic)
        before = eng.stats().probe_resolved
        batch, got = eng.schedule_profiles(w.R, [dict(profile=0), dict(profile=pid)], **w.kw)
        resolved = eng.stats().probe_resolved - before
        assert (resolved > 0) == (generic == 0)  # the sparse path takes the hash kernel's records; the generic kernels do not
        assert_run(got[0], want0, ("profile 0", generic))
        assert_run(got[1], want1, ("subset", generic))
        assert np.array_equal(batch["total_blocks"], want0["total_blocks"])
        assert np.isin(got[1]["pick"], w.members).all()
    eng.set_debug(1, 0)
    _, alone = eng.schedule_profiles(w.R, [dict(profile=pid)], **w.kw)
    assert_run(alone[0], want1, "subset alone")
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_mode", TIE_MODES)
@pytest.mark.parametrize("variant", W.MINMAX_VARIANTS)
def test_member_minmax(pkg, minmax_worlds, variant, tie_mode):
    """queue / running min/max over the members: a bucket table valid only because of the subset, member ranges that make
    the masked kernels scan, bases near 2^40; with a run mask, without one (the member-folded terms of the sparse path) and
    under pick modes 1 and 2; the subset written with bits at or above M, bits past max_endpoints and too few words"""
    w, idx = minmax_worlds[variant]
    seed = 0x3A3A + tie_mode
    eng = engine(pkg, w, W.QUEUE_RUNNING, tie_mode, seed)
    pick_mode = {0: 0}
    for pm in (0, 1, 2):
        pid = eng.add_profile(W.QUEUE_RUNNING, pick_mode=pm)
        pick_mode[pid] = pm
    rng = np.random.Generator(np.random.PCG64(7 + tie_mode))
    rm = W.short_run_mask(w.R, w.M, rng, (w.M + 31) // 32)
    want_all = {m is None: W.oracle_run(w, W.QUEUE_RUNNING, tie_mode, seed, run_mask=m, idx=idx) for m in (None, rm)}
    for name, words, eff in W.minmax_encodings(w):
        for p in (1, 2, 3):
            eng.set_profile_endpoints(p, words)
        eng.set_snapshot(**w.sd)
        eff_bits = W.bits(w.M, eff)
        for mask in (None, rm):
            runs = [dict(profile=p, cand_mask=mask) for p in range(4)]
            _, got = eng.schedule_profiles(w.R, runs, **w.kw)
            assert_run(got[0], want_all[mask is None], (name, "profile 0", mask is None))
            for p in (1, 2, 3):
                want = W.oracle_run(w, W.QUEUE_RUNNING, tie_mode, W.seed_of(seed, p), pick_mode[p], eff_bits, mask, idx=idx)
                assert_run(got[p], want, (name, p, mask is None))
                assert np.isin(got[p]["pick"], list(eff) + [-1]).all()
                if mask is None and p == 1:  # the sparse path: the generic kernels agree
                    eng.set_debug(1, 1)
                    _, gen = eng.schedule_profiles(w.R, [dict(profile=1)], **w.kw)
                    eng.set_debug(1, 0)
                    assert_run(gen[0], want, (name, "generic"))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
SPLITS = [(1, 1), (3, 2), (4, 3), (6, 4)]


@pytest.mark.parametrize("tie_mode", TIE_MODES)
def test_sliced_device_batches_with_profile_runs(pkg, sliced_world, tie_mode):
    """R = 12288 cut into 1, 3, 4 and 6 slices over 1..4 streams, eagerly and inside a CUDA graph: each slice writes its
    share of every run's outputs (its own scratch, its own subset rows for deferred and via-rows requests)"""
    import torch
    w, idx = sliced_world
    R, M = w.R, w.M
    seed = 0x511CE + tie_mode
    profs = W.sliced_profiles(M)
    eng = engine(pkg, w, profs[0][0], tie_mode, seed)
    for p in (1, 2, 3):
        assert eng.add_profile(profs[p][0], pick_mode=profs[p][1]) == p
    for p, (_, _, sub) in enumerate(profs):
        eng.set_profile_endpoints(p, sub)
    eng.set_snapshot(**w.sd)
    wants = [W.oracle_run(w, sc, tie_mode, W.seed_of(seed, p), pm, sub, idx=idx) for p, (sc, pm, sub) in enumerate(profs)]
    h, n = w.batch_hashes()
    dev = to_device(w.kw)
    s = torch.cuda.Stream()

    def run(split, streams, want_hashes, graph=False):
        eng.set_debug(5, split)
        eng.set_debug(6, streams)
        runs = device_runs(R, range(4))
        out = dict(total_blocks=torch.zeros(R, dtype=torch.int16, device="cuda"))
        if want_hashes:
            out["hashes_out"] = torch.zeros((R, W.MAX_BLOCKS), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        l0 = eng.stats().kernel_launches
        with torch.cuda.stream(s):
            eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, out=out, **dev)
        s.synchronize()
        launches = eng.stats().kernel_launches - l0
        if graph:  # the eager call above sized every slice's scratch
            for r in runs:
                r["pick"].fill_(-7)
            out["total_blocks"].zero_()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, out=out, **dev)
            g.replay()
            torch.cuda.synchronize()
        got = [host(r) for r in runs]
        what = (split, streams, want_hashes, graph)
        for p in range(4):
            assert_run(got[p], wants[p], what + (p,))
        assert np.array_equal(out["total_blocks"].cpu().numpy().astype(np.uint16), n), what
        if want_hashes:
            assert np.array_equal(out["hashes_out"].cpu().numpy().view(np.uint64), h), what
        return got, launches

    for want_hashes in (False, True):
        base, prev = None, -1
        for split, streams in SPLITS:
            got, launches = run(split, streams, want_hashes)
            assert launches > prev, (split, streams, launches)  # every slice launches its own kernels
            prev = launches
            if base is None:
                base = got
            for g_, b_ in zip(got, base):
                assert_run(g_, b_, ("against K = 1", split, streams))
    run(6, 4, False, graph=True)
    run(4, 3, True, graph=True)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_mode", TIE_MODES)
def test_producers_feed_profiles_beyond_zero(pkg, producer_world, tie_mode):
    """the in-flight counters feed a token-load profile and the running-request queues a latency profile, both >= 1 and
    with a subset: every mutation, on the host or the device, prepares those profiles again; profile 0 reads neither"""
    import torch
    w, idx = producer_world
    M, R = w.M, w.R
    seed = 0x9A0D + tie_mode
    eng = engine(pkg, w, W.HEADLINE, tie_mode, seed)
    tracker, queues = I.Tracker(), Q.Queues(M)
    rng = np.random.Generator(np.random.PCG64(60 + tie_mode))
    olat = o.make_latency_params(**W.LAT_COEF)
    want0 = W.oracle_run(w, W.HEADLINE, tie_mode, seed, idx=idx)

    def snap(tokens=None):
        mn, cnt = queues.get(M)
        return w.snap(inflight_tokens=tracker.get(M)[1] if tokens is None else tokens, min_tpot_slo=Q.canonical(mn),
                      dispatched=cnt)

    def want(p, tokens=None):
        sn = snap(tokens)
        if p == 1:
            return W.oracle_run(w, W.TOKEN_PROFILE, tie_mode, W.seed_of(seed, 1), subset=subsets[1], snap=sn, idx=idx)
        return W.oracle_run(w, W.LATENCY_PROFILE, tie_mode, W.seed_of(seed, 2), subset=subsets[2], snap=sn, latency=olat,
                            idx=idx)

    def check(what, tokens=None, profiles=(0, 1, 2)):
        _, got = eng.schedule_profiles(R, [dict(profile=p) for p in profiles], **w.kw)
        for p, g in zip(profiles, got):
            assert_run(g, want0 if p == 0 else want(p, tokens), (what, p))
        return got

    # the counters move before the token-load profile exists: add_profile prepares it with the current counters
    ep = rng.integers(-1, M, 400).astype(np.int32)
    tok = rng.integers(0, 4000, 400).astype(np.int64)
    eng.inflight_add(ep, tok)
    tracker.add(ep, tok)
    subsets = {1: None, 2: None}
    assert eng.add_profile(W.TOKEN_PROFILE) == 1
    check("add_profile after the counters moved", profiles=(0, 1))
    # the first latency profile: refused until the next set_snapshot prepares the latency fold-in
    eng.set_latency_params(pkg.latency_params(**W.LAT_COEF))
    assert eng.add_profile(W.LATENCY_PROFILE) == 2
    with pytest.raises(pkg.EppscoreError) as ex:
        eng.schedule_profiles(R, [dict(profile=0), dict(profile=2)], **w.kw)
    assert ex.value.code == ERR_INVALID
    eng.set_snapshot(**w.sd)
    check("latency profile after set_snapshot")
    subsets = {1: w.token_subset, 2: w.latency_subset}
    eng.set_profile_endpoints(1, subsets[1])
    eng.set_profile_endpoints(2, subsets[2])
    eng.set_snapshot(**w.sd)
    check("subsets")

    keys = iter(range(1, 1 << 30))
    added = []
    for step in range(9):
        n_ = 300
        e_ = rng.integers(-1, M, n_).astype(np.int32)
        t_ = rng.integers(0, 5000, n_).astype(np.int64)
        on_dev = step % 2 == 1
        if step in (0, 1):
            eng.inflight_add(torch.from_numpy(e_).cuda() if on_dev else e_, torch.from_numpy(t_).cuda() if on_dev else t_,
                             device=on_dev)
            tracker.add(e_, t_)
            added.append((e_, t_))
            what = "inflight_add"
        elif step in (2, 3):
            e0, t0 = added[step - 2]
            eng.inflight_release(torch.from_numpy(e0[:150]).cuda() if on_dev else e0[:150],
                                 torch.from_numpy(t0[:150]).cuda() if on_dev else t0[:150], device=on_dev)
            tracker.release(e0[:150], t0[:150])
            what = "inflight_release"
        elif step == 4:
            m = int(np.argmax(tracker.get(M)[1]))  # the endpoint with the most tokens in flight
            eng.inflight_remove_endpoint(m)
            tracker.remove(m)
            what = "inflight_remove_endpoint"
        elif step in (5, 6):
            k_ = np.array([next(keys) for _ in range(n_)], np.uint64)
            tp = rng.choice([0.0, 15.0, 22.0, 31.0], n_)
            eng.running_add(torch.from_numpy(e_).cuda() if on_dev else e_, torch.from_numpy(k_.view(np.int64)).cuda() if on_dev else k_,
                            torch.from_numpy(tp).cuda() if on_dev else tp, device=on_dev, want_added=not on_dev)
            queues.add(e_, k_, tp)
            added.append((e_, k_))
            what = "running_add"
        else:
            e0, k0 = added[2 + (step - 7)]
            eng.running_remove(torch.from_numpy(e0[:200]).cuda() if on_dev else e0[:200],
                               torch.from_numpy(k0[:200].view(np.int64)).cuda() if on_dev else k0[:200], device=on_dev,
                               want_removed=not on_dev)
            queues.remove(e0[:200], k0[:200])
            what = "running_remove"
        torch.cuda.synchronize()
        check((what, "device" if on_dev else "host"))

    # a snapshot that carries inflight_tokens: the counters no longer feed profile 1
    own = rng.integers(0, 60000, M).astype(np.int64)
    eng.set_snapshot(**w.sd, inflight_tokens=own)
    check("snapshot tokens", tokens=own)
    eng.inflight_add(ep, tok)
    tracker.add(ep, tok)
    check("snapshot tokens after a mutation", tokens=own)

    # one captured graph: a device inflight_add, then the three runs; exact after each replay
    eng.set_snapshot(**w.sd)
    check("counters again")
    d_ep, d_tok = torch.from_numpy(ep).cuda(), torch.from_numpy(tok).cuda()
    dev = to_device(w.kw)
    runs = device_runs(R, (0, 1, 2))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)  # sizes the scratch outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.inflight_add(d_ep, d_tok, device=True, stream=s.cuda_stream)
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)
    for rep in range(2):
        g.replay()
        torch.cuda.synchronize()
        tracker.add(ep, tok)
        for p, r in zip((0, 1, 2), runs):
            assert_run(host(r), want0 if p == 0 else want(p), ("graph", rep, p))
    assert np.array_equal(eng.inflight_get(M)[1], tracker.get(M)[1])
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_mode", TIE_MODES)
def test_subset_lifecycle_and_captured_snapshot(pkg, deferral_world, tie_mode):
    """set_profile_endpoints takes effect at the next set_snapshot; a set_snapshot captured into a CUDA graph copies the subset
    as it stands at each replay (NULL: every endpoint), and a profile captured without a subset stays without one there"""
    import torch
    w, idx = deferral_world
    M, R = w.M, w.R
    seed = 0x5B5E + tie_mode
    eng = engine(pkg, w, W.HEADLINE, tie_mode, seed)
    pid = eng.add_profile(W.PREFILL)
    A, B, C = W.bits(M, range(0, M, 2)), W.bits(M, range(0, M, 3)), W.bits(M, range(1, M, 2))
    wants = {}

    def want(p, sub):
        key = (p, None if sub is None else sub.tobytes())
        if key not in wants:
            sc = W.HEADLINE if p == 0 else W.PREFILL
            wants[key] = W.oracle_run(w, sc, tie_mode, W.seed_of(seed, p), subset=sub, idx=idx)
        return wants[key]

    def eager(what, sub0, sub1):
        _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], **w.kw)
        assert_run(got[0], want(0, sub0), (what, 0))
        assert_run(got[1], want(pid, sub1), (what, pid))

    eager("no subset", None, None)
    eng.set_profile_endpoints(0, A)
    eager("set without set_snapshot", None, None)
    eng.set_snapshot(**w.sd)
    eager("after set_snapshot", A, None)
    eng.set_profile_endpoints(0, None)
    eager("None without set_snapshot", A, None)
    eng.set_snapshot(**w.sd)
    eager("None after set_snapshot", None, None)

    # capture set_snapshot(device=True) + schedule_profiles with profile 0 on A and profile pid without a subset
    eng.set_profile_endpoints(0, A)
    eng.set_snapshot(**w.sd)
    dsd = to_device(w.sd)
    dev = to_device(w.kw)
    runs = device_runs(R, (0, pid))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)  # sizes the scratch outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.set_snapshot(**dsd, device=True, stream=s.cuda_stream)
        eng.schedule_profiles(R, runs, device=True, stream=s.cuda_stream, **dev)

    def replay(what, sub0, sub1):
        for r in runs:
            r["pick"].fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert_run(host(runs[0]), want(0, sub0), (what, 0))
        assert_run(host(runs[1]), want(pid, sub1), (what, pid))

    replay("captured", A, None)
    eng.set_profile_endpoints(0, B)  # after a captured set_snapshot: no error, the next replay copies B
    replay("bits changed", B, None)
    eng.set_profile_endpoints(0, None)
    replay("subset removed", None, None)
    eng.set_profile_endpoints(pid, C)
    replay("subset on a profile captured without one", None, None)
    eng.set_profile_endpoints(0, B)
    replay("bits again", B, None)
    # outside the graph the subsets as set apply from the next set_snapshot
    eng.set_profile_endpoints(0, None)
    eng.set_snapshot(**w.sd)
    eager("eager after the graph", None, C)
    eng.close()
