"""Per-stream batch scratch (eppscore_reserve_stream / eppscore_release_stream), bit-exact against the CPU oracle: device
batches of every kind in flight on four reserved streams at once, graphs captured on a reserved stream replayed after larger
calls grew the shared scratch, batches on a reserved stream ordered with index commits, snapshots and producer updates, and
the edges of the two calls.  One world serves every test: M = 1024 endpoints, an index warmed on the headline prompt pool and
a system prompt cached on every endpoint, and four profiles (0 headline, 1 latency, 2 prefill on the even endpoints, 3
token load)."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import profile_worlds as W
from tests import topk_oracle as T
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_CAPACITY = -1, -3
M, PLEN, SEED = 1024, 2048, 0x5EED
LKW = dict(W.LAT_COEF, streaming_mode=1)
PROFILES = [W.HEADLINE, W.LATENCY_PROFILE, W.PREFILL, W.TOKEN_PROFILE]
MEMBERS = W.bits(M, range(0, M, 2))
POOL = 70  # prefix seed of the headline prompt pool


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


@pytest.fixture(scope="module")
def world():
    """the snapshot and the commits every engine and oracle index starts from"""
    rng = np.random.Generator(np.random.PCG64(71))
    seed = o.model_seed("stream-scratch")
    warm_p, _, _ = synth_prompts(2 * M, prompt_len=PLEN, seed=POOL)
    h, n = W.hash_rows(warm_p, PLEN, seed)
    commits = [(rng.integers(0, M, 2 * M).astype(np.int32), h, n)]
    system = rng.integers(97, 123, PLEN // 2, dtype=np.uint8)  # 16 blocks, cached on every endpoint: past the sparse pick's limit
    sys_p = np.concatenate([np.tile(system, (M, 1)), rng.integers(97, 123, (M, PLEN // 2), dtype=np.uint8)], axis=1)
    h, n = W.hash_rows(sys_p, PLEN, seed)
    commits.append((np.arange(M, dtype=np.int32), h, n))
    return dict(sd=synth_snapshot(M, seed=72), commits=commits, seed=seed, system=system)


def engine(pkg, world):
    eng = pkg.Engine(pkg.default_config(W.HEADLINE, max_endpoints=M, prefix_capacity=1 << 18, tie_seed=SEED,
                                        token_load_threshold=W.TOKEN_THR))
    eng.set_latency_params(pkg.latency_params(**LKW))
    for scorers in PROFILES[1:]:
        eng.add_profile(scorers)
    eng.set_profile_endpoints(2, MEMBERS)
    for pick, h, n in world["commits"]:
        eng.commit_picks(pick, h, n)
    eng.set_snapshot(**world["sd"])
    return eng


def index(world):
    idx = o.Index()
    for pick, h, n in world["commits"]:
        idx.commit(pick, h, n)
    return idx


def oracle(world, p, R, kw, idx, sd=None, cand_mask=None, tokens=None, **extra):
    """oracle_py.schedule_batch of profile p: its scorers and tie seed, its subset ∧ cand_mask, the in-flight tokens"""
    prof = o.make_profile([(W.SCORER[k], w) for k, w in PROFILES[p]], tie_seed=W.seed_of(SEED, p), token_load_threshold=W.TOKEN_THR,
                          latency=o.make_latency_params(**LKW) if p == 1 else None)
    mask = cand_mask
    if p == 2:
        mask = np.tile(MEMBERS, (R, 1)) if mask is None else mask & MEMBERS[None, :]
    snap = o.SnapshotData(**(world["sd"] if sd is None else sd), inflight_tokens=np.zeros(M, np.int64) if tokens is None else tokens)
    return o.schedule_batch(snap, prof, idx, R, cand_mask=mask, n_threads=16, **kw, **extra), prof


def headline(world, R, seed):
    p, off, _ = synth_prompts(R, prompt_len=PLEN, seed=seed, prefix_seed=POOL)
    return dict(prompt_bytes=p, prompt_off=off, model_seed=np.full(R, world["seed"], np.uint64), adapter_id=zipf_adapters(R, seed=seed))


def with_system_prompt(world, R, seed):
    """every other request opens with the system prompt cached on every endpoint"""
    kw = headline(world, R, seed)
    p = kw["prompt_bytes"].reshape(R, PLEN)
    p[::2, : PLEN // 2] = world["system"]
    return kw


def texty(world, R, seed):
    """headline prompts with spaces in their tails, for the device-counted field counts"""
    kw = headline(world, R, seed)
    p = kw["prompt_bytes"].reshape(R, PLEN)
    rng = np.random.Generator(np.random.PCG64(seed))
    tail = p[:, PLEN // 2:]
    tail[rng.random(tail.shape) < 0.15] = 32
    fields = np.array([o.count_fields(p[r].tobytes()) for r in range(R)], np.int32)
    return kw, fields


def dev(kw):
    """CUDA copies (unsigned words as the signed type of their width)"""
    import torch
    signed = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}
    return {k: torch.from_numpy(np.ascontiguousarray(v).view(signed.get(v.dtype, v.dtype))).cuda() for k, v in kw.items()}


def outputs(R, k=0, hashes=False):
    import torch
    out = dict(pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"), pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
               tie_count=torch.zeros(R, dtype=torch.int32, device="cuda"), total_blocks=torch.zeros(R, dtype=torch.int16, device="cuda"))
    if k:
        out.update(topk_pick=torch.zeros((R, k), dtype=torch.int32, device="cuda"),
                   topk_score=torch.zeros((R, k), dtype=torch.float64, device="cuda"))
    if hashes:
        out["hashes_out"] = torch.zeros((R, W.MAX_BLOCKS), dtype=torch.int64, device="cuda")
    return out


def host(out):
    got = {k: v.cpu().numpy() for k, v in out.items() if hasattr(v, "cpu")}
    if "total_blocks" in got:
        got["total_blocks"] = got["total_blocks"].view(np.uint16)
    return got


def assert_run(got, want, what, keys=("pick", "pick_score", "tie_count")):
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert np.array_equal(g.view(np.uint64) if g.dtype == np.float64 else g, w.view(np.uint64) if w.dtype == np.float64 else w), (what, k)


def assert_lists(got, want, prof, k, what):
    wm, ws = T.lists(want["weighted_out"], prof, k)
    assert np.array_equal(got["topk_pick"], wm), what
    assert np.array_equal(got["topk_score"].view(np.uint64), ws.view(np.uint64)), what


def runs(R, profiles):
    import torch
    return [dict(profile=p, pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"),
                 pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
                 tie_count=torch.zeros(R, dtype=torch.int32, device="cuda")) for p in profiles]


# ---------------------------------------------------------------------------------------------------------------------------
def test_concurrent_batches_on_reserved_streams(pkg, world):
    """Four reserved streams, each launched with no host synchronisation in between: the sparse headline batch (64K x 1024, the
    hash kernel's probe records), a masked full-matrix latency batch with device-counted fields, a two-profile batch whose
    subset profile defers requests to member rows, and a k = 4 then a k = 16 (wide) top-k batch.  Then two streams running
    the headline batch on the same input buffers."""
    import torch
    eng, idx = engine(pkg, world), index(world)
    RA, RB, RC, RD = 65536, 4096, 4096, 2048
    ka = headline(world, RA, 80)
    kb, fields = texty(world, RB, 81)
    rng = np.random.Generator(np.random.PCG64(82))
    slo = dict(ttft_slo=rng.choice([0.0, 140.0, 400.0, 1e6], RB), tpot_slo=rng.choice([0.0, 18.0, 24.0, 30.0, 80.0], RB))
    mask_b = W.short_run_mask(RB, M, rng, M // 32)
    kc = with_system_prompt(world, RC, 83)
    kd = headline(world, RD, 84)
    want_a, _ = oracle(world, 0, RA, ka, idx)
    want_b, _ = oracle(world, 1, RB, dict(kb, input_tokens=fields, **slo), idx, cand_mask=mask_b)
    want_c = [oracle(world, p, RC, kc, idx)[0] for p in (0, 2)]
    want_d, prof0 = oracle(world, 0, RD, kd, idx, want_scores=True)
    da, db, dc, dd = dev(ka), dev(dict(kb, **slo)), dev(kc), dev(kd)
    dmask = dev(dict(m=mask_b))["m"]
    streams = [torch.cuda.Stream() for _ in range(5)]
    for s, r in zip(streams, (RA, RB, RC, RD, RA)):
        eng.reserve_stream(s, r)
    oa, oa2, od4, od16 = outputs(RA), outputs(RA), outputs(RD, 4), outputs(RD, 16)
    rb, rc = runs(RB, (1,)), runs(RC, (0, 2))
    rb[0]["cand_mask"] = dmask
    torch.cuda.synchronize()
    r0 = eng.stats().probe_resolved
    eng.schedule(RA, device=True, stream=streams[0].cuda_stream, out=oa, **da)
    eng.schedule_profiles(RB, rb, device=True, stream=streams[1].cuda_stream, **db)
    eng.schedule_profiles(RC, rc, device=True, stream=streams[2].cuda_stream, **dc)
    eng.schedule(RD, topk=4, device=True, stream=streams[3].cuda_stream, out=od4, **dd)
    eng.schedule(RD, topk_wide=16, device=True, stream=streams[3].cuda_stream, out=od16, **dd)
    torch.cuda.synchronize()
    assert eng.stats().probe_resolved != r0  # the headline batch took the probe records
    assert_run(host(oa), want_a, "headline", ("pick", "pick_score", "tie_count", "total_blocks"))
    assert_run(host(rb[0]), want_b, "latency, masked, counted fields")
    assert_run(host(rc[0]), want_c[0], "system prompt, profile 0")
    assert_run(host(rc[1]), want_c[1], "system prompt, subset profile")
    assert np.isin(rc[1]["pick"].cpu().numpy(), np.arange(0, M, 2)).all()
    for k, o_ in ((4, od4), (16, od16)):
        got = host(o_)
        assert_run(got, want_d, f"top-{k}")
        assert_lists(got, want_d, prof0, k, f"top-{k} lists")
    # two streams, the same input buffers
    for o_ in (oa, oa2):
        o_["pick"].fill_(-7)
    torch.cuda.synchronize()
    eng.schedule(RA, device=True, stream=streams[0].cuda_stream, out=oa, **da)
    eng.schedule(RA, device=True, stream=streams[4].cuda_stream, out=oa2, **da)
    torch.cuda.synchronize()
    for what, o_ in (("first", oa), ("second", oa2)):
        assert_run(host(o_), want_a, ("same inputs", what), ("pick", "pick_score", "tie_count", "total_blocks"))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
def test_graphs_on_reserved_streams_survive_larger_calls(pkg, world):
    """A batch and a wide top-k batch captured on reserved streams; larger device batches on an unreserved stream and host
    batches then grow the shared scratch; new inputs written into the captured buffers; the replays match the oracle."""
    import torch
    eng, idx = engine(pkg, world), index(world)
    R, RL = 2048, 16384
    s, sw, u = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    eng.reserve_stream(s, R)
    eng.reserve_stream(sw.cuda_stream, R)  # (a raw handle works as well)
    first, second = headline(world, R, 90), headline(world, R, 91)
    d = dev(first)
    out, outw = outputs(R), outputs(R, 16)
    graphs = []
    for st, o_, kw in ((s, out, {}), (sw, outw, dict(topk_wide=16))):
        st.wait_stream(torch.cuda.current_stream())
        eng.schedule(R, device=True, stream=st.cuda_stream, out=o_, **kw, **d)  # outside the capture: the wide call allocates sw's score rows
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            eng.schedule(R, device=True, stream=st.cuda_stream, out=o_, **kw, **d)
        graphs.append(g)
    # larger calls outside the captures: the shared scratch grows (hashes, probe records, wide rows, both host chunk sets)
    big = headline(world, RL, 92)
    dbig = dev(big)
    u.wait_stream(torch.cuda.current_stream())
    eng.schedule(RL, device=True, stream=u.cuda_stream, out=outputs(RL), **dbig)
    eng.schedule(RL, topk_wide=16, device=True, stream=u.cuda_stream, out=outputs(RL, 16), **dbig)
    u.synchronize()
    eng.schedule(RL, **big)
    eng.schedule(RL, topk_wide=16, **big)
    for k, v in dev(second).items():
        d[k].copy_(v)
    for o_ in (out, outw):
        o_["pick"].fill_(-7)
    torch.cuda.synchronize()
    for g in graphs:
        g.replay()
    torch.cuda.synchronize()
    want, prof0 = oracle(world, 0, R, second, idx, want_scores=True)
    assert_run(host(out), want, "replayed batch", ("pick", "pick_score", "tie_count", "total_blocks"))
    got = host(outw)
    assert_run(got, want, "replayed wide batch")
    assert_lists(got, want, prof0, 16, "replayed wide lists")
    del graphs
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
def test_reserved_stream_batches_order_with_mutations(pkg, world):
    """batch -> device commit on a second stream -> batch -> set_snapshot -> batch -> inflight_add -> batch, the batches on
    a reserved stream queued behind a ~1 s spin and nothing synchronised by the test until the end: every batch sees exactly
    the mutations issued before it (the oracle's sequential replay), and the index ends equal to the oracle's."""
    import torch
    eng, idx = engine(pkg, world), index(world)
    R = 4096
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    eng.reserve_stream(s, R)
    kws = [headline(world, R, 100 + i) for i in range(4)]
    ds = [dev(k) for k in kws]
    outs = [runs(R, (0, 3)) for _ in range(4)]
    batch_out = [outputs(R, hashes=True) for _ in range(4)]
    sd2 = synth_snapshot(M, seed=73)
    rng = np.random.Generator(np.random.PCG64(74))
    ep, tok = rng.integers(-1, M, 3000).astype(np.int32), rng.integers(0, 40000, 3000).astype(np.int64)

    def batch(i):
        b = batch_out[i]
        eng.schedule_profiles(R, outs[i], device=True, stream=s.cuda_stream, out=dict(total_blocks=b["total_blocks"], hashes_out=b["hashes_out"]),
                              **ds[i])

    torch.cuda.synchronize()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000_000)
    batch(0)
    s2.wait_stream(s)
    eng.commit_picks_device(outs[0][0]["pick"], batch_out[0]["hashes_out"], batch_out[0]["total_blocks"], touch_bound=R * W.MAX_BLOCKS,
                            stream=s2.cuda_stream)
    batch(1)
    eng.set_snapshot(**sd2)
    batch(2)
    eng.inflight_add(ep, tok)
    batch(3)
    torch.cuda.synchronize()
    tracker = I.Tracker()
    wants = []
    for i in range(4):
        if i == 3:
            tracker.add(ep, tok)
        sd = world["sd"] if i < 2 else sd2
        wants.append([oracle(world, p, R, kws[i], idx, sd=sd, tokens=tracker.get(M)[1], want_hashes=(p == 0))[0] for p in (0, 3)])
        if i == 0:
            w0 = wants[0][0]
            idx.commit(w0["pick"], w0["hashes_out"], w0["total_blocks"])
    for i in range(4):
        for j, p in enumerate((0, 3)):
            assert_run(host(outs[i][j]), wants[i][j], (f"batch {i}", p))
        assert np.array_equal(host(batch_out[i])["total_blocks"], wants[i][0]["total_blocks"]), i
    assert (wants[1][0]["pick"] != oracle(world, 0, R, kws[1], index(world))[0]["pick"]).any()  # the commit moved picks
    assert eng.stats().prefix_live_hashes == idx.num_hashes()
    for m in range(0, M, 7):
        assert eng.prefix_lru_keys(m) == idx.lru_keys(m), m
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
def test_reserve_and_release_edges(pkg, world):
    import torch
    eng, idx = engine(pkg, world), index(world)
    R = 1024
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    eng.reserve_stream(s, R, max_blocks=16)

    def code(fn, *a, **kw):
        with pytest.raises(pkg.EppscoreError) as ex:
            fn(*a, **kw)
        return ex.value.code

    kw1 = headline(world, R + 1, 110)
    d1 = dev(kw1)
    # R = max_R passes; R = max_R + 1 and more blocks than reserved are refused, and nothing is written
    first = dict(prompt_bytes=kw1["prompt_bytes"], prompt_off=kw1["prompt_off"][: R + 1], model_seed=kw1["model_seed"][:R],
                 adapter_id=kw1["adapter_id"][:R])
    out = outputs(R)
    eng.schedule(R, device=True, stream=s.cuda_stream, out=out, max_blocks=16, **d1)
    torch.cuda.synchronize()
    assert_run(host(out), oracle(world, 0, R, first, idx, max_blocks=16)[0], "R = max_R", ("pick", "pick_score", "tie_count", "total_blocks"))
    out = outputs(R + 1)
    assert code(eng.schedule, R + 1, device=True, stream=s.cuda_stream, out=out, max_blocks=16, **d1) == ERR_CAPACITY
    assert code(eng.schedule, R, device=True, stream=s.cuda_stream, out={k: v[:R] for k, v in out.items()}, max_blocks=17, **d1) == ERR_CAPACITY
    assert code(eng.schedule, R, device=True, stream=s.cuda_stream, out={k: v[:R] for k, v in out.items()}, **d1) == ERR_CAPACITY  # config: 256
    torch.cuda.synchronize()
    assert (out["pick"] == -7).all() and (out["tie_count"] == 0).all() and (out["total_blocks"] == 0).all()
    # ERR_INVALID
    assert code(eng.reserve_stream, None, 8) == ERR_INVALID
    assert code(eng.reserve_stream, u, 0) == ERR_INVALID
    assert code(eng.reserve_stream, u, 8, max_blocks=65536) == ERR_INVALID
    assert code(eng.reserve_stream, u, 8, max_blocks=-1) == ERR_INVALID
    assert code(eng.reserve_stream, s, 8) == ERR_INVALID  # already reserved
    assert code(eng.release_stream, u) == ERR_INVALID     # not reserved
    assert code(eng.release_stream, None) == ERR_INVALID
    x = torch.zeros(4, device="cuda")

    def under_capture(cap, fn, *arg):
        g = torch.cuda.CUDAGraph()
        cap.wait_stream(torch.cuda.current_stream())
        with torch.cuda.graph(g, stream=cap):
            x.add_(1)
            return code(fn, *arg)

    assert under_capture(u, eng.reserve_stream, u, 8) == ERR_INVALID  # the stream itself is being captured
    assert under_capture(s, eng.release_stream, s) == ERR_INVALID
    assert under_capture(s, eng.reserve_stream, u, 8) == ERR_INVALID  # a reserved stream is being captured
    # EPPSCORE_MAX_STREAMS: s and seven more, then one too many
    extra = [torch.cuda.Stream() for _ in range(pkg.MAX_STREAMS)]
    for st in extra[:-1]:
        eng.reserve_stream(st, 64)
    assert code(eng.reserve_stream, extra[-1], 64) == ERR_CAPACITY
    for st in extra[:-1]:
        eng.release_stream(st)
    # after a release the stream runs on the shared scratch, with no limit of its own
    eng.release_stream(s)
    out = outputs(R + 1)
    eng.schedule(R + 1, device=True, stream=s.cuda_stream, out=out, **d1)
    torch.cuda.synchronize()
    assert_run(host(out), oracle(world, 0, R + 1, kw1, idx)[0], "released", ("pick", "pick_score", "tie_count", "total_blocks"))
    eng.close()


def test_slicing_keys_do_not_cut_reserved_stream_batches(pkg, world):
    import torch
    eng, idx = engine(pkg, world), index(world)
    R = 8192
    s, u = torch.cuda.Stream(), torch.cuda.Stream()
    eng.reserve_stream(s, R)
    kw = headline(world, R, 120)
    d = dev(kw)
    want = oracle(world, 0, R, kw, idx)[0]

    def launches(st):
        out = outputs(R)
        st.wait_stream(torch.cuda.current_stream())
        l0 = eng.stats().kernel_launches
        eng.schedule(R, device=True, stream=st.cuda_stream, out=out, **d)
        torch.cuda.synchronize()
        assert_run(host(out), want, st is s, ("pick", "pick_score", "tie_count", "total_blocks"))
        return eng.stats().kernel_launches - l0

    whole = launches(s)
    eng.set_debug(5, 4)
    eng.set_debug(6, 3)
    assert launches(s) == whole
    assert launches(u) > whole  # the keys cut the same batch on an unreserved stream
    eng.close()


def test_destroy_with_reserved_streams(pkg, world):
    """destroying an engine waits for the batches still queued on its reserved streams before it frees their scratch"""
    import torch
    eng, idx = engine(pkg, world), index(world)
    R = 4096
    kw = headline(world, R, 130)
    d = dev(kw)
    want = oracle(world, 0, R, kw, idx)[0]
    streams = [torch.cuda.Stream() for _ in range(2)]
    outs = [outputs(R) for _ in streams]
    torch.cuda.synchronize()
    for st, out in zip(streams, outs):
        eng.reserve_stream(st, R)
        with torch.cuda.stream(st):
            torch.cuda._sleep(500_000_000)
        eng.schedule(R, device=True, stream=st.cuda_stream, out=out, **d)
    eng.close()
    torch.cuda.synchronize()
    for out in outs:
        assert_run(host(out), want, "after destroy", ("pick", "pick_score", "tie_count", "total_blocks"))
