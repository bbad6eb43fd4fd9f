"""The running-request queues of the predicted-latency producer on the GPU (eppscore_running_*): the reference's cases through
the device ABI, 200K random operations against the queue oracle after every call, dog-piling on one endpoint, churn that must
not grow the table, and the closed loop schedule -> running_add -> running_remove (round k-2) with a latency profile,
bit-exact against the CPU oracle whose snapshot takes min_tpot_slo / dispatched from the queue oracle — plain, masked, top-k
and inside a CUDA graph, with the in-flight producer updating on a third stream."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q
from tests import topk_oracle as T
from tests.helpers import synth_ragged_prompts, synth_snapshot
from tests.test_running_cpu import golden, run_case

pytestmark = pytest.mark.gpu

LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01, streaming_mode=1)


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _same_view(eng, q, M, what):
    got_m, got_c = eng.running_get(M)
    want_m, want_c = q.get(M)
    assert np.array_equal(got_c, want_c), what
    assert np.array_equal(got_m.view(np.uint64), Q.canonical(want_m).view(np.uint64)), what


def _u8(n):
    """a zeroed uint8[n] output; the fill (on torch's stream) is complete before the engine's stream writes it"""
    import torch
    out = torch.zeros(max(n, 1), dtype=torch.uint8, device="cuda:0")[:n]
    torch.cuda.synchronize()
    return out


def _host(t):
    """a device output read after every stream has finished (the engine's own stream does not order with torch's)"""
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.mark.parametrize("device", [False, True])
def test_reference_cases_through_the_device_abi(pkg, device):
    import torch
    for case in golden()["cases"]:
        eng = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=64))

        def add(m, k, t):
            if not device:
                return bool(eng.running_add(np.array([m], np.int32), np.array([k], np.uint64), np.array([t]))[0])
            out = _u8(1)
            eng.running_add(_dev(np.array([m], np.int32)), _dev(np.array([k], np.uint64)), _dev(np.array([t])), device=True, out=out)
            torch.cuda.synchronize()
            return bool(out.cpu()[0])

        def remove(m, k):
            if not device:
                return bool(eng.running_remove(np.array([m], np.int32), np.array([k], np.uint64))[0])
            out = _u8(1)
            eng.running_remove(_dev(np.array([m], np.int32)), _dev(np.array([k], np.uint64)), device=True, out=out)
            torch.cuda.synchronize()
            return bool(out.cpu()[0])

        run_case(case, add, remove, lambda: eng.running_get(64))
        eng.close()


TPOTS = np.array([0.0, -0.0, 5.0, 18.0, 22.0, 22.0, 40.0, np.inf, -1.0, 1e-300])


@pytest.mark.parametrize("max_endpoints", [1024, 8192])
def test_random_operations_against_the_oracle(pkg, max_endpoints):
    """200K operations: adds and removes with duplicate keys inside a call and across calls, key 0, negative tpot, -0.0, 0,
    +Inf, removes of absent keys, remove_endpoint; host and device arrays.  Every endpoint's min and count bit-equal to the
    oracle after every call, and added_out / removed_out equal to the oracle's."""
    import torch
    E = max_endpoints
    eng = pkg.Engine(pkg.default_config([("kv", 1), ("latency", 1)], max_endpoints=E))
    q = Q.Queues(E)
    rng = np.random.Generator(np.random.PCG64(E + 1))
    pool = 6000
    n_ops, step = 0, 0
    seen = set()  # kinds of minimum the views went through
    while n_ops < 200_000:
        kind = rng.choice(["add", "remove", "drop"], p=[0.55, 0.43, 0.02])
        device = bool(step % 2)
        if kind == "drop":
            m = int(rng.integers(0, E))
            eng.running_remove_endpoint(m)
            q.remove_endpoint(m)
            n_ops += 1
        else:
            R = int(rng.integers(1, 4000))
            hot = rng.integers(0, E, 3)
            ep = np.where(rng.random(R) < rng.random(), rng.choice(hot, R), rng.integers(-1, E, R)).astype(np.int32)
            key = rng.integers(0, pool, R).astype(np.uint64)
            if kind == "add":
                tp = rng.choice(TPOTS, R)
                want = q.add(ep, key, tp)
                if device:
                    out = _u8(R)
                    eng.running_add(_dev(ep), _dev(key), _dev(tp), device=True, out=out)
                    got = _host(out).astype(bool)
                else:
                    got = eng.running_add(ep, key, tp)
            else:
                want = q.remove(ep, key)
                if device:
                    out = _u8(R)
                    eng.running_remove(_dev(ep), _dev(key), device=True, out=out)
                    got = _host(out).astype(bool)
                else:
                    got = eng.running_remove(ep, key)
            assert np.array_equal(got, want), (step, kind)
            n_ops += R
        _same_view(eng, q, E, (step, kind))
        mn, cnt = q.get(E)
        seen |= {"inf"} if (mn == np.inf).any() else set()
        seen |= {"zero"} if ((mn == 0) & (cnt > 0)).any() else set()
        seen |= {"positive"} if ((mn > 0) & (mn < np.inf)).any() else set()
        step += 1
    assert seen == {"inf", "zero", "positive"} and q.get(E)[1].sum() > 1000
    # invalid entries: refused on host arrays (nothing applied), skipped and reported on device arrays
    with pytest.raises(pkg.EppscoreError):
        eng.running_add(np.array([0, E], np.int32), np.array([pool + 1, pool + 2], np.uint64))
    with pytest.raises(pkg.EppscoreError):
        eng.running_add(np.array([0, 1], np.int32), np.array([pool + 1, pool + 2], np.uint64), np.array([1.0, np.nan]))
    _same_view(eng, q, E, "refused")
    eng.running_add(_dev(np.array([0, E, 1], np.int32)), _dev(np.array([pool + 1, pool + 2, pool + 3], np.uint64)),
                    _dev(np.array([3.0, 1.0, np.nan])), device=True)
    with pytest.raises(pkg.EppscoreError):
        eng.running_get(E)
    q.add([0], [pool + 1], [3.0])
    _same_view(eng, q, E, "skipped")
    with pytest.raises(pkg.EppscoreError):
        eng.running_remove_endpoint(E)
    with pytest.raises(pkg.EppscoreError):
        eng.running_get(E + 1)
    eng.close()


def test_dog_piling_and_the_minimum_leaving_piece_by_piece(pkg):
    E, R = 1024, 65536
    eng = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=E))
    q = Q.Queues(E)
    rng = np.random.Generator(np.random.PCG64(3))
    ep = np.full(R, 7, np.int32)
    key = rng.permutation(R).astype(np.uint64) + 1
    cls = rng.choice([10.0, 20.0, 30.0], R)
    assert np.array_equal(_host(eng.running_add(_dev(ep), _dev(key), _dev(cls), device=True, out=_u8(R))).astype(bool),
                          q.add(ep, key, cls))
    _same_view(eng, q, E, "added")
    for c in (10.0, 20.0):  # the minimum class leaves in four pieces; the minimum moves only with the last one
        idx = np.nonzero(cls == c)[0]
        for i, piece in enumerate(np.array_split(rng.permutation(idx), 4)):
            got = eng.running_remove(_dev(ep[piece]), _dev(key[piece]), device=True, out=_u8(len(piece)))
            assert _host(got).all() and q.remove(ep[piece], key[piece]).all()
            mn, cnt = eng.running_get(E)
            assert mn[7] == (c if i < 3 else c + 10.0), (c, i)
            _same_view(eng, q, E, (c, i))
    eng.close()


def test_churn_does_not_grow_the_table(pkg):
    """1M add / remove cycles with at most 64K live entries: after warm-up the capacity never exceeds its first value."""
    E, R = 1024, 65536
    eng = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=E))
    rng = np.random.Generator(np.random.PCG64(5))
    prev = None
    caps = []
    for k in range(16):
        ep = rng.integers(0, E, R).astype(np.int32)
        key = (np.arange(R) + 1 + k * R).astype(np.uint64)
        tp = rng.choice([0.0, 18.0, 25.0], R)
        if prev is not None:
            eng.running_remove(_dev(prev[0]), _dev(prev[1]), device=True)
        eng.running_add(_dev(ep), _dev(key), _dev(tp), device=True)
        prev = (ep, key)
        caps.append(eng.running_reserve(0))
        mn, cnt = eng.running_get(E)
        assert cnt.sum() == R and np.array_equal(cnt, np.bincount(ep, minlength=E)), k
    assert max(caps[2:]) <= caps[1], caps
    eng.close()


M, R, ROUNDS, MB = 256, 4096, 5, 32
SCORERS = [("kv", 1), ("prefix", 1), ("latency", 2), ("token_load", 1)]
THR = 50000.0


def _workload(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    prompts, off = synth_ragged_prompts(R, max_len=1500, seed=seed, groups=24, shared=512)
    kw = dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64),
              input_tokens=rng.integers(0, 6000, R).astype(np.int32), ttft_slo=rng.choice([0.0, 140.0, 400.0, 1e6], R),
              tpot_slo=rng.choice([0.0, 18.0, 24.0, 30.0, 80.0], R))
    return kw, np.diff(off).astype(np.int64)


def _masks(rng):
    bits = rng.random((R, M)) < 0.9
    bits[:, 0] = False
    return (bits.reshape(R, M // 32, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


def _config(pkg, **kw):
    filt = [(pkg.FILTER_SLO_HEADROOM_TIER, (0.3,))]
    return pkg.default_config(SCORERS, filters=filt, max_endpoints=M, max_blocks=MB, prefix_capacity=1 << 16,
                              token_load_threshold=THR, tie_mode=1, tie_seed=13, **kw)


def _profile(pkg):
    return o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], latency=o.make_latency_params(**LAT_COEF),
                          filters=[(pkg.FILTER_SLO_HEADROOM_TIER, (0.3,))], token_load_threshold=THR, tie_mode=1, tie_seed=13)


@pytest.mark.parametrize("variant", ["plain", "masked", "topk", "graph"])
def test_closed_loop_with_latency_profile_matches_oracle(pkg, variant):
    """5 rounds of device schedule -> running_add(pick, keys, tpot_slo) -> running_remove(round k-2), with inflight_add on a
    third stream; picks, scores, tie counts (and top-k lists) bit-equal to the oracle fed by the queue oracle and tracker."""
    import torch
    k_top = 3 if variant == "topk" else 0
    eng = pkg.Engine(_config(pkg))
    eng.set_latency_params(pkg.latency_params(**LAT_COEF))
    sd = synth_snapshot(M, seed=9)
    eng.set_snapshot(**sd)
    if variant == "graph":
        eng.running_reserve(16 * R)
    prof = _profile(pkg)
    idx, q, tracker = o.Index(), Q.Queues(M), I.Tracker()
    rng = np.random.Generator(np.random.PCG64(4))
    dev = torch.device("cuda:0")
    s_batch = torch.cuda.Stream()
    s_upd = torch.cuda.Stream() if variant in ("masked", "graph") else s_batch
    s_inf = torch.cuda.Stream() if variant in ("masked", "graph") else s_batch
    picks, keys, mins = [], [], []
    for k in range(ROUNDS):
        kw, lens = _workload(100 + k)
        mask = _masks(rng) if variant == "masked" else None
        d_in = {key: _dev(v) for key, v in kw.items()}
        if mask is not None:
            d_in["cand_mask"] = _dev(mask)
        key = (np.arange(R) + 1 + k * R).astype(np.uint64)
        key[::97] = 0  # requests without an x-request-id are not tracked
        d_key, d_tok = _dev(key), _dev(lens)
        out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                   tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                   hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
        if k_top:
            out["topk_pick"] = torch.empty((R, k_top), dtype=torch.int32, device=dev)
            out["topk_score"] = torch.empty((R, k_top), dtype=torch.float64, device=dev)

        def batch():
            eng.schedule(R, device=True, stream=s_batch.cuda_stream, out=out, topk=k_top, **d_in)

        def update():
            eng.running_add(out["pick"], d_key, d_in["tpot_slo"], device=True, stream=s_upd.cuda_stream)
            if k >= 2:
                eng.running_remove(picks[k - 2], keys[k - 2], device=True, stream=s_upd.cuda_stream)

        def inflight():
            eng.inflight_add(out["pick"], d_tok, device=True, stream=s_inf.cuda_stream)

        torch.cuda.synchronize()
        if variant == "graph":
            batch()  # warm: the engine's scratch for this shape exists before the capture
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s_upd):
                s_batch.wait_stream(s_upd)
                batch()
                s_upd.wait_stream(s_batch)
                update()
                s_inf.wait_stream(s_upd)  # inside a capture the graph's edges order the producers' mutations
                inflight()
                s_upd.wait_stream(s_inf)
            g.replay()
            torch.cuda.synchronize()
            eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], touch_bound=R * MB, stream=s_batch.cuda_stream)
        else:
            batch()
            eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], touch_bound=R * MB, stream=s_batch.cuda_stream)
            s_upd.wait_stream(s_batch)
            s_inf.wait_stream(s_batch)
            update()     # the engine orders the two producers' mutations itself (they may be on different streams)
            inflight()
        torch.cuda.synchronize()
        picks.append(out["pick"].clone())
        keys.append(d_key)
        qmin, qcnt = q.get(M)
        snap = o.SnapshotData(**sd, min_tpot_slo=Q.canonical(qmin), dispatched=qcnt, inflight_tokens=tracker.get(M)[1])
        want = o.schedule_batch(snap, prof, idx, R, cand_mask=mask, max_blocks=MB, want_hashes=True, want_scores=bool(k_top),
                                n_threads=8, **kw)
        what = (variant, k)
        assert np.array_equal(out["pick"].cpu().numpy(), want["pick"]), what
        assert np.array_equal(out["pick_score"].cpu().numpy().view(np.uint64), want["pick_score"].view(np.uint64)), what
        assert np.array_equal(out["tie_count"].cpu().numpy(), want["tie_count"]), what
        if k_top:
            wm, ws = T.lists(want["weighted_out"], prof, k_top)
            assert np.array_equal(out["topk_pick"].cpu().numpy(), wm), what
            assert np.array_equal(out["topk_score"].cpu().numpy().view(np.uint64), ws.view(np.uint64)), what
        idx.commit(want["pick"], want["hashes_out"], want["total_blocks"])
        q.add(want["pick"], key, kw["tpot_slo"])
        if k >= 2:
            q.remove(picks[k - 2].cpu().numpy(), keys[k - 2].cpu().numpy())
        tracker.add(want["pick"], lens)
        _same_view(eng, q, M, what)
        assert np.array_equal(eng.inflight_get(M)[1], tracker.get(M)[1]), what
        mins.append(q.get(M))
    mn, cnt = mins[-1]
    assert (mn > 0).any() and ((mn == 0) & (cnt > 0)).any()  # tightened endpoints and endpoints a tpot-0 request untightened
    eng.close()


def test_snapshot_arrays_take_precedence_and_no_adds_changes_nothing(pkg):
    kw, _ = _workload(7)
    prof = _profile(pkg)
    sd = synth_snapshot(M, seed=3)
    rng = np.random.Generator(np.random.PCG64(2))
    own_min = rng.choice([0.0, 20.0, 26.0], M)
    own_cnt = rng.integers(0, 3, M).astype(np.int32)

    def same(got, want, what):
        for key in ("pick", "tie_count"):
            assert np.array_equal(got[key], want[key]), (what, key)
        assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what

    def oracle(**extra):
        return o.schedule_batch(o.SnapshotData(**sd, **extra), prof, None, R, max_blocks=MB, n_threads=8, **kw)

    eng = pkg.Engine(_config(pkg))
    eng.set_latency_params(pkg.latency_params(**LAT_COEF))
    eng.set_snapshot(**sd)
    same(eng.schedule(R, **kw), oracle(), "no adds")  # empty queues score exactly like absent arrays
    ep = rng.integers(0, M, 3000).astype(np.int32)
    eng.running_add(ep, np.arange(1, 3001, dtype=np.uint64), rng.choice([0.0, 15.0, 22.0], 3000))
    mn, cnt = eng.running_get(M)
    assert cnt.sum() == 3000
    same(eng.schedule(R, **kw), oracle(min_tpot_slo=mn, dispatched=cnt), "queues")
    # a snapshot that carries both arrays ignores the queues, before and after they change
    eng.set_snapshot(**sd, min_tpot_slo=own_min, dispatched=own_cnt)
    want = oracle(min_tpot_slo=own_min, dispatched=own_cnt)
    same(eng.schedule(R, **kw), want, "snapshot arrays")
    eng.running_remove(ep[:1000], np.arange(1, 1001, dtype=np.uint64))
    eng.running_remove_endpoint(int(ep[2000]))
    same(eng.schedule(R, **kw), want, "snapshot arrays after updates")
    # field by field: one array from the snapshot, the other from the queues
    mn, cnt = eng.running_get(M)
    eng.set_snapshot(**sd, min_tpot_slo=own_min)
    same(eng.schedule(R, **kw), oracle(min_tpot_slo=own_min, dispatched=cnt), "min from snapshot")
    eng.set_snapshot(**sd, dispatched=own_cnt)
    same(eng.schedule(R, **kw), oracle(min_tpot_slo=mn, dispatched=own_cnt), "count from snapshot")
    eng.close()


def test_one_captured_graph_replayed_across_growth_and_compaction(pkg):
    """One CUDA graph (running_add of this round, running_remove of the last) replayed 40 times with new contents in its
    buffers: its tombstones exceed the table several times over, so the device compacts it inside the replays, and eager
    adds between replays grow the table twice.  The queues equal to the oracle after every replay and every eager call."""
    import torch
    M_, R_ = 256, 2048
    eng = pkg.Engine(_config(pkg))
    eng.set_latency_params(pkg.latency_params(**LAT_COEF))
    eng.set_snapshot(**synth_snapshot(M_, seed=5))
    cap0 = eng.running_reserve(3 * R_)
    q = Q.Queues(M_)
    rng = np.random.Generator(np.random.PCG64(8))
    dev = torch.device("cuda:0")
    ep_add = torch.full((R_,), -1, dtype=torch.int32, device=dev)
    key_add = torch.zeros(R_, dtype=torch.int64, device=dev)
    tp_add = torch.zeros(R_, dtype=torch.float64, device=dev)
    ep_rm, key_rm = torch.full_like(ep_add, -1), torch.zeros_like(key_add)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.running_add(ep_add, key_add, tp_add, device=True, stream=s.cuda_stream)
        eng.running_remove(ep_rm, key_rm, device=True, stream=s.cuda_stream)
    prev = None
    caps = [cap0]
    for i in range(40):
        ep = rng.integers(-1, M_, R_).astype(np.int32)
        key = (np.arange(R_) + 1 + i * R_).astype(np.uint64)
        key[rng.random(R_) < 0.05] = key[0]  # duplicates inside the call
        tp = rng.choice([0.0, 15.0, 22.0, 40.0], R_)
        ep_add.copy_(_dev(ep))
        key_add.copy_(_dev(key.view(np.int64)))
        tp_add.copy_(_dev(tp))
        if prev is not None:
            ep_rm.copy_(_dev(prev[0]))
            key_rm.copy_(_dev(prev[1].view(np.int64)))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        q.add(ep, key, tp)
        if prev is not None:
            q.remove(*prev)
        prev = (ep, key)
        _same_view(eng, q, M_, ("replay", i))
        if i in (10, 25):  # an eager add large enough to grow the table, then its removal
            big_ep = rng.integers(0, M_, 8 * R_ * (1 + i // 25)).astype(np.int32)
            big_key = (np.arange(len(big_ep)) + 10 ** 9 + i * 10 ** 6).astype(np.uint64)
            big_tp = rng.choice([5.0, 30.0], len(big_ep))
            assert np.array_equal(eng.running_add(big_ep, big_key, big_tp), q.add(big_ep, big_key, big_tp))
            caps.append(eng.running_reserve(0))
            _same_view(eng, q, M_, ("eager add", i))
            assert np.array_equal(eng.running_remove(big_ep, big_key), q.remove(big_ep, big_key))
            _same_view(eng, q, M_, ("eager remove", i))
    assert caps[0] < caps[1] < caps[2], caps
    eng.close()


def test_host_track_running_requests_on_gpu(pkg):
    import os
    import subprocess
    lib = _pkg.load_build().build()
    olib = Q.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "_build", "host_running_test_gpu")
    src = os.path.join(root, "tests", "cpp", "host_running_test.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", src, "-o", exe, "-pthread",
                           "-L" + os.path.dirname(lib), "-leppscore", "-L" + os.path.dirname(olib), "-lrunning_oracle",
                           "-Wl,-rpath," + os.path.dirname(lib) + ":" + os.path.dirname(olib)])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host running: all checks passed" in r.stdout
