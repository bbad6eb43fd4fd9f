"""The in-flight load producer on the GPU (eppscore_estimate_tokens, eppscore_inflight_*): the estimator at its rounding
boundaries, the counters under 200K random updates against a dict model, and the closed loop schedule -> commit -> estimate ->
add (-> release two rounds later) with a token-load profile, bit-exact against the CPU oracle whose snapshot takes
inflight_tokens from its own tracker — on the sparse path, the full-matrix path, the top-k lists and inside a CUDA graph with
the batch and the update on different streams."""
import os
import subprocess

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import topk_oracle as T
from tests.helpers import synth_ragged_prompts, synth_snapshot, zipf_adapters
from tests.test_inflight_cpu import integer_estimate

pytestmark = pytest.mark.gpu

SCORERS = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 2)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def test_estimator_rounding_boundaries_host_and_device(pkg):
    import torch
    eng = pkg.Engine(pkg.default_config([("token_load", 1)], max_endpoints=64))
    cases = [(0, -1, c) for c in range(2050)]                               # every residue of chars mod 4
    cases += [(0, h, c) for h in list(range(0, 40)) + [2 ** 31 - 1] for c in (0, 2, 6, -1)]  # odd / even hints, hint 0
    cases += [(s, -1, c) for s in list(range(-3, 10)) + [2 ** 40 + 3] for c in (-1, 0, 7)]
    size, hint, chars = (np.array(x) for x in zip(*cases))
    want = I.estimate(size, hint, chars)
    assert np.array_equal(want, [integer_estimate(*c) for c in cases])
    R = len(cases)
    assert np.array_equal(eng.estimate_tokens(R, size, hint, chars), want)
    out = torch.zeros(R, dtype=torch.int64, device="cuda:0")
    eng.estimate_tokens(R, _dev(size.astype(np.int64)), _dev(hint.astype(np.int32)), _dev(chars.astype(np.int32)), device=True, out=out)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)
    # NULL arrays: size 0, hint -1, chars 0 (body present)
    for kw in (dict(), dict(request_size_bytes=size), dict(token_hint=hint), dict(prompt_chars=chars)):
        w = I.estimate(kw.get("request_size_bytes"), kw.get("token_hint"), kw.get("prompt_chars"), R=R)
        assert np.array_equal(eng.estimate_tokens(R, **kw), w), list(kw)
        d = {k: _dev(v.astype(np.int64 if k == "request_size_bytes" else np.int32)) for k, v in kw.items()}
        out.zero_()
        eng.estimate_tokens(R, device=True, out=out, **d)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), w), list(kw)
    eng.close()


@pytest.mark.parametrize("max_endpoints", [1024, 8192])
def test_random_updates_against_a_dict_model(pkg, max_endpoints):
    """200K add / release / remove operations, host and device arrays, skewed and uniform endpoints, negative counts; then
    64K adds on one endpoint.  Every counter equal to the model after every step."""
    import torch
    E = max_endpoints
    eng = pkg.Engine(pkg.default_config([("kv", 1), ("token_load", 1)], max_endpoints=E))
    rng = np.random.Generator(np.random.PCG64(E))
    req, tok = {}, {}  # the dict model: endpoint -> counter (absent = 0)
    n_ops, step = 0, 0
    while n_ops < 200_000:
        kind = rng.choice(["add", "release", "remove"], p=[0.5, 0.42, 0.08])
        if kind == "remove":
            m = int(rng.integers(0, E))
            eng.inflight_remove_endpoint(m)
            req.pop(m, None)
            tok.pop(m, None)
            n_ops += 1
        else:
            R = int(rng.integers(1, 9000))
            hot = rng.integers(0, E, 3)
            ep = np.where(rng.random(R) < rng.random(), rng.choice(hot, R), rng.integers(-1, E, R)).astype(np.int32)
            tk = rng.integers(0, 1 << 40, R).astype(np.int64) if rng.random() < 0.7 else None
            sign = 1 if kind == "add" else -1
            device = bool(step % 2)
            args = (_dev(ep), None if tk is None else _dev(tk)) if device else (ep, tk)
            (eng.inflight_add if sign > 0 else eng.inflight_release)(*args, device=device)
            for r in np.nonzero(ep >= 0)[0]:
                m = int(ep[r])
                req[m] = req.get(m, 0) + sign
                tok[m] = tok.get(m, 0) + sign * (int(tk[r]) if tk is not None else 0)
            n_ops += R
        step += 1
        if step % 7 == 0 or n_ops >= 200_000:
            got_r, got_t = eng.inflight_get(E)
            want_r = np.array([req.get(m, 0) for m in range(E)], np.int64)
            want_t = np.array([tok.get(m, 0) for m in range(E)], np.int64)
            assert np.array_equal(got_r, want_r) and np.array_equal(got_t, want_t), step
    assert min(req.values()) < 0 and min(tok.values()) < 0  # releases outran adds somewhere
    # dog-piling: 64K picks on one endpoint, host and device arrays
    R = 65536
    ep = np.full(R, E - 1, np.int32)
    tk = rng.integers(0, 1 << 20, R).astype(np.int64)
    base_r, base_t = (x[E - 1] for x in eng.inflight_get(E))
    eng.inflight_add(ep, tk)
    eng.inflight_add(_dev(ep), _dev(tk), device=True)
    eng.inflight_release(_dev(ep[: R // 2]), _dev(tk[: R // 2]), device=True)
    got_r, got_t = eng.inflight_get(E)
    assert got_r[E - 1] == base_r + R + R // 2
    assert got_t[E - 1] == base_t + 2 * int(tk.sum()) - int(tk[: R // 2].sum())
    # an endpoint >= max_endpoints: refused on host arrays (nothing applied), skipped and reported on device arrays
    before = eng.inflight_get(E)
    with pytest.raises(pkg.EppscoreError):
        eng.inflight_add(np.array([0, E], np.int32), np.array([5, 5], np.int64))
    eng.inflight_add(_dev(np.array([0, E], np.int32)), _dev(np.array([5, 5], np.int64)), device=True)
    with pytest.raises(pkg.EppscoreError):
        eng.inflight_get(E)
    after = eng.inflight_get(E)
    assert after[0][0] == before[0][0] + 1 and after[1][0] == before[1][0] + 5
    with pytest.raises(pkg.EppscoreError):
        eng.inflight_remove_endpoint(E)
    with pytest.raises(pkg.EppscoreError):
        eng.inflight_get(E + 1)
    eng.close()


M, R, ROUNDS, THR, MB = 256, 4096, 5, 6000.0, 32


def _workload(seed):
    prompts, off = synth_ragged_prompts(R, max_len=1500, seed=seed, groups=24, shared=512)
    lens = np.diff(off).astype(np.int32)
    return dict(prompt_bytes=prompts, prompt_off=off, model_seed=np.full(R, 0x5EED, np.uint64),
                adapter_id=zipf_adapters(R, seed=seed)), lens


def _masks(rng):
    bits = rng.random((R, M)) < 0.9
    bits[:, 0] = False
    return (bits.reshape(R, M // 32, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)


@pytest.mark.parametrize("variant", ["sparse", "masked", "topk", "graph"])
def test_closed_loop_with_token_load_matches_oracle(pkg, variant):
    """5 rounds of schedule -> commit_picks_device -> estimate_tokens -> inflight_add, releasing round k-2, all on the device;
    picks, scores and tie counts (and the top-k lists) bit-equal to the oracle fed by its own tracker"""
    import torch
    k_top = 3 if variant == "topk" else 0
    eng = pkg.Engine(pkg.default_config(SCORERS, max_endpoints=M, token_load_threshold=THR, max_blocks=MB, prefix_capacity=1 << 16))
    sd = synth_snapshot(M, seed=9)
    eng.set_snapshot(**sd)
    prof = o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], token_load_threshold=THR)
    idx, tracker = o.Index(), I.Tracker()
    rng = np.random.Generator(np.random.PCG64(4))
    dev = torch.device("cuda:0")
    s_batch = torch.cuda.Stream()
    s_upd = torch.cuda.Stream() if variant in ("masked", "graph") else s_batch  # the update on another stream than the batch
    loads, picks, ests = [], [], []
    for k in range(ROUNDS):
        kw, lens = _workload(100 + k)
        mask = _masks(rng) if variant == "masked" else None
        d_in = {key: _dev(v) for key, v in kw.items()}
        if mask is not None:
            d_in["cand_mask"] = _dev(mask)
        d_len = _dev(lens)
        out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                   tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
                   hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev))
        if k_top:
            out["topk_pick"] = torch.empty((R, k_top), dtype=torch.int32, device=dev)
            out["topk_score"] = torch.empty((R, k_top), dtype=torch.float64, device=dev)
        est = torch.empty(R, dtype=torch.int64, device=dev)

        def batch():
            eng.schedule(R, device=True, stream=s_batch.cuda_stream, out=out, topk=k_top, **d_in)

        def update():
            eng.estimate_tokens(R, prompt_chars=d_len, device=True, stream=s_upd.cuda_stream, out=est)
            eng.inflight_add(out["pick"], est, device=True, stream=s_upd.cuda_stream)
            if k >= 2:
                eng.inflight_release(picks[k - 2], ests[k - 2], device=True, stream=s_upd.cuda_stream)

        def commit():
            eng.commit_picks_device(out["pick"], out["hashes_out"], out["total_blocks"], touch_bound=R * MB, stream=s_batch.cuda_stream)

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
            g.replay()
            torch.cuda.synchronize()
            commit()
        else:
            batch()
            commit()
            s_upd.wait_stream(s_batch)
            update()
        torch.cuda.synchronize()
        picks.append(out["pick"].clone())
        ests.append(est.clone())
        # the oracle: the same round on a snapshot whose InFlightLoad.Tokens is the tracker's
        snap = o.SnapshotData(**sd, inflight_tokens=tracker.get(M)[1])
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
        w_est = I.estimate(None, None, lens)
        assert np.array_equal(est.cpu().numpy(), w_est), what
        tracker.add(want["pick"], w_est)
        if k >= 2:
            tracker.release(picks[k - 2].cpu().numpy(), ests[k - 2].cpu().numpy())
        got_r, got_t = eng.inflight_get(M)
        want_r, want_t = tracker.get(M)
        assert np.array_equal(got_r, want_r) and np.array_equal(got_t, want_t), what
        loads.append(int(want_t.max()))
    assert max(loads) > THR  # the loads reached the threshold: some endpoints' token-load term was 0
    eng.close()


def test_snapshot_tokens_take_precedence_and_no_adds_changes_nothing(pkg):
    kw, _ = _workload(7)
    prof = o.make_profile([(pkg.SCORER[s], w) for s, w in SCORERS], token_load_threshold=THR)
    sd = synth_snapshot(M, seed=3)
    cfg = dict(max_endpoints=M, token_load_threshold=THR, max_blocks=MB, prefix_capacity=1 << 16)

    def same(got, want, what):
        for key in ("pick", "tie_count"):
            assert np.array_equal(got[key], want[key]), (what, key)
        assert np.array_equal(got["pick_score"].view(np.uint64), want["pick_score"].view(np.uint64)), what

    # no adds: the token-load profile returns what it returns with the attribute absent
    eng = pkg.Engine(pkg.default_config(SCORERS, **cfg))
    eng.set_snapshot(**sd)
    base = o.schedule_batch(o.SnapshotData(**sd), prof, None, R, max_blocks=MB, n_threads=8, **kw)
    same(eng.schedule(R, **kw), base, "no adds")
    # a snapshot that carries inflight_tokens ignores the counters, before and after they change
    eng.inflight_add(np.arange(M // 2, dtype=np.int32), np.full(M // 2, 10 ** 6, np.int64))
    own = np.random.Generator(np.random.PCG64(2)).integers(0, 2 * int(THR), M).astype(np.int64)
    want = o.schedule_batch(o.SnapshotData(**sd, inflight_tokens=own), prof, None, R, max_blocks=MB, n_threads=8, **kw)
    eng.set_snapshot(**sd, inflight_tokens=own)
    same(eng.schedule(R, **kw), want, "snapshot tokens")
    eng.inflight_release(np.arange(M // 2, dtype=np.int32), np.full(M // 2, 3, np.int64))
    eng.inflight_remove_endpoint(1)
    same(eng.schedule(R, **kw), want, "snapshot tokens after updates")
    # back to a snapshot without them: the counters are read again
    eng.set_snapshot(**sd)
    req, tok = eng.inflight_get(M)
    want = o.schedule_batch(o.SnapshotData(**sd, inflight_tokens=tok), prof, None, R, max_blocks=MB, n_threads=8, **kw)
    same(eng.schedule(R, **kw), want, "counters again")
    assert (tok[: M // 2] > THR).sum() == M // 2 - 1 and tok[1] == 0
    eng.close()


def test_host_producer_on_gpu(pkg):
    lib = _pkg.load_build().build()
    exe = os.path.join(ROOT, "tests", "cpp", "_build", "host_inflight_test_gpu")
    src = os.path.join(ROOT, "tests", "cpp", "host_inflight_test.cpp")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", src, "-o", exe, "-pthread",
                           "-L" + os.path.dirname(lib), "-leppscore", "-Wl,-rpath," + os.path.dirname(lib)])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host inflight: all checks passed" in r.stdout
