"""Host-array forms against their device forms, and the refusals of the entry points that stage host arrays.

- eppscore_hash_prompts and eppscore_count_fields on device arrays, on a caller stream that is not the engine's, equal their
  host forms bit for bit, with prompt_len, offsets that are not 16-byte aligned, and R = 1 and R > 65 536.
- A host-array eppscore_schedule_batch_inorder with the host chunk (debug key 3) well below R equals the same call without
  it and the sequential reference, in-flight counters included: an in-order batch runs as one piece whatever that key says.
- Each entry point returns the code it returns for each refused call, and a refused producer call leaves the counters as they
  were.  Where several refusals apply, the first in the call's order decides."""
import ctypes as C

import numpy as np
import pytest

import _pkg
from tests.helpers import synth_snapshot
from tests.test_gpu_inorder import FOUR, MB, World

pytestmark = pytest.mark.gpu

OK, INVALID, CAPACITY, NO_SNAPSHOT = 0, -1, -3, -4


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _p(x):
    return None if x is None else x.ctypes.data


def _prompts(R, seed):
    """R prompts of words and spaces with gaps between them, so offsets are not 16-byte aligned and prompt_len is shorter
    than the distance to the next offset."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lens = rng.integers(0, 400, size=R).astype(np.int32)
    gaps = rng.integers(0, 9, size=R)
    off = np.zeros(R + 1, np.int64)
    off[1:] = np.cumsum(lens + gaps) + 3
    off[0] = 3
    data = rng.choice(np.frombuffer(b"abcdefgh \t\n ", np.uint8), size=int(off[-1]) + 5)
    seeds = rng.integers(0, 2 ** 63, size=R, dtype=np.int64).astype(np.uint64)
    return data, off, lens, seeds


@pytest.mark.parametrize("R", [1, 65536 + 4099])
def test_hash_and_count_device_forms_equal_host_forms(pkg, R):
    import torch
    eng = pkg.Engine(pkg.default_config(max_endpoints=64))
    lib = pkg.lib()
    data, off, lens, seeds = _prompts(R, seed=R)
    bc, mb = 64, 16
    hashes, nh = eng.hash_prompts(data, off, seeds, prompt_len=lens, block_chars=bc, max_blocks=mb)
    fields = eng.count_fields(data, off, lens)
    assert nh.max() > 0 and fields.max() > 0
    s = torch.cuda.Stream()
    d_data, d_off, d_len, d_seed = _dev(data), _dev(off), _dev(lens), _dev(seeds)
    d_hash = torch.zeros((R, mb), dtype=torch.int64, device="cuda")
    d_nh = torch.zeros(R, dtype=torch.int16, device="cuda")
    d_fields = torch.zeros(R, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert lib.eppscore_hash_prompts(eng._h, R, 1, d_data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), d_seed.data_ptr(), bc, mb,
                                     d_hash.data_ptr(), d_nh.data_ptr(), s.cuda_stream) == OK
    assert lib.eppscore_count_fields(eng._h, R, 1, d_data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), d_fields.data_ptr(),
                                     s.cuda_stream) == OK
    s.synchronize()
    assert np.array_equal(d_hash.cpu().numpy().view(np.uint64), hashes)
    assert np.array_equal(d_nh.cpu().numpy().view(np.uint16), nh)
    assert np.array_equal(d_fields.cpu().numpy(), fields)
    eng.close()


def test_host_inorder_runs_as_one_piece_whatever_the_host_chunk(pkg):
    R = 3000
    chunked, whole = World(pkg, 1024, FOUR, seed=7), World(pkg, 1024, FOUR, seed=7)
    chunked.eng.set_debug(3, 512)
    kw = chunked.workload(R, 12)
    mask = chunked.masks(R)
    tok = chunked.tokens(R)
    for rnd in range(2):
        got = chunked.eng.schedule_inorder(R, tokens=tok, cand_mask=mask, max_blocks=MB, request_base=rnd * R, want_hashes=True, **kw)
        same = whole.eng.schedule_inorder(R, tokens=tok, cand_mask=mask, max_blocks=MB, request_base=rnd * R, want_hashes=True, **kw)
        for k in got:
            assert np.array_equal(np.asarray(got[k]), np.asarray(same[k])), (rnd, k)
        want = chunked.reference(R, tok, request_base=rnd * R, cand_mask=mask, want_hashes=True, **kw)
        chunked.check(got, want, rnd)
        assert np.array_equal(got["hashes_out"], want["hashes_out"])
        assert all(np.array_equal(x, y) for x, y in zip(chunked.eng.inflight_get(1024), whole.eng.inflight_get(1024)))
    chunked.eng.close()
    whole.eng.close()


def _batch(pkg, R, location, outs, stream=None, **fields):
    b = pkg.Batch()
    b.struct_size = C.sizeof(pkg.Batch)
    b.R = R
    b.location = location
    b.stream = stream
    b.pick, b.pick_score, b.tie_count = outs
    for k, v in fields.items():
        setattr(b, k, v)
    return b


def test_inorder_refusals_in_the_parents_order(pkg):
    import torch
    lib = pkg.lib()
    M, R = 128, 64
    tok = np.arange(R, dtype=np.int64)
    host = [np.zeros(R, np.int32), np.zeros(R, np.float64), np.zeros(R, np.int32)]
    h_outs = [_p(x) for x in host]
    dev = [torch.zeros(R, dtype=t, device="cuda") for t in (torch.int32, torch.float64, torch.int32)]
    d_outs = [x.data_ptr() for x in dev]
    d_tok = _dev(tok)
    s = torch.cuda.Stream()

    # no snapshot yet: a device call on a stream reserved for fewer requests than R is refused for the snapshot
    eng = pkg.Engine(pkg.default_config([("kv", 1), ("token_load", 1)], max_endpoints=M))
    eng.reserve_stream(s.cuda_stream, R // 2, 16)
    call = lambda b, t=d_tok.data_ptr(): lib.eppscore_schedule_batch_inorder(eng._h, C.byref(b), t)
    assert call(_batch(pkg, R, 1, d_outs, s.cuda_stream)) == NO_SNAPSHOT
    assert call(_batch(pkg, R, 0, h_outs), _p(tok)) == NO_SNAPSHOT
    assert call(_batch(pkg, R, 2, h_outs), _p(tok)) == INVALID  # location comes before the snapshot
    assert call(_batch(pkg, R, 1, [d_outs[0], None, d_outs[2]], s.cuda_stream)) == INVALID
    assert call(_batch(pkg, -1, 1, d_outs, s.cuda_stream)) == INVALID
    assert call(_batch(pkg, 0, 1, d_outs, s.cuda_stream)) == OK
    eng.set_snapshot(**synth_snapshot(M, seed=2))
    prompts, off = np.full(4096, ord("x"), np.uint8), np.arange(0, 4096 + 1, 64, dtype=np.int64)[:R + 1]
    d_prompts = _dev(prompts)
    # with a snapshot: the stream's reservation; prompt_off before it
    assert call(_batch(pkg, R, 1, d_outs, s.cuda_stream)) == CAPACITY
    assert call(_batch(pkg, R, 1, d_outs, s.cuda_stream, prompt_bytes=d_prompts.data_ptr())) == INVALID
    assert call(_batch(pkg, R // 2, 1, d_outs, s.cuda_stream, prompt_bytes=d_prompts.data_ptr(), prompt_off=_dev(off).data_ptr(),
                       max_blocks=64)) == CAPACITY
    # the R x M outputs come before the location and the snapshot
    assert call(_batch(pkg, R, 2, h_outs, scores_out=_p(np.zeros((R, M)))), _p(tok)) == INVALID
    # host arrays: prompt_off, then hashes_out without prompt bytes
    assert call(_batch(pkg, R, 0, h_outs, prompt_bytes=_p(prompts)), _p(tok)) == INVALID
    assert call(_batch(pkg, R, 0, h_outs, hashes_out=_p(np.zeros((R, 256), np.uint64))), _p(tok)) == INVALID
    s.synchronize()
    assert not any(x.any() for x in eng.inflight_get(M))  # nothing ran
    # the plain batch on the same stream: refused for its reservation, before the snapshot is consulted
    eng2 = pkg.Engine(pkg.default_config([("kv", 1)], max_endpoints=M))
    eng2.reserve_stream(s.cuda_stream, R // 2, 16)
    assert lib.eppscore_schedule_batch(eng2._h, C.byref(_batch(pkg, R, 1, d_outs, s.cuda_stream))) == CAPACITY
    eng2.release_stream(s.cuda_stream)
    eng2.close()
    eng.release_stream(s.cuda_stream)
    eng.close()


def test_staged_entry_point_refusals(pkg):
    lib = pkg.lib()
    M = 64
    eng = pkg.Engine(pkg.default_config([("kv", 1), ("prefix", 1), ("token_load", 1)], max_endpoints=M, max_blocks=16))
    eng.set_snapshot(**synth_snapshot(M, seed=3))
    h = eng._h
    R, k, stride = 4, 2, 3
    data = np.frombuffer(b"a b c d " * 64, np.uint8)
    off = np.arange(0, 5 * 64, 64, dtype=np.int64)
    hashes = np.arange(R * stride, dtype=np.uint64).reshape(R, stride) + 1
    nh = np.full(R, stride, np.uint16)
    nh_long = nh.copy()
    nh_long[2] = stride + 1
    eps = np.zeros((R, k), np.int32)
    out16, out32, out64 = np.zeros(R * 256, np.uint16), np.zeros(R * k, np.int32), np.zeros(R * 256, np.uint64)
    pick = np.zeros(R, np.int32)
    far = 1 << 20  # past every endpoint row
    bad_pick = np.array([0, 1, far, 2], np.int32)
    picks2 = (C.c_void_p * 2)(_p(pick), _p(bad_pick))
    ep_bad = np.array([1, far, 2, 3], np.int32)
    table = [
        ("hash_prompts max_blocks", lib.eppscore_hash_prompts(h, R, 0, _p(data), _p(off), None, None, 64, 70000, _p(out64), _p(out16), None), CAPACITY),
        ("hash_prompts NULL", lib.eppscore_hash_prompts(h, R, 0, None, _p(off), None, None, 64, 16, _p(out64), _p(out16), None), INVALID),
        ("hash_prompts R = 0", lib.eppscore_hash_prompts(h, 0, 0, None, None, None, None, 64, 70000, None, None, None), OK),
        ("count_fields R < 0", lib.eppscore_count_fields(h, -1, 0, _p(data), _p(off), None, _p(out32), None), INVALID),
        ("count_fields NULL", lib.eppscore_count_fields(h, R, 0, _p(data), _p(off), None, None, None), INVALID),
        ("estimate_tokens NULL", lib.eppscore_estimate_tokens(h, R, 0, None, None, None, None, None), INVALID),
        ("prefix_match location", lib.eppscore_prefix_match(h, R, k, 2, _p(hashes), _p(nh), stride, _p(eps), _p(out16), None), INVALID),
        ("prefix_match k", lib.eppscore_prefix_match(h, R, 0, 0, _p(hashes), _p(nh), stride, _p(eps), _p(out16), None), INVALID),
        ("prefix_match stride", lib.eppscore_prefix_match(h, R, k, 0, _p(hashes), _p(nh), 0, _p(eps), _p(out16), None), INVALID),
        ("prefix_match n_hashes", lib.eppscore_prefix_match(h, R, k, 0, _p(hashes), _p(nh_long), stride, _p(eps), _p(out16), None), INVALID),
        ("predict_latency no latency scorer", lib.eppscore_predict_latency(h, R, k, 0, _p(hashes), _p(nh), stride, None, None, None, _p(eps),
                                                                           _p(out64), None, None), INVALID),
        ("commit_picks stride", lib.eppscore_commit_picks(h, R, _p(pick), _p(hashes), _p(nh), 0, None), INVALID),
        ("commit_picks pick range", lib.eppscore_commit_picks(h, R, _p(bad_pick), _p(hashes), _p(nh), stride, None), INVALID),
        ("commit_picks n_hashes", lib.eppscore_commit_picks(h, R, _p(pick), _p(hashes), _p(nh_long), stride, None), INVALID),
        ("commit_picks_profiles pick range", lib.eppscore_commit_picks_profiles(h, R, 2, picks2, _p(hashes), _p(nh), stride, None, 0, 0,
                                                                                None), INVALID),
        ("commit_picks_profiles n_picks", lib.eppscore_commit_picks_profiles(h, R, 0, picks2, _p(hashes), _p(nh), stride, None, 0, 0, None),
         INVALID),
        ("prefix_add n", lib.eppscore_prefix_add(h, _p(np.zeros(70000, np.uint64)), 70000, 1, 0), CAPACITY),
        ("prefix_add endpoint", lib.eppscore_prefix_add(h, _p(hashes), 3, far, 0), INVALID),
        ("prefix_apply endpoint", lib.eppscore_prefix_apply(h, R, _p(hashes), _p(ep_bad), _p(np.zeros(R, np.uint8))), CAPACITY),
    ]
    for what, got, want in table:
        assert got == want, (what, got, want)
    assert not eng.prefix_get(1)  # nothing was committed
    # producer calls: refused before anything moves
    eng.inflight_add(np.array([1, 2], np.int32), np.array([10, 20], np.int64))
    before = eng.inflight_get(M)
    assert lib.eppscore_inflight_add(h, R, 0, _p(ep_bad), _p(np.ones(R, np.int64)), None) == INVALID
    assert lib.eppscore_inflight_release(h, R, 0, _p(ep_bad), _p(np.ones(R, np.int64)), None) == INVALID
    assert lib.eppscore_inflight_add(h, R, 0, None, None, None) == INVALID
    assert all(np.array_equal(x, y) for x, y in zip(before, eng.inflight_get(M)))
    eng.close()

    lat = pkg.Engine(pkg.default_config([("latency", 1)], max_endpoints=M, max_blocks=16))
    lat.set_latency_params(pkg.latency_params())
    lat.set_snapshot(**synth_snapshot(M, seed=3))
    keys = np.arange(R, dtype=np.uint64)
    lat.running_add(np.array([1, 2], np.int32), keys[:2], np.array([0.5, 0.25]))
    before = lat.running_get(M)
    tpot_nan = np.array([0.1, np.nan, 0.1, 0.1])
    assert lib.eppscore_running_add(lat._h, R, 0, _p(ep_bad), _p(keys), _p(np.ones(R)), None, None) == INVALID
    assert lib.eppscore_running_add(lat._h, R, 0, _p(np.ones(R, np.int32)), _p(keys), _p(tpot_nan), None, None) == INVALID
    assert lib.eppscore_running_remove(lat._h, R, 0, _p(ep_bad), _p(keys), None, None) == INVALID
    assert all(np.array_equal(x, y) for x, y in zip(before, lat.running_get(M)))
    info = np.zeros(R * k * 48, np.uint8)
    assert lib.eppscore_predict_latency(lat._h, R, k, 0, _p(hashes), _p(nh_long), stride, None, None, None, _p(eps), _p(info), None,
                                        None) == INVALID
    assert lib.eppscore_predict_latency(lat._h, R, k, 0, _p(hashes), _p(nh), 0, None, None, None, _p(eps), _p(info), None,
                                        None) == INVALID
    assert lib.eppscore_predict_latency(lat._h, R, k, 3, _p(hashes), _p(nh), stride, None, None, None, _p(eps), _p(info), None,
                                        None) == INVALID
    lat.close()
