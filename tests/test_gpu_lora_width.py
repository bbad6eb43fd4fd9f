"""LoRA affinity past 64 adapters on the device, bit for bit against the oracle through the C ABI.

Every snapshot comes from tests/test_lora_width_cpu.wide_lora: adapters a and a ^ 64 are in different classes on every
endpoint, so a kernel that reads word 0 only, or the wrong word stride, changes the results; every batch asks for ids on both
sides of each word edge, past the dictionary (A and A_cap) and at 2^31 - 1.  Each check runs every route that applies: the
sparse pick (a small prefix index, so some requests take exceptions and the rest the summary route), the full matrix with
scores_out, masked, top-k 3, wide top-k 16, and weighted-random and random twins.

  A  max_adapters 65 / 128 / 1000 with W = A_cap / 64 and W - 1 words, M 33 / 1024 / 4097, lora-only and headline profiles
  B  one engine through W = 16 -> 2 -> no LoRA arrays -> lora_words 0 -> 1 -> 16, and a refused W = 17
  C  device-resident snapshots (W = 4) from a side stream, two profiles with their own endpoint subsets, a captured graph
  D  max_adapters 4096 with 8192 requests over 4096 adapters
  E  the host layer's program (tests/cpp/host_lora_width_test.cpp) on the engine"""
import os
import subprocess

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import topk_oracle
from tests.helpers import zipf_adapters
from tests.test_gpu_score_edges import BASIC, DIAG, assert_same, random_mask, uhashes
from tests.test_lora_width_cpu import edge_ids, wide_lora

pytestmark = pytest.mark.gpu

LORA_ONLY = [("lora", 1)]
HEADLINE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
PROFILES = {"lora": LORA_ONLY, "headline": HEADLINE}
GOLDEN = 0x9E3779B97F4A7C15
SEED = 99
RUN = ("pick", "pick_score", "tie_count")  # the per-profile outputs


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def oracle_sd(sd):
    """the oracle's view of a snapshot: lora_words 0 is 'no LoRA arrays' there"""
    if sd.get("lora_active") is not None and sd["lora_active"].shape[1] == 0:
        sd = dict(sd, lora_active=None, lora_waiting=None)
    return o.SnapshotData(**sd)


def request_ids(R, W, a_cap, seed):
    """the edge ids (twice), then Zipf over the snapshot's A = 64 W adapters"""
    edges = edge_ids(W, a_cap) * 2
    rest = zipf_adapters(R - len(edges), A=max(64 * W, 1), seed=seed)
    return np.concatenate([np.array(edges, np.int32), rest]).astype(np.int32)


class WideCase:
    """A max-score engine and its weighted-random and random twins over one snapshot, and the oracle's mirror."""

    def __init__(self, pkg, scorers, max_adapters, max_ep, tie_mode=0, prefix_capacity=1 << 14):
        self.scorers, self.tie_mode = scorers, tie_mode
        self.engines, self.profiles = [], []
        for mode in (0, 1, 2):
            self.engines.append(pkg.Engine(pkg.default_config(scorers, max_endpoints=max_ep, max_adapters=max_adapters, tie_mode=tie_mode,
                                                              tie_seed=SEED, pick_mode=mode, prefix_capacity=prefix_capacity)))
            self.profiles.append(o.make_profile([(pkg.SCORER[k], w) for k, w in scorers], tie_mode=tie_mode, tie_seed=SEED, pick_mode=mode))
        self.idx = o.Index()

    def set_snapshot(self, sd, **kw):
        for eng in self.engines:
            eng.set_snapshot(**sd, **kw)
        self.snap = oracle_sd(sd)

    def add(self, hashes, endpoint):
        h = np.ascontiguousarray(hashes, np.uint64)
        for eng in self.engines:
            eng.prefix_add(h, int(endpoint))
        self.idx.add(h, int(endpoint))

    def close(self):
        for eng in self.engines:
            eng.close()

    def oracle(self, R, mode=0, **kw):
        return o.schedule_batch(self.snap, self.profiles[mode], self.idx, R, want_match=True, want_scores=True, n_threads=8, **kw)

    def check(self, R, kw, mask, where):
        """every route; returns the oracle's unmasked result"""
        eng = self.engines[0]
        want = self.oracle(R, **kw)
        assert_same(eng.schedule(R, **kw), want, BASIC, f"{where} sparse")
        assert_same(eng.schedule(R, want_match=True, want_scores=True, **kw), want, DIAG, f"{where} full matrix")
        for k, arg in ((3, "topk"), (16, "topk_wide")):
            wm, ws = topk_oracle.lists(want["weighted_out"], self.profiles[0], k)
            got = eng.schedule(R, **{arg: k}, **kw)
            assert np.array_equal(got["topk_pick"], wm), f"{where} top-k {k}"
            assert np.array_equal(got["topk_score"].view(np.uint64), ws.view(np.uint64)), f"{where} top-k {k} scores"
        want_m = self.oracle(R, cand_mask=mask, **kw)
        assert_same(eng.schedule(R, cand_mask=mask, **kw), want_m, BASIC, f"{where} masked")
        assert_same(eng.schedule(R, cand_mask=mask, want_scores=True, **kw), want_m, BASIC + ("scores_out",), f"{where} masked diag")
        wm, _ = topk_oracle.lists(want_m["weighted_out"], self.profiles[0], 3)
        assert np.array_equal(eng.schedule(R, topk=3, cand_mask=mask, **kw)["topk_pick"], wm), f"{where} masked top-k"
        for mode in (1, 2):
            assert_same(self.engines[mode].schedule(R, **kw), self.oracle(R, mode=mode, **kw), BASIC, f"{where} pick mode {mode}")
            assert_same(self.engines[mode].schedule(R, cand_mask=mask, **kw), self.oracle(R, mode=mode, cand_mask=mask, **kw), BASIC,
                        f"{where} pick mode {mode} masked")
        return want


def prefix_world(case, M, R, rng, n_hashes=16):
    """8 chains, each cached on 1..6 endpoints, one on more than the sparse pick's exception limit; requests on a chain or on
    an unknown prompt"""
    chains = uhashes(rng, (8, n_hashes))
    for g in range(8):
        n_eps = min(M, 40 if g == 0 else int(rng.integers(1, 7)))
        for ep in rng.choice(M, size=n_eps, replace=False):
            case.add(chains[g, : int(rng.integers(1, n_hashes + 1))], ep)
    gi = rng.integers(0, 9, R)
    hashes = np.where(gi[:, None] < 8, chains[np.minimum(gi, 7)], uhashes(rng, (R, n_hashes)))
    return hashes, rng.integers(0, n_hashes + 1, R).astype(np.uint16)


def check_ids_past_word0(want, ids):
    assert (ids >= 64).any() and (want["pick"][ids >= 64] >= 0).all()


# ------------------------------------------------------------------------------------------ A. widths and geometries
@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("profile", list(PROFILES))
@pytest.mark.parametrize("M", [33, 1024, 4097])
@pytest.mark.parametrize("max_adapters", [65, 128, 1000])
def test_lora_widths_and_geometries(pkg, max_adapters, M, profile, tie_mode):
    a_cap = (max_adapters + 63) // 64 * 64
    R = 333 if M <= 1024 else 205
    rng = np.random.Generator(np.random.PCG64(max_adapters * 10 + M + tie_mode))
    case = WideCase(pkg, PROFILES[profile], max_adapters, M, tie_mode=tie_mode)
    hashes, nh = prefix_world(case, M, R, rng)
    mask = random_mask(rng, R, M, 0.6)
    W = a_cap // 64
    for w in [W, W - 1] if W > 1 else [W]:
        sd, _ = wide_lora(M, w, seed=M + w, focus=edge_ids(w, a_cap), tie_heavy=True)
        case.set_snapshot(sd)
        ids = request_ids(R, w, a_cap, seed=w)
        want = case.check(R, dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=ids), mask, f"A_cap={a_cap} W={w} M={M}")
        check_ids_past_word0(want, ids)
    case.close()


# ------------------------------------------------------------------------------------------ B. snapshot transitions
def test_lora_width_transitions_on_one_engine(pkg):
    """Rows of adapters past the new A still hold the previous snapshot's classes; every id in [new A, old A) must score as
    an unknown adapter.  A snapshot wider than the engine is refused and leaves the previous one in place."""
    M, R, a_cap = 1000, 411, 1024
    rng = np.random.Generator(np.random.PCG64(4242))
    case = WideCase(pkg, HEADLINE, a_cap, 1024, tie_mode=1)
    hashes, nh = prefix_world(case, M, R, rng)
    mask = random_mask(rng, R, M, 0.6)
    ids = request_ids(R, 16, a_cap, seed=16)
    kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=ids)
    base, _ = wide_lora(M, 16, seed=7, focus=edge_ids(16, a_cap), tie_heavy=True)
    plain = {k: base[k] for k in ("kv_usage", "queue", "running", "lora_nmodels", "lora_max")}
    last = None
    for step in (16, 2, "none", 0, 1, 16):
        if step == "none":
            sd = dict(plain)
        elif step == 0:
            sd = dict(plain, lora_active=np.zeros((M, 0), np.uint64), lora_waiting=np.zeros((M, 0), np.uint64))
        else:
            sd, _ = wide_lora(M, step, seed=100 + step, focus=edge_ids(step, a_cap), tie_heavy=True)
        case.set_snapshot(sd)
        want = case.check(R, kw, mask, f"step {step}")
        check_ids_past_word0(want, ids)
        last = want
    wide, _ = wide_lora(M, 17, seed=117)
    for eng in case.engines:
        with pytest.raises(pkg.EppscoreError) as ex:
            eng.set_snapshot(**wide)
        assert ex.value.code == -3
    assert_same(case.engines[0].schedule(R, **kw), last, BASIC, "after the refused snapshot")
    assert_same(case.engines[0].schedule(R, want_match=True, want_scores=True, **kw), last, DIAG, "after the refused snapshot")
    case.close()


# ------------------------------------------------------------------------------------------ C. device-resident snapshots
def to_device(d):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in d.items()}


@pytest.mark.parametrize("pass_words", [True, False])
def test_device_snapshot_profiles_and_graph(pkg, pass_words):
    import torch
    M, R, W, a_cap = 777, 299, 4, 256
    rng = np.random.Generator(np.random.PCG64(5150 + pass_words))
    eng = pkg.Engine(pkg.default_config(HEADLINE, max_endpoints=1024, max_adapters=a_cap, tie_mode=1, tie_seed=SEED))
    second = [("kv", 1), ("lora", 3)]
    pid = eng.add_profile(second, pick_mode=1)
    idx = o.Index()
    chains = uhashes(rng, (6, 12))
    for g in range(6):
        for ep in rng.choice(M, size=int(rng.integers(1, 30)), replace=False):
            h = chains[g, : int(rng.integers(1, 13))]
            eng.prefix_add(h, int(ep))
            idx.add(h, int(ep))
    hashes = chains[rng.integers(0, 6, R)]
    nh = rng.integers(0, 13, R).astype(np.uint16)
    ids = request_ids(R, W, a_cap, seed=W)
    kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=ids)
    subsets = {0: np.arange(0, M, 2), pid: np.arange(0, M, 3)}
    mw = (M + 31) // 32
    sub_bits = {}
    for p, members in subsets.items():
        b = np.zeros(mw * 32, bool)
        b[members] = True
        sub_bits[p] = np.packbits(b.reshape(-1, 32), axis=1, bitorder="little").view("<u4").reshape(mw).astype(np.uint32)
        eng.set_profile_endpoints(p, sub_bits[p])
    words = dict(lora_words=W) if pass_words else {}

    def device_snapshot(sd, stream):
        with torch.cuda.stream(stream):
            dsd = to_device(sd)
        eng.set_snapshot(**dsd, device=True, stream=stream.cuda_stream, **words)
        return dsd

    def oracle(sd, scorers, p, mode):
        prof = o.make_profile([(pkg.SCORER[k], w) for k, w in scorers], tie_mode=1, tie_seed=(SEED ^ (p * GOLDEN)) & (2 ** 64 - 1),
                              pick_mode=mode)
        return o.schedule_batch(o.SnapshotData(**sd), prof, idx, R, want_scores=True, cand_mask=np.tile(sub_bits[p], (R, 1)), **kw)

    side = torch.cuda.Stream()
    sd, _ = wide_lora(M, W, seed=31, focus=edge_ids(W, a_cap), tie_heavy=True)
    keep = device_snapshot(sd, side)  # the engine reads device snapshots in place: kept until the next set_snapshot
    side.synchronize()
    want0, want1 = oracle(sd, HEADLINE, 0, 0), oracle(sd, second, pid, 1)
    check_ids_past_word0(want0, ids)
    _, got = eng.schedule_profiles(R, [dict(profile=0), dict(profile=pid)], **kw)
    assert_same(got[0], want0, RUN, "profile 0")
    assert_same(got[1], want1, RUN, "profile 1")
    _, got = eng.schedule_profiles(R, [dict(profile=0, topk=3), dict(profile=pid, topk=16)], **kw)
    assert_same(got[0], want0, RUN, "profile 0 lists")
    assert_same(got[1], want1, RUN, "profile 1 lists")
    for g, want, scorers, p, mode, k in ((got[0], want0, HEADLINE, 0, 0, 3), (got[1], want1, second, pid, 1, 16)):
        prof = o.make_profile([(pkg.SCORER[s], w) for s, w in scorers], tie_mode=1, tie_seed=(SEED ^ (p * GOLDEN)) & (2 ** 64 - 1),
                              pick_mode=mode)
        wm, ws = topk_oracle.lists(want["weighted_out"], prof, k)
        assert np.array_equal(g["topk_pick"], wm) and np.array_equal(g["topk_score"].view(np.uint64), ws.view(np.uint64)), p

    # a graph that captures set_snapshot + schedule, replayed after the snapshot buffers are rewritten at the same W
    s = torch.cuda.Stream()
    dsd = to_device(sd)
    dev = to_device(kw)
    out = dict(pick=torch.full((R,), -7, dtype=torch.int32, device="cuda"), pick_score=torch.zeros(R, dtype=torch.float64, device="cuda"),
               tie_count=torch.zeros(R, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        eng.set_snapshot(**dsd, device=True, stream=s.cuda_stream, **words)
        eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **dev)  # sizes the scratch outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.set_snapshot(**dsd, device=True, stream=s.cuda_stream, **words)
        eng.schedule(R, device=True, stream=s.cuda_stream, out=out, **dev)
    for seed in (32, 33):
        sd2, _ = wide_lora(M, W, seed=seed, focus=edge_ids(W, a_cap), tie_heavy=True)
        for k, v in sd2.items():
            dsd[k].copy_(torch.from_numpy(np.ascontiguousarray(v)))
        out["pick"].fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        prof = o.make_profile([(pkg.SCORER[k], w) for k, w in HEADLINE], tie_mode=1, tie_seed=SEED)
        want = o.schedule_batch(o.SnapshotData(**sd2), prof, idx, R, cand_mask=np.tile(sub_bits[0], (R, 1)), **kw)
        assert_same({k: v.cpu().numpy() for k, v in out.items()}, want, RUN, f"replay {seed}")
    eng.close()


# ------------------------------------------------------------------------------------------ D. many adapters
def test_four_thousand_adapters(pkg):
    M, R, a_cap = 1024, 8192, 4096
    W = a_cap // 64
    rng = np.random.Generator(np.random.PCG64(4096))
    case = WideCase(pkg, HEADLINE, a_cap, M)
    hashes, nh = prefix_world(case, M, R, rng)
    sd, _ = wide_lora(M, W, seed=4096, focus=edge_ids(W, a_cap), tie_heavy=True)
    case.set_snapshot(sd)
    ids = request_ids(R, W, a_cap, seed=4096)
    eng = case.engines[0]
    kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=ids)
    got = eng.schedule(R, **kw)
    lists = eng.schedule(R, topk=3, **kw)
    rows = np.unique(np.concatenate([np.arange(len(edge_ids(W, a_cap)) * 2), rng.choice(R, 512, replace=False)]))
    want = case.oracle(len(rows), hashes_in=hashes[rows], n_hashes_in=nh[rows], adapter_id=ids[rows])
    assert_same({k: got[k][rows] for k in BASIC}, want, BASIC, "sparse")
    wm, ws = topk_oracle.lists(want["weighted_out"], case.profiles[0], 3)
    assert np.array_equal(lists["topk_pick"][rows], wm) and np.array_equal(lists["topk_score"][rows].view(np.uint64), ws.view(np.uint64))
    assert (ids[rows] >= 64).sum() > 50 and (ids[rows] >= 1024).any()
    case.close()


# ------------------------------------------------------------------------------------------ E. the host layer on the engine
def test_host_layer_lora_width_on_the_engine():
    from tests.test_lora_width_cpu import check_host_program_output
    b = _pkg.load_build()
    lib = b.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out_dir = os.path.join(root, "tests", "cpp", "_build")
    os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "host_lora_width_test_gpu")
    src = os.path.join(root, "tests", "cpp", "host_lora_width_test.cpp")
    host = os.path.join(root, "gateway-api-inference-extension_b200", "host")
    deps = [src, lib] + [os.path.join(host, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", src, "-o", exe, "-pthread", "-L" + os.path.dirname(lib),
                               "-leppscore", "-Wl,-rpath," + os.path.dirname(lib)])
    check_host_program_output(subprocess.run([exe], capture_output=True, text=True, timeout=900))
