"""eppscore_schedule_batch_inorder_index on the GPU, bit-exact against the sequential reference
(tests/inorder_index_reference.py: R single-request oracle schedules, each followed by the prefix match at its pick, the
in-flight add of its tokens and the Add of its blocks): picks, scores (as uint64), tie counts, totals, pick_match, the counters
afterwards and the WHOLE prefix index afterwards (every endpoint's LRU oldest -> newest, the set of every key ever committed,
len(hashToPods)) — at every cluster shape, every picker, with evictions inside the batch, sets moving to bitset rows and
emptied by eviction, candidate masks, supplied hashes with empty rows, batches over two slices, device arrays on a reserved
stream, a CUDA graph, a reserved index without room, a profile without the prefix scorer and a replica that replays the commits."""
import os
import re

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.helpers import synth_prompts, synth_ragged_prompts, synth_snapshot, zipf_adapters
from tests.inorder_index_reference import schedule_inorder_index
from tests.inorder_reference import schedule_inorder

pytestmark = pytest.mark.gpu

FULL = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 1)]
NO_PREFIX = [("queue", 2), ("kv", 2), ("lora", 1), ("token_load", 1)]
SPREAD = [("kv", 1), ("prefix", 1), ("token_load", 3)]  # the load outweighs a prefix: shared blocks reach many endpoints
THR = 8192.0
MB = 32
# kInOrderSliceBytes (csrc/capi.cu): the rows of a slice are this budget over 2 bytes per endpoint
_CAPI = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gateway-api-inference-extension_b200", "csrc",
                          "capi.cu")).read()
_m = re.search(r"constexpr size_t kInOrderSliceBytes = (\d+)ull << (\d+);", _CAPI)
SLICE_BYTES = int(_m.group(1)) << int(_m.group(2))


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")


def _u64(x):
    return np.ascontiguousarray(x).view(np.uint64)


class World:
    """An engine and its oracle twin: the same snapshot, the same warm-up batch committed in both indexes."""

    def __init__(self, pkg, M, scorers=FULL, pick_mode=0, tie_mode=1, seed=0, lru_default=31250, lru_max=0, warm=256,
                 max_endpoints=None):
        self.pkg, self.M = pkg, M
        self.eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=max_endpoints or max(M, 64), token_load_threshold=THR,
                                                 max_blocks=MB, prefix_capacity=1 << 16, pick_mode=pick_mode, tie_mode=tie_mode,
                                                 tie_seed=77, lru_capacity_default=lru_default, lru_capacity_max=lru_max))
        self.sd = synth_snapshot(M, seed=seed)
        self.eng.set_snapshot(**self.sd)
        self.prof = o.make_profile([(pkg.SCORER[s], w) for s, w in scorers], tie_mode=tie_mode, tie_seed=77,
                                   token_load_threshold=THR, pick_mode=pick_mode)
        self.idx, self.tracker = o.Index(lru_default), I.Tracker()
        self.rng = np.random.Generator(np.random.PCG64(seed + 5))
        self.keys = np.zeros(0, np.uint64)
        if warm:
            w = self.workload(warm, seed + 1, groups=8)
            got = self.eng.schedule(warm, want_hashes=True, max_blocks=MB, **w)
            self.eng.commit_picks(got["pick"], got["hashes_out"], got["total_blocks"])
            self.idx.commit(got["pick"], got["hashes_out"], got["total_blocks"])
            self.note_keys(got["pick"], got["hashes_out"], got["total_blocks"])

    def workload(self, R, seed, groups=16, new_groups=0, prompt_len=MB * 64):
        """Shared-prefix prompts: `groups` prefixes of the warm-up (prefix_seed 0) and `new_groups` fresh ones."""
        pb, off, _ = synth_prompts(R, prompt_len=prompt_len, groups=groups, shared=prompt_len // 2, seed=seed, prefix_seed=0)
        if new_groups:
            fresh, _, _ = synth_prompts(R, prompt_len=prompt_len, groups=new_groups, shared=prompt_len // 2, seed=seed + 7,
                                        prefix_seed=seed + 99)
            pb = pb.reshape(R, prompt_len)
            half = np.arange(R) % 2 == 1
            pb[half] = fresh.reshape(R, prompt_len)[half]
            pb = pb.reshape(-1)
        return dict(prompt_bytes=pb, prompt_off=off, model_seed=np.full(R, 5, np.uint64), adapter_id=zipf_adapters(R, seed=seed))

    def tokens(self, R):
        return self.rng.integers(0, 3000, size=R).astype(np.int64)

    def note_keys(self, pick, hashes, n):
        rows = np.asarray(pick) >= 0
        h = np.asarray(hashes)[rows]
        self.keys = np.union1d(self.keys, h[np.arange(h.shape[1])[None, :] < np.asarray(n)[rows][:, None]])

    def reference(self, R, tokens, caps=None, **kw):
        want, _ = schedule_inorder_index(self.sd, self.prof, self.idx, R, tokens, tracker=self.tracker, M=self.M,
                                         lru_capacity=caps, max_blocks=MB, **kw)
        self.note_keys(want["pick"], want["hashes"], want["total_blocks"])
        return want

    def check_outputs(self, got, want, what):
        for k in ("pick", "tie_count", "total_blocks", "pick_match"):
            assert np.array_equal(np.asarray(got[k]), want[k]), (what, k, np.flatnonzero(np.asarray(got[k]) != want[k])[:5])
        assert np.array_equal(_u64(got["pick_score"]), _u64(want["pick_score"])), what
        req, tok = self.eng.inflight_get(self.M)
        wreq, wtok = self.tracker.get(self.M)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), what

    def members(self, eng, idx_or_none, chunk=8192):
        out = np.zeros((len(self.keys), self.M), bool)
        for c0 in range(0, len(self.keys), chunk):
            k = np.ascontiguousarray(self.keys[c0:c0 + chunk], np.uint64)
            kw = dict(hashes_in=k[:, None], n_hashes_in=np.ones(len(k), np.uint16), want_match=True)
            if idx_or_none is None:
                m = eng.schedule(len(k), **kw)["match_blocks"]
            else:
                snap = o.SnapshotData(**self.sd)
                m = o.schedule_batch(snap, self.prof, idx_or_none, len(k), n_threads=8, **kw)["match_blocks"]
            out[c0:c0 + len(k)] = m[:, :self.M] > 0
        return out

    def check_index(self, what, eng=None):
        eng = eng or self.eng
        for m in range(self.M):
            assert eng.prefix_lru_keys(m) == self.idx.lru_keys(m), (what, "lru", m)
        got, want = self.members(eng, None), self.members(None, self.idx)
        bad = np.flatnonzero((got != want).any(axis=1))
        assert len(bad) == 0, (what, f"{len(bad)} of {len(self.keys)} sets differ")
        s = eng.stats()
        assert s.prefix_live_hashes == self.idx.num_hashes(), what
        return s

    def close(self):
        self.eng.close()


def run_host(w, R, tok, caps=None, request_base=0, **kw):
    got = w.eng.schedule_inorder_index(R, tokens=tok, lru_capacity=caps, max_blocks=MB, request_base=request_base, **kw)
    want = w.reference(R, tok, caps=caps, request_base=request_base, **kw)
    return got, want


def test_headline_world(pkg):
    """1024 endpoints, 4096 requests: half the shared-prefix groups new to a warmed index; queue/kv/prefix/lora + token-load.
    Most picks differ from the batch-wide in-order call on the same inputs."""
    M, R = 1024, 4096
    w = World(pkg, M, seed=1)
    kw = w.workload(R, 11, groups=8, new_groups=8)
    tok = w.tokens(R)
    # the batch-wide call on a twin engine with the same history
    twin = World(pkg, M, seed=1)
    wide = twin.eng.schedule_inorder(R, tokens=tok, max_blocks=MB, **kw)
    twin.close()
    got, want = run_host(w, R, tok, **kw)
    w.check_outputs(got, want, "headline")
    w.check_index("headline")
    differ = int((wide["pick"] != got["pick"]).sum())
    print(f"\nheadline: {differ} of {R} picks differ from the batch-wide in-order call")
    assert differ > R // 4, differ
    w.close()


@pytest.mark.parametrize("M", [256, 512, 1024, 2048, 4096, 8192])
def test_every_cluster_shape(pkg, M):
    R = 96
    w = World(pkg, M, seed=M, warm=64)
    kw = w.workload(R, 12, groups=4, new_groups=4)
    got, want = run_host(w, R, w.tokens(R), **kw)
    w.check_outputs(got, want, M)
    w.check_index(M)
    w.close()


@pytest.mark.parametrize("pick_mode,tie_mode", [(0, 0), (0, 1), (1, 1), (2, 1)])
def test_pickers(pkg, pick_mode, tie_mode):
    M, R = 512, 300
    w = World(pkg, M, pick_mode=pick_mode, tie_mode=tie_mode, seed=7)
    kw = w.workload(R, 13, groups=4, new_groups=6)
    got, want = run_host(w, R, w.tokens(R), **kw)
    w.check_outputs(got, want, (pick_mode, tie_mode))
    w.check_index((pick_mode, tie_mode))
    w.close()


def test_evictions_rows_and_per_endpoint_capacities(pkg):
    """LRUs smaller than a few calls (evictions inside the batch; a capacity 3 below n_hashes takes the sequential path), per
    endpoint capacities with LRUs created mid-batch, blocks reaching more than 10 endpoints (bitset rows) and sets emptied by
    eviction — each of which the test checks did happen, by replaying the reference's commits."""
    M, R = 64, 600
    w = World(pkg, M, scorers=SPREAD, seed=9, lru_default=40, lru_max=64, warm=0)
    caps = np.zeros(M, np.int32)
    caps[::3] = 29   # below one call's 32 blocks: the sequential path
    caps[1::3] = 64
    kw = w.workload(R, 14, groups=2, new_groups=3)
    got, want = run_host(w, R, w.tokens(R), caps=caps, **kw)
    w.check_outputs(got, want, "evictions")
    w.check_index("evictions")
    # the paths the batch took, from a replay of its commits on a fresh oracle index
    rep, widest, sequential = o.Index(40), 0, 0
    for r in range(R):
        p, n = int(want["pick"][r]), int(want["total_blocks"][r])
        if p < 0:
            continue
        rep.commit(want["pick"][r:r + 1], want["hashes"][r:r + 1], want["total_blocks"][r:r + 1], caps)
        sequential += int(caps[p] == 29 and n > 29)
        widest = max(widest, len(rep.get(int(want["hashes"][r, 0]))) if n else 0)
    assert sequential > 0, "no call took the sequential path"
    assert widest > 10, "no set reached a bitset row"
    assert rep.num_hashes() < len(w.keys), "no set was emptied by eviction"  # (every key was committed once)
    w.close()


def test_masks_hashes_in_empty_rows_and_unpicked(pkg):
    """cand_mask (rows without candidates give pick -1 and add nothing), a profile-0 endpoint subset, supplied hashes with
    empty rows and requests with 0 hashes."""
    M, R = 256, 400
    w = World(pkg, M, seed=15)
    sub = np.full(M // 32, 0xFFFFFFFF, np.uint32)
    sub[1] = 0x0000FFFF
    w.eng.set_profile_endpoints(0, sub)
    w.eng.set_snapshot(**w.sd)
    member = np.unpackbits(sub.view(np.uint8), bitorder="little").astype(bool)[:M]
    kw = w.workload(R, 16, groups=4, new_groups=4)
    h = w.eng.schedule(R, want_hashes=True, max_blocks=MB, **kw)
    n = h["total_blocks"].copy()
    n[::5] = 0
    mask = w.rng.integers(0, 2 ** 32, size=(R, M // 32), dtype=np.uint64).astype(np.uint32)
    mask[::7] = 0
    # the reference's profile subset: folded into the candidate masks
    mref = mask & np.packbits(member, bitorder="little").view(np.uint32)[None, :]
    tok = w.tokens(R)
    args = dict(hashes_in=h["hashes_out"], n_hashes_in=n, adapter_id=kw["adapter_id"])
    got = w.eng.schedule_inorder_index(R, tokens=tok, cand_mask=mask, **args)
    want = w.reference(R, tok, cand_mask=mref, **args)
    assert (want["pick"] == -1).any()
    w.check_outputs(got, want, "inputs")
    w.check_index("inputs")
    w.close()


def test_two_slices(pkg):
    """At 8192 endpoints a slice is kInOrderSliceBytes / (2 * 8192) rows: 52 requests more take two slices."""
    M = 8192
    rows = SLICE_BYTES // (2 * M)
    R = rows + 52
    w = World(pkg, M, seed=17, warm=64, max_endpoints=M)
    kw = w.workload(R, 18, groups=4, new_groups=4, prompt_len=256)
    got, want = run_host(w, R, w.tokens(R), **kw)
    w.check_outputs(got, want, "slices")
    w.check_index("slices")
    w.close()


def test_device_reserved_stream_and_graph(pkg):
    """device arrays on a reserved stream; then a CUDA graph on a reserved index, captured after one call outside the capture
    and replayed twice, equals two more rounds of the loop"""
    import torch
    M, R = 512, 512
    w = World(pkg, M, seed=19)
    w.eng.prefix_reserve()
    kw = w.workload(R, 20, groups=4, new_groups=4)
    tok = w.tokens(R)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream()
    w.eng.reserve_stream(s.cuda_stream, R, MB)
    d_in = {k: _dev(v) for k, v in kw.items()}
    d_tok = _dev(tok)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.uint16, device=dev),
               hashes_out=torch.zeros((R, MB), dtype=torch.int64, device=dev),
               pick_match=torch.empty(R, dtype=torch.uint16, device=dev))

    def step(base):
        w.eng.schedule_inorder_index(R, tokens=d_tok, device=True, stream=s.cuda_stream, out=out, max_blocks=MB,
                                     request_base=base, **d_in)

    def check(rnd):
        want = w.reference(R, tok, request_base=0, **kw)
        got = {k: v.cpu().numpy() for k, v in out.items()}
        w.check_outputs(got, want, ("device", rnd))
        assert np.array_equal(_u64(got["hashes_out"]), want["hashes"])
        w.check_index(("device", rnd))

    torch.cuda.synchronize()
    step(0)
    torch.cuda.synchronize()
    check(0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step(0)
    for rnd in (1, 2):
        g.replay()
        torch.cuda.synchronize()
        check(rnd)
    assert w.eng.stats().index_error == 0
    w.eng.release_stream(s.cuda_stream)
    w.close()


def test_reserved_index_without_room(pkg):
    """A slice without room is walked without commits: the index is unchanged, the outputs equal schedule_inorder's on the
    frozen index, and the next index call reports the skip."""
    M, R = 256, 200
    w = World(pkg, M, seed=23, warm=0)
    w.eng.prefix_reserve(live_hashes=16, touches_per_call=16, overflow_rows=16)
    kw = w.workload(R, 24, groups=2, new_groups=2)
    tok = w.tokens(R)
    got = w.eng.schedule_inorder_index(R, tokens=tok, max_blocks=MB, **kw)
    want, _ = schedule_inorder(w.sd, w.prof, w.idx, R, tok, tracker=w.tracker, M=M, max_blocks=MB, **kw)
    for k in ("pick", "tie_count", "total_blocks"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(_u64(got["pick_score"]), _u64(want["pick_score"]))
    assert w.eng.stats().prefix_live_hashes == 0
    assert all(w.eng.prefix_lru_len(m) == -1 for m in range(M))
    assert w.eng.stats().index_error & 4
    with pytest.raises(pkg.EppscoreError) as e:
        w.eng.schedule_inorder_index(R, tokens=tok, max_blocks=MB, **kw)
    assert e.value.code == -3
    w.close()


def test_without_prefix_scorer_and_replay(pkg):
    """Without the prefix scorer the call equals schedule_inorder followed by one batch commit; a second engine that replays
    (pick, hashes_out) through eppscore_commit_picks ends with an identical index."""
    M, R = 512, 700
    a = World(pkg, M, scorers=NO_PREFIX, seed=29)
    b = World(pkg, M, scorers=NO_PREFIX, seed=29)
    kw = a.workload(R, 30, groups=4, new_groups=4)
    tok = a.tokens(R)
    got = a.eng.schedule_inorder_index(R, tokens=tok, max_blocks=MB, want_hashes=True, **kw)
    plain = b.eng.schedule_inorder(R, tokens=tok, max_blocks=MB, want_hashes=True, **kw)
    for k in ("pick", "tie_count", "total_blocks", "hashes_out"):
        assert np.array_equal(got[k], plain[k]), k
    b.eng.commit_picks(plain["pick"], plain["hashes_out"], plain["total_blocks"])
    want = a.reference(R, tok, **kw)
    a.check_outputs(got, want, "no prefix")
    a.check_index("no prefix")
    a.check_index("replay", eng=b.eng)
    a.close()
    b.close()


def test_refusals(pkg):
    M, R = 128, 16
    w = World(pkg, M, seed=31, warm=0)
    kw = w.workload(R, 32)
    for flag in ("want_match", "want_scores"):
        with pytest.raises(ValueError):
            w.eng.schedule_inorder_index(R, **{flag: True}, **kw)
    w.close()
    eng = pkg.Engine(pkg.default_config([("latency", 1), ("prefix", 1)], max_endpoints=M))
    eng.set_latency_params(pkg.latency_params())
    eng.set_snapshot(**synth_snapshot(M, seed=1))
    with pytest.raises(pkg.EppscoreError) as e:
        eng.schedule_inorder_index(R, **kw)
    assert e.value.code == -1
    assert eng.stats().prefix_live_hashes == 0
    eng.close()


def test_host_program_on_the_engine(pkg):
    """SchedulerConfig::InOrderPrefixIndex of the C++ host layer (tests/cpp/host_inorder_index_test.cpp) on the engine itself:
    the batch equals a Scheduler fed one request at a time, the index is committed once, PrefixCacheMatchInfo is the match
    before each request's own Add, and the refusals."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cpp, pkgdir = os.path.join(root, "tests", "cpp"), os.path.join(root, "gateway-api-inference-extension_b200")
    import tempfile
    exe = os.path.join(tempfile.mkdtemp(), "host_inorder_index_engine")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread",
                           os.path.join(cpp, "host_inorder_index_test.cpp"), os.path.join(cpp, "engine_inorder_index_shim.cpp"),
                           "-I" + os.path.join(root, "include"), "-L" + pkgdir, "-leppscore", "-Wl,-rpath," + pkgdir,
                           "-Wl,--wrap=eppscore_schedule_batch_inorder_index", "-Wl,--wrap=eppscore_commit_picks", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host inorder index: all checks passed" in r.stdout
