"""eppscore_schedule_batch_inorder at the edges of its kernels, bit-exact against the sequential reference
(tests/inorder_reference.py): every cluster width of inorder_pick_kernel (each padded endpoint count from 256 to 8192, filled,
one past the previous one, and mostly empty); every scorer kind the kernel scores itself (running, endpoint columns, absent
pair columns), zero, negative and repeated weights in two profile orders, flat columns and queue values past 2^53; the
token-load threshold reached exactly, passed, at its default and with no tokens; counters moved by adds, releases and endpoint
removals between batches; the weighted-random picker emptying into its uniform fallback and the random picker at C = 1 and
C >= 8; tie-heavy snapshots with a tie seed whose both words are nonzero at C = 8 and 16; profile-0 subsets; LoRA classes past
64 adapters, full 256-block matches and wide block counters, supplied hashes with empty rows; a profile without a
load-dependent scorer against one plain batch and one inflight_add; and batches on several streams with no host sync between
them.  Every comparison is of exact bits (scores as uint64) or exact integers."""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests.helpers import synth_ragged_prompts, synth_snapshot, zipf_adapters
from tests.inorder_reference import schedule_inorder
from tests.test_gpu_inorder import FOUR, MB, THR, TL, World, _dev

pytestmark = pytest.mark.gpu

SEED = 0x9E3779B97F4A7C15  # tie seed with both 32-bit words nonzero
QR = [("queue", 1), ("running", 2), ("kv", 1), ("token_load", 1)]


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def mpad(max_endpoints):
    """the engine's padded endpoint count (kernels.cuh make_geo): 256, 512, then 1024 << {0..3}"""
    if max_endpoints <= 512:
        return 256 if max_endpoints <= 256 else 512
    return 1024 << max(0, (max_endpoints - 1).bit_length() - 10)


def cluster_of(max_endpoints):
    """(C, T) of inorder_pick_kernel: C = clamp(Mpad / 256, 1, 16) CTAs of T = Mpad / C threads (inorder_cluster_size on an
    H100, which grants the non-portable cluster size 16).  The engine does not report the shape, so the cases name it."""
    p = mpad(max_endpoints)
    C = min(max(p // 256, 1), 16)
    return C, p // C


class EdgeWorld(World):
    """tests/test_gpu_inorder.World with the engine options the edges need.  max_endpoints defaults to max(M, 64); `sd`
    replaces the synthetic snapshot (synth_snapshot(M, A, seed, tie_heavy)); `subset` is profile 0's endpoint mask
    (set_profile_endpoints before the snapshot; the reference composes it into cand_mask).  The counters are checked up to
    max_endpoints: nothing may move those past M."""

    def __init__(self, pkg, M, scorers, pick_mode=0, tie_mode=0, seed=0, *, max_endpoints=None, token_load_threshold=THR,
                 tie_seed=77, tie_heavy=False, A=64, max_blocks=MB, sd=None, subset=None):
        self.pkg, self.M, self.A, self.mb = pkg, M, A, max_blocks
        self.me = max(M, 64) if max_endpoints is None else max_endpoints
        self.subset = subset
        wide = dict(max_adapters=64 * ((A + 63) // 64)) if A > 64 else {}  # the snapshot's lora_words * 64 adapters
        self.eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=self.me, token_load_threshold=token_load_threshold,
                                                 max_blocks=max_blocks, prefix_capacity=1 << 16, pick_mode=pick_mode,
                                                 tie_mode=tie_mode, tie_seed=tie_seed, **wide))
        self.sd = synth_snapshot(M, A=A, seed=seed, tie_heavy=tie_heavy) if sd is None else sd
        if subset is not None:
            self.eng.set_profile_endpoints(0, subset)
        self.eng.set_snapshot(**self.sd)
        self.prof = o.make_profile([(pkg.SCORER[s], w) for s, w in scorers], tie_mode=tie_mode, tie_seed=tie_seed,
                                   token_load_threshold=token_load_threshold, pick_mode=pick_mode)
        self.idx, self.tracker = o.Index(), I.Tracker()
        self.rng = np.random.Generator(np.random.PCG64(seed + 5))
        w = self.workload(256, seed + 1)
        warm = self.eng.schedule(256, want_hashes=True, max_blocks=max_blocks, **w)
        self.eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
        self.idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])

    def workload(self, R, seed):
        pb, off = synth_ragged_prompts(R, max_len=min(self.mb, MB) * 64, seed=seed)
        return dict(prompt_bytes=pb, prompt_off=off, model_seed=np.full(R, 5, np.uint64),
                    adapter_id=zipf_adapters(R, A=self.A, seed=seed))

    def cand(self, R, mask=None):
        """the reference's candidates: profile 0's subset ∧ cand_mask (None when neither is set)"""
        if self.subset is None:
            return mask
        mw = (self.M + 31) // 32
        sub = np.zeros(mw, np.uint32)
        n = min(mw, np.asarray(self.subset).size)
        sub[:n] = np.asarray(self.subset, np.uint32)[:n]
        out = np.tile(sub, (R, 1))
        return out if mask is None else out & mask

    def reference(self, R, tokens, request_base=0, cand_mask=None, **kw):
        want, _ = schedule_inorder(self.sd, self.prof, self.idx, R, tokens, tracker=self.tracker, request_base=request_base,
                                   max_blocks=self.mb, cand_mask=self.cand(R, cand_mask), **kw)
        return want

    def check(self, got, want, what):
        for k in ("pick", "tie_count", "total_blocks"):
            assert np.array_equal(np.asarray(got[k]), want[k]), (what, k)
        assert np.array_equal(np.asarray(got["pick_score"]).view(np.uint64), want["pick_score"].view(np.uint64)), what
        req, tok = self.eng.inflight_get(self.me)
        wreq, wtok = self.tracker.get(self.me)
        assert np.array_equal(req, wreq) and np.array_equal(tok, wtok), what


def run(w, R, tok, mask=None, rounds=1, kw=None, seed=3, what="", **extra):
    """`rounds` in-order batches of the same R requests (request_base moving on), each checked against the reference; returns
    the last (got, want)"""
    kw = w.workload(R, seed) if kw is None else kw
    for rnd in range(rounds):
        got = w.eng.schedule_inorder(R, tokens=tok, cand_mask=mask, max_blocks=w.mb, request_base=rnd * R, **kw)
        want = w.reference(R, tok, request_base=rnd * R, cand_mask=mask, **kw, **extra)
        w.check(got, want, (what, rnd))
    return got, want


def tied_endpoints(w, want, tok, load0, kw):
    """(r, endpoints) for every request r with tie_count > 1: the set its pick was drawn from, by a single-request oracle
    schedule with the token counters the picks of requests 0..r-1 left (load0: the counters before the batch)"""
    load = np.array(load0, np.int64)
    for r in range(len(want["pick"])):
        if want["tie_count"][r] > 1:
            a, b = int(kw["prompt_off"][r]), int(kw["prompt_off"][r + 1])
            x = o.schedule_batch(o.SnapshotData(**w.sd, inflight_tokens=load), w.prof, w.idx, 1, request_base=r, max_blocks=w.mb,
                                 want_tie_set=True, prompt_bytes=np.ascontiguousarray(kw["prompt_bytes"][a:b]),
                                 prompt_off=np.array([0, b - a], np.int64), model_seed=kw["model_seed"][r:r + 1],
                                 adapter_id=kw["adapter_id"][r:r + 1])
            assert x["pick"][0] == want["pick"][r]
            yield r, np.nonzero(np.unpackbits(x["tie_set"][0].view(np.uint8), bitorder="little")[:w.M])[0]
        if want["pick"][r] >= 0:
            load[want["pick"][r]] += tok[r]


def spread(M, n):
    """n endpoints < M spread evenly, so that they fall in different CTAs whenever the cluster has several"""
    return sorted({int(x) for x in np.linspace(0, M - 1, n)})


def rows_with(M, R, members):
    mw = (M + 31) // 32
    m = np.zeros((R, mw), np.uint32)
    for e in members:
        m[:, e >> 5] |= np.uint32(1 << (e & 31))
    return m


# ---------------------------------------------------------------------------------------------------------------------------
# every cluster width

CLUSTER_CASES = [  # (M, max_endpoints, R, scorers, pick_mode, tie_mode, masked)
    (256, 256, 1500, FOUR, 0, 1, True),       # M fills Mpad 256
    (257, 257, 1500, FOUR, 1, 0, False),      # one past Mpad 256
    (512, 512, 1000, FOUR, 0, 0, True),       # fills Mpad 512
    (513, 513, 1000, TL, 2, 1, False),        # one past Mpad 512
    (1025, 1025, 600, FOUR, 1, 1, True),      # one past Mpad 1024
    (2048, 2048, 500, FOUR, 0, 1, False),     # fills Mpad 2048
    (2049, 2049, 400, TL, 1, 0, True),        # one past Mpad 2048
    (4096, 4096, 250, FOUR, 0, 0, True),      # fills Mpad 4096
    (300, 4096, 2000, TL, 0, 1, False),       # Mpad 4096 with 14 of its 16 CTAs holding no endpoint
    (300, 8192, 2000, TL, 1, 1, True),        # Mpad 8192 with 15 of its 16 CTAs holding no endpoint
]


def _cluster_id(case):
    M, me, R, scorers, pm, tm, masked = case
    C, T = cluster_of(me)
    return f"Mpad{mpad(me)}-C{C}xT{T}-M{M}-R{R}-{'tl' if scorers is TL else 'four'}-pick{pm}-tie{tm}{'-masked' if masked else ''}"


@pytest.mark.parametrize("M,me,R,scorers,pick_mode,tie_mode,masked", CLUSTER_CASES, ids=[_cluster_id(c) for c in CLUSTER_CASES])
def test_cluster_shapes_match_sequential_reference(pkg, M, me, R, scorers, pick_mode, tie_mode, masked):
    """the cluster width the engine derives from max_endpoints (C = clamp(Mpad / 256, 1, 16)), with endpoints past M holding
    counters from an earlier inflight_add: those come back unchanged"""
    w = EdgeWorld(pkg, M, scorers, pick_mode, tie_mode, seed=M + me, max_endpoints=me)
    far = np.array(sorted({m for m in (M, M + 1, M + 257, me - 1) if M <= m < me}), np.int32)
    if far.size:
        w.eng.inflight_add(far, np.full(far.size, 1234, np.int64))
        w.tracker.add(far, np.full(far.size, 1234, np.int64))
    mask = w.masks(R) if masked else None
    got, want = run(w, R, w.tokens(R), mask, rounds=2, seed=4, what=(M, me, R))
    if far.size:
        assert (w.eng.inflight_get(me)[1][far] == 1234).all()
    C, T = cluster_of(me)
    if C > 1:  # the picks reach past the first CTA (else the cluster merge is not exercised)
        assert (want["pick"] >= T).any() or M <= T
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# scorer kinds and weights

def _snap(kind, M, seed):
    sd = synth_snapshot(M, seed=seed)
    rng = np.random.Generator(np.random.PCG64(seed + 17))
    if kind == "cols":  # values outside [0, 1] too: the range is enforced before the weight
        sd["endpoint_cols"] = [rng.uniform(-0.25, 1.25, M) for _ in range(4)]
    elif kind == "flat":  # mx == mn for both min / max columns on every candidate set, and one kv value
        sd.update(queue=np.full(M, 7, np.int64), running=np.full(M, 3, np.int64), kv_usage=np.full(M, 0.5))
    elif kind == "spread":  # ranges past 2^53: (double)(mx - q) rounds; |values| < 2^61, so no int64 difference overflows
        sd.update(queue=rng.integers(-2 ** 61, 2 ** 61, M, dtype=np.int64),
                  running=(2 ** 60 + rng.integers(0, 2 ** 55, M, dtype=np.int64)) * rng.choice([-1, 1], M))
    return sd


def _mask(kind, w, R):
    if kind == "rand":
        return w.masks(R)
    if kind == "one":  # one candidate per request, every third row; the rest random
        m = w.masks(R)
        e = w.rng.integers(0, w.M, R)
        for r in range(0, R, 3):
            m[r] = 0
            m[r, e[r] >> 5] = np.uint32(1 << (e[r] & 31))
        return m
    return None


SIGNED = [("token_load", 1), ("kv", 0), ("queue", -1), ("token_load", -0.25), ("prefix", 3), ("lora", 0.5), ("running", 0.75)]
SCORER_CASES = {  # name: (M, max_endpoints, R, scorers, snapshot, mask, pick_mode, tie_mode)
    "running-C2": (300, 512, 600, [("running", 1), ("token_load", 1)], "synth", "rand", 0, 0),
    "queue+running-C8": (1500, 2048, 300, QR, "synth", "rand", 0, 1),
    "cols-C4": (700, 1024, 500, [("col0", 1), ("col1", -0.5), ("col2", 2), ("col3", 1), ("token_load", 1)], "cols", None, 0, 1),
    "pairs-C16": (300, 4096, 800, [("pair0", 1.5), ("kv", 1), ("pair1", -2), ("token_load", 1)], "synth", "rand", 0, 0),
    "signed-order-a-C4": (600, 1024, 500, SIGNED, "synth", "rand", 0, 1),
    "signed-order-b-C4": (600, 1024, 500, SIGNED[::-1], "synth", "rand", 0, 1),
    "signed-weighted-random-C8": (1100, 2048, 300, SIGNED[2:] + SIGNED[:2], "synth", "rand", 1, 0),
    "flat-C1": (200, 256, 800, [("queue", 2), ("running", 1), ("kv", 1), ("token_load", 1)], "flat", "rand", 0, 0),
    "one-candidate-C4": (1000, 1024, 400, QR + [("prefix", 2)], "synth", "one", 0, 1),
    "int64-spread-C8": (1200, 2048, 300, [("queue", 1), ("running", 1), ("token_load", 0.001)], "spread", "rand", 0, 0),
}


@pytest.mark.parametrize("name", list(SCORER_CASES))
def test_scorer_kinds_and_weights(pkg, name):
    M, me, R, scorers, snap, mk, pm, tm = SCORER_CASES[name]
    seed = sum(map(ord, name))
    w = EdgeWorld(pkg, M, scorers, pm, tm, seed=seed, max_endpoints=me, tie_seed=SEED, sd=_snap(snap, M, seed))
    mask = _mask(mk, w, R)
    run(w, R, w.tokens(R), mask, rounds=2, what=name)
    if snap == "spread":
        assert int(w.sd["queue"].max()) - int(w.sd["queue"].min()) > 2 ** 53
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the token-load threshold and the counters

@pytest.mark.parametrize("me", [256, 2048], ids=lambda me: f"C{cluster_of(me)[0]}")
@pytest.mark.parametrize("case", ["small", "exact", "default", "no-tokens"])
def test_threshold_edges(pkg, case, me):
    M = me
    cand = spread(M, 6)
    scorers = {"small": [("kv", 0.5), ("token_load", 1)], "exact": TL, "default": [("token_load", 2), ("kv", 1)],
               "no-tokens": FOUR}[case]
    thr = {"small": 300.0, "exact": 1000.0, "default": 0.0, "no-tokens": THR}[case]
    w = EdgeWorld(pkg, M, scorers, 0, 0, seed=me + len(case), max_endpoints=me, token_load_threshold=thr)
    if case == "small":  # endpoints saturate within the batch, then stay at 0
        R = 200
        tok = w.rng.integers(0, 121, R).astype(np.int64)
        run(w, R, tok, rows_with(M, R, cand), what=case)
        assert (w.tracker.get(M)[1] > thr).sum() >= 3
    elif case == "exact":  # 250 tokens at a time: after four picks each candidate holds exactly the threshold
        R = 4 * len(cand)
        tok = np.full(R, 250, np.int64)
        run(w, R, tok, rows_with(M, R, cand), what=case)
        assert (w.tracker.get(M)[1][cand] == 1000).all()
        run(w, R, tok, rows_with(M, R, cand), what=case + "-past")  # every candidate at 0: ties until the batch ends
    elif case == "default":  # threshold 0 is 4194304 on both sides; estimates of that size pass it
        R = 80
        tok = w.rng.integers(0, 3_000_000, R).astype(np.int64)
        run(w, R, tok, rows_with(M, R, cand), what=case)
        assert (w.tracker.get(M)[1] > 4194304).any()
    else:  # tokens=None: every pick is counted as a request, no token is added
        R = 300
        got, want = run(w, R, None, w.masks(R), what=case)
        req, tok = w.eng.inflight_get(M)
        assert int(req.sum()) == int((want["pick"] >= 0).sum()) > 0 and not tok.any()
    w.eng.close()


def test_counters_moved_between_batches(pkg):
    """adds, releases that leave token counters negative and endpoint removals, on the engine and the tracker alike, before
    and between in-order batches"""
    M, R = 1024, 300
    w = EdgeWorld(pkg, M, FOUR + [("running", 0.5)], 0, 1, seed=91, token_load_threshold=4000.0, tie_seed=SEED)
    eps = np.array(spread(M, 12), np.int32)

    def both(op, endpoint, tokens=None):
        getattr(w.eng, "inflight_" + op)(endpoint, tokens)
        getattr(w.tracker, op)(endpoint, tokens)

    both("add", eps, np.arange(1, 13, dtype=np.int64) * 500)
    both("release", eps[:4], np.full(4, 9000, np.int64))           # below zero before the first batch
    kw = w.workload(R, 5)
    tok = w.tokens(R)
    for rnd in range(3):
        got = w.eng.schedule_inorder(R, tokens=tok, max_blocks=MB, request_base=rnd * R, **kw)
        w.check(got, w.reference(R, tok, request_base=rnd * R, **kw), rnd)
        sel = np.nonzero(got["pick"] >= 0)[0]
        both("release", got["pick"][sel[:50]], tok[sel[:50]] + 7)  # a little more than was added
        e = int(got["pick"][sel[-1]])
        w.eng.inflight_remove_endpoint(e)
        w.tracker.remove(e)
        both("release", np.array([e], np.int32), np.array([300 + rnd], np.int64))
        both("add", eps[rnd::3], None)                             # requests counted, no tokens
        req, tk = w.eng.inflight_get(M)
        wreq, wtk = w.tracker.get(M)
        assert np.array_equal(req, wreq) and np.array_equal(tk, wtk), rnd
        assert (tk < 0).any()
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the stochastic pickers

@pytest.mark.parametrize("me", [256, 2048], ids=lambda me: f"C{cluster_of(me)[0]}")
@pytest.mark.parametrize("case", ["weighted-to-uniform", "nonpositive-weighted", "random"])
def test_pickers(pkg, case, me):
    M = me
    if case == "weighted-to-uniform":  # scores reach 0 as the candidates saturate: the A-Res state empties mid-batch
        w = EdgeWorld(pkg, M, TL, 1, 0, seed=me + 1, max_endpoints=me, token_load_threshold=300.0, tie_seed=SEED)
        R = 120
        got, want = run(w, R, w.rng.integers(40, 160, R).astype(np.int64), rows_with(M, R, spread(M, 8)), what=case)
        assert (want["pick_score"] > 0).any() and ((want["pick"] >= 0) & (want["pick_score"] == 0)).any()
        assert (want["tie_count"][want["pick_score"] == 0] == 8).all()  # the uniform draw is over every candidate
    elif case == "nonpositive-weighted":  # no score is ever > 0: every request takes the uniform draw
        w = EdgeWorld(pkg, M, [("kv", -1), ("token_load", -0.5), ("queue", -2), ("prefix", 0)], 1, 1, seed=me + 2, max_endpoints=me,
                  tie_seed=SEED)
        R = 400
        got, want = run(w, R, w.tokens(R), w.masks(R), rounds=2, what=case)
        assert (want["pick_score"][want["pick"] >= 0] <= 0).all()
    else:
        w = EdgeWorld(pkg, M, FOUR, 2, 0, seed=me + 3, max_endpoints=me, tie_seed=SEED)
        R = 400
        got, want = run(w, R, w.tokens(R), w.masks(R), rounds=2, what=case)
    C, T = cluster_of(me)
    if C > 1:
        assert len(set((want["pick"][want["pick"] >= 0] // T).tolist())) > 1  # picks from several CTAs
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# ties across CTAs

@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("me", [2048, 4096], ids=lambda me: f"C{cluster_of(me)[0]}")
def test_ties_across_ctas(pkg, me, tie_mode):
    M, R = me, 300
    w = EdgeWorld(pkg, M, [("kv", 1), ("token_load", 1)], 0, tie_mode, seed=me + tie_mode, max_endpoints=me, tie_seed=SEED,
              tie_heavy=True)
    assert SEED >> 32 and SEED & 0xFFFFFFFF
    kw, tok = w.workload(R, 3), w.tokens(R)
    load0 = w.tracker.get(M)[1].copy()
    got, want = run(w, R, tok, kw=kw, what=(me, tie_mode))
    C, T = cluster_of(me)
    crossing = 0
    for r, members in tied_endpoints(w, want, tok, load0, kw):
        assert len(members) == want["tie_count"][r]
        crossing += len(set((members // T).tolist())) > 1
    assert crossing >= 10, crossing
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# profile-0 subsets

@pytest.mark.parametrize("masked", [False, True], ids=["subset", "subset+mask"])
@pytest.mark.parametrize("where", ["one-cta", "spread"])
def test_profile0_subset(pkg, where, masked):
    M, R = 2048, 400
    C, T = cluster_of(M)
    members = [m for m in range(2 * T, 3 * T) if m % 3 == 0] if where == "one-cta" else [m for m in range(M) if m % 5 in (0, 2)]
    sub = np.zeros(M // 32, np.uint32)
    for m in members:
        sub[m >> 5] |= np.uint32(1 << (m & 31))
    w = EdgeWorld(pkg, M, QR + [("prefix", 2)], 0, 1, seed=len(where) + masked, tie_seed=SEED, subset=sub)
    mask = None
    if masked:
        mask = w.masks(R)
        mask[3::11] = ~sub  # subset ∧ mask empty: pick -1, no counter moves
    got, want = run(w, R, w.tokens(R), mask, rounds=2, what=(where, masked))
    assert set(want["pick"][want["pick"] >= 0].tolist()) <= set(members)
    if masked:
        assert (got["pick"][3::11] == -1).all() and (got["tie_count"][3::11] == 0).all()
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# adapters and blocks

@pytest.mark.parametrize("A", [100, 200])
def test_adapters_past_64(pkg, A):
    M, R = 600, 500
    w = EdgeWorld(pkg, M, FOUR, 0, 1, seed=A, max_endpoints=1024, A=A)
    kw = w.workload(R, 6)
    ad = kw["adapter_id"]
    W64 = 64 * ((A + 63) // 64)
    ad[::9] = -1
    ad[1::9] = A            # past the adapters any endpoint holds, inside the dictionary's words
    ad[2::9] = W64 - 1
    ad[3::9] = W64          # past the dictionary
    ad[4::9] = 100000
    ad[5::9] = A - 1
    assert (ad >= 64).sum() > R // 4
    run(w, R, w.tokens(R), w.masks(R), rounds=2, kw=kw, what=A)
    w.eng.close()


def _long_prompts(n, nbytes, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    pb = rng.integers(97, 123, size=n * nbytes, dtype=np.uint8)
    return pb, np.arange(n + 1, dtype=np.int64) * nbytes


@pytest.mark.parametrize("mb,me", [(256, 256), (256, 2048), (320, 1024)], ids=["mb256-C1", "mb256-C8", "mb320-wide-C4"])
def test_full_matches(pkg, mb, me):
    """prompts committed in a warm-up batch and sent again: every block matches on the warm-up pick.  At max_blocks 256 that is
    a count of 256 (the 8-bit counters' wrap to 0); past 256 the counters are 16-bit"""
    M, K = me - 7, 24
    w = EdgeWorld(pkg, M, FOUR, 0, 1, seed=mb + me, max_endpoints=me, max_blocks=mb)
    pb, off = _long_prompts(K, mb * 64 + 50, mb)
    seeds = np.full(K, 5, np.uint64)
    warm = w.eng.schedule(K, prompt_bytes=pb, prompt_off=off, model_seed=seeds, want_hashes=True, max_blocks=mb)
    w.eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    w.idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    assert (warm["total_blocks"] == mb).all()
    R = 2 * K
    pb2 = np.concatenate([pb, _long_prompts(K, 3000, mb + 1)[0]])
    off2 = np.concatenate([off, off[-1] + np.arange(1, K + 1, dtype=np.int64) * 3000])
    kw = dict(prompt_bytes=pb2, prompt_off=off2, model_seed=np.full(R, 5, np.uint64), adapter_id=np.full(R, -1, np.int32))
    got, want = run(w, R, np.full(R, 100, np.int64), rounds=2, kw=kw, what=(mb, me))
    assert (want["total_blocks"][:K] == mb).all()
    w.eng.close()


def test_hashes_in_with_empty_rows(pkg):
    M, R = 500, 400
    w = EdgeWorld(pkg, M, FOUR, 0, 0, seed=8, max_endpoints=512)
    kw = w.workload(R, 9)
    h = w.eng.schedule(R, want_hashes=True, max_blocks=MB, **kw)
    n = h["total_blocks"].copy()
    n[::4] = 0
    hin = dict(hashes_in=h["hashes_out"], n_hashes_in=n, adapter_id=kw["adapter_id"])
    tok = w.tokens(R)
    got = w.eng.schedule_inorder(R, tokens=tok, **hin)
    want = w.reference(R, tok, **hin)
    w.check(got, want, "hashes_in")
    assert (got["total_blocks"][::4] == 0).all() and got["total_blocks"].any()
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# a profile without a load-dependent scorer: one plain batch and one inflight_add

@pytest.mark.parametrize("me,pick_mode,R", [(4096, 0, 3000), (8192, 1, 3000), (2048, 2, 4000)],
                         ids=["C16xT256-max", "C16xT512-weighted", "C8-random"])
def test_load_independent_profile_equals_one_batch(pkg, me, pick_mode, R):
    """no token-load scorer: in arrival order or all at once the scores are the same, so the in-order call equals one
    eppscore_schedule_batch, and its counters one eppscore_inflight_add of those picks (no Python reference involved)"""
    M = me
    scorers = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
    w = EdgeWorld(pkg, M, scorers, pick_mode, 1, seed=me + pick_mode, max_endpoints=me, tie_seed=SEED)
    kw = w.workload(R, 10)
    mask = w.masks(R)
    tok = w.tokens(R)
    plain = w.eng.schedule(R, cand_mask=mask, max_blocks=MB, request_base=77, **kw)
    got = w.eng.schedule_inorder(R, tokens=tok, cand_mask=mask, max_blocks=MB, request_base=77, **kw)
    for k in ("pick", "tie_count", "total_blocks"):
        assert np.array_equal(got[k], plain[k]), k
    assert np.array_equal(got["pick_score"].view(np.uint64), plain["pick_score"].view(np.uint64))
    twin = pkg.Engine(pkg.default_config(scorers, max_endpoints=me))
    twin.inflight_add(got["pick"], tok)
    a, b = w.eng.inflight_get(me), twin.inflight_get(me)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert (got["pick"] == -1).any() and a[0].sum() == (got["pick"] >= 0).sum()
    twin.close()
    w.eng.close()


# ---------------------------------------------------------------------------------------------------------------------------
# stream order of device-location calls

@pytest.mark.parametrize("between", ["nothing", "inflight_add", "plain_schedule"])
def test_streams_without_host_sync(pkg, between):
    """in-order batches on a reserved and an unreserved stream back to back (with an inflight_add on a third stream, or a plain
    batch on another stream, in between), no host synchronisation until the end: the engine orders them as producer updates,
    so the outputs equal the sequential reference over the calls in issue order"""
    import torch
    M, R = 1024, 300
    scorers = FOUR
    w = EdgeWorld(pkg, M, scorers, 0, 1, seed=55 + len(between), tie_seed=SEED)
    dev = torch.device("cuda:0")
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    w.eng.reserve_stream(s1.cuda_stream, R, MB)
    batches = []
    for i in range(2):
        kw = w.workload(R, 20 + i)
        d = {k: _dev(v) for k, v in kw.items()}
        mask, tok = w.masks(R), w.tokens(R)
        d["cand_mask"], dtok = _dev(mask), _dev(tok)
        out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                   tie_count=torch.empty(R, dtype=torch.int32, device=dev),
                   total_blocks=torch.empty(R, dtype=torch.uint16, device=dev))
        batches.append((kw, d, mask, tok, dtok, out))
    add_ep = np.array(spread(M, 40), np.int32)
    add_tok = np.arange(40, dtype=np.int64) * 311
    d_ep, d_tok = _dev(add_ep), _dev(add_tok)
    plain = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
                 tie_count=torch.empty(R, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()  # inputs staged; from here on only the engine orders the calls

    (kw0, d0, m0, t0, dt0, o0), (kw1, d1, m1, t1, dt1, o1) = batches
    w.eng.schedule_inorder(R, tokens=dt0, device=True, stream=s1.cuda_stream, out=o0, max_blocks=MB, request_base=0, **d0)
    if between == "inflight_add":
        w.eng.inflight_add(d_ep, d_tok, device=True, stream=s3.cuda_stream)
    elif between == "plain_schedule":
        w.eng.schedule(R, device=True, stream=s2.cuda_stream, out=plain, max_blocks=MB, request_base=5000, **d1)
    w.eng.schedule_inorder(R, tokens=dt1, device=True, stream=s2.cuda_stream, out=o1, max_blocks=MB, request_base=R, **d1)
    torch.cuda.synchronize()

    want0 = w.reference(R, t0, request_base=0, cand_mask=m0, **kw0)
    w0 = {k: v.cpu().numpy() for k, v in o0.items()}
    for k in ("pick", "tie_count", "total_blocks"):
        assert np.array_equal(w0[k], want0[k]), k
    assert np.array_equal(w0["pick_score"].view(np.uint64), want0["pick_score"].view(np.uint64))
    if between == "inflight_add":
        w.tracker.add(add_ep, add_tok)
    elif between == "plain_schedule":  # sees the counters batch 0 left
        snap = o.SnapshotData(**w.sd, inflight_tokens=w.tracker.get(M)[1])
        wp = o.schedule_batch(snap, w.prof, w.idx, R, request_base=5000, max_blocks=MB, cand_mask=m1, **kw1)
        gp = {k: v.cpu().numpy() for k, v in plain.items()}
        for k in ("pick", "tie_count"):
            assert np.array_equal(gp[k], wp[k]), k
        assert np.array_equal(gp["pick_score"].view(np.uint64), wp["pick_score"].view(np.uint64))
    want1 = w.reference(R, t1, request_base=R, cand_mask=m1, **kw1)
    w.check({k: v.cpu().numpy() for k, v in o1.items()}, want1, between)
    w.eng.release_stream(s1.cuda_stream)
    w.eng.close()
