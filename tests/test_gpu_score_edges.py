"""The scoring kernels (pick_sparse.cu, the score_matrix.cu family and the dense kernels) against the oracle at the thresholds
where they change representation or take a shortcut, bit for bit, through the C ABI.  Every threshold comes from
tests/score_constants.py, which parses it out of the sources.

  A  every engine geometry (log_epl, J) x snapshot M x three profiles x 8/16-bit match counters, on every route
  B  pick_sparse: the exception table's deferral limit and slot count, probe collisions, the lane-group probe rounds, the
     uniform-set shortcut, slot-table probing past emptied sets, mixed warps, T == gmax
  C  8-bit against 16-bit match counters and the 256-entry LUTs (lut2d, lut_p, lut_l, the affinity filter, top-k)
  D  the latency bucket's reciprocal fast path and its 64-bit truncation"""
import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests import topk_oracle
from tests.helpers import synth_snapshot, zipf_adapters
from tests.score_constants import score_constants

pytestmark = pytest.mark.gpu

K = score_constants()

HEADLINE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]                     # one folded term
WIDE = [("prefix", 3), ("kv", 2), ("running", 1), ("token_load", 1), ("col0", 1.5), ("lora", 1), ("queue", 2)]  # unfolded terms
LATENCY = [("kv", 1), ("latency", 2)]                                                  # behind both device filters
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01, streaming_mode=1)
TOKEN_THRESHOLD = 4096.0
BASIC = ("pick", "pick_score", "tie_count", "total_blocks")
DIAG = BASIC + ("match_blocks", "scores_out")


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


def assert_same(got, want, keys=BASIC, where=""):
    for k in keys:
        g, w = got[k], want["weighted_out" if k == "scores_out" else k]
        if g.dtype.kind == "f":
            if k == "scores_out":  # the oracle's candidates (after the device filters, which the engine reports as scored)
                keep = ~np.isnan(w)
                assert np.array_equal(g[keep].view(np.uint64), w[keep].view(np.uint64)), f"{where}: {k}"
            else:
                assert np.array_equal(g.view(np.uint64), w.view(np.uint64)), f"{where}: {k}"
        else:
            assert np.array_equal(g, w), f"{where}: {k}"


def filters_of(pkg, scorers):
    if ("latency", 2) not in scorers:
        return []
    return [(pkg.FILTER_PREFIX_AFFINITY, (0.5, 0.1, 5000.0)), (pkg.FILTER_SLO_HEADROOM_TIER, (0.3,))]


class Case:
    """One engine (and, optionally, a weighted-random twin) and the oracle's mirror of its snapshot and index."""

    def __init__(self, pkg, scorers, max_ep, M, *, tie_mode=0, seed=0, lat=None, random_twin=False, tie_heavy=False,
                 prefix_capacity=1 << 14):
        self.pkg, self.scorers, self.M = pkg, scorers, M
        filt = filters_of(pkg, scorers)
        lat_on = any(k == "latency" for k, _ in scorers)
        lkw = dict(LAT_COEF, **(lat or {}))
        rng = np.random.Generator(np.random.PCG64(seed + 17))
        sd = synth_snapshot(M, seed=seed, tie_heavy=tie_heavy)
        if tie_heavy:
            sd["kv_usage"] = np.round(sd["kv_usage"], 1)
        if any(k == "col0" for k, _ in scorers):
            sd["endpoint_cols"] = (np.round(rng.random(M) * 1.4 - 0.2, 2),)
        if any(k == "token_load" for k, _ in scorers):
            sd["inflight_tokens"] = rng.integers(0, 8000, M).astype(np.int64)
        if lat_on:
            sd["min_tpot_slo"] = rng.choice([0.0, 22.0, 26.5, 60.0], M)
            sd["dispatched"] = rng.integers(0, 3, M).astype(np.int32)
            sd["prefill_role"] = (rng.random(M) < 0.1).astype(np.uint8)
        self.snap = o.SnapshotData(**sd)
        self.engines = []
        self.profiles = []
        for mode in ((0, 1) if random_twin else (0,)):
            eng = pkg.Engine(pkg.default_config(scorers, filters=filt, max_endpoints=max_ep, tie_mode=tie_mode, tie_seed=99,
                                                pick_mode=mode, token_load_threshold=TOKEN_THRESHOLD,
                                                prefix_capacity=prefix_capacity))
            if lat_on:
                eng.set_latency_params(pkg.latency_params(**lkw))
            eng.set_snapshot(**sd)
            self.engines.append(eng)
            self.profiles.append(o.make_profile([(pkg.SCORER[k], w) for k, w in scorers], tie_mode=tie_mode, tie_seed=99,
                                                latency=o.make_latency_params(**lkw) if lat_on else None,
                                                token_load_threshold=TOKEN_THRESHOLD, pick_mode=mode, filters=filt))
        self.idx = o.Index()

    def add(self, hashes, endpoint):
        h = np.ascontiguousarray(hashes, np.uint64)
        for eng in self.engines:
            eng.prefix_add(h, int(endpoint))
        self.idx.add(h, int(endpoint))

    def remove_endpoint(self, endpoint):
        for eng in self.engines:
            eng.prefix_remove_endpoint(int(endpoint))
        self.idx.remove_pod(int(endpoint))

    def close(self):
        for eng in self.engines:
            eng.close()

    def oracle(self, R, mode=0, **kw):
        return o.schedule_batch(self.snap, self.profiles[mode], self.idx, R, want_match=True, want_scores=True,
                                want_tie_set=True, n_threads=8, **kw)

    def check(self, R, kw, *, masked=None, dense=None, topk=True, diag=True, where=""):
        """Every route of the ABI that applies to the profile; returns the oracle's unmasked result."""
        eng = self.engines[0]
        lat_on = any(k == "latency" for k, _ in self.scorers)
        want = self.oracle(R, **kw)
        keys = DIAG if kw.get("hashes_in") is not None or kw.get("prompt_bytes") is not None else BASIC + ("scores_out",)
        assert_same(eng.schedule(R, **kw), want, BASIC, f"{where} sparse/plain")          # pick_sparse (+ deferred pass)
        if diag:
            assert_same(eng.schedule(R, want_match=True, want_scores=True, **kw), want, keys, f"{where} full matrix")
        if topk:
            wm, ws = topk_oracle.lists(want["weighted_out"], self.profiles[0], 3)
            got = eng.schedule(R, topk=3, **kw)
            assert np.array_equal(got["topk_pick"], wm) and np.array_equal(got["topk_score"].view(np.uint64), ws.view(np.uint64)), \
                f"{where} top-k"
        if len(self.engines) > 1:
            want_r = self.oracle(R, mode=1, **kw)
            assert_same(self.engines[1].schedule(R, **kw), want_r, BASIC, f"{where} weighted-random")
            if masked is not None:
                want_rm = self.oracle(R, mode=1, cand_mask=masked, **kw)
                assert_same(self.engines[1].schedule(R, cand_mask=masked, **kw), want_rm, BASIC, f"{where} weighted-random masked")
        if masked is not None:
            want_m = self.oracle(R, cand_mask=masked, **kw)
            assert_same(eng.schedule(R, cand_mask=masked, **kw), want_m, BASIC, f"{where} masked")
            assert_same(eng.schedule(R, cand_mask=masked, want_match=True, want_scores=True, **kw), want_m, keys, f"{where} masked diag")
            if topk:
                wm, ws = topk_oracle.lists(want_m["weighted_out"], self.profiles[0], 3)
                got = eng.schedule(R, topk=3, cand_mask=masked, **kw)
                assert np.array_equal(got["topk_pick"], wm), f"{where} masked top-k"
        if dense is not None and not lat_on:
            feat, total = dense
            dkw = dict(dense_feat=feat, dense_total=total, adapter_id=kw.get("adapter_id"))
            want_d = self.oracle(R, **dkw)
            assert_same(eng.schedule(R, **dkw), want_d, BASIC, f"{where} dense fast")
            assert_same(eng.schedule(R, want_match=True, want_scores=True, **dkw), want_d, DIAG, f"{where} dense generic")
            if masked is not None:
                want_dm = self.oracle(R, cand_mask=masked, **dkw)
                assert_same(eng.schedule(R, cand_mask=masked, want_scores=True, **dkw), want_dm, BASIC + ("scores_out",),
                            f"{where} dense masked")
        return want


def random_mask(rng, R, M, density=0.5):
    bits = rng.random((R, M)) < density
    bits[0, :] = False
    mask = np.zeros((R, max(1, (M + 31) // 32)), np.uint32)
    for w in range((M + 31) // 32):
        chunk = bits[:, w * 32:(w + 1) * 32]
        mask[:, w] = (chunk * (1 << np.arange(chunk.shape[1], dtype=np.uint64))).sum(axis=1).astype(np.uint32)
    return mask


def lat_request_kw(rng, R):
    return dict(input_tokens=rng.integers(0, 6000, R).astype(np.int32), ttft_slo=rng.choice([0.0, 90.0, 200.0, 1e6], R),
                tpot_slo=rng.choice([0.0, 18.0, 30.0, 80.0], R))


def uhashes(rng, shape, low=None):
    """distinct-looking 64-bit block hashes (never 0); low: force these low 40 bits (slot-table collisions)"""
    h = rng.integers(1, 1 << 62, size=shape, dtype=np.int64).astype(np.uint64)
    if low is not None:
        h = (h & ~np.uint64((1 << 40) - 1)) | np.uint64(low)
    return h


# ------------------------------------------------------------------------------------------ A. geometry sweep
GEOMETRIES = [1, 33, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192]
PROFILES = {"headline": HEADLINE, "wide": WIDE, "latency": LATENCY}


@pytest.mark.parametrize("max_blocks", [64, 300])
@pytest.mark.parametrize("profile", list(PROFILES))
@pytest.mark.parametrize("max_ep", GEOMETRIES)
def test_geometry_sweep(pkg, max_ep, profile, max_blocks):
    """Every geometry the ABI accepts launches and returns the oracle's results on every route: the shared-memory layout of
    the full-matrix and generic dense kernels must fit the device at Mpad 8192 with many terms and 16-bit counters."""
    scorers = PROFILES[profile]
    lat_on = profile == "latency"
    R = 256 if max_ep > 2048 else 384
    assert (max_blocks > K.narrow_counter_max) == (max_blocks == 300)
    Ms = [max_ep] + ([max_ep - 7] if max_ep > 32 and (max_ep - 7) % 32 else [])
    for M in Ms:
        rng = np.random.Generator(np.random.PCG64(max_ep * 7 + M + max_blocks))
        case = Case(pkg, scorers, max_ep, M, seed=M, random_twin=True)
        # prefix chains: 16 groups cached on a few endpoints each (endpoints >= M included when the snapshot is smaller), one
        # group on more than kExcMax endpoints, so the sparse kernel defers its requests
        groups = uhashes(rng, (16, max_blocks))
        for g in range(16):
            n_eps = K.exc_max + 8 if g == 0 else int(rng.integers(1, 14))
            for ep in rng.choice(max_ep, size=min(n_eps, max_ep), replace=False):
                case.add(groups[g, : int(rng.integers(1, max_blocks + 1))], ep)
        gi = rng.integers(0, 17, R)  # group 16: unknown prompt
        hashes = np.where(gi[:, None] < 16, groups[np.minimum(gi, 15)], uhashes(rng, (R, max_blocks)))
        nh = rng.integers(0, max_blocks + 1, R).astype(np.uint16)
        nh[:4] = [0, 1, max_blocks, max_blocks]
        kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=zipf_adapters(R, seed=M))
        if lat_on:
            kw.update(lat_request_kw(rng, R))
        mask = random_mask(rng, R, M)
        dense = None
        if not lat_on:
            w0 = case.oracle(R, **kw)
            feat = np.zeros((R, M, 4), np.float32)
            feat[:, :, 0] = w0["match_blocks"]
            feat[:, :, 1] = rng.integers(0, 4, (R, M))
            dense = (feat, nh.copy())
        want = case.check(R, kw, masked=mask, dense=dense, where=f"max_ep={max_ep} M={M}")
        if M > K.exc_max + 8 and not lat_on:
            assert ((want["match_blocks"] > 0).sum(axis=1) > K.exc_max).any()  # some request was deferred
        case.close()


# ------------------------------------------------------------------------------------------ B. pick_sparse edges
SPARSE_EPS = {1: 1000, 2: 2000, 4: 4000, 8: 8000}   # J -> max_endpoints


def exc_home(m):
    return ((m * 0x9E3779B1) & 0xFFFFFFFF) >> (32 - (K.exc_slots.bit_length() - 1))


def chain_case(case, rng, members_per_hash):
    """A chain of fresh hashes, hash i cached on members_per_hash[i] (None: not cached); returns the chain."""
    chain = uhashes(rng, len(members_per_hash))
    for h, eps in zip(chain, members_per_hash):
        for ep in (eps or ()):
            case.add([h], ep)
    return chain


def pack(chains):
    R = len(chains)
    stride = max(1, max(len(c) for c in chains))
    hashes = np.zeros((R, stride), np.uint64)
    nh = np.zeros(R, np.uint16)
    for r, c in enumerate(chains):
        hashes[r, : len(c)] = c
        nh[r] = len(c)
    return hashes, nh


def split_sets(eps, size):
    return [list(eps[i:i + size]) for i in range(0, len(eps), size)]


@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("J", [1, 2, 4, 8])
def test_sparse_exception_table_limits(pkg, J, tie_mode):
    """Distinct matched endpoints at kExcMax-1, kExcMax, kExcMax+1 and kExcSlots+1, reached through inline sets, through one
    bitset row, and with the overflow crossing inside a row; also with endpoints whose exception-table homes collide, so
    probe runs are long and wrap past the last slot."""
    max_ep = SPARSE_EPS[J]
    rng = np.random.Generator(np.random.PCG64(J * 10 + tie_mode))
    case = Case(pkg, HEADLINE, max_ep, max_ep, tie_mode=tie_mode, seed=J, tie_heavy=True, prefix_capacity=1 << 16)
    # endpoints ordered by exception-table home starting at slot kExcSlots-8: long runs that wrap at the last slot
    start = K.exc_slots - 8
    colliding = sorted(range(max_ep), key=lambda m: ((exc_home(m) - start) % K.exc_slots, m))
    chains, targets = [], []
    for n in (K.exc_max - 1, K.exc_max, K.exc_max + 1, K.exc_slots + 1):
        for pool in ("random", "colliding"):
            eps = rng.choice(max_ep, size=n, replace=False) if pool == "random" else np.array(colliding[:n])
            rng.shuffle(eps)
            inline = split_sets(eps, K.inline_eps)
            row = [list(eps)]
            split = n - (K.inline_eps * 2)
            crossing = split_sets(eps[:split], K.inline_eps) + [list(eps[split:])]
            for sets in (inline, row, crossing):
                chains.append(chain_case(case, rng, sets))
                targets.append(n)
    R = len(chains)
    hashes, nh = pack(chains)
    kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=zipf_adapters(R, seed=J))
    want = case.check(R, kw, topk=False, where=f"J={J}")
    assert np.array_equal((want["match_blocks"] > 0).sum(axis=1), np.array(targets))
    case.close()


def probe_positions(G):
    U = K.probe_unroll
    return sorted({0, 1, G - 1, G, G + 1, U * G - 1, U * G, U * G + 1, 2 * U * G})


@pytest.mark.parametrize("J", [1, 2, 4])
def test_sparse_probe_rounds_and_first_miss(pkg, J):
    """Matched length and first miss at every edge of the G-lane, U-hash probe rounds; a block cached after the first miss
    must not count."""
    max_ep = SPARSE_EPS[J]
    G = K.geo(max_ep)[3]
    assert G == {1: 8, 2: 16, 4: 32}[J]
    rng = np.random.Generator(np.random.PCG64(J + 100))
    case = Case(pkg, HEADLINE, max_ep, max_ep, seed=J + 100, prefix_capacity=1 << 16)
    S = [int(x) for x in rng.choice(max_ep, 3, replace=False)]
    chains, expect = [], []
    for p in probe_positions(G):
        n = 2 * K.probe_unroll * G + 3
        chains.append(chain_case(case, rng, [S] * p + [None] + [S + [int(rng.integers(max_ep))]] * (n - p - 1)))
        expect.append(p)
        if p > 0:  # the chain ends at p: everything matched
            chains.append(chain_case(case, rng, [S] * p))
            expect.append(p)
    R = len(chains)
    hashes, nh = pack(chains)
    want = case.check(R, dict(hashes_in=hashes, n_hashes_in=nh), where=f"G={G}")
    assert np.array_equal(want["match_blocks"].max(axis=1), np.array(expect))
    case.close()


@pytest.mark.parametrize("J", [1, 2, 4])
def test_sparse_uniform_shortcut_switch(pkg, J):
    """The uniform-set shortcut hands over to the exception table at every probe-round edge, for each kind of change of the
    set: one member past the first two, the count only, 2 <-> 3 members (the second half of the slot), kInlineEps <->
    kInlineEps+1 members (an inline set becomes a bitset row)."""
    max_ep = SPARSE_EPS[J]
    G = K.geo(max_ep)[3]
    rng = np.random.Generator(np.random.PCG64(J + 200))
    case = Case(pkg, HEADLINE, max_ep, max_ep, seed=J + 200, tie_heavy=True, prefix_capacity=1 << 17)
    E = K.inline_eps
    chains = []
    for p in probe_positions(G):
        if p == 0:
            continue
        base = sorted(int(x) for x in rng.choice(max_ep - 1, E + 1, replace=False))
        variants = [
            (base[:5], base[:4] + [base[5]]),       # a member past the first two
            (base[:3], base[:4]),                   # the count only
            (base[:2], base[:3]), (base[:3], base[:2]),
            (base[:E], base[:E + 1]), (base[:E + 1], base[:E]),
        ]
        for a, b in variants:
            n = p + int(rng.integers(1, 2 * K.probe_unroll * G))
            chains.append(chain_case(case, rng, [a] * p + [b] * (n - p)))
    R = len(chains)
    hashes, nh = pack(chains)
    case.check(R, dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=zipf_adapters(R, seed=J)), where=f"G={G}")
    case.close()


def test_sparse_slot_table_probing(pkg):
    """Block hashes that collide in their low bits share one probe chain of the slot table; a set emptied by
    prefix_remove_endpoint in the middle of the chain reads as a miss, and probes for later keys walk past it."""
    max_ep = 1000
    rng = np.random.Generator(np.random.PCG64(300))
    case = Case(pkg, HEADLINE, max_ep, max_ep, seed=300, prefix_capacity=1 << 12)
    low = 0x12345
    coll = uhashes(rng, 12, low=low)
    sole = 977  # the only member of hashes 3 and 7, removed below; endpoint 5 holds every other hash
    for i, h in enumerate(coll):
        for ep in ([sole] if i in (3, 7) else [5] + [int(x) for x in rng.choice(np.arange(6, 900), i % 4, replace=False)]):
            case.add([h], ep)
    case.remove_endpoint(sole)
    chains = [coll[:3], coll[:6], coll[4:7], coll[8:], coll[[0, 1, 2, 8, 9]], coll[[8, 7, 9]], coll[[11, 10, 9]]]
    chains += [np.concatenate([coll[i:i + 1], uhashes(rng, 3, low=low)]) for i in (0, 5, 11)]
    R = len(chains)
    hashes, nh = pack(chains)
    want = case.check(R, dict(hashes_in=hashes, n_hashes_in=nh))
    assert want["match_blocks"][1].max() == 3 and want["match_blocks"][3].max() == 4
    case.close()


@pytest.mark.parametrize("J", [1, 2, 4])
def test_sparse_mixed_warps(pkg, J):
    """No-match, uniform, table and deferred requests interleaved at every phase of the 32/G requests of a warp, with R large
    enough that every lane group serves several requests: a small-table request right after a deferred one must find its
    exception table reset."""
    import torch
    max_ep = SPARSE_EPS[J]
    G = K.geo(max_ep)[3]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    R = 3 * sms * 8 * (32 // G) * 4   # > 2 grid strides of the sparse kernel at up to 4 resident CTAs of 8 warps per SM
    rng = np.random.Generator(np.random.PCG64(J + 400))
    case = Case(pkg, HEADLINE, max_ep, max_ep, seed=J + 400, prefix_capacity=1 << 16)
    S = [int(x) for x in rng.choice(max_ep, 4, replace=False)]
    uniform = chain_case(case, rng, [S] * 40)
    table = chain_case(case, rng, [S] * 5 + [S[:2]] * 10 + [[int(rng.integers(max_ep))]] * 5)
    deferred = chain_case(case, rng, [list(rng.choice(max_ep, K.exc_max + 5, replace=False))] * 3)
    short = chain_case(case, rng, [S[1:]] * 7)
    unknown = uhashes(rng, 20)
    kinds = [unknown, uniform, table, deferred, short]
    pick = (np.arange(R) * 3 + np.arange(R) // 7) % 5   # period coprime with the lane groups of a warp
    chains = [kinds[k][: int(rng.integers(1, len(kinds[k]) + 1)) if k != 3 else 3] for k in pick]
    hashes, nh = pack(chains)
    want = case.check(R, dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=zipf_adapters(R, seed=J)), topk=False, diag=False,
                      where=f"G={G}")
    assert ((want["match_blocks"] > 0).sum(axis=1) > K.exc_max).sum() >= R // 6  # deferred requests everywhere
    case.close()


@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("w_prefix", [0.0, 1e-18])
def test_sparse_exceptions_at_gmax(pkg, tie_mode, w_prefix):
    """T == gmax: a prefix weight of 0, or one so small that the sum absorbs it, leaves every exception at its zero-match
    score; exceptions inside and outside the precomputed arg-max set."""
    max_ep = 1000
    scorers = [("kv", 1), ("prefix", w_prefix), ("lora", 1)]
    rng = np.random.Generator(np.random.PCG64(500 + tie_mode))
    case = Case(pkg, scorers, max_ep, max_ep, tie_mode=tie_mode, seed=500, tie_heavy=True, prefix_capacity=1 << 16)
    R = 600
    chains = []
    for r in range(R):
        n_eps = int(rng.integers(1, K.exc_max + 4))
        chains.append(chain_case(case, rng, split_sets(rng.choice(max_ep, n_eps, replace=False), K.inline_eps)))
    hashes, nh = pack(chains)
    kw = dict(hashes_in=hashes, n_hashes_in=nh, adapter_id=zipf_adapters(R, seed=5))
    want = case.check(R, kw, topk=False)
    ts = want["tie_set"]
    exc = want["match_blocks"] > 0
    in_ts = np.zeros_like(exc)
    for m in range(max_ep):
        in_ts[:, m] = (ts[:, m >> 5] >> np.uint32(m & 31)) & 1
    assert (exc & in_ts).any() and (exc & ~in_ts).any()
    case.close()


# ------------------------------------------------------------------------------------------ C. counter width, LUT bypass
@pytest.mark.parametrize("profile", ["headline", "latency"])
def test_counter_width_and_lut_edges(pkg, profile):
    """hash_stride on both sides of the 8/16-bit counter split with one endpoint matching 255..4096 blocks, and totals on
    both sides of kLutMax on every route that switches on it (lut2d, lut_p, lut_l, the affinity filter's threshold, top-k)."""
    scorers = PROFILES[profile]
    M = 300
    cut, lut = K.narrow_counter_max, K.lut_max
    rng = np.random.Generator(np.random.PCG64(600))
    case = Case(pkg, scorers, M, M, seed=600, prefix_capacity=1 << 14)
    long_chain = uhashes(rng, 4096)
    lengths = sorted({lut - 1, lut, lut + 1, cut - 1, cut, cut + 1, 1000, 4096})
    for i, L in enumerate(lengths):
        case.add(long_chain[:L], 17 + i)
    case.add(long_chain[: lut // 2], 250)
    for stride in sorted({cut, cut + 1, 1000, 4096}):
        ns = [n for n in sorted({lut - 1, lut, lut + 1, cut - 1, cut, cut + 1, 1000, 4096, stride}) if n <= stride]
        R = 3 * len(ns)
        hashes = np.tile(long_chain[:stride], (R, 1))
        nh = np.array([n for n in ns for _ in range(3)], np.uint16)
        kw = dict(hashes_in=hashes, n_hashes_in=nh)
        if profile == "latency":
            kw.update(lat_request_kw(rng, R))
        want = case.check(R, kw, masked=random_mask(rng, R, M, 0.7), where=f"stride={stride}")
        assert want["match_blocks"].max() == max(ns)
    case.close()


def test_prompt_bytes_small_blocks_wide_counters(pkg):
    """block_chars = 4 and more than 256 blocks per prompt: the hash path feeds the 16-bit counters and the LUT bypass."""
    M, R, mb = 200, 300, 300
    scorers = HEADLINE
    eng = pkg.Engine(pkg.default_config(scorers, max_endpoints=M, block_chars=4, max_blocks=mb, prefix_capacity=1 << 16))
    rng = np.random.Generator(np.random.PCG64(700))
    sd = synth_snapshot(M, seed=700)
    eng.set_snapshot(**sd)
    snap, prof, idx = o.SnapshotData(**sd), o.make_profile([(pkg.SCORER[k], w) for k, w in scorers]), o.Index()
    base = rng.integers(97, 123, size=(4, 4 * mb + 40), dtype=np.uint8)
    lens = rng.integers(4 * 250, 4 * mb + 40, R)
    data = np.concatenate([base[r % 4, : lens[r]] for r in range(R)])
    off = np.zeros(R + 1, np.int64)
    off[1:] = np.cumsum(lens)
    seeds = np.full(R, eng.model_seed("tiny"), np.uint64)
    kw = dict(prompt_bytes=data, prompt_off=off, model_seed=seeds)
    warm = o.schedule_batch(snap, prof, idx, R, block_chars=4, max_blocks=mb, want_hashes=True, **kw)
    idx.commit(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    eng.commit_picks(warm["pick"], warm["hashes_out"], warm["total_blocks"])
    want = o.schedule_batch(snap, prof, idx, R, block_chars=4, max_blocks=mb, want_match=True, want_scores=True, **kw)
    assert_same(eng.schedule(R, **kw), want, BASIC)
    assert_same(eng.schedule(R, want_match=True, want_scores=True, **kw), want, DIAG)
    assert want["total_blocks"].max() > K.lut_max and want["match_blocks"].max() > K.lut_max
    eng.close()


# ------------------------------------------------------------------------------------------ D. latency buckets
@pytest.mark.parametrize("strategy_most", [0, 1])
@pytest.mark.parametrize("weights", [(1.0, -0.5), (1.0, -0.99999999), (1e-9, 1.0)], ids=["w1_m05", "w1_m099999999", "w1e9_1"])
def test_latency_bucket_weights(pkg, weights, strategy_most):
    """Latency weights outside [0, 1] after normalisation (alpha up to 1e8): the reciprocal fast path must hand over to the
    exact divides, and int(x) must not saturate or wrap below 2^63."""
    M, R = 256, 512
    lat = dict(ttft_weight=weights[0], tpot_weight=weights[1], strategy_most=strategy_most)
    rng = np.random.Generator(np.random.PCG64(800))
    case = Case(pkg, [("latency", 1)], M, M, seed=800, lat=lat)
    chains = uhashes(rng, (8, 32))
    for g in range(8):
        for ep in rng.choice(M, 5, replace=False):
            case.add(chains[g, : int(rng.integers(1, 33))], ep)
    kw = dict(hashes_in=chains[rng.integers(0, 8, R)], n_hashes_in=rng.integers(0, 33, R).astype(np.uint16))
    kw.update(lat_request_kw(rng, R))
    case.check(R, kw, masked=random_mask(rng, R, M, 0.6), topk=False)
    case.close()


@pytest.mark.parametrize("strategy_most", [0, 1])
def test_latency_composite_extreme_weights(pkg, strategy_most):
    """The composite fallback with weights (1, -0.99999999, 0): 100 * composite reaches about 1e10, past 32 bits."""
    M, R = 256, 512
    lat = dict(has_predictions=0, composite_kv=1.0, composite_queue=-0.99999999, composite_prefix=0.0,
               strategy_most=strategy_most)
    rng = np.random.Generator(np.random.PCG64(900))
    case = Case(pkg, [("latency", 1)], M, M, seed=900, lat=lat)
    kw = lat_request_kw(rng, R)
    want = case.check(R, kw, masked=random_mask(rng, R, M, 0.6), topk=False)
    assert np.nanmax(want["weighted_out"]) == 1.0
    case.close()
