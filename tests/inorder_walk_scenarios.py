"""Inputs for the edge tests of the in-order index and latency walks (csrc/inorder_kernel.cu: inorder_walk<RND, IDX, LAT>), shared
by the CPU check of the scenarios themselves (tests/test_inorder_walk_scenarios_cpu.py) and the GPU tests
(tests/test_gpu_inorder_index_edges.py, tests/test_gpu_inorder_latency_edges.py).  Pure numpy plus the CPU oracle: the same case
gives the same batches on both sides, and the CPU check fails when a case drifts off the edge it names.

Every boundary comes from constants parsed out of the sources: the probe round (kCommitThreads: the index walk probes that many
blocks per round), the commit chunk (kChunkMax), the inline set size (kInlineEps) and the slice rows (kInOrderSliceBytes)."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q
from tests.helpers import synth_ragged_prompts, synth_snapshot
from tests.index_scenarios import CSRC, index_constants

_IC = index_constants()
T = _IC.commit_threads   # blocks probed per round of the index walk, and threads of its CTAs
CHUNK = _IC.chunk_max    # touches per parallel chunk of IndexProgram::commit
with open(os.path.join(CSRC, "prefix_table.cuh")) as _f:
    INLINE_EPS = int(re.search(r"constexpr\s+int\s+kInlineEps\s*=\s*(\d+)\s*;", _f.read()).group(1))
with open(os.path.join(CSRC, "capi.cu")) as _f:
    _m = re.search(r"constexpr size_t kInOrderSliceBytes = (\d+)ull << (\d+);", _f.read())
SLICE_BYTES = int(_m.group(1)) << int(_m.group(2))

SEED = 0x9E3779B97F4A7C15  # tie seed with both 32-bit words nonzero
THR = 8192.0
MB = 32
FULL = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1), ("token_load", 1)]
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01)


def mpad(max_endpoints):
    """the engine's padded endpoint count (kernels.cuh make_geo): 256, 512, then 1024 << {0..3}"""
    if max_endpoints <= 512:
        return 256 if max_endpoints <= 256 else 512
    return 1024 << max(0, (max_endpoints - 1).bit_length() - 10)


def index_cluster(max_endpoints):
    """(C, T) of the index walk: CTAs of T threads, C = 1 up to Mpad T, then Mpad / T (launch_inorder_index)"""
    p = mpad(max_endpoints)
    return (1 if p <= T else p // T), T


def flight_cluster(max_endpoints):
    """(C, T) of the in-flight walk: C = clamp(Mpad / 256, 1, 16) CTAs of Mpad / C threads (inorder_cluster_size on an H100)"""
    p = mpad(max_endpoints)
    C = min(max(p // 256, 1), 16)
    return C, p // C


def slice_rows(max_endpoints):
    """rows of one slice of an in-order call: kInOrderSliceBytes over 2 bytes per padded endpoint"""
    return max(1, SLICE_BYTES // (2 * mpad(max_endpoints)))


class KeyGen:
    """Distinct nonzero block keys: splitmix64 of a counter (a bijection, so never a repeat within one generator)."""

    def __init__(self, stream):
        self.next = (stream & 0xFFFF) << 40

    def __call__(self, n):
        x = (np.arange(self.next, self.next + n, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        self.next += n
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
        return np.where(x == 0, np.uint64(1), x)


def mask_rows(M, cands):
    """uint32 [R, ceil(M / 32)] candidate masks from one list of endpoints per request (None: every endpoint)"""
    mw = (M + 31) // 32
    m = np.zeros((len(cands), mw), np.uint32)
    for r, c in enumerate(cands):
        if c is None:
            m[r] = 0xFFFFFFFF
            if M % 32:
                m[r, -1] = (1 << (M % 32)) - 1
            continue
        for e in c:
            m[r, e >> 5] |= np.uint32(1 << (e & 31))
    return m


def rows_array(rows, stride=None):
    """(hashes uint64 [R, stride], n uint16 [R]) from a list of key arrays"""
    stride = stride or max(1, max(len(h) for h in rows))
    H = np.zeros((len(rows), stride), np.uint64)
    n = np.zeros(len(rows), np.uint16)
    for r, h in enumerate(rows):
        H[r, :len(h)] = h
        n[r] = len(h)
    return H, n


@dataclass
class Batch:
    R: int
    kw: dict                      # schedule arguments: hashes_in / n_hashes_in or prompts, cand_mask, adapter_id, SLOs ...
    tokens: np.ndarray
    caps: np.ndarray | None = None  # lru_capacity [M]
    key: np.ndarray | None = None   # request keys (latency form)
    meta: dict = field(default_factory=dict)  # what the CPU check asserts about the batch


@dataclass
class Case:
    name: str
    M: int
    E: int                        # max_endpoints
    scorers: list
    sd: dict                      # SnapshotData keyword arguments (no queue view, no inflight tokens)
    pick_mode: int = 0
    tie_mode: int = 1
    lru_default: int = 31250
    lru_max: int = 0
    threshold: float = THR
    seeds: list = field(default_factory=list)   # (keys, endpoint, lru capacity): prefix_add / Index.add, in order
    live: tuple | None = None     # (endpoint, key, tpot) running entries added before the batches
    lat: dict | None = None       # latency parameters (LAT_COEF + overrides); None: no latency scorer
    batches: list = field(default_factory=list)

    def profile(self):
        from _pkg import load
        pkg = load()
        lat = o.make_latency_params(**self.lat) if self.lat is not None else None
        return o.make_profile([(pkg.SCORER[s], w) for s, w in self.scorers], tie_mode=self.tie_mode, tie_seed=SEED,
                              token_load_threshold=self.threshold, pick_mode=self.pick_mode, latency=lat)


def seed_oracle(case, idx):
    for keys, ep, cap in case.seeds:
        idx.add(keys, ep, cap)


def first_miss(idx, h):
    """the first block of h whose set is empty in the oracle index (len(h): every block is held somewhere)"""
    for k, x in enumerate(h):
        if not idx.get(int(x)):
            return k
    return len(h)


# ---------------------------------------------------------------------------------------------------------------------------
# index walk: probe rounds

PROBE = [("queue", 1), ("kv", 1), ("prefix", 20), ("lora", 1), ("token_load", 1)]  # a match outweighs the other scorers
MISS_AT = [0, T - 1, T, T + 1, 2 * T - 1, 2 * T, 2 * T + 1, None]  # None: every block hits (the walk runs past the end)
PROBE_N = 3 * T + 7                                                  # four rounds, the last partial


def probe_case(M, seed=0, E=None):
    """Supplied rows of PROBE_N blocks, each seeded on its own owner endpoint except for the block at its first miss, plus: a
    row whose round-2 miss is a set emptied by eviction (cnt == 0), a row with a bitset-row set in round 2, and rows whose
    owner is the 10th / 9th inline member of sets in every round (the last staged member word).  Rows twice over in a mixed
    order, so consecutive requests leave and enter rounds at different parities; each request's candidates are its owner and a
    decoy that holds nothing."""
    E = E or max(M, 64)
    kg, rng = KeyGen(seed + 1), np.random.Generator(np.random.PCG64(seed))
    owners = [int(x) for x in np.linspace(INLINE_EPS + 2, M - 1, 2 * (len(MISS_AT) + 4))]
    seeds, rows, expect, kinds = [], [], [], []
    oi = iter(owners)
    for rep in range(2):
        for p in MISS_AT:
            e, h = next(oi), kg(PROBE_N)
            seeds.append((h if p is None else np.delete(h, p), e, 0))
            rows.append((h, e))
            expect.append(PROBE_N if p is None else p)
            kinds.append(f"miss{p}")
        # emptied set at T + 5: held by an endpoint of LRU capacity 4, then evicted by 4 newer keys there
        e, h = next(oi), kg(PROBE_N)
        x = (e + M // 3) % M
        seeds += [(h[T + 5:T + 6], x, 4), (kg(4), x, 4), (np.delete(h, T + 5), e, 0)]
        rows.append((h, e))
        expect.append(T + 5)
        kinds.append("emptied")
        # a bitset-row set at T + 9 (INLINE_EPS + 1 members over the cluster), the first miss at 3T
        e, h = next(oi), kg(PROBE_N)
        for m in np.linspace(0, M - 1, INLINE_EPS + 1).astype(int):
            if m != e:
                seeds.append((h[T + 9:T + 10], int(m), 0))
        seeds.append((np.delete(h, 3 * T), e, 0))
        rows.append((h, e))
        expect.append(3 * T)
        kinds.append("bitset")
        # owner as the last inline member: INLINE_EPS and INLINE_EPS - 1 members, the owner the largest id
        for members in (INLINE_EPS, INLINE_EPS - 1):
            e, h = next(oi), kg(PROBE_N)
            at = [3, T + 3, 2 * T + 3, 3 * T + 3]
            lower = np.linspace(0, e - 1, members - 1).astype(int)
            for m in lower:
                seeds.append((h[at], int(m), 0))
            seeds.append((h, e, 0))
            rows.append((h, e))
            expect.append(PROBE_N)
            kinds.append(f"inline{members}")
    order = rng.permutation(len(rows))
    rows, expect, kinds = [rows[i] for i in order], [expect[i] for i in order], [kinds[i] for i in order]
    H, n = rows_array([h for h, _ in rows])
    cands = [[e, (e + M // 2) % M] for _, e in rows]
    R = len(rows)
    b = Batch(R, dict(hashes_in=H, n_hashes_in=n, cand_mask=mask_rows(M, cands)), rng.integers(0, 3000, R).astype(np.int64),
              meta=dict(first_miss=expect, kinds=kinds, owner=[e for _, e in rows]))
    return Case(f"probe-C{index_cluster(E)[0]}", M, E, PROBE, synth_snapshot(M, seed=seed), seeds=seeds, batches=[b])


# ---------------------------------------------------------------------------------------------------------------------------
# index walk: commits past one chunk

def chunk_case(M=8192, seed=0):
    """Calls of CHUNK - 1, CHUNK, CHUNK + 1 and 2 CHUNK + 1 blocks at the default capacity (one to three chunks), and at endpoints
    of capacity CHUNK - 1, CHUNK and CHUNK + 1 (chunked when the call fits, sequential_call when it does not), with rows that
    re-touch keys earlier requests of the batch committed; a 2 CHUNK + 1 call picked in the cluster's last CTA is then probed
    by the next requests, whose picks see pick_match past 255 and past 512."""
    C, TT = index_cluster(M)
    kg, rng = KeyGen(seed + 7), np.random.Generator(np.random.PCG64(seed))
    last = (C - 1) * TT + 37          # an endpoint of the last CTA
    a0, a1, a2 = 5, TT + 11, 2 * TT + 3 if C > 2 else 200
    p1, p2, p3 = (C // 2) * TT + 1, (C // 2) * TT + 2, (C // 2) * TT + 3
    caps = np.zeros(M, np.int32)
    caps[[p1, p2, p3]] = [CHUNK - 1, CHUNK, CHUNK + 1]
    k = [kg(n) for n in (CHUNK - 1, CHUNK, CHUNK + 1)]
    long_ = np.concatenate([k[2], kg(CHUNK)])                       # re-touches request 2's keys, then new ones
    rows = [
        (k[0], [a0]),                                              # one chunk less one
        (k[1], [a1]),                                              # one whole chunk
        (k[2], [a2]),                                              # a chunk and one
        (long_, [last]),                                           # 2 CHUNK + 1 in the last CTA
        (np.concatenate([long_[:1000], kg(50)]), [last, a0]),      # probes it: pick_match 1000 at `last`
        (np.concatenate([long_[:300], kg(9)]), [last]),            # pick_match 300
        (long_, [a1, last]),                                       # the whole call again
        (kg(CHUNK), [p1]),                                         # longer than p1's LRU: sequential_call
        (k[1], [p1]),                                              # again: evictions inside the call
        (kg(CHUNK), [p2]),                                         # exactly p2's LRU: chunked
        (np.concatenate([k[0][:CHUNK - 1], kg(2)]), [p2]),         # CHUNK + 1 at p2: sequential, evicting
        (kg(CHUNK + 1), [p3]),                                     # exactly p3's LRU
        (long_, [p3]),                                             # 2 CHUNK + 1 at p3: sequential
        (np.concatenate([long_[:CHUNK], k[0][:10]]), None),       # free pick, probing everything above
    ]
    H, n = rows_array([h for h, _ in rows])
    R = len(rows)
    b = Batch(R, dict(hashes_in=H, n_hashes_in=n, cand_mask=mask_rows(M, [c for _, c in rows])),
              rng.integers(0, 3000, R).astype(np.int64), caps=caps, meta=dict(last=last, caps_at=(p1, p2, p3)))
    return Case(f"chunks-C{C}", M, M, FULL, synth_snapshot(M, seed=seed + 3), lru_max=CHUNK + 1, batches=[b])


# ---------------------------------------------------------------------------------------------------------------------------
# index walk: bitset rows over a 16-CTA cluster

def bitset_case(M=8192, seed=0):
    """Blocks shared by every request, picked in turn at 24 endpoints spread over every CTA: their sets grow past INLINE_EPS
    members into a bitset row inside the batch; then the same endpoints take rows of new keys longer than their LRU
    (capacity 40), which evicts the shared blocks and empties the rows."""
    kg, rng = KeyGen(seed + 11), np.random.Generator(np.random.PCG64(seed))
    shared = kg(12)
    eps = [int(x) for x in np.linspace(0, M - 1, 24)]
    rows, cands = [], []
    for e in eps:
        rows.append(np.concatenate([shared, kg(8)]))
        cands.append([e])
    for e in eps:                                                  # each shared block's set at 24 members: probed here
        rows.append(np.concatenate([shared, kg(20)]))
        cands.append([e, eps[(eps.index(e) + 5) % len(eps)]])
    for e in eps:
        rows.append(kg(MB))
        cands.append([e])
    H, n = rows_array(rows)
    R = len(rows)
    b = Batch(R, dict(hashes_in=H, n_hashes_in=n, cand_mask=mask_rows(M, cands)), rng.integers(0, 3000, R).astype(np.int64),
              meta=dict(shared=shared, eps=eps))
    return Case(f"bitset-C{index_cluster(M)[0]}", M, M, [("kv", 1), ("prefix", 2), ("token_load", 1)],
                synth_snapshot(M, seed=seed + 5), lru_default=40, batches=[b])


# ---------------------------------------------------------------------------------------------------------------------------
# pickers and ties over several CTAs (both walks)

def prompts_batch(M, R, seed, groups=4):
    rng = np.random.Generator(np.random.PCG64(seed))
    pb, off = synth_ragged_prompts(R, max_len=MB * 64, seed=seed, groups=groups, shared=512)
    kw = dict(prompt_bytes=pb, prompt_off=off, model_seed=np.full(R, 5, np.uint64),
              adapter_id=rng.integers(-1, 64, R).astype(np.int32))
    return Batch(R, kw, rng.integers(0, 3000, R).astype(np.int64))


PICKERS = {  # name: (scorers, pick_mode, tie_mode, threshold)
    "max-tie0": ([("kv", 1), ("prefix", 1), ("token_load", 1)], 0, 0, THR),
    "max-tie1": ([("kv", 1), ("prefix", 1), ("token_load", 1)], 0, 1, THR),
    "weighted": ([("kv", -2), ("prefix", 0.5), ("token_load", 1)], 1, 1, 300.0),  # loads past 300: the uniform draw
    "random": ([("kv", 1), ("prefix", 1), ("token_load", 1)], 2, 0, THR),
}


def picker_case(name, M, R=300, seed=0, lat=False):
    scorers, pm, tm, thr = PICKERS[name]
    if lat:
        scorers = scorers + [("latency", 1)]
    b = prompts_batch(M, R, seed + 1)
    if pm == 1:  # eight candidates over the cluster: they saturate within the batch, and scores fall to <= 0
        b.kw["cand_mask"] = mask_rows(M, [[int(x) for x in np.linspace(0, M - 1, 8)]] * R)
    c = Case(f"{name}-M{M}", M, M, scorers, synth_snapshot(M, seed=seed, tie_heavy=True), pick_mode=pm, tie_mode=tm,
             threshold=thr, batches=[b])
    if lat:
        add_latency(c, seed, predictions=0)  # the composite: flat, so ties are the rule
    return c


def add_latency(case, seed, predictions=1, **lat):
    """A latency profile for the case: parameters, request keys, SLOs and running entries on a third of the endpoints."""
    rng = np.random.Generator(np.random.PCG64(seed + 101))
    case.lat = dict(LAT_COEF, streaming_mode=1, **dict(dict(has_predictions=predictions), **lat))
    if not any(s == "latency" for s, _ in case.scorers):
        case.scorers = case.scorers + [("latency", 2)]
    kbase = 1 << 20
    for i, b in enumerate(case.batches):
        b.key = np.arange(kbase, kbase + b.R, dtype=np.uint64)
        kbase += b.R
        b.kw.setdefault("ttft_slo", rng.choice([0.0, 60.0, 140.0, 400.0, 1e6], b.R))
        b.kw.setdefault("tpot_slo", rng.choice([0.0, 14.0, 18.0, 24.0, 30.0, 80.0], b.R))
        b.kw.setdefault("input_tokens", rng.integers(0, 6000, b.R).astype(np.int32))
    if case.live is None:
        ep = rng.integers(0, case.M, case.M // 3 + 1).astype(np.int32)
        case.live = (ep, np.arange(1, len(ep) + 1, dtype=np.uint64), rng.choice([0.0, 12.0, 20.0, 35.0], len(ep)))
    return case


# ---------------------------------------------------------------------------------------------------------------------------
# the sequential reference over a case

class Ref:
    """The oracle side of a case: index (seeded), in-flight tracker, running queues (with the case's live entries)."""

    def __init__(self, case: Case):
        self.case = case
        self.prof = case.profile()
        self.idx = o.Index(case.lru_default)
        seed_oracle(case, self.idx)
        self.tracker = I.Tracker()
        self.q = Q.Queues(case.E)
        if case.live is not None:
            self.live_added = self.q.add(*case.live)

    def run(self, b: Batch, index_form=True, request_base=0):
        from tests.inorder_index_reference import schedule_inorder_index
        from tests.inorder_latency_reference import schedule_inorder_latency
        c = self.case
        if c.lat is not None:
            want, _ = schedule_inorder_latency(c.sd, self.prof, self.idx if index_form else None, b.R, self.q, tokens=b.tokens,
                                               request_key=b.key, tracker=self.tracker, M=c.M, lru_capacity=b.caps,
                                               index_form=index_form, max_blocks=MB, request_base=request_base, **b.kw)
        else:
            want, _ = schedule_inorder_index(c.sd, self.prof, self.idx, b.R, b.tokens, tracker=self.tracker, M=c.M,
                                             lru_capacity=b.caps, max_blocks=MB, request_base=request_base, **b.kw)
        return want


def tiers(case: Case, b: Batch, want, index_form=False):
    """Replays a latency batch on the oracle (with the picks and adds the reference made) and returns per request: the lowest
    tier among its candidates, its candidates in that tier, and whether the |TTFT| / |TPOT| headroom ranges of that tier are
    degenerate (<= 1e-9).  Valid for cases with predictions on and no prefix-dependent TTFT (index_form False)."""
    lp = o.make_latency_params(**case.lat)
    q = Q.Queues(case.E)
    if case.live is not None:
        q.add(*case.live)
    tracker = I.Tracker()
    out = []
    M = case.M
    for r in range(b.R):
        mn, cnt = q.get(M)
        snap = o.SnapshotData(**case.sd, min_tpot_slo=Q.canonical(mn), dispatched=cnt, inflight_tokens=tracker.get(M)[1])
        kw = {k: v[r:r + 1] for k, v in b.kw.items() if k in ("input_tokens", "ttft_slo", "tpot_slo", "cand_mask")}
        x = o.schedule_batch(snap, case.profile(), None, 1, want_pred=True, max_blocks=MB, **kw)
        assert x["pick"][0] == want["pick"][r]
        cand = np.ones(M, bool) if "cand_mask" not in b.kw else \
            np.unpackbits(b.kw["cand_mask"][r].view(np.uint8), bitorder="little")[:M].astype(bool)
        rank = np.full(M, 9)
        hT, hP = np.zeros(M), np.zeros(M)
        tslo = float(b.kw["ttft_slo"][r]) if "ttft_slo" in b.kw else 0.0
        pslo = float(b.kw["tpot_slo"][r]) if "tpot_slo" in b.kw else 0.0
        for m in np.flatnonzero(cand):
            neutral = not case.lat.get("streaming_mode", 0) or bool(case.sd.get("prefill_role", np.zeros(M))[m])
            v = o.latency_validate(lp, x["pred_out"][0, m, 0], x["pred_out"][0, m, 1], tslo, pslo, float(Q.canonical(mn)[m]), neutral)
            hT[m], hP[m] = v["ttft_headroom"], v["headroom"]
            tn, pn = hT[m] < 0, hP[m] < 0
            rank[m] = 0 if not (tn or pn) else (1 if cnt[m] == 0 else (4 if tn and pn else (3 if tn else 2)))
        low = int(rank[cand].min()) if cand.any() else 9
        inn = np.flatnonzero(cand & (rank == low))
        rT = np.ptp(np.abs(hT[inn])) if len(inn) else 0.0
        rP = np.ptp(np.abs(hP[inn])) if len(inn) else 0.0
        out.append(dict(rank=low, members=inn, tdeg=bool(rT <= 1e-9), pdeg=bool(rP <= 1e-9)))
        p = int(want["pick"][r])
        if p >= 0:
            if b.key is not None:
                q.add(want["pick"][r:r + 1], b.key[r:r + 1], b.kw["tpot_slo"][r:r + 1] if "tpot_slo" in b.kw else None)
            tracker.add(want["pick"][r:r + 1], b.tokens[r:r + 1])
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# latency walk: parameters, tiers and queue values

def lat_base(M, E, R, seed, scorers=None, **lat):
    rng = np.random.Generator(np.random.PCG64(seed))
    b = Batch(R, dict(input_tokens=rng.integers(0, 6000, R).astype(np.int32),
                      ttft_slo=rng.choice([0.0, 60.0, 140.0, 400.0, 1e6], R),
                      tpot_slo=rng.choice([0.0, 14.0, 18.0, 24.0, 30.0, 80.0], R)),
              rng.integers(0, 3000, R).astype(np.int64), key=np.arange(1000, 1000 + R, dtype=np.uint64))
    c = Case("", M, E, scorers or [("kv", 1), ("latency", 2), ("token_load", 1)], synth_snapshot(M, seed=seed), batches=[b])
    add_latency(c, seed, **lat)
    return c


PARAMS = {  # name: latency overrides (predictions on unless has_predictions is given)
    "most": dict(strategy_most=1),
    "buffer0.5": dict(slo_buffer_factor=0.5),
    "buffer1.3": dict(slo_buffer_factor=1.3),
    "w1-0": dict(ttft_weight=1.0, tpot_weight=0.0),
    "w0-1": dict(ttft_weight=0.0, tpot_weight=1.0),
    "w0-0": dict(ttft_weight=0.0, tpot_weight=0.0),
    "w1-neg": dict(ttft_weight=1.0, tpot_weight=-0.99999999),
    "composite": dict(has_predictions=0, composite_kv=0.25, composite_queue=2.0, composite_prefix=0.5),
    "composite-nonpos": dict(has_predictions=0, composite_kv=1.0, composite_queue=-1.5, composite_prefix=0.25),
}


def param_case(name, M, E, R=240, seed=0):
    c = lat_base(M, E, R, seed + len(name), **PARAMS[name])
    c.name = name
    b = c.batches[0]
    rng = np.random.Generator(np.random.PCG64(seed + 9))
    if name == "most":  # loose SLOs (tier 0) and impossible ones (tiers past 0) in one batch
        b.kw["ttft_slo"] = rng.choice([1.0, 1e6], R)
        b.kw["tpot_slo"] = rng.choice([1e-3, 1e3], R)
    if name.startswith("composite"):  # negative queue values, and (second case) a range past 2^53
        q = c.sd["queue"].astype(np.int64) - 6
        if name == "composite-nonpos":
            q = rng.integers(-2 ** 61, 2 ** 61, M, dtype=np.int64)
        c.sd["queue"] = q
        c.scorers = [("kv", 1), ("latency", 2), ("queue", 1), ("token_load", 1)]
    return c


def tier_case(M, E, R=300, seed=0, one_cta=None):
    """SLOs from impossible to loose and running entries on most endpoints, so the lowest tier of some request is each of
    ranks 0-4; one_cta = (lo, hi): the candidates outside [lo, hi) are busy (tier 1 impossible there) and hold SLOs they
    cannot meet in both dimensions, so the lowest tier's members sit only in [lo, hi)."""
    c = lat_base(M, E, R, seed)
    c.name = "tiers"
    rng = np.random.Generator(np.random.PCG64(seed + 17))
    b = c.batches[0]
    busy = np.setdiff1d(np.arange(M), np.arange(0, M, 7)).astype(np.int32)
    c.live = (busy, np.arange(1, len(busy) + 1, dtype=np.uint64), np.full(len(busy), 30.0))
    b.kw["ttft_slo"] = rng.choice([1.0, 60.0, 400.0, 1e6], R)
    b.kw["tpot_slo"] = rng.choice([1e-3, 12.0, 20.0, 1e3], R)
    cands = []
    for r in range(R):
        k = r % 5
        if k == 0:
            cands.append([int(rng.integers(0, M))])                                  # single candidate
        elif k == 1:
            cands.append([int(x) for x in rng.choice(busy, 6, replace=False)])       # busy only: tiers 2-4 reachable
        else:
            cands.append(None)
    # the one-side-degenerate ranges: two candidates with equal |TTFT headroom| and different TPOT bounds (one idle, no
    # running queue), two prefill-role candidates (TPOT headroom 0) with different TTFTs, and two identical candidates
    sd = c.sd
    sd["kv_usage"][[2, 7]] = sd["kv_usage"][[1, 3]]
    sd["queue"][[2, 3, 7]] = sd["queue"][1], 0, 0
    sd["running"][[2, 3, 7]] = sd["running"][1], 0, 0
    sd["prefill_role"] = np.zeros(M, np.uint8)
    sd["prefill_role"][[4, 5]] = 1
    sd["kv_usage"][5] = sd["kv_usage"][4] / 2
    for r, pair in ((2, [3, 7]), (3, [4, 5]), (4, [1, 2])):
        cands[r] = pair
        b.kw["ttft_slo"][r], b.kw["tpot_slo"][r] = 1e6, 1e3
    b.kw["cand_mask"] = mask_rows(M, cands)
    if one_cta is not None:
        lo, hi = one_cta
        q = c.sd["queue"].copy()
        q[:lo] += 400  # TTFT and TPOT past any SLO outside [lo, hi)
        q[hi:] += 400
        c.sd["queue"] = q
        c.sd["running"] = np.where((np.arange(M) >= lo) & (np.arange(M) < hi), c.sd["running"], c.sd["running"] + 400)
        b.kw["ttft_slo"] = rng.choice([140.0, 400.0, 1e6], R)
        b.kw["tpot_slo"] = rng.choice([24.0, 80.0, 1e3], R)
        b.kw["cand_mask"] = mask_rows(M, [None] * R)
        c.name = "tiers-one-cta"
    return c


SPECIAL_TPOT = [-0.0, 0.0, np.inf, 5e-324, 1e308]


def queue_case(M, E, R=200, seed=0):
    """tpot -0.0, +0.0, +Inf, the smallest subnormal and 1e308 among the SLOs; one endpoint (`down`) taking a run of adds whose
    tpot falls every time, another (`flat`) many adds at one value that is its minimum; live entries on endpoints in
    [M, E) that the call must leave alone."""
    c = lat_base(M, E, R, seed)
    c.name = "queue-values"
    rng = np.random.Generator(np.random.PCG64(seed + 23))
    b = c.batches[0]
    down, flat = 3, M - 2
    tp = rng.choice(SPECIAL_TPOT + [14.0, 30.0], R)
    cands = [None] * R
    for i, r in enumerate(range(0, 40, 2)):     # the falling run
        cands[r] = [down]
        tp[r] = 100.0 - 4.0 * i
    for r in range(1, 40, 2):                   # equal minima
        cands[r] = [flat]
        tp[r] = 7.0
    b.kw["tpot_slo"] = tp
    b.kw["cand_mask"] = mask_rows(M, cands)
    ep = list(rng.integers(0, M, M // 4 + 1))
    far = [m for m in (M, M + 1, E - 1) if M <= m < E]
    ep += far
    tps = list(rng.choice([0.0, 12.0, 35.0], len(ep)))
    ep.append(flat)
    tps.append(9.0)  # the flat endpoint's minimum before the batch is above the batch's equal minima
    c.live = (np.array(ep, np.int32), np.arange(1, len(ep) + 1, dtype=np.uint64), np.array(tps))
    b.meta = dict(down=down, flat=flat, far=far)
    return c


def repeat_keys_case(M, E, seed=0):
    """A call over two slices whose second slice repeats keys of the first: on the same endpoint (refused) and on another
    endpoint (added)."""
    rows = slice_rows(E)
    R = rows + 40
    c = lat_base(M, E, R, seed)
    c.name = "keys-across-slices"
    b = c.batches[0]
    a, z = 1, M - 1
    cands = [None] * R
    for i in range(20):
        cands[i] = [a]
        cands[rows + i] = [a]          # same key, same endpoint: refused
        b.key[rows + i] = b.key[i]
        cands[20 + i] = [a]
        cands[rows + 20 + i] = [z]     # same key, another endpoint: added
        b.key[rows + 20 + i] = b.key[20 + i]
    b.kw["cand_mask"] = mask_rows(M, cands)
    b.kw["tpot_slo"] = np.abs(b.kw["tpot_slo"])
    b.meta = dict(rows=rows)
    return c
