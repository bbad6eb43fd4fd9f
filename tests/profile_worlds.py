"""Worlds for the scheduler-profile edge tests (tests/test_gpu_profile_edges.py): a snapshot, the prefix-index history that
warms it and a test batch, built from the CPU oracle alone so that tests/test_profile_worlds_cpu.py can check, without a GPU,
that each world reaches the edge its GPU test is about.  Everything is seeded: the same world comes out on every machine."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from oracle import oracle_py as o
from tests.helpers import synth_prompts, synth_snapshot, zipf_adapters

GOLDEN = 0x9E3779B97F4A7C15
SCORER = dict(queue=o.SCORER_QUEUE, kv=o.SCORER_KV_CACHE, prefix=o.SCORER_PREFIX, lora=o.SCORER_LORA,
              running=o.SCORER_RUNNING, latency=o.SCORER_LATENCY, token_load=o.SCORER_TOKEN_LOAD)
HEADLINE = [("queue", 2), ("kv", 2), ("prefix", 3), ("lora", 1)]
PREFILL = [("kv", 1), ("prefix", 2)]
QUEUE_RUNNING = [("queue", 1), ("running", 1.5), ("prefix", 2)]
EXC_MAX = 44        # distinct endpoints a sparse-pick request holds before it is deferred (pick_sparse.cu kExcMax)
INLINE_EPS = 10     # endpoints a table slot holds inline; larger sets live in bitset rows
SLICE_MIN = 2048    # a device batch is cut into K slices only while R / K >= this
LAT_COEF = dict(ttft_intercept=12.5, ttft_kv=80.0, ttft_input=0.031, ttft_waiting=7.25, ttft_running=1.5,
                ttft_prefix=-40.0, tpot_intercept=9.0, tpot_kv=11.0, tpot_input=0.0007, tpot_waiting=0.9,
                tpot_running=0.35, tpot_generated=0.01)
TOKEN_THR = 50000.0
BLOCK, MAX_BLOCKS = 64, 256


def seed_of(seed, p):
    """tie seed of profile p (include/eppscore.h: eppscore_profile)"""
    return (seed ^ (p * GOLDEN)) & (2 ** 64 - 1)


def bits(M, members, words=None):
    """uint32 natural-order bitmask of `members` in `words` words (default ceil(M/32))"""
    words = max((M + 31) // 32, 1) if words is None else words
    out = np.zeros(words, np.uint32)
    for m in members:
        out[m >> 5] |= np.uint32(1 << (m & 31))
    return out


def members_of(mask, M):
    """endpoints < M whose bit is set in a natural-order mask (missing words are 0)"""
    mask = np.asarray(mask, np.uint32)
    return [m for m in range(M) if (m >> 5) < mask.size and (int(mask[m >> 5]) >> (m & 31)) & 1]


def hash_rows(prompts, prompt_len, seed):
    """block hashes [R, MAX_BLOCKS] and counts [R] of R equal-length prompts (flattened bytes), by the oracle"""
    P = np.asarray(prompts, np.uint8).reshape(-1, prompt_len)
    h = np.zeros((len(P), MAX_BLOCKS), np.uint64)
    n = np.zeros(len(P), np.uint16)
    for r, p in enumerate(P):
        x = o.hash_prompt(p.tobytes(), seed, BLOCK, MAX_BLOCKS)
        h[r, :len(x)] = x
        n[r] = len(x)
    return h, n


def oracle_run(world, scorers, tie_mode, seed, pick_mode=0, subset=None, run_mask=None, snap=None, latency=None, idx=None):
    """oracle_py.schedule_batch of one run: `subset` a natural-order endpoint mask (any number of words: bits at or past M and
    missing words count as 0), the candidates of request r subset ∧ run_mask[r]"""
    M, R = world.M, world.R
    prof = o.make_profile([(SCORER[k], w) for k, w in scorers], tie_mode=tie_mode, tie_seed=seed, pick_mode=pick_mode,
                          latency=latency, token_load_threshold=TOKEN_THR)
    mask = None
    if subset is not None or run_mask is not None:
        mw = (M + 31) // 32
        mask = np.full((R, mw), 0xFFFFFFFF, np.uint32)
        if subset is not None:
            mask &= bits(M, members_of(subset, M))[None, :]
        if run_mask is not None:
            mask &= run_mask
    return o.schedule_batch(world.snap() if snap is None else snap, prof, world.index() if idx is None else idx, R,
                            cand_mask=mask, n_threads=8, **world.kw)


class World(SimpleNamespace):
    """M, R, max_endpoints, sd (snapshot arrays), warm [(pick, hashes, n_hashes)] committed in order, kw (the test batch)"""

    def snap(self, **extra):
        return o.SnapshotData(**self.sd, **extra)

    def index(self):
        idx = o.Index()
        for pick, h, n in self.warm:
            idx.commit(pick, h, n)
        return idx

    def commit(self, prompts, prompt_len, picks):
        h, n = hash_rows(prompts, prompt_len, self.model_seed)
        self.warm.append((np.asarray(picks, np.int32), h, n))

    def batch_hashes(self):
        return hash_rows(self.kw["prompt_bytes"], self.prompt_len, self.model_seed)


def _new(M, R, prompt_len=1024, max_endpoints=None, **kw):
    return World(M=M, R=R, max_endpoints=max_endpoints or M, prompt_len=prompt_len, warm=[],
                 model_seed=o.model_seed("profile-edges"), **kw)


def _batch(w, prompts, adapters, **extra):
    R = w.R
    w.kw = dict(prompt_bytes=np.ascontiguousarray(prompts, np.uint8).reshape(-1),
                prompt_off=np.arange(R + 1, dtype=np.int64) * w.prompt_len, model_seed=np.full(R, w.model_seed, np.uint64),
                adapter_id=np.asarray(adapters, np.int32), **extra)


def _rand_prompts(rng, n, length):
    return rng.integers(97, 123, size=(n, length), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. a subset that drops the zero-match arg-max
ARGMAX_SCORERS = [("queue", 2), ("kv", 2), ("prefix", 1), ("lora", 1)]
ARGMAX_ADAPTERS = [0, 1, 2, 3, 4, 5, 6, -1]


def world_argmax():
    """M = 200, members = the even endpoints.  Every endpoint has queue 5 and kv 0.5 (zero-match score 2 + 1 + 0 + lora), except
    the hand-placed ones below; with scorers queue 2, kv 2, prefix 1, lora 1 the zero-match score G[a][m] of adapter row a is
      row 0: non-members 1, 3 active (4.0); every member 3.0
      row 1: non-member 5 active with kv 0.25 (4.5), non-member 7 active (4.0); every member 3.0
      row 2: non-member 9 waiting (3.6); every member 3.0
      row 3: non-members 11, 13 active (4.0), member 14 active with kv 0.75 (3.5): one member at the member maximum
      row 4: non-member 15 and member 16 active (4.0): the member maximum ties with a non-member
      row 5: members 20, 22, 24 active (4.0), non-member 21 active with kv 0.25 (4.5): three members at the member maximum
      rows 6.. and the unknown adapter: non-members 5, 21 (kv 0.25, 3.5); every member 3.0
    Test prompts (R = 400, kinds x adapters cover every pair): F fully cached on member 30 (4.0 = the member maximum of rows
    4 and 5: exceptions that tie), W fully cached on member 20, P 12 of 16 blocks on member 40 and non-member 41 (3.75), N cached
    on non-members only, U unmatched."""
    M, R = 200, 400
    w = _new(M, R, members=list(range(0, M, 2)))
    kv = np.full(M, 0.5)
    kv[[5, 21]] = 0.25
    kv[14] = 0.75
    act = np.zeros((M, 1), np.uint64)
    wai = np.zeros((M, 1), np.uint64)
    for a, eps in {0: [1, 3], 1: [5, 7], 3: [11, 13, 14], 4: [15, 16], 5: [20, 21, 22, 24]}.items():
        for m in eps:
            act[m, 0] |= np.uint64(1 << a)
    wai[9, 0] |= np.uint64(1 << 2)
    w.sd = dict(kv_usage=kv, queue=np.full(M, 5, np.int64), running=np.full(M, 3, np.int64), lora_active=act,
                lora_waiting=wai, lora_nmodels=np.zeros(M, np.int32), lora_max=np.zeros(M, np.int32))
    rng = np.random.Generator(np.random.PCG64(11))
    L = w.prompt_len
    full_f, full_w = _rand_prompts(rng, 6, L), _rand_prompts(rng, 6, L)
    pre_p, pre_n = _rand_prompts(rng, 1, 768)[0], _rand_prompts(rng, 1, 768)[0]
    w.commit(full_f, L, [30] * 6)
    w.commit(full_w, L, [20] * 6)
    warm_p = np.concatenate([np.tile(pre_p, (2, 1)), _rand_prompts(rng, 2, L - 768)], axis=1)
    w.commit(warm_p, L, [40, 41])
    warm_n = np.concatenate([np.tile(pre_n, (4, 1)), _rand_prompts(rng, 4, L - 768)], axis=1)
    w.commit(warm_n, L, [1, 3, 5, 7])
    prompts = np.empty((R, L), np.uint8)
    w.kind = np.array(["FWPNU"[r % 5] for r in range(R)])
    adapters = np.array([ARGMAX_ADAPTERS[(r // 5) % len(ARGMAX_ADAPTERS)] for r in range(R)], np.int32)
    for r in range(R):
        k = w.kind[r]
        if k == "F":
            prompts[r] = full_f[r % 6]
        elif k == "W":
            prompts[r] = full_w[r % 6]
        elif k in "PN":
            prompts[r, :768] = pre_p if k == "P" else pre_n
            prompts[r, 768:] = _rand_prompts(rng, 1, L - 768)[0]
        else:
            prompts[r] = _rand_prompts(rng, 1, L)[0]
    _batch(w, prompts, adapters)
    return w


# ---------------------------------------------------------------------------------------------------------------------------
# 2. deferral on a subset profile
DEFER_CLASSES = "abcdef"


def world_deferral():
    """M = 512, members = the even endpoints, a synthetic snapshot.  Six request classes, 40 requests each (new tails on a
    768-byte cached prefix, so 12 of 16 blocks match):
      a  the prefix is cached on 30 members and 30 non-members       (60 distinct endpoints: deferred, members among them)
      b  on 50 non-members                                          (deferred, no member)
      c  on 20 members and 30 non-members                           (20 members, 50 endpoints in all: deferred)
      d  the first 8 blocks on 19 endpoints, blocks 8.. on 3 of them (bitset-row slots, then inline sets)
      e  on 2 members and 1 non-member, every block the same set     (the hash kernel resolves it)
      f  nothing cached"""
    M, R = 512, 240
    w = _new(M, R, members=list(range(0, M, 2)))
    w.sd = synth_snapshot(M, seed=21)
    rng = np.random.Generator(np.random.PCG64(22))
    L = w.prompt_len
    ev, od = rng.permutation(np.arange(0, M, 2)), rng.permutation(np.arange(1, M, 2))
    sets = dict(a=np.concatenate([ev[:30], od[:30]]), b=od[30:80], c=np.concatenate([ev[30:50], od[80:110]]),
                e=np.array([ev[50], ev[51], od[110]]))
    d_wide, d_narrow = np.concatenate([ev[52:60], od[111:119]]), np.array([ev[60], od[119], od[120]])
    w.sets = dict(sets, d=np.concatenate([d_wide, d_narrow]))
    prefixes = {c: _rand_prompts(rng, 1, 768)[0] for c in "abcdef"}
    for c in "abce":
        eps = sets[c]
        warm = np.concatenate([np.tile(prefixes[c], (len(eps), 1)), _rand_prompts(rng, len(eps), L - 768)], axis=1)
        w.commit(warm, L, eps)
    # class d: 512-byte prompts (the first 8 blocks of the prefix) on d_wide, whole prompts on d_narrow
    warm = np.concatenate([np.tile(prefixes["d"], (3, 1)), _rand_prompts(rng, 3, L - 768)], axis=1)
    w.commit(warm, L, d_narrow)
    w.commit(np.tile(prefixes["d"][:512], (len(d_wide), 1)), 512, d_wide)
    w.cls = np.array([DEFER_CLASSES[r % 6] for r in range(R)])
    prompts = np.empty((R, L), np.uint8)
    for r in range(R):
        prompts[r, :768] = prefixes[w.cls[r]]
        prompts[r, 768:] = _rand_prompts(rng, 1, L - 768)[0]
    _batch(w, prompts, zipf_adapters(R, seed=23))
    return w


# ---------------------------------------------------------------------------------------------------------------------------
# 3. masked min/max over members
MINMAX_VARIANTS = ("bucket_by_subset", "scan", "big_base")


def world_minmax(variant):
    """M = 200 (not a multiple of 32) in an engine of max_endpoints 256; members = endpoints m with m % 3 != 0.
      bucket_by_subset  queue / running ranges over all endpoints >= 256, over the members < 256: the value-bucket table
                        is valid only because of the subset
      scan              member ranges >= 256: the masked kernels scan
      big_base          member values near 2^40 with ranges < 256 (non-members far below): the table's base is not small"""
    M, R = 200, 256
    w = _new(M, R, max_endpoints=256, members=[m for m in range(M) if m % 3])
    rng = np.random.Generator(np.random.PCG64(31 + MINMAX_VARIANTS.index(variant)))
    mem = np.array([m % 3 != 0 for m in range(M)])
    q, run = np.zeros(M, np.int64), np.zeros(M, np.int64)
    if variant == "bucket_by_subset":
        q[mem] = 1000 + rng.integers(0, 200, mem.sum())
        q[~mem] = rng.choice([0, 5000], (~mem).sum())
        run[mem] = 50 + rng.integers(0, 100, mem.sum())
        run[~mem] = 10000 + rng.integers(0, 5, (~mem).sum())
    elif variant == "scan":
        q[mem] = rng.integers(0, 100000, mem.sum())
        q[~mem] = rng.integers(0, 10, (~mem).sum())
        run[mem] = rng.integers(0, 2000, mem.sum())
        run[~mem] = rng.integers(0, 10, (~mem).sum())
    else:
        q[mem] = 2 ** 40 + rng.integers(0, 250, mem.sum())
        q[~mem] = rng.integers(0, 100, (~mem).sum())
        run[mem] = 2 ** 40 + 12345 + rng.integers(0, 200, mem.sum())
        run[~mem] = 2 ** 41 + rng.integers(0, 100, (~mem).sum())
    sd = synth_snapshot(M, seed=32)
    sd.update(kv_usage=np.round(rng.random(M), 1), queue=q, running=run)
    w.sd = sd
    L = w.prompt_len
    pw, _, _ = synth_prompts(60, prompt_len=L, groups=6, shared=768, seed=33, prefix_seed=34)
    w.commit(pw, L, rng.integers(0, M, 60))
    pt, _, _ = synth_prompts(R, prompt_len=L, groups=8, shared=768, seed=35, prefix_seed=34)
    _batch(w, pt, zipf_adapters(R, seed=36))
    return w


def minmax_encodings(w):
    """the member set written four ways: (name, mask words, effective members)"""
    M, mem = w.M, w.members
    above = bits(256, mem, 8)
    above |= bits(256, range(M, 256), 8)               # bits at or above M (< max_endpoints): no endpoint there
    past = np.zeros(12, np.uint32)
    past[:7] = bits(M, mem)
    past[8:] = 0xFFFFFFFF                               # bits past max_endpoints: ignored
    short = bits(M, mem)[:3]                            # fewer than Mpad / 32 words: the missing words are 0
    return [("plain", bits(M, mem), mem), ("above_M", above, mem), ("past_max", past, mem),
            ("short", short, [m for m in mem if m < 96])]


def short_run_mask(R, M, rng, words):
    """a run mask of `words` words per request in an [R, ceil(M/32)] array (the rest 0) — the oracle's view of it"""
    mw = (M + 31) // 32
    b = np.zeros((R, mw * 32), bool)
    b[:, :M] = rng.random((R, M)) < 0.6
    m = (b.reshape(R, mw, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)
    m[:, words:] = 0
    return m


def value_range(v, members):
    v = np.asarray(v, np.int64)[list(members)]
    return int(v.max()) - int(v.min())


# ---------------------------------------------------------------------------------------------------------------------------
# 4. sliced device batches with profile runs
SLICE_R, SLICE_M = 12288, 1024


def world_sliced():
    """R = 12288 (six slices of 2048), M = 1024: the test batch of test_gpu_profiles.build_world, scaled up.  Pool a is cached
    on a few endpoints per prefix, pool b's two prefixes on 60 endpoints each (deferred), pool c is not cached."""
    M, R = SLICE_M, SLICE_R
    w = _new(M, R)
    w.sd = synth_snapshot(M, seed=41)
    rng = np.random.Generator(np.random.PCG64(41))
    L = w.prompt_len
    pa, _, ga = synth_prompts(240, prompt_len=L, groups=40, shared=768, seed=41, prefix_seed=100)
    pb, _, _ = synth_prompts(120, prompt_len=L, groups=2, shared=768, seed=42, prefix_seed=200)
    w.commit(pa, L, np.where(ga < 20, 2 * ((ga * 7 + np.arange(240)) % (M // 2)) + 1, rng.integers(0, M, 240)))
    w.commit(pb, L, rng.permutation(M)[:120])
    qa, _, _ = synth_prompts(6144, prompt_len=L, groups=40, shared=768, seed=47, prefix_seed=100)
    qb, _, _ = synth_prompts(3072, prompt_len=L, groups=2, shared=768, seed=48, prefix_seed=200)
    qc, _, _ = synth_prompts(3072, prompt_len=L, groups=4, shared=768, seed=49, prefix_seed=300)
    prompts = np.concatenate([qa, qb, qc]).reshape(R, L)
    perm = rng.permutation(R)          # the pools spread over every slice
    w.pool = np.repeat(np.array(list("abc")), [6144, 3072, 3072])[perm]
    _batch(w, prompts[perm], zipf_adapters(R, seed=43))
    return w


def sliced_profiles(M):
    """(scorers, pick_mode, subset) of profiles 0..3"""
    return [(HEADLINE, 0, bits(M, range(0, M, 2))),
            (PREFILL, 0, bits(M, range(1, M, 2))),
            ([("kv", 1), ("prefix", 2)], 1, bits(M, range(0, M, 3))),
            ([("queue", 1), ("kv", 1), ("prefix", 1)], 0, None)]


# ---------------------------------------------------------------------------------------------------------------------------
# 5. producers feeding profiles >= 1
TOKEN_PROFILE = [("kv", 1), ("token_load", 2), ("prefix", 1)]
LATENCY_PROFILE = [("latency", 1), ("kv", 0.5)]


def world_producers():
    """M = 256, R = 512 requests with latency inputs, an index warmed on a few prefixes"""
    M, R = 256, 512
    w = _new(M, R)
    w.sd = synth_snapshot(M, seed=51)
    rng = np.random.Generator(np.random.PCG64(51))
    L = w.prompt_len
    pw, _, _ = synth_prompts(80, prompt_len=L, groups=8, shared=768, seed=52, prefix_seed=53)
    w.commit(pw, L, rng.integers(0, M, 80))
    pt, _, _ = synth_prompts(R, prompt_len=L, groups=10, shared=768, seed=54, prefix_seed=53)
    _batch(w, pt, zipf_adapters(R, seed=55), input_tokens=rng.integers(0, 6000, R).astype(np.int32),
           ttft_slo=rng.choice([0.0, 140.0, 400.0, 1e6], R), tpot_slo=rng.choice([0.0, 18.0, 24.0, 30.0, 80.0], R))
    w.token_subset = bits(M, range(0, M, 2))
    w.latency_subset = bits(M, range(M // 4, M))
    return w
