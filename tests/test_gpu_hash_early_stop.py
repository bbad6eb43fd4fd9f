"""The probing hash kernel (hash_warp_kernel<BC, true>) streams, chains and probes each request's blocks in chunks of
kProbeChunk and stops loading a request's bytes at its first miss while the request is still resolvable.  This checks it
against the oracle bit for bit (pick, score, tie count, total_blocks and the engine's count of resolved requests) with first
misses at every position relative to the chunk and 32-block window edges, set changes and bitset rows inside and after the
first chunk, trailing partial blocks after a full match and after an early miss, and batch sizes across the tile edge.
Every miss leaves the blocks after it in the index, so a walk that ran past the first miss, or a chunk chained from the
wrong value, changes the matched count and with it the pick or its score (the prefix scorer dominates the profile)."""
import os
import re

import numpy as np
import pytest

import _pkg
from oracle import oracle_py as o
from tests.helpers import synth_snapshot, zipf_adapters
from tests.score_constants import score_constants

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "gateway-api-inference-extension_b200", "csrc", "hash_kernel.cu")) as f:
    KC = int(re.search(r"constexpr int kProbeChunk = (\d+);", f.read()).group(1))
INLINE = score_constants().inline_eps
MB, M = 256, 1000
PROFILE = [("kv", 1), ("prefix", 2)]
SEED0 = 0x5851F42D4C957F2D
KEYS = ("pick", "pick_score", "tie_count", "total_blocks")
N = 3 * KC + 3     # full blocks of a prompt that spans three chunks
NW = 32 + 2 * KC   # full blocks of a prompt that spans two 32-block windows


def specs():
    """(kind, full blocks, first miss or None, where the set changes or None, trailing partial block, resolvable)."""
    out = []
    for n in (N, NW):
        for miss in sorted({0, 1, KC - 1, KC, KC + 1, 2 * KC, n - 1}) + [None]:
            out.append(("miss", n, miss, None, False, True))
    for miss in (31, 32, 33, 32 + KC - 1, 32 + KC):
        out.append(("miss", NW, miss, None, False, True))
    for kind in ("diff", "row"):            # a second set (inline / a bitset row) from block `at` up to the miss
        for at in (1, KC - 1, KC, KC + 1, 2 * KC):
            out.append((kind, N, at + KC if at + KC < N else None, at, False, False))
        out.append((kind, NW, 33, 32, False, False))
    out.append(("row", N, KC + 2, 0, False, False))     # a bitset row as the first hit
    for miss in (0, KC - 1, KC + 1, None):              # a trailing partial block after an early miss / a full match
        out.append(("tail", N, miss, None, True, False))
    out.append(("tail", 0, None, None, True, True))     # shorter than one block: no full block, no trailing one
    out.append(("miss", 0, None, None, False, True))    # empty
    return out


class World:
    def __init__(self, pkg, bc, seed):
        self.pkg, self.bc = pkg, bc
        self.rng = np.random.Generator(np.random.PCG64(seed))
        sd = synth_snapshot(M, seed=seed)
        self.eng = pkg.Engine(pkg.default_config(PROFILE, max_endpoints=M, block_chars=bc, max_blocks=MB, prefix_capacity=1 << 16))
        self.eng.set_snapshot(**sd)
        self.snap = o.SnapshotData(**sd)
        self.prof = o.make_profile([(pkg.SCORER[k], w) for k, w in PROFILE])
        self.idx = o.Index()
        self.templates = [self._template(*s) for s in specs()]

    def _add(self, h, ep):
        h = np.ascontiguousarray(h, np.uint64)
        if len(h):
            self.eng.prefix_add(h, int(ep))
            self.idx.add(h, int(ep))

    def _template(self, kind, n, miss, at, tail, resolvable):
        rng, bc = self.rng, self.bc
        L = n * bc + (int(rng.integers(1, bc)) if tail else 0)
        body = rng.integers(97, 123, L, dtype=np.uint8)
        h, _ = self.pkg.Engine.hash_prompts_host(body, np.array([0, L], np.int64), np.full(1, SEED0, np.uint64),
                                                 block_chars=bc, max_blocks=MB)
        h = h[0, :n]
        end = n if miss is None else miss
        S = [int(x) for x in rng.choice(M - 1, int(rng.integers(1, 3)), replace=False)]
        if kind == "row" and at == 0:
            S = [int(x) for x in rng.choice(M - 1, INLINE + 2, replace=False)]
        for ep in S:
            self._add(h[:end], ep)
            if miss is not None:
                self._add(h[miss + 1:], ep)  # blocks past the first miss are indexed: only the walk's stop hides them
        if kind in ("diff", "row") and at > 0:
            extra = [M - 1] if kind == "diff" else [int(x) for x in rng.choice(M - 1, INLINE + 2, replace=False) if x not in S]
            for ep in extra:
                self._add(h[at:end], ep)
        return body, resolvable

    def batch(self, R):
        """Row r takes template perm[r]: every tile mixes resolved rows that stop early with rows that stream to the end."""
        perm = self.rng.integers(0, len(self.templates), R)
        rows = [self.templates[i] for i in perm]
        lens = np.array([len(b) for b, _ in rows], np.int32)
        off = np.zeros(R + 1, np.int64)
        off[1:] = np.cumsum(lens)
        seeds = np.full(R, SEED0, np.uint64)
        ad = zipf_adapters(R, seed=R)
        data = np.concatenate([b for b, _ in rows]) if R else np.zeros(0, np.uint8)
        # 16-byte aligned starts, so every row takes the kernel's fast path
        starts = (-(-off[:-1] // 16)) * 16 + 16 * np.arange(R)
        packed = np.zeros(int(starts[-1] + lens[-1]) + 16, np.uint8)
        for r in range(R):
            packed[starts[r]:starts[r] + lens[r]] = rows[r][0]
        ekw = dict(prompt_bytes=packed, prompt_off=np.append(starts, len(packed)).astype(np.int64), prompt_len=lens,
                   model_seed=seeds, adapter_id=ad)
        okw = dict(prompt_bytes=data, prompt_off=off, model_seed=seeds, adapter_id=ad)
        return ekw, okw, sum(res for _, res in rows)


@pytest.fixture(scope="module")
def pkg():
    _pkg.load_build().build()
    return _pkg.load()


@pytest.fixture(scope="module", params=[64, 96], ids=["bc64", "bc96"])
def world(request, pkg):
    w = World(pkg, request.param, seed=1000 + request.param)
    yield w
    w.eng.close()


def test_specs_reach_their_edges():
    """The first misses and set changes sit at the chunk and window edges they name."""
    got = {(k, n, m) for k, n, m, _, _, _ in specs()}
    for m in (0, KC - 1, KC, KC + 1, N - 1, None):
        assert ("miss", N, m) in got
    for m in (31, 32, 33, NW - 1):
        assert ("miss", NW, m) in got
    assert {a for k, _, _, a, _, _ in specs() if k == "diff"} >= {1, KC - 1, KC, KC + 1}
    assert {a for k, _, _, a, _, _ in specs() if k == "row"} >= {0, 1, KC - 1, KC, KC + 1}


@pytest.mark.parametrize("R", [1, 31, 32, 33, 63, 64, 65, 257, 4099])
def test_early_stop_against_oracle(world, R):
    ekw, okw, resolved_want = world.batch(R)
    want = o.schedule_batch(world.snap, world.prof, world.idx, R, block_chars=world.bc, max_blocks=MB, n_threads=8, **okw)
    eng = world.eng
    r0 = eng.stats().probe_resolved
    got = eng.schedule(R, **ekw)
    for k in KEYS:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        if g.dtype.kind == "f":
            g, w = g.view(np.uint64), w.astype(np.float64).view(np.uint64)
        bad = np.flatnonzero(g != w)
        assert bad.size == 0, f"bc={world.bc} R={R} {k}: {bad.size} rows differ, first {bad[:5]}"
    resolved = (eng.stats().probe_resolved - r0) % (1 << 32)
    assert resolved == resolved_want, f"bc={world.bc} R={R}: the hash kernel resolved {resolved} of {resolved_want}"
