"""Index states and queries for eppscore_prefix_match (matchLongestPrefix read at chosen endpoints), shared by the CPU emulator
test (tests/test_prefix_match_cpu.py) and the GPU test (tests/test_gpu_prefix_match.py).  A scenario is a list of commit batches
(tests/index_scenarios.Batch) and, after each, the queries to ask; the expected answer of a query is the oracle's
matchLongestPrefix (orc_match_longest_prefix) read at the listed endpoints, 0 for entries outside [0, limit)."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from tests.index_scenarios import Batch, _pack, grid_scenario


@dataclass
class Query:
    hashes: np.ndarray     # uint64 [R, stride]
    n_hashes: np.ndarray   # uint16 [R]
    endpoints: np.ndarray  # int32 [R, k]


@dataclass
class MatchScenario:
    name: str
    M: int                 # endpoints the commits use
    lru: int               # defaultLRUCapacityPerServer
    steps: list = field(default_factory=list)  # [(Batch, [Query, ...])]: commit, then ask
    caps: np.ndarray | None = None  # int32 [M] CacheNumBlocks per endpoint (0: default), or None
    lru_max: int = 0       # largest LRU capacity the commits name (0: lru)


def expected(idx, q: Query, limit: int) -> np.ndarray:
    """uint16 [R, k] from the oracle's indexer `idx`."""
    R, k = q.endpoints.shape
    out = np.zeros((R, k), np.uint16)
    for r in range(R):
        m = idx.match(q.hashes[r, : int(q.n_hashes[r])], limit)
        e = q.endpoints[r]
        ok = (e >= 0) & (e < limit)
        out[r, ok] = m[e[ok]]
    return out


def endpoint_lists(rng, R: int, k: int, M: int, limit: int) -> np.ndarray:
    """[R, k] lists: mostly endpoints in use, some -1 padding, some at or past `limit`."""
    e = rng.integers(0, M, size=(R, k)).astype(np.int32)
    u = rng.random((R, k))
    e[u < 0.1] = -1
    e[(u >= 0.1) & (u < 0.15)] = limit + rng.integers(0, 3)
    return e


def queries_for(b: Batch, rng, k: int, M: int, limit: int) -> Query:
    """The batch's own prompts, the same prompts with a fresh tail after a random cut, and prompts of fresh hashes."""
    R, stride = b.hashes.shape
    h = b.hashes.copy()
    nh = b.n_hashes.copy()
    kind = rng.integers(0, 3, size=R)
    for r in range(R):
        n = int(nh[r])
        if kind[r] == 1 and n:
            cut = int(rng.integers(0, n))
            h[r, cut:n] = rng.integers(1, 2 ** 63, size=n - cut, dtype=np.uint64)
        elif kind[r] == 2:
            h[r, :n] = rng.integers(1, 2 ** 63, size=n, dtype=np.uint64)
    return Query(h, nh, endpoint_lists(rng, R, k, M, limit))


# LRU capacities from 3 to 31 250: evictions empty sets all along the prompts
CHURN = [(6, 3, 300, 8, 0), (32, 5, 500, 12, 4), (8, 50, 1000, 64, 2), (16, 700, 1500, 40, 1), (64, 31250, 2000, 32, 0)]


def churn_scenario(M, lru, R, nmax, seed, k, limit, n_batches=3) -> MatchScenario:
    rng = np.random.Generator(np.random.PCG64(7000 + seed))
    k = min(k, limit)  # (k <= max_endpoints)
    sc = grid_scenario(M, lru, R, nmax, seed, n_batches=n_batches)
    steps = [(b, [queries_for(b, rng, k, M + 1, limit)]) for b in sc.batches]
    return MatchScenario(f"churn-lru{lru}", M + 1, lru, steps, sc.caps, sc.lru_max)


def _one(pick, h):
    return _pack([(pick, np.asarray(h, np.uint64))])


def crafted_scenarios(limit: int) -> list:
    """Edge states, each with one query per interesting prompt (k = every endpoint, -1 and limit added)."""
    rng = np.random.Generator(np.random.PCG64(4242))
    fresh = lambda n: rng.integers(1, 2 ** 63, size=n, dtype=np.uint64)  # noqa: E731
    out = []

    def query(prompts, M):
        stride = max([len(p) for p in prompts] + [1])
        h = np.zeros((len(prompts), stride), np.uint64)
        nh = np.zeros(len(prompts), np.uint16)
        for r, p in enumerate(prompts):
            h[r, : len(p)] = p
            nh[r] = len(p)
        eps = np.tile(np.array(list(range(M)) + [-1, limit, limit + 7], np.int32), (len(prompts), 1))
        return Query(h, nh, eps)

    # a set that grows past the 10 inline members into an overflow row, one Add per endpoint
    M = 14
    p = fresh(6)
    steps = [(_one(m, p[: 2 + m % 5]), []) for m in range(M)]
    steps[-1] = (steps[-1][0], [query([p, p[:3], p[2:], fresh(4)], M)])
    out.append(MatchScenario("inline-to-row", M, 31250, steps))

    # a universal prefix: every endpoint holds it, each with its own tail
    M = 40
    u = fresh(20)
    tails = [fresh(5) for _ in range(M)]
    steps = [(_one(m, np.concatenate([u, tails[m]])), []) for m in range(M)]
    steps[-1] = (steps[-1][0], [query([np.concatenate([u, tails[3]]), u[:7], np.concatenate([u, fresh(3)])], M)])
    out.append(MatchScenario("universal-prefix", M, 31250, steps))

    # an emptied set in the middle of a prompt stops the walk; hits after the first miss do not count.  Endpoint 0 (LRU of 3)
    # holds h1, then h0 and h2; a fourth block evicts h1, whose set is now empty.  Endpoint 1 holds h2 only.
    M = 3
    h = fresh(3)
    z = fresh(1)
    steps = [(_one(0, h[1:2]), []), (_one(0, [h[0], h[2]]), []), (_one(1, h[2:3]), []),
             (_one(0, z), [query([h, h[:1], h[2:], np.concatenate([h[:1], fresh(1), h[2:]])], M)])]
    out.append(MatchScenario("emptied-mid-prompt", M, 3, steps))

    # an endpoint that holds only some of the hit blocks: its count is every hit block it holds, not a run
    M = 3
    p = fresh(8)
    steps = [(_one(0, p), []), (_one(1, p[[0, 2, 5]]), []), (_one(2, p[1:2]), [query([p, p[:4], p[:0]], M)])]
    out.append(MatchScenario("partial-holder", M, 31250, steps))

    # 0 hashes, and prompts of 256 and 1000 hashes: counts past 255
    M = 4
    p = fresh(1000)
    steps = [(_one(0, p), []), (_one(1, p[:300]), []), (_one(2, p[:256]), []),
             (_one(3, []), [query([p, p[:256], p[:0], np.concatenate([p[:600], fresh(400)])], M)])]
    out.append(MatchScenario("long-prompts", M, 31250, steps))
    return out
