"""The probing hash kernel (hash_warp_kernel<BC, true>: a warp hashes a tile of 32 requests, then walks each row's blocks
through the prefix index in rounds of slot loads) at its tile, half-tile and round edges, against the oracle bit for bit.
Every row has its own prompt and its own endpoint set, and the rows of a tile mix every way a request can leave the probe: resolved
(no match, a miss at the first block, at the last block of a 32-block pass, past one pass, a full match of 1 to 70 blocks,
an empty or sub-block prompt) or handed to pick_sparse (a different set partway, a bitset row as the first hit, a trailing
partial block, an unaligned start).  A probe result consumed for the wrong block changes the matched count of a row that
misses; one consumed for the wrong row changes its set; both change the pick or its score (the prefix scorer dominates
the profile).  Batch sizes cut the last tile and its halves at every edge; block_chars 96 runs the kernel's generic
block size; the hashes_out route checks the hashes the kernel writes and n_hashes."""
import numpy as np
import pytest

from oracle import oracle_py as o
from tests.helpers import synth_snapshot, zipf_adapters
from tests.score_constants import score_constants
from tests.test_gpu_score_edges import BASIC, assert_same, pkg  # noqa: F401

pytestmark = pytest.mark.gpu

K = score_constants()
MB, M = 256, 1000
PROFILE = [("kv", 1), ("prefix", 2)]
SEED0 = 0x9E3779B97F4A7C15
# (kind, full blocks, parameter): miss = first absent block, diff = first block of the second set
SPECS = [("none", 0, 0), ("short", 0, 0), ("none", 1, 0), ("none", 20, 0), ("full", 1, 0), ("full", 31, 0), ("full", 32, 0),
         ("full", 33, 0), ("full", 64, 0), ("full", 70, 0), ("miss", 32, 31), ("miss", 33, 31), ("miss", 33, 32), ("miss", 31, 15),
         ("miss", 16, 15), ("miss", 17, 16), ("miss", 64, 40), ("miss", 70, 63), ("miss", 40, 1), ("diff", 32, 13), ("diff", 40, 33),
         ("diff", 20, 1), ("diff", 64, 31), ("row", 12, 0), ("row", 40, 0), ("tail", 5, 0), ("tail", 32, 0), ("tail", 0, 0),
         ("unaligned", 10, 0), ("unaligned", 33, 0)]
NTEMPLATES = 97  # distinct prompts; row r uses prompt r % 97, so neighbouring rows always differ


class World:
    """One engine at a block size, the oracle's mirror of its snapshot and index, and NTEMPLATES prompts with their blocks
    entered in both indexes."""

    def __init__(self, pkg, bc, seed):
        self.pkg, self.bc = pkg, bc
        self.rng = np.random.Generator(np.random.PCG64(seed))
        sd = synth_snapshot(M, seed=seed)
        self.eng = pkg.Engine(pkg.default_config(PROFILE, max_endpoints=M, block_chars=bc, max_blocks=MB, prefix_capacity=1 << 16))
        self.eng.set_snapshot(**sd)
        self.snap = o.SnapshotData(**sd)
        self.prof = o.make_profile([(pkg.SCORER[k], w) for k, w in PROFILE])
        self.idx = o.Index()
        self.templates = self._templates()

    def add(self, hashes, ep):
        h = np.ascontiguousarray(hashes, np.uint64)
        self.eng.prefix_add(h, int(ep))
        self.idx.add(h, int(ep))

    def _templates(self):
        rng, bc = self.rng, self.bc
        order = [SPECS[i % len(SPECS)] for i in rng.permutation(NTEMPLATES)]
        # the last rows of the first half-tile and tile, and the first rows after them, leave the probe in different ways
        order[15], order[16], order[31], order[32] = ("miss", 32, 31), ("diff", 32, 13), ("row", 12, 0), ("none", 5, 0)
        out = []
        for kind, n, par in order:
            L = n * bc + (int(rng.integers(1, bc)) if kind == "tail" else 0) + (int(rng.integers(1, bc)) if kind == "short" else 0)
            body = rng.integers(97, 123, L, dtype=np.uint8)
            h, nh = self.pkg.Engine.hash_prompts_host(body, np.array([0, L], np.int64), np.full(1, SEED0, np.uint64),
                                                      block_chars=bc, max_blocks=MB)
            h = h[0, :n]
            S = [int(x) for x in rng.choice(M - 1, int(rng.integers(1, 3)), replace=False)]
            segs = {"full": [(0, n, S)], "miss": [(0, par, S)], "diff": [(0, par, S), (par, n, S + [M - 1])],
                    "row": [(0, n, [int(x) for x in rng.choice(M - 1, K.inline_eps + 2, replace=False)])],
                    "tail": [(0, n, S)], "unaligned": [(0, n, S)]}.get(kind, [])
            for b0, b1, eps in segs:
                for ep in eps:
                    if b1 > b0:
                        self.add(h[b0:b1], ep)
            # resolvable: an aligned start without a trailing partial block (a prompt shorter than one block has neither)
            out.append((kind, body, kind not in ("diff", "row", "unaligned") and not (kind == "tail" and n > 0)))
        return out

    def batch(self, R):
        """Rows r -> prompt r % NTEMPLATES: engine arguments (16-byte aligned starts unless 'unaligned', lengths through
        prompt_len), oracle arguments (the same prompts packed) and the number of rows the probe resolves."""
        rows = [self.templates[r % NTEMPLATES] for r in range(R)]
        chunks, offs, pos = [], [], 0
        for kind, body, _ in rows:
            pad = (-pos) % 16 + (int(self.rng.integers(1, 16)) if kind == "unaligned" else 0)
            chunks.append(np.full(pad, 32, np.uint8))
            pos += pad
            offs.append(pos)
            chunks.append(body)
            pos += len(body)
        lens = np.array([len(b) for _, b, _ in rows], np.int32)
        data = np.concatenate(chunks)
        off = np.array(offs + [pos], np.int64)
        poff = np.zeros(R + 1, np.int64)
        poff[1:] = np.cumsum(lens)
        seeds = np.full(R, SEED0, np.uint64)
        ad = zipf_adapters(R, seed=R)
        ekw = dict(prompt_bytes=data, prompt_off=off, prompt_len=lens, model_seed=seeds, adapter_id=ad)
        okw = dict(prompt_bytes=np.concatenate([b for _, b, _ in rows]), prompt_off=poff, model_seed=seeds, adapter_id=ad)
        return ekw, okw, sum(res for _, _, res in rows)

    def oracle(self, R, okw, **kw):
        return o.schedule_batch(self.snap, self.prof, self.idx, R, block_chars=self.bc, max_blocks=MB, n_threads=8, **okw, **kw)


@pytest.fixture(scope="module", params=[64, 96], ids=["bc64", "bc96"])
def world(request, pkg):  # noqa: F811
    w = World(pkg, request.param, seed=request.param)
    yield w
    w.eng.close()


@pytest.mark.parametrize("R", [1, 15, 16, 17, 31, 32, 33, 63, 65, 97 * 3 + 5, 65536])
def test_subtile_records_and_hashes(world, R):
    """Records route (picks, scores, ties, n_hashes and the resolved count) and the hashes_out route at every batch edge."""
    if R == 65536 and world.bc != 64:
        pytest.skip("the headline batch size runs at the headline block size")
    ekw, okw, resolved_want = world.batch(R)
    want = world.oracle(R, okw, want_hashes=True)
    eng = world.eng
    r0 = eng.stats().probe_resolved
    assert_same(eng.schedule(R, **ekw), want, BASIC, f"R={R} bc={world.bc} records")
    resolved = (eng.stats().probe_resolved - r0) % (1 << 32)
    assert resolved == resolved_want, f"R={R} bc={world.bc}: the hash kernel resolved {resolved} of {resolved_want}"
    got = eng.schedule(R, want_hashes=True, **ekw)
    assert_same(got, want, BASIC + ("hashes_out",), f"R={R} bc={world.bc} hashes_out")
    assert (eng.stats().probe_resolved - r0) % (1 << 32) == resolved_want  # the hashes_out batch takes no records


def test_subtile_graph_on_reserved_stream(world):
    """The batch captured in a CUDA graph on a reserved stream and replayed gives the oracle's picks and resolves the same
    rows on every replay."""
    import torch
    R = 2048 + 33
    ekw, okw, resolved_want = world.batch(R)
    want = world.oracle(R, okw)
    eng, dev = world.eng, torch.device("cuda", 0)
    t = {k: torch.from_numpy(np.ascontiguousarray(v).view(np.int64) if v.dtype == np.uint64 else np.ascontiguousarray(v)).to(dev)
         for k, v in ekw.items()}
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.int16, device=dev))
    s = torch.cuda.Stream(device=dev)
    eng.reserve_stream(s, R)

    def step():
        eng.schedule(R, prompt_bytes=t["prompt_bytes"], prompt_off=t["prompt_off"], prompt_len=t["prompt_len"], model_seed=t["model_seed"],
                     adapter_id=t["adapter_id"], device=True, stream=s.cuda_stream, out=out)

    def got():
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()} | {"total_blocks": out["total_blocks"].cpu().numpy().view(np.uint16)}

    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        assert_same(got(), want, BASIC, f"bc={world.bc} direct on the reserved stream")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
        for v in out.values():
            v.zero_()
        torch.cuda.synchronize()
        r0 = eng.stats().probe_resolved
        for _ in range(3):
            g.replay()
        assert_same(got(), want, BASIC, f"bc={world.bc} graph replay")
        assert (eng.stats().probe_resolved - r0) % (1 << 32) == 3 * resolved_want
    del g
