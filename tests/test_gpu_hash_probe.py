"""The hash kernel's probe of the prefix index (hash_warp_kernel<BC, true>) and pick_sparse's use of its records, against the
oracle bit for bit.  Batches come as prompt bytes, so the device hashes them; the index holds chosen sets for the blocks of
chosen prompts, so every way a request can leave the probe shows up: resolved (no match, a first-block miss, a uniform set of
1, 2, 3 or 10 members, matched in part, in full or across chunks, up to an emptied set, a key past another one's home slot)
or handed to pick_sparse's own probe (a different set partway, a bitset row, more than kExcMax endpoints, a trailing partial
block, an unaligned start) — mixed inside one warp's tile of 32 requests.  The engine's count of resolved
requests shows that the record route is the one taken."""
import numpy as np
import pytest

from tests.helpers import synth_snapshot, zipf_adapters
from tests.score_constants import score_constants
from tests.test_gpu_score_edges import BASIC, HEADLINE, SPARSE_EPS, WIDE, Case, assert_same, pkg  # noqa: F401

pytestmark = pytest.mark.gpu

K = score_constants()
BC, MB = 64, 256
EP = [("kv", 1), ("prefix", 2)]
PROFILES = {"EPL": HEADLINE, "EP": EP, "generic": WIDE}
KINDS = ("none", "first_miss", "uni1", "uni2", "uni3", "uni10", "part", "full256", "miss_chunk2", "diff", "diff_chunk2",
         "row", "many", "emptied", "tail", "unaligned", "collide")
RESOLVED = {"none", "first_miss", "uni1", "uni2", "uni3", "uni10", "part", "full256", "miss_chunk2", "emptied", "collide"}


def colliding_pairs(case, rng, seeds0, n):
    """n pairs of one-block prompts whose hashes share a home slot of the engine's table (h & mask): the second one entered
    lies past the first on the probe chain."""
    slots = 2 * case.engines[0].stats().prefix_capacity  # the table holds `capacity` hashes at load 0.5
    N = max(8192, int(3 * np.sqrt(2 * n * slots)))  # ~ N^2 / (2 slots) pairs
    cand = rng.integers(97, 123, (N, BC), dtype=np.uint8)
    off = np.arange(0, (N + 1) * BC, BC, dtype=np.int64)
    h, _ = case.pkg.Engine.hash_prompts_host(cand.reshape(-1), off, np.full(N, seeds0, np.uint64), block_chars=BC, max_blocks=MB)
    home = h[:, 0] & np.uint64(slots - 1)
    first, pairs = {}, []
    for i, x in enumerate(home.tolist()):
        if x in first:
            pairs.append((first.pop(x), i))
        else:
            first[x] = i
    assert len(pairs) >= n, "not enough colliding homes"
    return slots, [(cand[i], cand[j], h[i, 0], h[j, 0]) for i, j in pairs[:n]]


def build_batch(case, rng, R, max_ep, sole):
    """R prompts, request r of kind KINDS[(7r + r // 32) % len(KINDS)] (every tile holds a different mix), with their block
    sets entered in the index; endpoint `sole` holds the blocks that are emptied afterwards.  Returns the kinds, the engine's
    arguments (16-byte aligned starts unless 'unaligned', lengths through prompt_len) and the oracle's (the same prompts,
    packed back to back)."""
    kinds = [KINDS[(r * 7 + r // 32) % len(KINDS)] for r in range(R)]
    seed0 = 0x9E3779B97F4A7C15
    slots, pairs = colliding_pairs(case, rng, seed0, kinds.count("collide"))
    nblocks = {"full256": MB, "miss_chunk2": 70, "diff_chunk2": 70, "many": 8}
    prompts, chunks, offs, pos = [], [], [], 0
    for k in kinds:
        n = nblocks.get(k, int(rng.integers(2, 40)))
        L = n * BC + (int(rng.integers(1, BC)) if k == "tail" else 0)
        pad = (-pos) % 16 + (int(rng.integers(1, 16)) if k == "unaligned" else 0)
        chunks.append(rng.integers(97, 123, pad, dtype=np.uint8))
        pos += pad
        offs.append(pos)
        prompts.append(pairs.pop()[:] if k == "collide" else rng.integers(97, 123, L, dtype=np.uint8))
        body = prompts[-1][1] if k == "collide" else prompts[-1]
        chunks.append(body)
        pos += len(body)
    lens = np.array([len(p[1]) if k == "collide" else len(p) for p, k in zip(prompts, kinds)], np.int32)
    data = np.concatenate(chunks)
    off = np.array(offs + [pos], np.int64)
    seeds = np.full(R, seed0, np.uint64)
    hashes, nh = case.pkg.Engine.hash_prompts_host(data, off, seeds, prompt_len=lens, block_chars=BC, max_blocks=MB)
    pick_set = lambda s: [int(x) for x in rng.choice(max_ep - 2, s, replace=False)]  # noqa: E731
    for r, k in enumerate(kinds):
        h, n = hashes[r], int(nh[r])
        nfull = int(lens[r]) // BC
        S = pick_set(int(rng.integers(1, 5)))
        if k == "none":
            continue
        if k == "collide":
            partner, mine = prompts[r][2], prompts[r][3]
            assert (partner & np.uint64(slots - 1)) == (mine & np.uint64(slots - 1)) and mine == h[0]
            for ep in S:
                case.add([partner], ep)
            segs = [(0, 1, S)]
        elif k == "first_miss":
            segs = [(1, n, S)]
        elif k.startswith("uni"):
            segs = [(0, n, pick_set(int(k[3:])))]
        elif k == "part":
            segs = [(0, int(rng.integers(0, n + 1)), S)]
        elif k == "full256":
            segs = [(0, n, S)]
        elif k == "miss_chunk2":
            segs = [(0, 33, S), (34, n, S)]
        elif k == "diff":
            p = int(rng.integers(1, n))
            segs = [(0, p, S), (p, n, S + [max_ep - 1])]
        elif k == "diff_chunk2":
            segs = [(0, 37, S), (37, n, S + [max_ep - 1])]
        elif k == "row":
            segs = [(0, n, pick_set(K.inline_eps + 2))]
        elif k == "many":
            segs = [(b, b + 1, pick_set(K.inline_eps)) for b in range(min(n, 6))]
        elif k == "emptied":
            p = int(rng.integers(0, n))
            segs = [(0, p, S), (p + 1, n, S)]
            case.add(h[p:p + 1], sole)
        else:  # tail, unaligned: a uniform set over the full blocks
            segs = [(0, nfull, S)]
        for b0, b1, eps in segs:
            for ep in eps:
                if b1 > b0:
                    case.add(h[b0:b1], ep)
    case.remove_endpoint(sole)
    assert 2 * case.engines[0].stats().prefix_capacity == slots  # no rebuild moved the homes
    packed = np.concatenate([p[1] if k == "collide" else p for p, k in zip(prompts, kinds)])
    poff = np.zeros(R + 1, np.int64)
    poff[1:] = np.cumsum(lens)
    ad = zipf_adapters(R, seed=R)
    ekw = dict(prompt_bytes=data, prompt_off=off, prompt_len=lens, model_seed=seeds, adapter_id=ad)
    okw = dict(prompt_bytes=packed, prompt_off=poff, model_seed=seeds, adapter_id=ad)
    return kinds, ekw, okw


def check_routes(case, R, ekw, okw, kinds, where):
    eng = case.engines[0]
    want = case.oracle(R, want_hashes=True, **okw)
    r0 = eng.stats().probe_resolved
    assert_same(eng.schedule(R, **ekw), want, BASIC, f"{where} records")
    resolved = (eng.stats().probe_resolved - r0) % (1 << 32)
    assert resolved == sum(k in RESOLVED for k in kinds), f"{where}: the hash kernel resolved {resolved} requests"
    got = eng.schedule(R, want_hashes=True, **ekw)
    assert_same(got, want, BASIC + ("hashes_out",), f"{where} hashes_out (no records)")
    return want


@pytest.mark.parametrize("tie_mode", [0, 1])
@pytest.mark.parametrize("profile", ["EPL", "EP", "generic"])
@pytest.mark.parametrize("J", [1, 2, 4, 8])
def test_probe_records_every_kind(pkg, J, profile, tie_mode):
    """Every kind of request mixed in each tile, R not a multiple of 32, on every geometry, sequence and tie mode."""
    max_ep = SPARSE_EPS[J]
    rng = np.random.Generator(np.random.PCG64(J * 100 + tie_mode * 10 + len(profile)))
    case = Case(pkg, PROFILES[profile], max_ep, max_ep, tie_mode=tie_mode, seed=J, tie_heavy=True, prefix_capacity=1 << 16)
    R = 32 * 7 + 13
    kinds, ekw, kw = build_batch(case, rng, R, max_ep, sole=max_ep - 2)
    want = check_routes(case, R, ekw, kw, kinds, f"J={J} {profile}")
    matched = (want["match_blocks"] > 0).sum(axis=1)
    k = np.array(kinds)
    assert (matched[k == "many"] > K.exc_max).all()          # deferred to the full-matrix pass
    assert (want["match_blocks"].max(axis=1)[k == "full256"] == MB).all()
    assert (want["total_blocks"][k == "tail"] == ekw["prompt_len"][k == "tail"] // BC + 1).all()
    assert (ekw["prompt_off"][:-1][k == "unaligned"] % 16 != 0).all() and (ekw["prompt_off"][:-1][k != "unaligned"] % 16 == 0).all()
    if J == 1 and profile == "EPL" and tie_mode == 0:
        case.check(R, kw, topk=True, where="every route")      # the routes that never take records agree too (packed prompts)
    case.close()


def test_probe_graph_side_stream_and_slices(pkg):
    """The step as the benchmark runs it: device-resident inputs, the snapshot prepared on a second stream while the batch is
    hashed and probed, the whole step captured in a CUDA graph and replayed; then the same batch cut into slices over
    several streams (debug keys 5 and 6)."""
    import torch
    max_ep = SPARSE_EPS[1]
    rng = np.random.Generator(np.random.PCG64(4242))
    case = Case(pkg, HEADLINE, max_ep, max_ep, seed=42, prefix_capacity=1 << 19)
    R = 4 * 2048 + 77
    kinds, kw, okw = build_batch(case, rng, R, max_ep, sole=max_ep - 2)
    want = case.oracle(R, want_hashes=True, **okw)
    eng = case.engines[0]
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(np.ascontiguousarray(v).view(np.int64) if v.dtype == np.uint64 else np.ascontiguousarray(v)).to(dev)
         for k, v in kw.items()}
    snap = synth_snapshot(max_ep, seed=42)  # what Case set on the engine
    sd = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in snap.items()}
    stream, side = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    out = dict(pick=torch.empty(R, dtype=torch.int32, device=dev), pick_score=torch.empty(R, dtype=torch.float64, device=dev),
               tie_count=torch.empty(R, dtype=torch.int32, device=dev), total_blocks=torch.empty(R, dtype=torch.int16, device=dev))

    def step():
        side.wait_stream(stream)
        eng.set_snapshot(sd["kv_usage"].data_ptr(), sd["queue"].data_ptr(), sd["running"].data_ptr(), sd["lora_active"].data_ptr(),
                         sd["lora_waiting"].data_ptr(), sd["lora_nmodels"].data_ptr(), sd["lora_max"].data_ptr(), device=True,
                         stream=side.cuda_stream, M=max_ep, lora_words=snap["lora_active"].size // max_ep)
        eng.schedule(R, prompt_bytes=t["prompt_bytes"], prompt_off=t["prompt_off"], prompt_len=t["prompt_len"],
                     model_seed=t["model_seed"], adapter_id=t["adapter_id"], device=True, stream=stream.cuda_stream, out=out)

    def got():
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()} | {"total_blocks": out["total_blocks"].cpu().numpy().view(np.uint16)}

    with torch.cuda.stream(stream):
        r0 = eng.stats().probe_resolved
        step()
        assert_same(got(), want, BASIC, "direct")
        assert (eng.stats().probe_resolved - r0) % (1 << 32) == sum(k in RESOLVED for k in kinds)
        for v in out.values():
            v.zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            step()
        for _ in range(3):
            g.replay()
        assert_same(got(), want, BASIC, "graph")
        for split, streams in ((4, 2), (3, 3), (5, 4)):
            eng.set_debug(5, split)
            eng.set_debug(6, streams)
            for v in out.values():
                v.zero_()
            step()
            assert_same(got(), want, BASIC, f"sliced {split}x{streams}")
        eng.set_debug(5, 1)
    case.close()
