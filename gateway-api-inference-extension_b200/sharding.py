"""Host-side helpers for the multi-GPU layout (DESIGN.md §7): the request batch shards by request with no
data-path collective; the endpoint snapshot is packed into ONE contiguous tile so that a single broadcast
(NCCL over NVLink on GPUs, gloo in the CPU tests) replicates it, and each rank's engine then ingests it in
place (eppscore_set_snapshot, location=1)."""
from __future__ import annotations

import numpy as np

# field order and dtypes of the packed tile (== eppscore_snapshot's arrays)
SNAPSHOT_FIELDS = (("kv_usage", np.float64), ("queue", np.int64), ("running", np.int64), ("lora_active", np.uint64),
                   ("lora_waiting", np.uint64), ("lora_nmodels", np.int32), ("lora_max", np.int32))
# optional per-endpoint arrays (latency fold-in, token-load scorer); packed after the mandatory ones when present
OPTIONAL_FIELDS = (("min_tpot_slo", np.float64), ("dispatched", np.int32), ("prefill_role", np.uint8),
                   ("inflight_tokens", np.int64))


def snapshot_layout(M: int, lora_words: int, optional=()):
    """[(name, byte offset, nbytes, dtype, shape)] — every field starts 16-byte aligned.
    optional: names from OPTIONAL_FIELDS that the tile carries (every rank must pass the same tuple)."""
    out, off = [], 0
    for name, dt in SNAPSHOT_FIELDS + tuple(f for f in OPTIONAL_FIELDS if f[0] in optional):
        shape = (M, lora_words) if name in ("lora_active", "lora_waiting") else (M,)
        nbytes = int(np.prod(shape)) * np.dtype(dt).itemsize
        out.append((name, off, nbytes, np.dtype(dt), shape))
        off += (nbytes + 15) // 16 * 16
    return out, off


def pack_snapshot(snap: dict):
    M = len(snap["kv_usage"])
    lw = int(np.asarray(snap["lora_active"]).size // M) if M else 1
    layout, total = snapshot_layout(M, lw, tuple(n for n, _ in OPTIONAL_FIELDS if snap.get(n) is not None))
    buf = np.zeros(total, np.uint8)
    for name, off, nbytes, dt, shape in layout:
        buf[off:off + nbytes] = np.ascontiguousarray(snap[name], dtype=dt).reshape(-1).view(np.uint8)
    return buf, layout


def unpack_snapshot(buf: np.ndarray, layout):
    return {name: buf[off:off + nbytes].view(dt).reshape(shape) for name, off, nbytes, dt, shape in layout}


def shard_range(R_total: int, rank: int, world: int):
    """Contiguous request shard of a global batch; request_base = start keeps tie priorities shard-invariant."""
    start = R_total * rank // world
    stop = R_total * (rank + 1) // world
    return start, stop


def gather_commit_stream(dist, pick, n_hashes, hashes, g_pick, g_nh, g_hash):
    """The exchange step of the closed loop (DESIGN.md §7): every rank contributes its shard's PreRequest records — pick
    i32[R], block count u16[R], block hashes u64[R, B] — and receives all shards concatenated in RANK order, which is global
    request order when shard r holds requests [r*R, (r+1)*R).  The prefix index is a deterministic function of the ordered
    commit stream (approximateprefix/plugin.go:169-197, indexer.go:52-83), so every rank that replays the gathered stream with
    eppscore_commit_picks_device holds the same index.  Torch tensors (CUDA with NCCL, CPU with gloo); g_* are the
    preallocated [world*R ...] outputs.  NCCL has no 16-bit integer type: the counts travel as bytes."""
    import torch
    dist.all_gather_into_tensor(g_pick, pick)
    dist.all_gather_into_tensor(g_nh.view(torch.uint8), n_hashes.view(torch.uint8))
    dist.all_gather_into_tensor(g_hash, hashes)
    return g_pick, g_nh, g_hash


def gather_inflight_stream(dist, endpoint, tokens, g_endpoint, g_tokens):
    """The in-flight load counterpart (inflightload/producer.go:101-169): every rank contributes its shard's updates —
    endpoint i32[R] (-1: none), estimated tokens i64[R] — and receives every shard's, which it applies with one
    eppscore_inflight_add (or _release) of world*R entries.  The counters are sums of integer adds, so the order of the
    gathered stream does not matter, only that the set is complete: every rank then holds the counters of one process that
    applied all updates.  g_* are the preallocated [world*R] outputs."""
    dist.all_gather_into_tensor(g_endpoint, endpoint)
    dist.all_gather_into_tensor(g_tokens, tokens)
    return g_endpoint, g_tokens


def gather_running_stream(dist, endpoint, request_key, g_endpoint, g_key, tpot_slo=None, g_tpot=None):
    """The running-request queue counterpart (predictedlatency/requestcontrol_hooks.go:73-86,219): every rank contributes its
    shard's adds — endpoint i32[R] (-1: none), request key u64[R], tpot_slo f64[R] — or its removes (tpot_slo None), and
    receives every shard's in rank order, which it applies with one eppscore_running_add (or _remove) of world*R entries.
    Unlike the in-flight counters these updates do not commute when keys repeat (the first add of a key wins, a remove before
    an add finds nothing), so every replica must apply the same concatenation in global request order, as the commit stream
    does: shard r's requests are global requests [r*R, (r+1)*R).  Keys must be unique across shards; the caller assigns them
    (e.g. rank in the top bits, or a key derived from the globally unique x-request-id).  g_* are the preallocated [world*R]
    outputs; the keys travel as int64 (same bits)."""
    dist.all_gather_into_tensor(g_endpoint, endpoint)
    dist.all_gather_into_tensor(g_key, request_key)
    if tpot_slo is not None:
        dist.all_gather_into_tensor(g_tpot, tpot_slo)
    return g_endpoint, g_key, g_tpot
