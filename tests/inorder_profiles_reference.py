"""Sequential reference of eppscore_schedule_batch_inorder_profiles (test infrastructure only): R consecutive single-request
Schedule calls over several profile runs on the CPU oracle, each followed, when the primary run picked, by what PreRequest
records for it: the prefix match at every run's pick before the request's Adds (Index.match), the in-flight add of its tokens
at every run's pick (Tracker.add, producer.go:106-119) and, in the index form, the Adds of its blocks at the primary pick and
then at the prefill pick (Index.commit, approximateprefix/plugin.go:177-197)."""
from __future__ import annotations

import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I

GOLDEN = 0x9E3779B97F4A7C15


def seed_of(seed: int, p: int) -> int:
    """tie seed of profile p (include/eppscore.h: eppscore_profile)"""
    return (seed ^ (p * GOLDEN)) & (2 ** 64 - 1)


def subset_rows(M: int, R: int, subset=None, cand_mask=None):
    """candidate rows [R, ceil(M/32)] of a run: its natural-order endpoint subset ∧ its cand_mask, or None for every endpoint"""
    if subset is None and cand_mask is None:
        return None
    mw = max((M + 31) // 32, 1)
    rows = np.full((R, mw), 0xFFFFFFFF, np.uint32)
    if subset is not None:
        s = np.zeros(mw, np.uint32)
        sub = np.asarray(subset, np.uint32)
        s[:min(mw, sub.size)] = sub[:mw]
        rows &= s[None, :]
    if cand_mask is not None:
        rows &= np.asarray(cand_mask, np.uint32).reshape(R, mw)
    return rows


def schedule_inorder_profiles(snapshot: dict, runs, index, R: int, tokens=None, tracker: I.Tracker | None = None,
                              M: int | None = None, *, ordered_index=False, primary_run=0, prefill_run=-1, run_mask=None,
                              lru_capacity=None, tie_mode=o.TIE_LOWEST_INDEX, tie_seed=0, token_load_threshold=0.0,
                              prompt_bytes=None, prompt_off=None, model_seed=None, hashes_in=None, n_hashes_in=None,
                              adapter_id=None, request_base=0, block_chars=64, max_blocks=256):
    """runs: [{"profile": id, "scorers": [(kind, w)], "pick_mode": 0, "subset": natural-order mask or None,
    "cand_mask": [R, ceil(M/32)] or None}].  ordered_index: the index form (request r's prefix scorer sees the Adds of requests
    0..r-1); otherwise `index` stays as it is (the in-flight form scores against the frozen index).
    Returns (batch outputs {total_blocks, hashes}, [per-run {pick, pick_score, tie_count, pick_match}], tracker)."""
    M = len(snapshot["kv_usage"]) if M is None else M
    tracker = I.Tracker() if tracker is None else tracker
    tokens = np.zeros(R, np.int64) if tokens is None else np.asarray(tokens, np.int64)
    stride = hashes_in.shape[1] if hashes_in is not None else max_blocks
    profs = [o.make_profile(u["scorers"], tie_mode=tie_mode, tie_seed=seed_of(tie_seed, u["profile"]),
                            pick_mode=u.get("pick_mode", 0), token_load_threshold=token_load_threshold) for u in runs]
    rows = [subset_rows(M, R, u.get("subset"), u.get("cand_mask")) for u in runs]
    out = dict(total_blocks=np.zeros(R, np.uint16), hashes=np.zeros((R, stride), np.uint64))
    outs = [dict(pick=np.full(R, -1, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32),
                 pick_match=np.zeros(R, np.uint16)) for _ in runs]
    for r in range(R):
        _, tok = tracker.get(M)
        snap = o.SnapshotData(**snapshot, inflight_tokens=tok)
        kw = dict(request_base=request_base + r, block_chars=block_chars, max_blocks=max_blocks)
        if prompt_bytes is not None and hashes_in is None:
            a, b = int(prompt_off[r]), int(prompt_off[r + 1])
            kw.update(prompt_bytes=np.ascontiguousarray(prompt_bytes[a:b]), prompt_off=np.array([0, b - a], np.int64),
                      want_hashes=True)
            if model_seed is not None:
                kw["model_seed"] = model_seed[r:r + 1]
        if hashes_in is not None:
            kw.update(hashes_in=hashes_in[r:r + 1], n_hashes_in=n_hashes_in[r:r + 1])
        if adapter_id is not None:
            kw["adapter_id"] = adapter_id[r:r + 1]
        bits = 0xF if run_mask is None else int(run_mask[r])
        w = None
        for i, prof in enumerate(profs):
            mask = None if rows[i] is None else rows[i][r:r + 1]
            if not (bits >> i) & 1:  # the handler did not pick this run: no candidate
                mask = np.zeros((1, max((M + 31) // 32, 1)), np.uint32)
            w = o.schedule_batch(snap, prof, index, 1, cand_mask=mask, **kw)
            outs[i]["pick"][r] = w["pick"][0]
            outs[i]["pick_score"][r] = w["pick_score"][0]
            outs[i]["tie_count"][r] = w["tie_count"][0]
        n = int(w["total_blocks"][0])
        out["total_blocks"][r] = n
        h = hashes_in[r] if hashes_in is not None else (w["hashes_out"][0] if "hashes_out" in w else np.zeros(stride, np.uint64))
        out["hashes"][r, :n] = h[:n]
        if outs[primary_run]["pick"][r] < 0:
            continue
        picked = [int(x["pick"][r]) for x in outs if x["pick"][r] >= 0]
        match = index.match(out["hashes"][r, :n], M) if n else np.zeros(M, np.uint16)
        for x in outs:
            if x["pick"][r] >= 0:
                x["pick_match"][r] = match[int(x["pick"][r])]
        tracker.add(np.array(picked, np.int32), np.full(len(picked), tokens[r], np.int64))
        if ordered_index:
            for j in (primary_run, prefill_run):
                if j >= 0 and outs[j]["pick"][r] >= 0:
                    index.commit(outs[j]["pick"][r:r + 1], out["hashes"][r:r + 1], out["total_blocks"][r:r + 1], lru_capacity)
    return out, outs, tracker
