"""Sequential reference of eppscore_schedule_batch_inorder_index (test infrastructure only): R consecutive single-request
schedules on the CPU oracle, each followed by what PreRequest records for it — the prefix match at its pick before its own Add
(Index.match), the in-flight add of its tokens (Tracker.add) and the Add of its blocks at the pick (Index.commit) — so request
r + 1 is scored against the index and the load requests 0..r left."""
from __future__ import annotations

import numpy as np

from tests import inflight_oracle as I
from tests.inorder_reference import schedule_inorder


def schedule_inorder_index(snapshot: dict, profile, index, R: int, tokens=None, tracker: I.Tracker | None = None,
                           M: int | None = None, lru_capacity=None, *, prompt_bytes=None, prompt_off=None, model_seed=None,
                           hashes_in=None, n_hashes_in=None, adapter_id=None, cand_mask=None, request_base=0, block_chars=64,
                           max_blocks=256):
    """Returns (outputs, tracker): pick / pick_score / tie_count / total_blocks / pick_match [R] and hashes [R, stride] (the
    blocks each request committed: hashes_out for prompts, hashes_in when supplied), with `index` and `tracker` (a fresh one
    when None) advanced by every request.  snapshot: SnapshotData keyword arguments without inflight_tokens."""
    M = len(snapshot["kv_usage"]) if M is None else M
    tracker = I.Tracker() if tracker is None else tracker
    tokens = np.zeros(R, np.int64) if tokens is None else np.asarray(tokens, np.int64)
    stride = hashes_in.shape[1] if hashes_in is not None else max_blocks
    out = dict(pick=np.zeros(R, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32),
               total_blocks=np.zeros(R, np.uint16), pick_match=np.zeros(R, np.uint16), hashes=np.zeros((R, stride), np.uint64))
    for r in range(R):
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
        if cand_mask is not None:
            kw["cand_mask"] = cand_mask[r:r + 1]
        w, tracker = schedule_inorder(snapshot, profile, index, 1, tokens[r:r + 1], tracker=tracker, M=M, **kw)
        for k in ("pick", "pick_score", "tie_count", "total_blocks"):
            out[k][r] = w[k][0]
        n = int(w["total_blocks"][0])
        h = hashes_in[r] if hashes_in is not None else (w["hashes_out"][0] if "hashes_out" in w else np.zeros(stride, np.uint64))
        out["hashes"][r, :n] = h[:n]
        p = int(w["pick"][0])
        if p >= 0:
            out["pick_match"][r] = index.match(out["hashes"][r, :n], M)[p] if n else 0
            index.commit(w["pick"][:1], out["hashes"][r:r + 1], w["total_blocks"][:1], lru_capacity)
    return out, tracker
