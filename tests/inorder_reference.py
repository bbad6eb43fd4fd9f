"""Sequential reference of eppscore_schedule_batch_inorder (test infrastructure only): R consecutive single-request schedules
on the CPU oracle, each with the snapshot's inflight_tokens taken from the in-flight producer oracle (tests/inflight_oracle.py),
each followed by PreRequest's add of that request's tokens on its pick — the reference's Schedule + PreRequest sequence."""
from __future__ import annotations

import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I


def schedule_inorder(snapshot: dict, profile, index, R: int, tokens=None, tracker: I.Tracker | None = None, M: int | None = None,
                     *, prompt_bytes=None, prompt_off=None, model_seed=None, hashes_in=None, n_hashes_in=None, adapter_id=None,
                     cand_mask=None, request_base=0, block_chars=64, max_blocks=256, want_hashes=False):
    """Returns (outputs, tracker): pick / pick_score / tie_count / total_blocks [R] (and hashes_out [R, max_blocks]), with
    `tracker` (a fresh one when None) advanced by every pick.  snapshot: SnapshotData keyword arguments without inflight_tokens."""
    M = len(snapshot["kv_usage"]) if M is None else M
    tracker = I.Tracker() if tracker is None else tracker
    tokens = np.zeros(R, np.int64) if tokens is None else np.asarray(tokens, np.int64)
    out = dict(pick=np.zeros(R, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32),
               total_blocks=np.zeros(R, np.uint16))
    if want_hashes:
        out["hashes_out"] = np.zeros((R, max_blocks), np.uint64)
    for r in range(R):
        _, tok = tracker.get(M)
        snap = o.SnapshotData(**snapshot, inflight_tokens=tok)
        kw = {}
        if prompt_bytes is not None:
            a, b = int(prompt_off[r]), int(prompt_off[r + 1])
            kw.update(prompt_bytes=np.ascontiguousarray(prompt_bytes[a:b]), prompt_off=np.array([0, b - a], np.int64))
        if model_seed is not None:
            kw["model_seed"] = model_seed[r:r + 1]
        if hashes_in is not None:
            kw.update(hashes_in=hashes_in[r:r + 1], n_hashes_in=n_hashes_in[r:r + 1])
        if adapter_id is not None:
            kw["adapter_id"] = adapter_id[r:r + 1]
        if cand_mask is not None:
            kw["cand_mask"] = cand_mask[r:r + 1]
        w = o.schedule_batch(snap, profile, index, 1, request_base=request_base + r, block_chars=block_chars,
                             max_blocks=max_blocks, want_hashes=want_hashes, **kw)
        for k in out:
            out[k][r] = w[k][0]
        if w["pick"][0] >= 0:
            tracker.add(w["pick"][:1], tokens[r:r + 1])
    return out, tracker
