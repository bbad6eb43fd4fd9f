"""Sequential reference of eppscore_schedule_batch_inorder_latency (test infrastructure only): R consecutive single-request
schedules on the CPU oracle, each with a snapshot whose min_tpot_slo / dispatched come from the running-request queue oracle
(tests/running_oracle.py) and whose inflight_tokens come from the in-flight producer oracle (tests/inflight_oracle.py), each
followed by what PreRequest records for it: the queue add of (pick, key, tpot), the in-flight add of its tokens and, in the
index form, the prefix match at its pick before its own Add and the Add of its blocks (Index.commit)."""
from __future__ import annotations

import numpy as np

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q


def schedule_inorder_latency(snapshot: dict, profile, index, R: int, queues: Q.Queues, tokens=None, request_key=None,
                             tracker: I.Tracker | None = None, M: int | None = None, lru_capacity=None, index_form=False, *,
                             prompt_bytes=None, prompt_off=None, model_seed=None, hashes_in=None, n_hashes_in=None,
                             adapter_id=None, cand_mask=None, input_tokens=None, ttft_slo=None, tpot_slo=None, request_base=0,
                             block_chars=64, max_blocks=256):
    """Returns (outputs, tracker): pick / pick_score / tie_count / total_blocks / added [R] (and pick_match in the index form),
    with `queues`, `tracker` (a fresh one when None) and, in the index form, `index` advanced by every request.  snapshot:
    SnapshotData keyword arguments without min_tpot_slo, dispatched and inflight_tokens.  request_key None: nothing is added."""
    M = len(snapshot["kv_usage"]) if M is None else M
    tracker = I.Tracker() if tracker is None else tracker
    tokens = np.zeros(R, np.int64) if tokens is None else np.asarray(tokens, np.int64)
    out = dict(pick=np.zeros(R, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32),
               total_blocks=np.zeros(R, np.uint16), added=np.zeros(R, bool), pick_match=np.zeros(R, np.uint16))
    for r in range(R):
        mn, cnt = queues.get(M)
        snap = o.SnapshotData(**snapshot, min_tpot_slo=Q.canonical(mn), dispatched=cnt, inflight_tokens=tracker.get(M)[1])
        kw = dict(request_base=request_base + r, block_chars=block_chars, max_blocks=max_blocks)
        if prompt_bytes is not None and hashes_in is None:
            a, b = int(prompt_off[r]), int(prompt_off[r + 1])
            kw.update(prompt_bytes=np.ascontiguousarray(prompt_bytes[a:b]), prompt_off=np.array([0, b - a], np.int64),
                      want_hashes=True)
            if model_seed is not None:
                kw["model_seed"] = model_seed[r:r + 1]
        if hashes_in is not None:
            kw.update(hashes_in=hashes_in[r:r + 1], n_hashes_in=n_hashes_in[r:r + 1])
        for name, v in (("adapter_id", adapter_id), ("cand_mask", cand_mask), ("input_tokens", input_tokens),
                        ("ttft_slo", ttft_slo), ("tpot_slo", tpot_slo)):
            if v is not None:
                kw[name] = v[r:r + 1]
        if input_tokens is None and prompt_bytes is not None:  # len(strings.Fields(prompt)), as the engine counts it
            kw["input_tokens"] = np.array([o.count_fields(bytes(prompt_bytes[int(prompt_off[r]):int(prompt_off[r + 1])]))], np.int32)
        w = o.schedule_batch(snap, profile, index, 1, **kw)
        for k in ("pick", "pick_score", "tie_count", "total_blocks"):
            out[k][r] = w[k][0]
        p = int(w["pick"][0])
        if p < 0:
            continue
        if request_key is not None:
            tp = None if tpot_slo is None else tpot_slo[r:r + 1]
            out["added"][r] = queues.add(w["pick"][:1], request_key[r:r + 1], tp)[0]
        tracker.add(w["pick"][:1], tokens[r:r + 1])
        if index_form:
            n = int(w["total_blocks"][0])
            h = hashes_in[r] if hashes_in is not None else (w["hashes_out"][0] if "hashes_out" in w else np.zeros(1, np.uint64))
            hs = np.zeros((1, max(n, 1)), np.uint64)
            hs[0, :n] = h[:n]
            out["pick_match"][r] = index.match(hs[0, :n], M)[p] if n else 0
            index.commit(w["pick"][:1], hs, w["total_blocks"][:1], lru_capacity)
    return out, tracker
