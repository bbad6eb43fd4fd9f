"""Thin Python face of the C ABI (include/eppscore.h).  No arithmetic happens here: numpy arrays /
torch tensors are only handed to libeppscore.so as pointers."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import Batch, Config, EppscoreError, LatencyParams, Profile, ProfileRun, SCORER, Snapshot, Stats, TopK


def default_config(scorers=None, filters=(), **kw) -> Config:
    """scorers: list of (kind name | int, weight) in profile order; default = reference default config
    (queue 2, kv 2, prefix 3; pkg/epp/config/loader/defaults.go:46-103)."""
    cfg = Config()
    capi.lib().eppscore_config_default(C.byref(cfg))
    if scorers is not None:
        if len(scorers) > capi.MAX_SCORERS:
            raise ValueError("too many scorers")
        cfg.n_scorers = len(scorers)
        for i, (k, w) in enumerate(scorers):
            cfg.scorer_kind[i] = SCORER[k] if isinstance(k, str) else int(k)
            cfg.scorer_weight[i] = float(w)
    cfg.n_filters = len(filters)  # [(kind, (params...))] device-side filters, in order
    for i, (k, par) in enumerate(filters):
        cfg.filter_kind[i] = int(k)
        for j, v in enumerate(par):
            cfg.filter_param[i][j] = float(v)
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise TypeError(f"unknown config field {k}")
        setattr(cfg, k, v)
    return cfg


def latency_params(**kw) -> LatencyParams:
    """eppscore_latency_params with the reference defaults (predictedlatency/plugin.go:128-136,
    scorer/latency/plugin.go:83-90); keyword arguments override fields."""
    p = LatencyParams()
    capi.lib().eppscore_latency_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise TypeError(f"unknown latency field {k}")
        setattr(p, k, v)
    return p


# eppscore_latency_info as a numpy structured dtype (48 bytes, the C layout)
LATENCY_INFO_DTYPE = np.dtype([("ttft", "<f8"), ("tpot", "<f8"), ("ttft_headroom", "<f8"), ("tpot_headroom", "<f8"),
                               ("prefix_cache_score", "<f8"), ("dispatched", "<i4"), ("present", "u1"), ("ttft_valid", "u1"),
                               ("tpot_valid", "u1"), ("reserved", "u1")])
assert LATENCY_INFO_DTYPE.itemsize == C.sizeof(capi.LatencyInfo) == 48


def _is_torch(x) -> bool:
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _stream_handle(stream):
    """the raw cudaStream_t of a torch.cuda.Stream; raw handles and None pass through"""
    return getattr(stream, "cuda_stream", stream)


class _Args:
    """Keeps converted arrays alive for the duration of a call and yields raw pointers."""

    def __init__(self, device: bool):
        self.device = device
        self.keep = []

    def ptr(self, x, dtype):
        if x is None:
            return None
        if self.device:
            if isinstance(x, int):
                return x
            if not _is_torch(x) or not x.is_cuda:
                raise TypeError("device-location call needs CUDA tensors or raw device pointers")
            if not x.is_contiguous():
                raise ValueError("tensor must be contiguous")
            self.keep.append(x)
            return x.data_ptr()
        if _is_torch(x):
            x = x.numpy()
        a = np.ascontiguousarray(x, dtype=dtype)
        self.keep.append(a)
        return a.ctypes.data


class Engine:
    """One engine per CUDA device (eppscore_create)."""

    def __init__(self, config: Config | None = None, device: int = 0):
        self._lib = capi.lib()
        self.cfg = config if config is not None else default_config()
        h = C.c_void_p()
        rc = self._lib.eppscore_create(device, C.byref(self.cfg), C.byref(h))
        if rc != 0:
            raise EppscoreError(rc, (self._lib.eppscore_last_error(None) or b"").decode())
        self._h = h
        self.M = 0

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_h", None):
            self._lib.eppscore_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise EppscoreError(rc, (self._lib.eppscore_last_error(self._h) or b"").decode())
        return rc

    def stats(self) -> Stats:
        s = Stats()
        self._check(self._lib.eppscore_get_stats(self._h, C.byref(s)))
        return s

    def set_debug(self, key: int, value: int):
        self._check(self._lib.eppscore_set_debug(self._h, key, value))

    def set_latency_params(self, params: LatencyParams):
        """Takes effect at the next set_snapshot."""
        self._check(self._lib.eppscore_set_latency_params(self._h, C.byref(params)))

    # ------------------------------------------------------------------ snapshot
    def set_snapshot(self, kv_usage, queue, running=None, lora_active=None, lora_waiting=None, lora_nmodels=None,
                     lora_max=None, endpoint_cols=(), epoch=0, device=False, stream=None, M=None, lora_words=None,
                     min_tpot_slo=None, dispatched=None, prefill_role=None, inflight_tokens=None):
        a = _Args(device)
        s = Snapshot()
        s.struct_size = C.sizeof(Snapshot)
        if M is None:
            M = int(kv_usage.shape[0]) if hasattr(kv_usage, "shape") else len(kv_usage)
        s.M = M
        if lora_words is None:
            if lora_active is None:
                lora_words = 0
            else:
                n = int(np.prod(lora_active.shape)) if hasattr(lora_active, "shape") else len(lora_active)
                lora_words = (n // M) if M else 1
        s.lora_words = lora_words
        s.location = 1 if device else 0
        s.kv_usage = a.ptr(kv_usage, np.float64)
        s.queue = a.ptr(queue, np.int64)
        s.running = a.ptr(running, np.int64)
        s.lora_active = a.ptr(lora_active, np.uint64)
        s.lora_waiting = a.ptr(lora_waiting, np.uint64)
        s.lora_nmodels = a.ptr(lora_nmodels, np.int32)
        s.lora_max = a.ptr(lora_max, np.int32)
        for i, c in enumerate(endpoint_cols):
            s.endpoint_col[i] = a.ptr(c, np.float64)
        s.epoch = epoch
        s.stream = stream
        s.min_tpot_slo = a.ptr(min_tpot_slo, np.float64)
        s.dispatched = a.ptr(dispatched, np.int32)
        s.prefill_role = a.ptr(prefill_role, np.uint8)
        s.inflight_tokens = a.ptr(inflight_tokens, np.int64)
        self._check(self._lib.eppscore_set_snapshot(self._h, C.byref(s)))
        self.M = M

    # ------------------------------------------------------------------ the hot path
    def schedule(self, R, *, prompt_bytes=None, prompt_off=None, prompt_len=None, model_seed=None, hashes_in=None,
                 n_hashes_in=None, hash_stride=0, adapter_id=None, cand_mask=None, dense_feat=None, dense_total=None,
                 block_chars=0, max_blocks=0, request_base=0, want_match=False, want_total=True, want_hashes=False,
                 want_scores=False, input_tokens=None, ttft_slo=None, tpot_slo=None, want_pred=False, want_filter_mask=False,
                 topk=0, topk_wide=0, device=False, stream=None, out=None, _inorder=None):
        """Host mode (device=False): numpy in, returns dict of numpy outputs (copies inside the call).
        Device mode: CUDA tensors / raw pointers in; `out` must hold preallocated CUDA tensors
        (pick int32[R], pick_score float64[R], tie_count int32[R], optional match_blocks/total_blocks/hashes_out);
        the call is asynchronous on `stream`.
        topk=k (1..8): also the first k endpoints of every request's pick order (maxNumOfEndpoints, eppscore_topk):
        topk_pick int32[R, k] (-1 padded) and topk_score float64[R, k]; in device mode `out` holds them.
        topk_wide=k (1..max_endpoints): the same lists for any k (eppscore_schedule_batch_topk_wide), returned the same way."""
        if topk and topk_wide:
            raise ValueError("topk and topk_wide are exclusive")
        call, topk = ((self._lib.eppscore_schedule_batch_topk_wide, topk_wide) if topk_wide else
                      (self._lib.eppscore_schedule_batch_topk, topk))
        a = _Args(device)
        if _inorder is not None and len(_inorder) > 2:  # schedule_inorder_latency: (tokens, InOrderIndex | None, InOrderRunning)
            tok, ix, q = a.ptr(_inorder[0], np.int64), _inorder[1], _inorder[2]
            q.request_key = a.ptr(_inorder[3], np.uint64)
            call = lambda h, bp: self._lib.eppscore_schedule_batch_inorder_latency(h, bp, tok, None if ix is None else C.byref(ix),
                                                                                   C.byref(q))
        elif _inorder is not None and len(_inorder) > 1:  # schedule_inorder_index: (tokens, InOrderIndex)
            tok, ix = a.ptr(_inorder[0], np.int64), _inorder[1]
            call = lambda h, bp: self._lib.eppscore_schedule_batch_inorder_index(h, bp, tok, C.byref(ix))
        elif _inorder is not None:  # schedule_inorder: (tokens,)
            tok = a.ptr(_inorder[0], np.int64)
            call = lambda h, bp: self._lib.eppscore_schedule_batch_inorder(h, bp, tok)
        else:
            call = self._lib.eppscore_schedule_batch if not topk else call
        b = Batch()
        b.struct_size = C.sizeof(Batch)
        b.R = R
        b.location = 1 if device else 0
        b.request_base = request_base
        b.prompt_bytes = a.ptr(prompt_bytes, np.uint8)
        b.prompt_off = a.ptr(prompt_off, np.int64)
        b.prompt_len = a.ptr(prompt_len, np.int32)
        b.model_seed = a.ptr(model_seed, np.uint64)
        b.hashes_in = a.ptr(hashes_in, np.uint64)
        b.n_hashes_in = a.ptr(n_hashes_in, np.uint16)
        if hashes_in is not None and not hash_stride:
            hash_stride = int(hashes_in.shape[1])
        b.hash_stride = hash_stride
        b.block_chars = block_chars
        b.max_blocks = max_blocks
        b.adapter_id = a.ptr(adapter_id, np.int32)
        b.cand_mask = a.ptr(cand_mask, np.uint32)
        b.dense_feat = a.ptr(dense_feat, np.float32)
        b.dense_total = a.ptr(dense_total, np.uint16)
        b.input_tokens = a.ptr(input_tokens, np.int32)
        b.ttft_slo = a.ptr(ttft_slo, np.float64)
        b.tpot_slo = a.ptr(tpot_slo, np.float64)
        b.stream = stream
        if device:
            if out is None:
                raise ValueError("device mode needs preallocated outputs")
            b.pick = a.ptr(out["pick"], None)
            b.pick_score = a.ptr(out["pick_score"], None)
            b.tie_count = a.ptr(out["tie_count"], None)
            b.match_blocks = a.ptr(out.get("match_blocks"), None)
            b.total_blocks = a.ptr(out.get("total_blocks"), None)
            b.hashes_out = a.ptr(out.get("hashes_out"), None)
            b.scores_out = a.ptr(out.get("scores_out"), None)
            b.pred_out = a.ptr(out.get("pred_out"), None)
            b.filter_mask_out = a.ptr(out.get("filter_mask_out"), None)
            if topk:
                t = self._topk(topk, a.ptr(out["topk_pick"], None), a.ptr(out["topk_score"], None))
                self._check(call(self._h, C.byref(b), C.byref(t)))
            else:
                self._check(call(self._h, C.byref(b)))
            return out
        M = self.M
        mb = max_blocks or self.cfg.max_blocks
        res = dict(pick=np.full(R, -2, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32))
        if want_total:
            res["total_blocks"] = np.zeros(R, np.uint16)
        if want_match:
            res["match_blocks"] = np.zeros((R, M), np.uint16)
        if want_hashes:
            res["hashes_out"] = np.zeros((R, mb), np.uint64)
        if want_scores:
            res["scores_out"] = np.zeros((R, M), np.float64)
        if want_pred:
            res["pred_out"] = np.zeros((R, M, 2), np.float64)
        if want_filter_mask:
            res["filter_mask_out"] = np.zeros((R, max((M + 31) // 32, 1)), np.uint32)
        for k, v in res.items():
            setattr(b, k, v.ctypes.data)
        if topk:
            res["topk_pick"] = np.full((R, topk), -1, np.int32)
            res["topk_score"] = np.zeros((R, topk), np.float64)
            t = self._topk(topk, res["topk_pick"].ctypes.data, res["topk_score"].ctypes.data)
            self._check(call(self._h, C.byref(b), C.byref(t)))
        else:
            self._check(call(self._h, C.byref(b)))
        return res

    def schedule_inorder(self, R, tokens=None, **kw):
        """eppscore_schedule_batch_inorder: `schedule` for profile 0 with request r scored against the in-flight load that
        requests 0..r-1 were sent with, and each pick's tokens (int64[R], None = 0) added to the counters in order.  Takes the
        arguments of `schedule` except the R x M outputs, dense rows and top-k lists; host mode returns the same dict, device
        mode fills `out` asynchronously on `stream` (tokens then a CUDA tensor)."""
        for k in ("want_match", "want_scores", "want_pred", "want_filter_mask", "topk", "topk_wide"):
            if kw.get(k):
                raise ValueError(f"schedule_inorder does not take {k}")
        return self.schedule(R, _inorder=(tokens,), **kw)

    def schedule_inorder_index(self, R, tokens=None, lru_capacity=None, **kw):
        """eppscore_schedule_batch_inorder_index: `schedule_inorder` with request r also scored against the prefix index as
        requests 0..r-1's commits left it, and each request's blocks committed at its pick inside the call (do not commit the
        batch again).  lru_capacity: host int32[M] CacheNumBlocks or None.  Host mode returns the `schedule_inorder` dict plus
        pick_match uint16[R] (matchBlocks at each pick before its own Add); device mode fills `out` asynchronously on `stream`,
        pick_match included when `out` has it."""
        for k in ("want_match", "want_scores", "want_pred", "want_filter_mask", "topk", "topk_wide"):
            if kw.get(k):
                raise ValueError(f"schedule_inorder_index does not take {k}")
        x = capi.InOrderIndex()
        x.struct_size = C.sizeof(capi.InOrderIndex)
        caps = None if lru_capacity is None else np.ascontiguousarray(lru_capacity, np.int32)
        x.lru_capacity = None if caps is None else caps.ctypes.data
        if kw.get("device"):
            out = kw.get("out") or {}
            pm = out.get("pick_match")
            x.pick_match = None if pm is None else _Args(True).ptr(pm, None)
            return self.schedule(R, _inorder=(tokens, x), **kw)
        pick_match = np.zeros(R, np.uint16)
        x.pick_match = pick_match.ctypes.data
        res = self.schedule(R, _inorder=(tokens, x), **kw)
        res["pick_match"] = pick_match
        return res

    def schedule_inorder_latency(self, R, tokens=None, request_key=None, index=False, lru_capacity=None, **kw):
        """eppscore_schedule_batch_inorder_latency: `schedule_inorder` (index=True: `schedule_inorder_index`) for a profile 0 with
        the latency scorer, request r's latency scorer seeing the running-request queues after requests 0..r-1 were added to
        them: each request joins its pick's queue inside the call with key request_key[r] (uint64[R]; None: the queues are read,
        never changed) and tpot tpot_slo[r].  Host mode returns the `schedule_inorder(_index)` dict plus added bool[R]; device
        mode fills `out` asynchronously on `stream`, with added_out (uint8[R]) and pick_match when `out` has them."""
        for k in ("want_match", "want_scores", "want_pred", "want_filter_mask", "topk", "topk_wide"):
            if kw.get(k):
                raise ValueError(f"schedule_inorder_latency does not take {k}")
        x = None
        if index:
            x = capi.InOrderIndex()
            x.struct_size = C.sizeof(capi.InOrderIndex)
            caps = None if lru_capacity is None else np.ascontiguousarray(lru_capacity, np.int32)
            x.lru_capacity = None if caps is None else caps.ctypes.data
        q = capi.InOrderRunning()
        q.struct_size = C.sizeof(capi.InOrderRunning)
        if kw.get("device"):
            out = kw.get("out") or {}
            dev = _Args(True)
            if x is not None:
                pm = out.get("pick_match")
                x.pick_match = None if pm is None else dev.ptr(pm, None)
            ad = out.get("added_out")
            q.added_out = None if ad is None else dev.ptr(ad, None)
            return self.schedule(R, _inorder=(tokens, x, q, request_key), **kw)
        added = np.zeros(max(R, 1), np.uint8)
        q.added_out = added.ctypes.data
        pick_match = np.zeros(max(R, 1), np.uint16)
        if x is not None:
            x.pick_match = pick_match.ctypes.data
        res = self.schedule(R, _inorder=(tokens, x, q, request_key), **kw)
        res["added"] = added[:R].astype(bool)
        if x is not None:
            res["pick_match"] = pick_match[:R]
        return res

    # ------------------------------------------------------------------ several scheduler profiles
    def add_profile(self, scorers, pick_mode=0, filters=()) -> int:
        """eppscore_add_profile: scorers [(kind name | int, weight)] in profile order, the picker and the device-side
        filters [(kind, (params...))]; everything else is the engine's.  Returns the profile id."""
        if len(scorers) > capi.MAX_SCORERS or len(filters) > 4:
            raise ValueError("too many scorers or filters")
        p = Profile()
        p.struct_size = C.sizeof(Profile)
        p.n_scorers = len(scorers)
        for i, (k, w) in enumerate(scorers):
            p.scorer_kind[i] = SCORER[k] if isinstance(k, str) else int(k)
            p.scorer_weight[i] = float(w)
        p.pick_mode = pick_mode
        p.n_filters = len(filters)
        for i, (k, par) in enumerate(filters):
            p.filter_kind[i] = int(k)
            for j, v in enumerate(par):
                p.filter_param[i][j] = float(v)
        pid = C.c_int32()
        self._check(self._lib.eppscore_add_profile(self._h, C.byref(p), C.byref(pid)))
        return pid.value

    def set_profile_endpoints(self, profile: int, mask=None):
        """The profile's endpoint subset as a uint32 bitmask over endpoint rows (None: every endpoint); applied by the next
        set_snapshot."""
        a = _Args(False)
        words = 0 if mask is None else int(np.asarray(mask).size)
        self._check(self._lib.eppscore_set_profile_endpoints(self._h, profile, a.ptr(mask, np.uint32), words))

    def schedule_profiles(self, R, runs, *, prompt_bytes=None, prompt_off=None, prompt_len=None, model_seed=None, hashes_in=None,
                          n_hashes_in=None, hash_stride=0, adapter_id=None, dense_feat=None, dense_total=None, block_chars=0,
                          max_blocks=0, request_base=0, want_match=False, want_total=True, want_hashes=False, input_tokens=None,
                          ttft_slo=None, tpot_slo=None, device=False, stream=None, out=None, _inorder=None):
        """eppscore_schedule_batch_profiles: one hash stage, then one Filter -> Score -> Pick per run.  runs: list of dicts
        {"profile": id, "cand_mask": optional, "want_scores" / "want_pred" / "want_filter_mask": optional bools (host mode)};
        in device mode each run dict also holds its preallocated outputs (pick, pick_score, tie_count, optional scores_out,
        pred_out, filter_mask_out) and `out` the batch's (total_blocks, match_blocks, hashes_out).
        A run's "topk": k (0..max_endpoints) also asks for the first k endpoints of its pick order; any k > 0 makes the call
        eppscore_schedule_batch_profiles_topk.  Host mode returns them as topk_pick int32[R, k] (-1 padded) and topk_score
        float64[R, k] in the run's outputs dict; device mode takes them preallocated in the run dict under the same names.
        Host mode returns (batch outputs dict, [per-run outputs dict])."""
        a = _Args(device)
        b = Batch()
        b.struct_size = C.sizeof(Batch)
        b.R = R
        b.location = 1 if device else 0
        b.request_base = request_base
        b.prompt_bytes = a.ptr(prompt_bytes, np.uint8)
        b.prompt_off = a.ptr(prompt_off, np.int64)
        b.prompt_len = a.ptr(prompt_len, np.int32)
        b.model_seed = a.ptr(model_seed, np.uint64)
        b.hashes_in = a.ptr(hashes_in, np.uint64)
        b.n_hashes_in = a.ptr(n_hashes_in, np.uint16)
        if hashes_in is not None and not hash_stride:
            hash_stride = int(hashes_in.shape[1])
        b.hash_stride = hash_stride
        b.block_chars = block_chars
        b.max_blocks = max_blocks
        b.adapter_id = a.ptr(adapter_id, np.int32)
        b.dense_feat = a.ptr(dense_feat, np.float32)
        b.dense_total = a.ptr(dense_total, np.uint16)
        b.input_tokens = a.ptr(input_tokens, np.int32)
        b.ttft_slo = a.ptr(ttft_slo, np.float64)
        b.tpot_slo = a.ptr(tpot_slo, np.float64)
        b.stream = stream
        arr = (ProfileRun * len(runs))()
        M = self.M
        mw = max((M + 31) // 32, 1)
        res_runs = []
        tarr = (TopK * len(runs))()
        with_lists = any(run.get("topk", 0) for run in runs)
        for i, run in enumerate(runs):
            x = arr[i]
            x.struct_size = C.sizeof(ProfileRun)
            x.profile = run["profile"]
            x.cand_mask = a.ptr(run.get("cand_mask"), np.uint32)
            tk = int(run.get("topk", 0))
            tarr[i].struct_size = C.sizeof(TopK)
            tarr[i].k = tk
            if device:
                for k in ("pick", "pick_score", "tie_count", "scores_out", "pred_out", "filter_mask_out"):
                    setattr(x, k, a.ptr(run.get(k), None))
                if tk:
                    tarr[i].endpoints = a.ptr(run.get("topk_pick"), None)
                    tarr[i].scores = a.ptr(run.get("topk_score"), None)
                continue
            o = dict(pick=np.full(R, -2, np.int32), pick_score=np.zeros(R, np.float64), tie_count=np.zeros(R, np.int32))
            if tk > 0:
                o["topk_pick"] = np.full((R, tk), -1, np.int32)
                o["topk_score"] = np.zeros((R, tk), np.float64)
                tarr[i].endpoints = o["topk_pick"].ctypes.data
                tarr[i].scores = o["topk_score"].ctypes.data
            if run.get("want_scores"):
                o["scores_out"] = np.zeros((R, M), np.float64)
            if run.get("want_pred"):
                o["pred_out"] = np.zeros((R, M, 2), np.float64)
            if run.get("want_filter_mask"):
                o["filter_mask_out"] = np.zeros((R, mw), np.uint32)
            for k, v in o.items():
                if not k.startswith("topk_"):
                    setattr(x, k, v.ctypes.data)
            res_runs.append(o)

        if _inorder is not None:  # schedule_inorder_profiles: (tokens, InOrderProfiles)
            tok, x = a.ptr(_inorder[0], np.int64), _inorder[1]
            x.run_mask = a.ptr(_inorder[2], np.uint8)
            for i, run in enumerate(runs):
                if device:
                    x.pick_match[i] = a.ptr(run.get("pick_match"), None)
                else:
                    res_runs[i]["pick_match"] = np.zeros(max(R, 1), np.uint16)
                    x.pick_match[i] = res_runs[i]["pick_match"].ctypes.data

        def call():
            if _inorder is not None:
                return self._lib.eppscore_schedule_batch_inorder_profiles(self._h, C.byref(b), tok, len(runs), arr, C.byref(x))
            if with_lists:
                return self._lib.eppscore_schedule_batch_profiles_topk(self._h, C.byref(b), len(runs), arr, tarr)
            return self._lib.eppscore_schedule_batch_profiles(self._h, C.byref(b), len(runs), arr)

        if device:
            if out is None:
                out = {}
            b.match_blocks = a.ptr(out.get("match_blocks"), None)
            b.total_blocks = a.ptr(out.get("total_blocks"), None)
            b.hashes_out = a.ptr(out.get("hashes_out"), None)
            self._check(call())
            return out, runs
        res = {}
        if want_total:
            res["total_blocks"] = np.zeros(R, np.uint16)
        if want_match:
            res["match_blocks"] = np.zeros((R, M), np.uint16)
        if want_hashes:
            res["hashes_out"] = np.zeros((R, max_blocks or self.cfg.max_blocks), np.uint64)
        for k, v in res.items():
            setattr(b, k, v.ctypes.data)
        self._check(call())
        if _inorder is not None:
            for o in res_runs:
                o["pick_match"] = o["pick_match"][:R]
        return res, res_runs

    def schedule_inorder_profiles(self, R, runs, tokens=None, index=False, primary_run=0, prefill_run=-1, run_mask=None,
                                  lru_capacity=None, **kw):
        """eppscore_schedule_batch_inorder_profiles: `schedule_profiles` with request r's runs scored against the in-flight load
        (index=True: and the prefix index) that requests 0..r-1 left, and, when the primary run picked, each run's pick counted
        with tokens[r] (int64[R], None = 0) and the primary and prefill picks' Adds made inside the call (do not commit the batch
        again).  run_mask: uint8[R], bit i = run i runs for request r (None: every run).  lru_capacity: host int32[M] or None.
        Takes the arguments of `schedule_profiles` except match_blocks and the runs' R x M outputs and lists.  Host mode returns
        (batch outputs, [run outputs]) with each run's pick_match uint16[R]; device mode fills the runs' outputs (pick_match when
        the run dict has it) asynchronously on `stream`."""
        if kw.get("want_match") or kw.get("dense_feat") is not None:
            raise ValueError("schedule_inorder_profiles does not take want_match or dense_feat")
        for run in runs:
            for k in ("want_scores", "want_pred", "want_filter_mask", "topk"):
                if run.get(k):
                    raise ValueError(f"schedule_inorder_profiles does not take a run's {k}")
        x = capi.InOrderProfiles()
        x.struct_size = C.sizeof(capi.InOrderProfiles)
        x.index = 1 if index else 0
        x.primary_run = primary_run
        x.prefill_run = prefill_run
        caps = None if lru_capacity is None else np.ascontiguousarray(lru_capacity, np.int32)
        x.lru_capacity = None if caps is None else caps.ctypes.data
        return self.schedule_profiles(R, runs, _inorder=(tokens, x, run_mask), **kw)

    @staticmethod
    def _topk(k, endpoints, scores) -> TopK:
        t = TopK()
        t.struct_size = C.sizeof(TopK)
        t.k = k
        t.endpoints = endpoints
        t.scores = scores
        return t

    def hash_prompts(self, prompt_bytes, prompt_off, model_seed=None, prompt_len=None, block_chars=0, max_blocks=0):
        R = len(prompt_off) - 1
        mb = max_blocks or self.cfg.max_blocks
        a = _Args(False)
        hashes = np.zeros((max(R, 1), mb), np.uint64)
        n = np.zeros(max(R, 1), np.uint16)
        self._check(self._lib.eppscore_hash_prompts(
            self._h, R, 0, a.ptr(prompt_bytes, np.uint8), a.ptr(prompt_off, np.int64), a.ptr(prompt_len, np.int32),
            a.ptr(model_seed, np.uint64), block_chars, max_blocks, hashes.ctypes.data, n.ctypes.data, None))
        return hashes[:R], n[:R]

    @staticmethod
    def hash_prompts_host(prompt_bytes, prompt_off, model_seed=None, prompt_len=None, block_chars=64, max_blocks=256, stride=0,
                          n_threads=0, out=None):
        """hashPrompt on the host cores (library worker pool).  Returns (hashes [R, stride], n_hashes [R])."""
        R = len(prompt_off) - 1
        stride = stride or max_blocks
        a = _Args(False)
        if out is None:
            out = (np.empty((max(R, 1), stride), np.uint64), np.empty(max(R, 1), np.uint16))
        rc = capi.lib().eppscore_hash_prompts_host(R, a.ptr(prompt_bytes, np.uint8), a.ptr(prompt_off, np.int64),
                                                   a.ptr(prompt_len, np.int32), a.ptr(model_seed, np.uint64), block_chars, max_blocks,
                                                   out[0].ctypes.data, stride, out[1].ctypes.data, n_threads)
        if rc != 0:
            raise EppscoreError(rc, "eppscore_hash_prompts_host")
        return out[0][:R], out[1][:R]

    def count_fields(self, prompt_bytes, prompt_off, prompt_len=None):
        """len(strings.Fields(prompt)) per request, computed on the device (host arrays in and out)."""
        R = len(prompt_off) - 1
        a = _Args(False)
        out = np.zeros(max(R, 1), np.int32)
        self._check(self._lib.eppscore_count_fields(self._h, R, 0, a.ptr(prompt_bytes, np.uint8), a.ptr(prompt_off, np.int64),
                                                    a.ptr(prompt_len, np.int32), out.ctypes.data, None))
        return out[:R]

    # ------------------------------------------------------------------ in-flight load producer
    def estimate_tokens(self, R, request_size_bytes=None, token_hint=None, prompt_chars=None, device=False, stream=None, out=None):
        """SimpleTokenEstimator.Estimate per request (eppscore_estimate_tokens): int64[R].  Host mode: numpy in, numpy out.
        Device mode: CUDA tensors / raw pointers in, `out` an int64[R] CUDA tensor, asynchronous on `stream`."""
        a = _Args(device)
        if device:
            if out is None:
                raise ValueError("device mode needs a preallocated out")
            o_ptr = a.ptr(out, None)
        else:
            out = np.zeros(max(R, 1), np.int64)
            o_ptr = out.ctypes.data
        self._check(self._lib.eppscore_estimate_tokens(self._h, R, 1 if device else 0, a.ptr(request_size_bytes, np.int64),
                                                       a.ptr(token_hint, np.int32), a.ptr(prompt_chars, np.int32), o_ptr, stream))
        return out if device else out[:R]

    def _inflight(self, fn, endpoint, tokens, device, stream):
        a = _Args(device)
        R = int(endpoint.shape[0]) if hasattr(endpoint, "shape") else len(endpoint)
        self._check(fn(self._h, R, 1 if device else 0, a.ptr(endpoint, np.int32), a.ptr(tokens, np.int64), stream))

    def inflight_add(self, endpoint, tokens=None, device=False, stream=None):
        """PreRequest for a batch: requests[endpoint[r]] += 1, tokens[endpoint[r]] += tokens[r] (endpoint -1: skipped)."""
        self._inflight(self._lib.eppscore_inflight_add, endpoint, tokens, device, stream)

    def inflight_release(self, endpoint, tokens=None, device=False, stream=None):
        """ResponseBody at end of stream: the reverse of inflight_add with the same estimates."""
        self._inflight(self._lib.eppscore_inflight_release, endpoint, tokens, device, stream)

    def inflight_remove_endpoint(self, endpoint):
        self._check(self._lib.eppscore_inflight_remove_endpoint(self._h, endpoint))

    def inflight_get(self, M=None):
        """(requests int64[M], tokens int64[M]): the counters after every earlier update; M defaults to max_endpoints."""
        M = self.cfg.max_endpoints if M is None else M
        req, tok = np.zeros(max(M, 1), np.int64), np.zeros(max(M, 1), np.int64)
        self._check(self._lib.eppscore_inflight_get(self._h, req.ctypes.data, tok.ctypes.data, M))
        return req[:M], tok[:M]

    # ------------------------------------------------------------------ running-request queues (predicted-latency producer)
    def _running(self, fn, endpoint, request_key, tpot_slo, device, stream, out, want_out, extra):
        a = _Args(device)
        R = int(endpoint.shape[0]) if hasattr(endpoint, "shape") else len(endpoint)
        if device:
            o_ptr = a.ptr(out, None)
        else:
            out = np.zeros(max(R, 1), np.uint8) if want_out else None
            o_ptr = out.ctypes.data if want_out else None
        args = [a.ptr(endpoint, np.int32), a.ptr(request_key, np.uint64)]
        if extra:
            args.append(a.ptr(tpot_slo, np.float64))
        self._check(fn(self._h, R, 1 if device else 0, *args, o_ptr, stream))
        if device:
            return out
        return out[:R].astype(bool) if want_out else None

    def running_add(self, endpoint, request_key, tpot_slo=None, device=False, stream=None, out=None, want_added=True):
        """PreRequest for a batch (eppscore_running_add): adds (endpoint[r], request_key[r], tpot_slo[r]); endpoint -1 is
        skipped.  Host mode returns added bool[R]; device mode writes `out` (a uint8[R] CUDA tensor) when given."""
        return self._running(self._lib.eppscore_running_add, endpoint, request_key, tpot_slo, device, stream, out, want_added, True)

    def running_remove(self, endpoint, request_key, device=False, stream=None, out=None, want_removed=True):
        """End of stream / TTL expiry for a batch (eppscore_running_remove); host mode returns removed bool[R]."""
        return self._running(self._lib.eppscore_running_remove, endpoint, request_key, None, device, stream, out, want_removed, False)

    def running_remove_endpoint(self, endpoint):
        self._check(self._lib.eppscore_running_remove_endpoint(self._h, endpoint))

    def running_get(self, M=None):
        """(min_tpot float64[M], count int32[M]): the queues' view after every earlier update; M defaults to max_endpoints."""
        M = self.cfg.max_endpoints if M is None else M
        mn, cnt = np.zeros(max(M, 1), np.float64), np.zeros(max(M, 1), np.int32)
        self._check(self._lib.eppscore_running_get(self._h, mn.ctypes.data, cnt.ctypes.data, M))
        return mn[:M], cnt[:M]

    def running_reserve(self, live_entries=0):
        """Room for live_entries entries (and calls of up to that many) before a graph capture; returns the capacity in
        entries (live_entries 0: only the query)."""
        return self._check(self._lib.eppscore_running_reserve(self._h, int(live_entries)))

    # ------------------------------------------------------------------ per-stream batch scratch
    def reserve_stream(self, stream, max_R, max_blocks=0):
        """eppscore_reserve_stream: `stream` (a torch.cuda.Stream or a raw cudaStream_t) gets its own batch scratch for
        device-location batches of up to max_R requests and max_blocks blocks per prompt (0: config.max_blocks), so its
        batches run concurrently with other streams' and graphs captured on it survive larger calls elsewhere."""
        self._check(self._lib.eppscore_reserve_stream(self._h, _stream_handle(stream), int(max_R), int(max_blocks)))

    def release_stream(self, stream):
        """eppscore_release_stream: waits for the stream's work, then frees its scratch."""
        self._check(self._lib.eppscore_release_stream(self._h, _stream_handle(stream)))

    @staticmethod
    def model_seed(model, salt=b"") -> int:
        if isinstance(model, str):
            model = model.encode()
        if isinstance(salt, str):
            salt = salt.encode()
        return capi.lib().eppscore_model_seed(model, len(model), salt, len(salt))

    # ------------------------------------------------------------------ prefix index
    def commit_picks(self, pick, hashes, n_hashes, lru_capacity=None):
        a = _Args(False)
        hashes = np.ascontiguousarray(hashes, np.uint64)
        stride = hashes.shape[1] if hashes.ndim == 2 else 0
        self._check(self._lib.eppscore_commit_picks(self._h, len(pick), a.ptr(pick, np.int32), a.ptr(hashes, np.uint64),
                                                    a.ptr(n_hashes, np.uint16), stride, a.ptr(lru_capacity, np.int32)))

    def commit_picks_device(self, pick, hashes, n_hashes, lru_capacity=None, touch_bound=0, stream=None):
        """PreRequest with DEVICE arrays (CUDA tensors / raw pointers), asynchronous and ordered on `stream`:
        pick int32[R], hashes uint64[R, stride], n_hashes uint16[R]; lru_capacity is a HOST array."""
        a = _Args(True)
        ah = _Args(False)
        R = int(pick.shape[0])
        stride = int(hashes.shape[1])
        self._check(self._lib.eppscore_commit_picks_device(self._h, R, a.ptr(pick, None), a.ptr(hashes, None), a.ptr(n_hashes, None),
                                                           stride, ah.ptr(lru_capacity, np.int32), int(touch_bound), stream))

    def commit_picks_profiles(self, picks, hashes, n_hashes, lru_capacity=None, device=False, touch_bound=0, stream=None):
        """PreRequest with several picks per request (eppscore_commit_picks_profiles): picks is a list of [R] arrays (the primary
        profile's first, then e.g. the "prefill" profile's); Adds run per request in list order.  device=True: CUDA tensors /
        raw pointers, asynchronous on `stream`; lru_capacity is always a HOST array."""
        a = _Args(device)
        ah = _Args(False)
        if device:
            R = int(picks[0].shape[0])
            stride = int(hashes.shape[1])
            hp, nhp = a.ptr(hashes, None), a.ptr(n_hashes, None)
            pp = [a.ptr(p, None) for p in picks]
        else:
            hashes = np.ascontiguousarray(hashes, np.uint64)
            R = len(picks[0])
            stride = hashes.shape[1] if hashes.ndim == 2 else 0
            hp, nhp = a.ptr(hashes, np.uint64), a.ptr(n_hashes, np.uint16)
            pp = [a.ptr(p, np.int32) for p in picks]
        arr = (C.c_void_p * len(pp))(*pp)
        self._check(self._lib.eppscore_commit_picks_profiles(self._h, R, len(pp), arr, hp, nhp, stride, ah.ptr(lru_capacity, np.int32),
                                                             1 if device else 0, int(touch_bound), stream))

    def prefix_reserve(self, live_hashes=0, touches_per_call=0, overflow_rows=0):
        """Sizes the prefix index up front (eppscore_prefix_reserve): from then on commits decide their room on the device,
        never wait on the host and may be captured into CUDA graphs.  0 picks the documented default of each size."""
        self._check(self._lib.eppscore_prefix_reserve(self._h, int(live_hashes), int(touches_per_call), int(overflow_rows)))

    def prefix_add(self, hashes, endpoint, lru_capacity=0):
        a = _Args(False)
        h = np.ascontiguousarray(hashes, np.uint64)
        self._check(self._lib.eppscore_prefix_add(self._h, a.ptr(h, np.uint64), len(h), endpoint, lru_capacity))

    def prefix_apply(self, hash_, endpoint, op):
        a = _Args(False)
        self._check(self._lib.eppscore_prefix_apply(self._h, len(hash_), a.ptr(hash_, np.uint64),
                                                    a.ptr(endpoint, np.int32), a.ptr(op, np.uint8)))

    def prefix_remove_endpoint(self, endpoint):
        self._check(self._lib.eppscore_prefix_remove_endpoint(self._h, endpoint))

    def prefix_get(self, hash_: int) -> set:
        words = (self.cfg.max_endpoints + 31) // 32 + 1
        words = max(words, 8)
        # geometry may pad beyond max_endpoints; ask for a generous number of words
        buf = np.zeros(512, np.uint32)
        n = self._check(self._lib.eppscore_prefix_get(self._h, int(hash_), buf.ctypes.data, len(buf)))
        s = {w * 32 + b for w in range(len(buf)) if buf[w] for b in range(32) if (int(buf[w]) >> b) & 1}
        assert len(s) == n, (s, n)
        return s

    def prefix_match(self, hashes, n_hashes, endpoints, device=False, stream=None, out=None):
        """PrefixCacheMatchInfo.matchBlocks at chosen endpoints (eppscore_prefix_match): endpoints is [R, k] (int32, -1 and
        entries >= max_endpoints give 0), hashes [R, stride] and n_hashes [R] as for the commit calls.  Host mode returns a
        uint16 array [R, k].  device=True: CUDA tensors / raw pointers, asynchronous on `stream`; `out` is a preallocated
        uint16 (torch.int16 / torch.uint16) tensor [R, k] that the call fills, and is returned."""
        a = _Args(device)
        if device:
            R, k = int(endpoints.shape[0]), int(endpoints.shape[1])
            stride = int(hashes.shape[1])
            if out is None:
                raise ValueError("device mode fills a preallocated `out` tensor")
            self._check(self._lib.eppscore_prefix_match(self._h, R, k, 1, a.ptr(hashes, None), a.ptr(n_hashes, None), stride,
                                                        a.ptr(endpoints, None), a.ptr(out, None), _stream_handle(stream)))
            return out
        endpoints = np.ascontiguousarray(endpoints, np.int32)
        hashes = np.ascontiguousarray(hashes, np.uint64)
        R, k = endpoints.shape
        stride = hashes.shape[1] if hashes.ndim == 2 else 0
        res = np.zeros((R, k), np.uint16)
        self._check(self._lib.eppscore_prefix_match(self._h, R, k, 0, a.ptr(hashes, np.uint64), a.ptr(n_hashes, np.uint16), stride,
                                                    a.ptr(endpoints, np.int32), res.ctypes.data, None))
        return res

    def predict_latency(self, hashes, n_hashes, endpoints, input_tokens=None, ttft_slo=None, tpot_slo=None, device=False,
                        stream=None, out=None, match_out=None):
        """The predicted-latency producer's LatencyPredictionInfo and prefix cache score at chosen endpoints
        (eppscore_predict_latency), from the current snapshot: endpoints is [R, k] (int32; -1 and entries outside [0, M) give
        present = 0), hashes [R, stride] and n_hashes [R] as for prefix_match, input_tokens / ttft_slo / tpot_slo [R] or None (0).
        Host mode returns a LATENCY_INFO_DTYPE array [R, k]; with match_out=True it returns (info, match), match the uint16
        array prefix_match gives.  device=True: CUDA tensors / raw pointers, asynchronous on `stream`; `out` is a preallocated
        tensor of R*k*48 bytes (e.g. torch.uint8 [R, k, 48]) that the call fills and returns, `match_out` an optional uint16 [R, k]
        tensor filled as prefix_match fills it."""
        a = _Args(device)
        if device:
            R, k = int(endpoints.shape[0]), int(endpoints.shape[1])
            stride = int(hashes.shape[1])
            if out is None:
                raise ValueError("device mode fills a preallocated `out` tensor")
            self._check(self._lib.eppscore_predict_latency(
                self._h, R, k, 1, a.ptr(hashes, None), a.ptr(n_hashes, None), stride, a.ptr(input_tokens, None),
                a.ptr(ttft_slo, None), a.ptr(tpot_slo, None), a.ptr(endpoints, None), a.ptr(out, None), a.ptr(match_out, None),
                _stream_handle(stream)))
            return out
        endpoints = np.ascontiguousarray(endpoints, np.int32)
        hashes = np.ascontiguousarray(hashes, np.uint64)
        R, k = endpoints.shape
        stride = hashes.shape[1] if hashes.ndim == 2 else 0
        info = np.zeros((R, k), LATENCY_INFO_DTYPE)
        match = np.zeros((R, k), np.uint16) if match_out else None
        self._check(self._lib.eppscore_predict_latency(
            self._h, R, k, 0, a.ptr(hashes, np.uint64), a.ptr(n_hashes, np.uint16), stride, a.ptr(input_tokens, np.int32),
            a.ptr(ttft_slo, np.float64), a.ptr(tpot_slo, np.float64), a.ptr(endpoints, np.int32), info.ctypes.data,
            None if match is None else match.ctypes.data, None))
        return (info, match) if match_out else info

    def prefix_lru_len(self, endpoint) -> int:
        return self._lib.eppscore_prefix_lru_len(self._h, endpoint)

    def prefix_lru_keys(self, endpoint):
        n = self.prefix_lru_len(endpoint)
        if n < 0:
            return None
        out = np.zeros(max(n, 1), np.uint64)
        self._lib.eppscore_prefix_lru_keys(self._h, endpoint, out.ctypes.data, len(out))
        return [int(x) for x in out[:n]]
