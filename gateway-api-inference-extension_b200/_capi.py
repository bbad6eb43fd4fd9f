"""ctypes declarations mirroring include/eppscore.h one-to-one."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
MAX_SCORERS = 8
MAX_ENDPOINT_COLS = 4
MAX_TOPK = 8
MAX_PROFILES = 4
MAX_STREAMS = 8

SCORER = {"queue": 0, "kv": 1, "prefix": 2, "lora": 3, "running": 4, "latency": 5, "token_load": 6,
          "col0": 8, "col1": 9, "col2": 10, "col3": 11, "pair0": 16, "pair1": 17}
TIE_LOWEST_INDEX, TIE_SEEDED_RANDOM = 0, 1
PICK_MAX_SCORE, PICK_WEIGHTED_RANDOM, PICK_RANDOM = 0, 1, 2
FILTER_PREFIX_AFFINITY, FILTER_SLO_HEADROOM_TIER = 1, 2

ERR_NAMES = {0: "OK", -1: "ERR_INVALID", -2: "ERR_CUDA", -3: "ERR_CAPACITY", -4: "ERR_NO_SNAPSHOT", -5: "ERR_NO_DEVICE"}


class EppscoreError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"eppscore {ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_scorers", C.c_int32), ("scorer_kind", C.c_int32 * MAX_SCORERS),
                ("scorer_weight", C.c_double * MAX_SCORERS), ("block_chars", C.c_int32), ("max_blocks", C.c_int32),
                ("tie_mode", C.c_int32), ("tie_seed", C.c_uint64), ("max_endpoints", C.c_int32),
                ("max_adapters", C.c_int32), ("prefix_capacity", C.c_int64), ("lru_capacity_default", C.c_int32),
                ("lru_capacity_max", C.c_int32), ("token_load_threshold", C.c_double), ("pick_mode", C.c_int32), ("n_filters", C.c_int32),
                ("filter_kind", C.c_int32 * 4), ("filter_param", (C.c_double * 3) * 4)]


class Profile(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_scorers", C.c_int32), ("scorer_kind", C.c_int32 * MAX_SCORERS),
                ("scorer_weight", C.c_double * MAX_SCORERS), ("pick_mode", C.c_int32), ("n_filters", C.c_int32),
                ("filter_kind", C.c_int32 * 4), ("filter_param", (C.c_double * 3) * 4)]


class ProfileRun(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("profile", C.c_int32), ("cand_mask", C.c_void_p), ("pick", C.c_void_p),
                ("pick_score", C.c_void_p), ("tie_count", C.c_void_p), ("scores_out", C.c_void_p), ("pred_out", C.c_void_p),
                ("filter_mask_out", C.c_void_p)]


class LatencyParams(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("has_predictions", C.c_int32),
                ("ttft_intercept", C.c_double), ("ttft_kv", C.c_double), ("ttft_input", C.c_double),
                ("ttft_waiting", C.c_double), ("ttft_running", C.c_double), ("ttft_prefix", C.c_double),
                ("tpot_intercept", C.c_double), ("tpot_kv", C.c_double), ("tpot_input", C.c_double),
                ("tpot_waiting", C.c_double), ("tpot_running", C.c_double), ("tpot_generated", C.c_double),
                ("slo_buffer_factor", C.c_double), ("streaming_mode", C.c_int32), ("strategy_most", C.c_int32),
                ("ttft_weight", C.c_double), ("tpot_weight", C.c_double), ("composite_kv", C.c_double),
                ("composite_queue", C.c_double), ("composite_prefix", C.c_double)]


class Snapshot(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("M", C.c_int32), ("lora_words", C.c_int32), ("location", C.c_int32),
                ("kv_usage", C.c_void_p), ("queue", C.c_void_p), ("running", C.c_void_p), ("lora_active", C.c_void_p),
                ("lora_waiting", C.c_void_p), ("lora_nmodels", C.c_void_p), ("lora_max", C.c_void_p),
                ("endpoint_col", C.c_void_p * MAX_ENDPOINT_COLS), ("epoch", C.c_uint64), ("stream", C.c_void_p),
                ("min_tpot_slo", C.c_void_p), ("dispatched", C.c_void_p), ("prefill_role", C.c_void_p),
                ("inflight_tokens", C.c_void_p)]


class Batch(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("R", C.c_int32), ("location", C.c_int32), ("reserved0", C.c_int32),
                ("request_base", C.c_int64), ("prompt_bytes", C.c_void_p), ("prompt_off", C.c_void_p),
                ("prompt_len", C.c_void_p), ("model_seed", C.c_void_p), ("hashes_in", C.c_void_p),
                ("n_hashes_in", C.c_void_p), ("hash_stride", C.c_int32), ("block_chars", C.c_int32),
                ("max_blocks", C.c_int32), ("reserved1", C.c_int32), ("adapter_id", C.c_void_p),
                ("cand_mask", C.c_void_p), ("dense_feat", C.c_void_p), ("dense_total", C.c_void_p),
                ("pick", C.c_void_p), ("pick_score", C.c_void_p), ("tie_count", C.c_void_p),
                ("match_blocks", C.c_void_p), ("total_blocks", C.c_void_p), ("hashes_out", C.c_void_p),
                ("scores_out", C.c_void_p), ("stream", C.c_void_p), ("input_tokens", C.c_void_p),
                ("ttft_slo", C.c_void_p), ("tpot_slo", C.c_void_p), ("pred_out", C.c_void_p),
                ("filter_mask_out", C.c_void_p)]


class TopK(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("k", C.c_int32), ("endpoints", C.c_void_p), ("scores", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("M", C.c_int32), ("epoch", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("prefix_hashes", C.c_int64), ("prefix_live_hashes", C.c_int64), ("prefix_capacity", C.c_int64),
                ("prefix_table_bytes", C.c_int64), ("lru_entries", C.c_int64), ("lru_bytes", C.c_int64),
                ("prefix_overflow_rows", C.c_int64), ("prefix_rebuilds", C.c_int64), ("index_error", C.c_uint32),
                ("probe_resolved", C.c_uint32)]


# every symbol include/eppscore.h declares: (name, restype, argtypes)
_P = C.c_void_p
ABI_SYMBOLS = [
    ("eppscore_abi_version", C.c_int32, []),
    ("eppscore_config_default", None, [C.POINTER(Config)]),
    ("eppscore_create", C.c_int32, [C.c_int32, C.POINTER(Config), C.POINTER(_P)]),
    ("eppscore_destroy", None, [_P]),
    ("eppscore_last_error", C.c_char_p, [_P]),
    ("eppscore_get_stats", C.c_int32, [_P, C.POINTER(Stats)]),
    ("eppscore_set_debug", C.c_int32, [_P, C.c_int32, C.c_int64]),
    ("eppscore_set_snapshot", C.c_int32, [_P, C.POINTER(Snapshot)]),
    ("eppscore_latency_params_default", None, [C.POINTER(LatencyParams)]),
    ("eppscore_set_latency_params", C.c_int32, [_P, C.POINTER(LatencyParams)]),
    ("eppscore_schedule_batch", C.c_int32, [_P, C.POINTER(Batch)]),
    ("eppscore_schedule_batch_topk", C.c_int32, [_P, C.POINTER(Batch), C.POINTER(TopK)]),
    ("eppscore_schedule_batch_topk_wide", C.c_int32, [_P, C.POINTER(Batch), C.POINTER(TopK)]),
    ("eppscore_add_profile", C.c_int32, [_P, C.POINTER(Profile), C.POINTER(C.c_int32)]),
    ("eppscore_set_profile_endpoints", C.c_int32, [_P, C.c_int32, _P, C.c_int32]),
    ("eppscore_schedule_batch_profiles", C.c_int32, [_P, C.POINTER(Batch), C.c_int32, C.POINTER(ProfileRun)]),
    ("eppscore_schedule_batch_profiles_topk", C.c_int32, [_P, C.POINTER(Batch), C.c_int32, C.POINTER(ProfileRun),
                                                          C.POINTER(TopK)]),
    ("eppscore_hash_prompts", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P]),
    ("eppscore_count_fields", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P]),
    ("eppscore_hash_prompts_host", C.c_int32, [C.c_int32, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32]),
    ("eppscore_model_seed", C.c_uint64, [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    ("eppscore_xxh64", C.c_uint64, [C.c_char_p, C.c_size_t, C.c_uint64]),
    ("eppscore_commit_picks", C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, _P]),
    ("eppscore_commit_picks_profiles", C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), _P, _P, C.c_int32, _P,
                                                   C.c_int32, C.c_int64, _P]),
    ("eppscore_prefix_reserve", C.c_int32, [_P, C.c_int64, C.c_int64, C.c_int64]),
    ("eppscore_prefix_add", C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32]),
    ("eppscore_prefix_apply", C.c_int32, [_P, C.c_int64, _P, _P, _P]),
    ("eppscore_prefix_remove_endpoint", C.c_int32, [_P, C.c_int32]),
    ("eppscore_prefix_get", C.c_int32, [_P, C.c_uint64, _P, C.c_int32]),
    ("eppscore_prefix_lru_len", C.c_int32, [_P, C.c_int32]),
    ("eppscore_prefix_lru_keys", C.c_int32, [_P, C.c_int32, _P, C.c_int32]),
    ("eppscore_commit_picks_device", C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32, _P, C.c_int64, _P]),
    ("eppscore_estimate_tokens", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P]),
    ("eppscore_inflight_add", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P]),
    ("eppscore_inflight_release", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P]),
    ("eppscore_inflight_remove_endpoint", C.c_int32, [_P, C.c_int32]),
    ("eppscore_inflight_get", C.c_int32, [_P, _P, _P, C.c_int32]),
    ("eppscore_running_add", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P]),
    ("eppscore_running_remove", C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P, _P, _P]),
    ("eppscore_running_remove_endpoint", C.c_int32, [_P, C.c_int32]),
    ("eppscore_running_get", C.c_int32, [_P, _P, _P, C.c_int32]),
    ("eppscore_running_reserve", C.c_int32, [_P, C.c_int64]),
    ("eppscore_reserve_stream", C.c_int32, [_P, _P, C.c_int32, C.c_int32]),
    ("eppscore_release_stream", C.c_int32, [_P, _P]),
    ("eppscore_host_alloc", _P, [C.c_size_t]),
    ("eppscore_host_free", None, [_P]),
]

_lib = None


def lib_path() -> str:
    return os.path.join(_HERE, "libeppscore.so")


def lib():
    """Loads libeppscore.so. Fails loudly when it has not been built: there is no fallback."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise ImportError(f"{path} is missing: build it with __graft_entry__.build() "
                              "(nvcc, sm_90a). The engine has no CPU/PyTorch fallback.")
        L = C.CDLL(path)
        for name, res, args in ABI_SYMBOLS:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib
