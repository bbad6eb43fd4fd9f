"""Thresholds of the scoring kernels (csrc/pick_sparse.cu, csrc/score_matrix.cu, csrc/kernels.cuh, csrc/prefix_table.cuh),
parsed out of the CUDA sources so that the edge cases of tests/test_gpu_score_edges.py move with the constants instead of
quietly testing interiors.  Pure Python: tests/test_score_constants_cpu.py checks that the parse succeeds."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gateway-api-inference-extension_b200", "csrc")


@dataclass(frozen=True)
class ScoreConstants:
    exc_slots: int        # kExcSlots: entries of pick_sparse's per-request exception table
    exc_max: int          # kExcMax: more distinct matched endpoints than this defer the request to the full-matrix kernel
    probe_unroll: int     # U: hashes each lane probes per round of pick_sparse
    group_div: int        # G = min(row_words / group_div, group_cap) lanes per request
    group_cap: int
    inline_eps: int       # kInlineEps: members a table slot holds inline; larger sets are bitset rows
    lut_max: int          # kLutMax: the prefix / latency LUTs cover totals up to this
    epl_bounds: tuple     # make_geo: max_endpoints <= epl_bounds[i] -> log_epl = epl_logs[i], else epl_logs[-1]
    epl_logs: tuple
    narrow_counter_max: int  # score_matrix: hash_stride above this switches the match counters from 8 to 16 bits

    def geo(self, max_endpoints: int):
        """make_geo (csrc/kernels.cuh): (log_epl, J, Mpad, G lanes per sparse request)"""
        log_epl = self.epl_logs[-1]
        for b, lg in zip(self.epl_bounds, self.epl_logs):
            if max_endpoints <= b:
                log_epl = lg
                break
        per_pass = 32 << log_epl
        need = max(1, -(-max_endpoints // per_pass))
        J = 1
        while J < need:
            J <<= 1
        rw = J * 32
        return log_epl, J, J * per_pass, min(rw // self.group_div, self.group_cap)


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _int(text, pattern, what):
    m = re.search(pattern, text)
    if not m:
        raise ValueError(f"cannot parse {what}")
    return int(m.group(1))


def score_constants() -> ScoreConstants:
    sparse, matrix, kern, table = _read("pick_sparse.cu"), _read("score_matrix.cu"), _read("kernels.cuh"), _read("prefix_table.cuh")
    slots = _int(sparse, r"constexpr\s+int\s+kExcSlots\s*=\s*(\d+)\s*;", "kExcSlots")
    emax = _int(sparse, r"constexpr\s+int\s+kExcMax\s*=\s*(\d+)\s*;", "kExcMax")
    u = _int(sparse, r"constexpr\s+int\s+U\s*=\s*(\d+)\s*;", "U")
    g = re.search(r"constexpr\s+int\s+G\s*=\s*\(RW\s*/\s*(\d+)\s*<\s*(\d+)\)\s*\?\s*RW\s*/\s*\1\s*:\s*\2\s*;", sparse)
    if not g:
        raise ValueError("cannot parse the lane-group rule G")
    eps = _int(table, r"constexpr\s+int\s+kInlineEps\s*=\s*(\d+)\s*;", "kInlineEps")
    lut = _int(kern, r"constexpr\s+int\s+kLutMax\s*=\s*(\d+)\s*;", "kLutMax")
    e = re.search(r"g\.log_epl\s*=\s*M\s*<=\s*(\d+)\s*\?\s*(\d+)\s*:\s*\(M\s*<=\s*(\d+)\s*\?\s*(\d+)\s*:\s*(\d+)\)\s*;", kern)
    if not e:
        raise ValueError("cannot parse make_geo's log_epl rule")
    if not re.search(r"while\s*\(J\s*<\s*need\)\s*J\s*<<=\s*1\s*;", kern):
        raise ValueError("cannot parse make_geo's J rule")
    wide = _int(matrix, r"const\s+bool\s+wide_cnt\s*=\s*a\.hash_stride\s*>\s*(\d+)\s*;", "the counter-width split")
    return ScoreConstants(slots, emax, u, int(g.group(1)), int(g.group(2)), eps, lut, (int(e.group(1)), int(e.group(3))),
                          (int(e.group(2)), int(e.group(4)), int(e.group(5))), wide)
