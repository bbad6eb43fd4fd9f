"""The host layer's maxNumOfEndpoints > 8 route on the CPU: tests/cpp/host_topk_wide_test.cpp runs the Scheduler against the
oracle-backed stand-in of the C ABI, built twice: with tests/cpp/oracle_backed_topk_wide.cpp (the library has
eppscore_schedule_batch_topk_wide) and with tests/cpp/oracle_backed_topk.cpp alone (it does not, as an older library).

  - weighted-random and random with k = 12 and 40: refused without the wide call, lists of min(k, n) distinct candidates with
    it (random: inclusion min(k/n, 1) +- 0.05);
  - max-score with lowest-index ties: the wide lists equal the score map's (pick first, then descending score, ties in
    ascending index);
  - max-score with seeded-random ties keeps the score-map route."""
import os
import subprocess

import numpy as np

from oracle import oracle_py as o
from tests import topk_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")
N_ENDPOINTS = 50


def _build(name, topk_src):
    o.build()
    topk_lib = T.build()
    exe = os.path.join(BUILD, name)
    main = os.path.join(CPP, "host_topk_wide_test.cpp")
    srcs = [main, os.path.join(CPP, "oracle_backed_abi.cpp"), os.path.join(CPP, topk_src)]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), os.path.join(CPP, "oracle_backed_topk.cpp"), topk_lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-ltopk_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-2000:] + r.stderr
    cases, cur = {}, None
    for line in r.stdout.splitlines()[:-1]:
        if line.startswith("case "):
            _, name, route = line.split()
            cur = cases[name] = {"route": route.split("=")[1], "lists": []}
        else:
            cur["lists"].append([(int(i), float(s)) for i, s in (p.split(":") for p in line.split())])
    return cases


def test_host_layer_lists_past_eight():
    wide = _run(_build("host_topk_wide_test", "oracle_backed_topk_wide.cpp"))
    old = _run(_build("host_topk_wide_test_no_wide", "oracle_backed_topk.cpp"))
    for k in (12, 40):
        for picker in ("weighted_random", "random"):
            name = f"{picker}_k{k}"
            assert old[name]["route"] == "refused", name  # a library without the wide call: refused when built, as before
            assert wide[name]["route"] == "wide", name
            lists = wide[name]["lists"]
            assert len(lists) == 2000
            for lst in lists:
                ids = [i for i, _ in lst]
                assert len(ids) == min(k, N_ENDPOINTS) and len(set(ids)) == len(ids), name
            if picker == "random":
                freq = np.bincount([i for lst in lists for i, _ in lst], minlength=N_ENDPOINTS) / len(lists)
                assert np.abs(freq - min(k / N_ENDPOINTS, 1.0)).max() <= 0.05, (name, freq)
    for name in ("max_score_lowest_index_k12", "max_score_lowest_index_k100"):
        assert wide[name]["route"] == "wide" and old[name]["route"] == "map", name
        assert wide[name]["lists"] == old[name]["lists"], name
        lst = wide[name]["lists"][0]
        assert len(lst) == (12 if name.endswith("k12") else N_ENDPOINTS)
        assert all((a[1], -a[0]) > (b[1], -b[0]) for a, b in zip(lst, lst[1:])), name  # descending score, ties ascending index
    name = "max_score_seeded_random_k12"
    assert wide[name]["route"] == "map" and old[name]["route"] == "map"
    assert wide[name]["lists"] == old[name]["lists"]
