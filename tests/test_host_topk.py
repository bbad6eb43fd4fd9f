"""The host layer's maxNumOfEndpoints route (Scheduler with k in 2..8 through eppscore_schedule_batch_topk, every picker).

On the CPU: the host test programs (host/host_test.cpp, tests/cpp/host_ids_test.cpp) linked against the oracle-backed
stand-in of the C ABI plus tests/cpp/oracle_backed_topk.cpp, which supplies eppscore_schedule_batch_topk from the CPU
oracle.  Without that file the host layer sees no top-k entry point (it is bound weakly) and takes the score-map route,
which tests/test_host_mirror_cpu.py covers.  On the GPU: the same program against libeppscore.so takes the top-k route."""
import os
import subprocess

import pytest

import _pkg
from oracle import oracle_py as o
from tests import topk_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")
DEPS = [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp", "coalescer.hpp")] + \
    [os.path.join(ROOT, "include", "eppscore.h"), os.path.join(ROOT, "oracle", "oracle.h"),
     os.path.join(CPP, "oracle_backed_abi.cpp"), os.path.join(CPP, "oracle_backed_topk.cpp")]


def _build(name, main_src):
    o.build()
    topk_lib = T.build()
    exe = os.path.join(BUILD, name)
    srcs = [main_src, os.path.join(CPP, "oracle_backed_abi.cpp"), os.path.join(CPP, "oracle_backed_topk.cpp")]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in DEPS + srcs + [topk_lib]):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-ltopk_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def test_host_topk_route_on_the_oracle_backed_abi():
    exe = _build("host_test_cpu_topk", os.path.join(HOST, "host_test.cpp"))
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("top-k stochastic pickers: checked") == 2 and "skipped" not in r.stdout
    assert "all checks passed" in r.stdout


def test_host_ids_on_the_topk_route():
    exe = _build("host_ids_test_topk", os.path.join(CPP, "host_ids_test.cpp"))
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host ids: all checks passed" in r.stdout


@pytest.mark.gpu
def test_host_topk_route_on_gpu():
    exe = _pkg.load_build().build_host_test()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("top-k stochastic pickers: checked") == 2 and "all checks passed" in r.stdout
