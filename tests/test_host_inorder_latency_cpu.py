"""SchedulerConfig::InOrderRunningRequests of the C++ host layer on the oracle-backed stand-in of the C ABI
(tests/cpp/host_inorder_latency_test.cpp): picks, in-flight counters, running-request queues and (with InOrderPrefixIndex) the
prefix index against a Scheduler fed one request at a time, one queue Add per request, ResponseComplete removing what the call
added, and every refusal; and, against a stand-in without eppscore_schedule_batch_inorder_latency, the refusal of a library
that lacks the call."""
import os
import subprocess

import pytest

from oracle import oracle_py as o
from tests import inflight_oracle as I
from tests import running_oracle as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")


def build(with_call: bool) -> str:
    """The program, linked against the stand-in.  oracle_backed_inflight.cpp and oracle_backed_running.cpp both hook
    eppscore_create and eppscore_set_snapshot: the running hook is compiled to call the in-flight one, which calls the stand-in."""
    o.build()
    lib = I.build()
    rlib = Q.build()
    exe = os.path.join(BUILD, "host_inorder_latency_test_cpu" if with_call else "host_inorder_latency_test_cpu_nocall")
    main = [os.path.join(CPP, "host_inorder_latency_test.cpp"),
            os.path.join(CPP, "oracle_backed_inorder_latency.cpp" if with_call else "oracle_backed_inorder.cpp")]
    deps = main + [os.path.join(CPP, f) for f in ("oracle_backed_abi.cpp", "oracle_backed_inorder.cpp", "oracle_backed_inflight.cpp",
                                                  "oracle_backed_running.cpp")] + \
        [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), lib, rlib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        os.makedirs(BUILD, exist_ok=True)
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        flags = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-pthread", "-I" + os.path.join(ROOT, "include")]
        tag = "" if with_call else "_nocall"
        inflight_o = os.path.join(BUILD, f"inorder_latency_inflight{tag}.o")
        running_o = os.path.join(BUILD, f"inorder_latency_running{tag}.o")
        subprocess.check_call(flags + ["-D__wrap_eppscore_create=inflight_hook_create",
                                       "-D__wrap_eppscore_set_snapshot=inflight_hook_set_snapshot", "-c",
                                       os.path.join(CPP, "oracle_backed_inflight.cpp"), "-o", inflight_o])
        subprocess.check_call(flags + ["-D__real_eppscore_create=inflight_hook_create",
                                       "-D__real_eppscore_set_snapshot=inflight_hook_set_snapshot", "-c",
                                       os.path.join(CPP, "oracle_backed_running.cpp"), "-o", running_o])
        subprocess.check_call(flags + (["-Wl,--wrap=eppscore_running_add"] if with_call else ["-DEPP_NO_INORDER_LATENCY_SYMBOL"]) +
                              main + [inflight_o, running_o] +
                              ["-L" + BUILD, "-linflight_oracle", "-lrunning_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


@pytest.mark.parametrize("with_call", [True, False])
def test_host_inorder_latency_on_the_oracle_backed_abi(with_call):
    r = subprocess.run([build(with_call)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "host inorder latency: all checks passed" in r.stdout
