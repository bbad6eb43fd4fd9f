"""SchedulerConfig::InOrderInFlightLoad / InOrderPrefixIndex with the Profiles list on the oracle-backed stand-in of the C ABI
(tests/cpp/host_inorder_profiles_test.cpp): picks, counters and the prefix index against the batch route fed one request at a
time, one in-order call per batch, no second count or commit in PreRequest, PrefixCacheMatchInfo from before each request's
Adds, the per-request error for another primary profile and the refusals; and, against a stand-in without
eppscore_schedule_batch_inorder_profiles, the refusal of a library that lacks the call."""
import os
import subprocess

import pytest

from oracle import oracle_py as o
from tests import inflight_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")


def build(with_call: bool) -> str:
    o.build()
    lib = I.build()
    exe = os.path.join(BUILD, "host_inorder_profiles_test" if with_call else "host_inorder_profiles_test_nocall")
    srcs = [os.path.join(CPP, "host_inorder_profiles_test.cpp"),
            os.path.join(CPP, "oracle_backed_inorder_profiles.cpp" if with_call else "oracle_backed_profiles.cpp"),
            os.path.join(CPP, "oracle_backed_inflight.cpp")]
    deps = srcs + [os.path.join(CPP, "oracle_backed_abi.cpp"), os.path.join(CPP, "oracle_backed_profiles.cpp")] + \
        [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-linflight_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


@pytest.mark.parametrize("with_call", [True, False])
def test_host_inorder_profiles_on_the_oracle_backed_abi(with_call):
    r = subprocess.run([build(with_call)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    out = r.stdout.splitlines()
    assert not any(line.startswith("FAIL") for line in out), out[:20]
    if with_call:
        for line in ("in-flight form checked", "index form checked", "primary checked", "refusals checked"):
            assert line in out, line
    else:
        assert any(line.startswith("refused ") and "eppscore_schedule_batch_inorder_profiles" in line for line in out), out
