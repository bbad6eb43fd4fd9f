"""The host layer's several-profile route with maxNumOfEndpoints lists and the latency scorer, on the CPU:
tests/cpp/host_profiles_topk_test.cpp runs the Scheduler against the oracle-backed stand-in of the C ABI, built twice: with
tests/cpp/oracle_backed_profiles_topk.cpp (the library has eppscore_schedule_batch_profiles_topk) and with
tests/cpp/oracle_backed_profiles.cpp alone (it does not, as an older library).  With it: decode lists of 3 and prefill lists of 1
equal filtered single-profile Schedulers, a latency decode profile with TrackRunningRequests queues only the primary target, and
two differing predicted-latency producers are refused.  Without it: the list config is refused when the Scheduler is built."""
import os
import subprocess

from oracle import oracle_py as o
from tests import running_oracle as Q
from tests import topk_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")


def _build(name, abi_src):
    o.build()
    libs = [Q.build(), T.build()]
    exe = os.path.join(BUILD, name)
    srcs = [os.path.join(CPP, "host_profiles_topk_test.cpp"), os.path.join(CPP, abi_src), os.path.join(CPP, "oracle_backed_running.cpp")]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), os.path.join(CPP, "oracle_backed_abi.cpp"),
         os.path.join(CPP, "oracle_backed_profiles.cpp")] + libs
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-lrunning_oracle", "-ltopk_oracle",
                               "-L" + oracle_dir, "-loracle", "-Wl,-rpath," + BUILD + ":" + oracle_dir,
                               "-Wl,--wrap=eppscore_create", "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    return r.stdout.splitlines()


def test_host_layer_lists_and_latency_with_several_profiles():
    with_lists = _run(_build("host_profiles_topk_test", "oracle_backed_profiles_topk.cpp"))
    without = _run(_build("host_profiles_topk_test_old", "oracle_backed_profiles.cpp"))
    for line in ("lists checked", "latency checked", "producers checked"):
        assert line in with_lists, line
    assert not any(line.startswith("FAIL") for line in with_lists)
    lists = [line.split()[1:] for line in with_lists if line.startswith("list ")]
    assert len(lists) == 48
    assert all(len(set(x[:3])) == 3 for x in lists)  # three distinct decode endpoints per request
    assert any(line.startswith("refused ") and "eppscore_schedule_batch_profiles_topk" in line for line in without)
