"""The host layer's LatencyPredictionInfo (SchedulerConfig::LatencyPredictionInfo) and PreRequest's dispatch record, on the CPU:
tests/cpp/host_latency_info_test.cpp runs the Scheduler against the oracle-backed stand-in of the C ABI, built twice: with
tests/cpp/oracle_backed_latency_info.cpp (the library has eppscore_predict_latency, implemented on orc_latency_predict /
orc_latency_validate) and with tests/cpp/oracle_backed_prefix_match.cpp alone (it does not, as an older library).  With it:
every SchedulingResult::TargetLatency entry of single-profile, top-k (3 and 12) and decode / prefill results equals the oracle's predict +
validate, also through a BatchingScheduler, the dispatch record takes TTFT at the prefill target, TPOT at the primary and 0 without a prediction, HavePredictions
= false leaves everything empty, two endpoints sharing a Name read the later one's values, and the option off makes no call.
Without it: the option is refused when the Scheduler is built."""
import os
import subprocess

from oracle import oracle_py as o
from tests import topk_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")


def _build(name, abi_src):
    o.build()
    libs = [T.build()]
    exe = os.path.join(BUILD, name)
    srcs = [os.path.join(CPP, "host_latency_info_test.cpp"), os.path.join(CPP, abi_src)]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp", "coalescer.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h")] + \
        [os.path.join(CPP, f) for f in ("oracle_backed_abi.cpp", "oracle_backed_profiles.cpp", "oracle_backed_profiles_topk.cpp",
                                        "oracle_backed_prefix_match.cpp", "oracle_backed_latency_info.cpp")] + libs
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        os.makedirs(BUILD, exist_ok=True)
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-ltopk_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-o", exe])
    return exe


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    return r.stdout.splitlines()


def test_host_latency_info_and_dispatch_record():
    out = _run(_build("host_latency_info_test", "oracle_backed_latency_info.cpp"))
    assert not any(line.startswith("FAIL") for line in out), out
    entries = {line.split()[1]: int(line.split()[3]) for line in out if line.startswith("single k=")}
    assert entries == {"k=1": 72, "k=3": 3 * 72, "k=12": 12 * 72}, entries
    assert any(line.startswith("nopred k=3") for line in out)
    assert any(line.startswith("pd entries") for line in out)
    names = [line.split() for line in out if line.startswith("names entries")]
    assert names and int(names[0][4]) > 0, names  # some requests went to the endpoint whose Name is shared
    assert "option off checked" in out
    assert any(line.startswith("coalescer entries") and int(line.split()[2]) > 0 for line in out)


def test_option_refused_without_the_symbol():
    out = _run(_build("host_latency_info_test_old", "oracle_backed_prefix_match.cpp"))
    assert any(line.startswith("refused ") and "eppscore_predict_latency" in line for line in out), out
