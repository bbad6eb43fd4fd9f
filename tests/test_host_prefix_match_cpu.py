"""The host layer's PrefixCacheMatchInfo (SchedulerConfig::PrefixMatchInfo) and PreRequest's prefix-indexer histograms, on the
CPU: tests/cpp/host_prefix_match_test.cpp runs the Scheduler against the oracle-backed stand-in of the C ABI, built twice: with
tests/cpp/oracle_backed_prefix_match.cpp (the library has eppscore_prefix_match) and with tests/cpp/oracle_backed_profiles_topk.cpp
alone (it does not, as an older library).  With it: every TargetEndpoints entry of single-profile, top-k (3 and 12) and
decode / prefill results equals the oracle's matchLongestPrefix, and the histograms equal a hand restatement of
RecordPrefixCacheMatch.  Without it: the option is refused when the Scheduler is built."""
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
    srcs = [os.path.join(CPP, "host_prefix_match_test.cpp"), os.path.join(CPP, abi_src)]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), os.path.join(CPP, "oracle_backed_abi.cpp"),
         os.path.join(CPP, "oracle_backed_profiles.cpp"), os.path.join(CPP, "oracle_backed_profiles_topk.cpp")] + libs
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


def test_host_prefix_match_info_and_metrics():
    out = _run(_build("host_prefix_match_test", "oracle_backed_prefix_match.cpp"))
    assert not any(line.startswith("FAIL") for line in out), out
    for line in ("edges checked", "autotune checked", "option off checked"):
        assert line in out, line
    entries = {line.split()[1]: int(line.split()[3]) for line in out if line.startswith("single k=")}
    assert set(entries) == {"k=1", "k=3", "k=12"} and entries["k=1"] == 96 and entries["k=3"] == 3 * 96 and entries["k=12"] == 12 * 96
    assert any(line.startswith("pd entries") for line in out)


def test_option_refused_without_the_symbol():
    out = _run(_build("host_prefix_match_test_old", "oracle_backed_profiles_topk.cpp"))
    assert any(line.startswith("refused ") and "eppscore_prefix_match" in line for line in out), out
