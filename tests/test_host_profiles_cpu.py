"""The host layer's several-profile route on the CPU: tests/cpp/host_profiles_test.cpp runs the Scheduler against the
oracle-backed stand-in of the C ABI, built twice: with tests/cpp/oracle_backed_profiles.cpp (the library has the profile calls)
and with tests/cpp/oracle_backed_abi.cpp alone (it does not, as an older library).  With them: a decode / prefill handler whose
picks equal filtered single-profile Schedulers, PreRequest's commits in reference order, the in-flight counts through
PreRequest / ResponseStarted / ResponseComplete, the multi-round refusal.  Without them: the multi-profile config is refused and
the single-profile output is unchanged."""
import os
import subprocess

from oracle import oracle_py as o
from tests import inflight_oracle as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gateway-api-inference-extension_b200", "host")
CPP = os.path.join(ROOT, "tests", "cpp")
BUILD = os.path.join(CPP, "_build")


def _build(name, abi_src):
    o.build()
    lib = I.build()
    exe = os.path.join(BUILD, name)
    srcs = [os.path.join(CPP, "host_profiles_test.cpp"), os.path.join(CPP, abi_src), os.path.join(CPP, "oracle_backed_inflight.cpp")]
    deps = srcs + [os.path.join(HOST, h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp")] + \
        [os.path.join(ROOT, "include", "eppscore.h"), os.path.join(CPP, "oracle_backed_abi.cpp"), lib]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        oracle_dir = os.path.join(ROOT, "oracle", "_build")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-pthread"] + srcs +
                              ["-I" + os.path.join(ROOT, "include"), "-L" + BUILD, "-linflight_oracle", "-L" + oracle_dir, "-loracle",
                               "-Wl,-rpath," + BUILD + ":" + oracle_dir, "-Wl,--wrap=eppscore_create",
                               "-Wl,--wrap=eppscore_set_snapshot", "-o", exe])
    return exe


def _run(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.rstrip().endswith("done"), r.stdout[-3000:] + r.stderr
    return r.stdout.splitlines()


def test_host_layer_several_profiles():
    with_profiles = _run(_build("host_profiles_test", "oracle_backed_profiles.cpp"))
    without = _run(_build("host_profiles_test_old", "oracle_backed_abi.cpp"))
    for line in ("picks checked", "commits checked", "inflight checked", "multi-round checked"):
        assert line in with_profiles, line
    assert not any(line.startswith("FAIL") for line in with_profiles)
    assert any(line.startswith("refused ") and "eppscore_add_profile" in line for line in without)
    single = [line for line in with_profiles if line.startswith("single ")]
    assert len(single) == 60 and single == [line for line in without if line.startswith("single ")]
