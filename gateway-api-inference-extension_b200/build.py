"""Builds libeppscore.so (sm_90a only) in-tree with nvcc.  No JIT, no torch extension machinery:
the C-ABI library has no torch types in it, so it is plain `nvcc -c` per source (in parallel) and one
`nvcc -shared` link."""
from __future__ import annotations

import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libeppscore.so")
SOURCES = ["capi.cu", "hash_kernel.cu", "prepare_kernel.cu", "score_generic.cu", "score_dense.cu", "pick_sparse.cu",
           "prefix_index.cu", "fields_kernel.cu", "host_path.cu", "inflight_kernel.cu", "running_kernel.cu"]
# score_matrix.cu holds 64 instantiations of one kernel template: compiled as eight objects (one (MASKED, DIAG) combination each,
# with and without top-k lists, -DEPP_MATRIX_PART=k) so that they build in parallel
PART_SOURCES = [("score_matrix.cu", f"score_matrix_p{k}.o", [f"-DEPP_MATRIX_PART={k}"]) for k in range(8)]
# host-only C++ compiled by g++ directly (AVX-512 intrinsics: kept away from nvcc's front end); the ISA flags apply to this
# file alone and its one entry point is only called after a run-time CPU check (host_path.cu)
CPP_SOURCES = [("host_hash_simd.cpp", ["-mavx512f", "-mavx512dq"])]
HEADERS = ["kernels.cuh", "device_common.cuh", "xxh64.cuh", "prefix_index.hpp", "prefix_table.cuh", "cuda_owners.hpp",
           os.path.join("..", "..", "include", "eppscore.h")]

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-O3", "-std=c++17",
    *GENCODE,
    "-lineinfo",
    "-fmad=false",            # never contract a*b+c: float64 parity with the reference (GOAMD64=v1 never fuses)
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off",
]


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return "nvcc"


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    for src, objname, defs in PART_SOURCES + [(s_, s_.replace(".cu", ".o"), []) for s_ in SOURCES]:  # the slow parts first
        obj = os.path.join(OBJ, objname)
        if force or _stale(obj, [os.path.join(CSRC, src)] + hdrs):
            jobs.append((src, obj, defs))

    def compile_one(job):
        src, obj, defs = job
        extra = os.environ.get("EPPSCORE_NVCC_EXTRA", "").split()  # experiments only (e.g. -DEPP_SPARSE_MINBLOCKS=5)
        cmd = [nvcc()] + NVCC_FLAGS + defs + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for src, r in ex.map(compile_one, jobs):
                if r.returncode != 0:
                    sys.stderr.write(r.stdout + r.stderr)
                    raise RuntimeError(f"nvcc failed on {src}")
                if verbose:
                    sys.stderr.write(r.stdout + r.stderr)
    cpp_built = False
    for src, isa in CPP_SOURCES:
        obj = os.path.join(OBJ, src.replace(".cpp", ".o"))
        if force or _stale(obj, [os.path.join(CSRC, src), os.path.abspath(__file__)]):
            r = subprocess.run(["g++", "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off"] + isa + ["-c", os.path.join(CSRC, src), "-o", obj],
                               capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"g++ failed on {src}")
            cpp_built = True
    objs = ([os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES] + [os.path.join(OBJ, o_) for _, o_, _ in PART_SOURCES] +
            [os.path.join(OBJ, s.replace(".cpp", ".o")) for s, _ in CPP_SOURCES])
    if force or jobs or cpp_built or _stale(LIB, objs):
        cmd = [nvcc(), "-shared", "-cudart", "static", *GENCODE, "-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("nvcc link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))


HOST_TEST = os.path.join(HERE, "host", "host_test")


def build_host_test(force: bool = False) -> str:
    """C++ host mirror tests (host/host_test.cpp): plain g++, linked against libeppscore.so."""
    build()
    src = os.path.join(HERE, "host", "host_test.cpp")
    deps = [src, LIB] + [os.path.join(HERE, "host", h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp", "coalescer.hpp")]
    if force or _stale(HOST_TEST, deps):
        cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", src, "-o", HOST_TEST, "-pthread", "-L" + HERE, "-leppscore",
               "-Wl,-rpath,$ORIGIN/.."]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("g++ failed building host_test")
    return HOST_TEST


HOST_BENCH = os.path.join(HERE, "host", "host_bench")


def build_host_bench(force: bool = False) -> str:
    """Host-layer timings (host/host_bench.cpp: config A through the product, coalescing-front latency); run by bench.py."""
    build()
    src = os.path.join(HERE, "host", "host_bench.cpp")
    deps = [src, LIB] + [os.path.join(HERE, "host", h) for h in ("epp_scheduler.hpp", "epp_types.hpp", "host_eval.hpp", "coalescer.hpp")]
    if force or _stale(HOST_BENCH, deps):
        cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", src, "-o", HOST_BENCH, "-pthread", "-L" + HERE, "-leppscore",
               "-Wl,-rpath,$ORIGIN/.."]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("g++ failed building host_bench")
    return HOST_BENCH
