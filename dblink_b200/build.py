"""Builds libdblink_b200.so in-tree with nvcc for sm_90a (explicit nvcc; no JIT cache).

Translation units: dbl_engine.cu (all kernels but the PCG-II link kernel), dbl_host.cpp (host-side model
construction), dbl_index_gpu.cu (attribute-index tables), dbl_posterior.cu (shared most probable clusters of a chain)
and dbl_link_inst.cu compiled once per attribute count A = 1..16 (k_link_pcg2<A, 0..A>);
objects are compiled in parallel and linked with `nvcc -shared`.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.environ.get("DBL_OBJ") or os.path.join(HERE, "build")
SO = os.environ.get("DBL_SO") or os.path.join(HERE, "libdblink_b200.so")  # DBL_SO / DBL_NVCC_FLAGS: experiment builds
MAX_A = 16

COMMON = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # the draw protocol is defined over individually rounded binary64 operations: no FMA contraction
    "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math,-O2,-pthread",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
] + os.environ.get("DBL_NVCC_FLAGS", "").split()


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.exists(p):
            return p
    return "nvcc"


def _deps():
    d = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    d.append(os.path.join(ROOT, "include", "dblink_b200.h"))
    d.append(os.path.abspath(__file__))
    return d


def units():
    u = [("dbl_engine.o", "dbl_engine.cu", []), ("dbl_host.o", "dbl_host.cpp", []),
         ("dbl_index_gpu.o", "dbl_index_gpu.cu", []), ("dbl_posterior.o", "dbl_posterior.cu", [])]
    for a in range(1, MAX_A + 1):
        u.append((f"dbl_link_a{a}.o", "dbl_link_inst.cu", [f"-DDBL_INST_A={a}"]))
    return u


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    return any(os.path.getmtime(d) > t for d in _deps() if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    os.makedirs(OBJ, exist_ok=True)
    nvcc = nvcc_path()
    newest = max(os.path.getmtime(d) for d in _deps() if os.path.exists(d))

    def compile_one(unit):
        obj, src, extra = unit
        out = os.path.join(OBJ, obj)
        if not force and os.path.exists(out) and os.path.getmtime(out) > newest:
            return out, ""
        cmd = [nvcc, "-c", "-o", out] + COMMON + extra + (["-Xptxas", "-v"] if verbose else []) + [os.path.join(CSRC, src)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src} {extra}:\n{res.stdout}{res.stderr}")
        return out, res.stderr

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, units()))
    if verbose:
        for _, err in results:
            sys.stderr.write(err)
    cmd = [nvcc, "-shared", "-o", SO, "-cudart", "static"] + [r[0] for r in results]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
