"""Build bitblas_b200/lib/libbitblas_b200.so with plain nvcc for sm_90a (H100), in-tree."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT_DIR = os.path.join(PKG, "lib")
OBJ_DIR = os.path.join(HERE, "build")
SOURCES = ["bb_api.cu", "bb_generic.cu", "bb_gemv.cu", "bb_gemv_slab.cu", "bb_gemm_ts.cu", "bb_grouped.cu", "bb_grouped_gemm.cu",
           "bb_moe.cu", "bb_permute.cu", "bb_prep.cu", "bb_quant.cu", "bb_gemm_fp8.cu", "bb_grouped_fp8.cu"]
HEADERS = ["bb_common.cuh", "bb_gemv_mma.cuh", "bb_gemm_ts.cuh", "bb_wgmma.inc", os.path.join(PKG, "..", "include", "bitblas_b200.h")]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v" if os.environ.get("BB_PTXAS_V") else "-O3"]


def lib_path() -> str:
    return os.path.join(OUT_DIR, "libbitblas_b200.so")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdrs = [h if os.path.isabs(h) else os.path.join(HERE, h) for h in HEADERS]
    hdrs.append(os.path.abspath(__file__))
    jobs = []
    objs = []
    for s in SOURCES:
        src = os.path.join(HERE, s)
        obj = os.path.join(OBJ_DIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            jobs.append(["nvcc", *FLAGS, "-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode:
            raise RuntimeError("nvcc failed for " + cmd[-3])
        return r

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    out = lib_path()
    if jobs or force or _stale(out, objs):
        run(["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out, *objs])
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
