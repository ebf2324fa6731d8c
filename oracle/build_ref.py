"""Build oracle/_ref/libbitblas_ref.so from the reference's OWN sources where they lie.

TEST INFRASTRUCTURE ONLY.  Compiles oracle/ref_shim.cu, which #includes
testing/cpp/lop3_type_conversion/fast_decoding.hpp of a microsoft/BitBLAS checkout (never copied into the repo; its
location is taken from $BITBLAS_REFERENCE_DIR), with plain nvcc (the reference's CMake/gtest build is not used).  Output
goes only to oracle/_ref/, which is git-ignored.  Without a reference checkout this is a no-op (an existing oracle/_ref is
used as is) and the tests that call into it skip.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.environ.get("BITBLAS_REFERENCE_DIR", "")
REF_INC = os.path.join(REF_DIR, "testing", "cpp", "lop3_type_conversion") if REF_DIR else ""
OUT_DIR = os.path.join(HERE, "_ref")
OUT = os.path.join(OUT_DIR, "libbitblas_ref.so")


def build(force: bool = False) -> str | None:
    if not REF_INC or not os.path.isdir(REF_INC):
        return OUT if os.path.exists(OUT) else None
    os.makedirs(OUT_DIR, exist_ok=True)
    src = os.path.join(HERE, "ref_shim.cu")
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= os.path.getmtime(src):
        return OUT
    cmd = ["nvcc", "-O2", "-shared", "-Xcompiler", "-fPIC", "-w",
           "-gencode", "arch=compute_90a,code=sm_90a", "-I", REF_INC, src, "-o", OUT]
    subprocess.run(cmd, check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
