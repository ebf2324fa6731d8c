"""Generate tests/golden/ref_decode_golden.npz by RUNNING the reference's LOP3 device decode functions on a GPU.

The device functions are the BitBLAS LOP3 decode library (bitblas/gpu/intrin/lop3.py, MIT, Microsoft) in the copy that
TileLang ships as tilelang/quantize/lop3.py: the same `decode_*` functions with the same signatures as the C++ test header
that oracle/ref_shim.cu includes.  The CUDA sources are read out of that installed module (nothing is copied into this
repository), placed in a temporary `fast_decoding.hpp` next to stubs for the header's host helpers (not used here), and
compiled together with oracle/ref_shim.cu unchanged; its kernels then run on the exact seeded inputs of the reference
comparisons in tests/test_gpu_decode_kat.py.  The outputs are stored with `source = "lop3"`.  One documented difference
from the C++ header: lop3.py's signed fp16 decodes subtract 2^(b-1) (MEDIAN 0x6408 / 0x6402), the C++ header 2^(b-1) - 1.

    python tests/golden/make_ref_decode_golden.py        # needs an sm_90a GPU, nvcc and an installed tilelang
"""
import ast
import ctypes
import importlib.util
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bitblas_oracle as O  # noqa: E402
import test_gpu_decode_kat as KAT  # noqa: E402  (input recipes shared with the tests)

SNIPPETS = ["decode_i4_to_f16", "decode_i4_to_f16_scale", "decode_i4_to_f16_scale_zeros_original",
            "decode_i4_to_f16_scale_zeros_rescale", "decode_i4_to_f16_scale_zeros_quantized", "decode_i2_to_f16",
            "decode_i2_to_f16_scale", "decode_i2_to_f16_scale_zeros_original", "decode_i2_to_f16_scale_zeros_rescale",
            "decode_i1_to_f16", "decode_i1s_to_i8s", "decode_i2s_to_i8s", "decode_i4s_to_i8s"]
PRELUDE = r"""
#pragma once
#include <cuda_fp16.h>
#include <cstdint>
#include <stdexcept>
__device__ __forceinline__ unsigned __pack_half2(const half x, const half y) {
  unsigned v0 = *((const unsigned short*)&x), v1 = *((const unsigned short*)&y);
  return (v1 << 16) | v0;
}
// host helpers of the C++ header: not part of the device library, never called by this generator
inline void general_compress(const int8_t*, int8_t*, int, int, bool) { throw std::runtime_error("unavailable"); }
inline void general_interleave_fp16(int8_t*, int8_t*, int, size_t, bool) { throw std::runtime_error("unavailable"); }
inline void general_interleave_int8(int8_t*, int8_t*, int, size_t, bool) { throw std::runtime_error("unavailable"); }
"""


def lop3_sources():
    spec = importlib.util.find_spec("tilelang")
    path = os.path.join(spec.submodule_search_locations[0], "quantize", "lop3.py")
    tree = ast.parse(open(path).read())
    consts = {t.id: node.value.value for node in tree.body if isinstance(node, ast.Assign)
              for t in node.targets if isinstance(t, ast.Name) and isinstance(node.value, ast.Constant)}
    return "\n".join(consts[k] for k in SNIPPETS)


def build(tmp):
    with open(os.path.join(tmp, "fast_decoding.hpp"), "w") as f:
        f.write(PRELUDE + lop3_sources())
    so = os.path.join(tmp, "libref_lop3.so")
    subprocess.run(["nvcc", "-O2", "-shared", "-Xcompiler", "-fPIC", "-w", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-I", tmp, os.path.join(ROOT, "oracle", "ref_shim.cu"), "-o", so], check=True)
    return KAT.bind_ref(ctypes.CDLL(so), host=False)   # 1-bit packing: the oracle's (pinned to the C++ helpers)


def main():
    with tempfile.TemporaryDirectory() as tmp:
        ref = build(tmp)
        out = {"source": np.array("lop3")}
        for name, fn in KAT.REF_CASES.items():
            for key, arr in fn(ref).items():
                out[f"{name}/{key}"] = arr
    dst = os.path.join(HERE, "ref_decode_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes,", len(out) - 1, "arrays")


if __name__ == "__main__":
    torch.cuda.init()
    main()
