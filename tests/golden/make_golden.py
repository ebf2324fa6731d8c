"""Generate golden vectors by RUNNING the reference's own numpy functions.

Loads bitblas/quantization/utils.py of the microsoft/BitBLAS checkout at $BITBLAS_REFERENCE_DIR standalone via importlib (it only needs numpy+torch),
runs general_compress / interleave_weight on seeded inputs and stores inputs+outputs in
tests/golden/quant_golden.npz.  Cases the reference itself cannot run are recorded as such:
  * interleave 2-bit/float16 raises OverflowError under NumPy 2 (np.int32(0xFF0000FF), utils.py:97)
  * interleave 1-bit/float16 returns the un-shuffled word (missing `return n8_weight`, utils.py:101-110)
those two layouts are pinned against the reference's C++ host function instead (oracle/_ref, see
tests/test_oracle_golden.py) and against vectors produced from it here (ref_cpp_* keys).
"""
import ctypes
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
spec = importlib.util.spec_from_file_location(
    "ref_quant_utils", os.path.join(os.environ["BITBLAS_REFERENCE_DIR"], "bitblas", "quantization", "utils.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

rng = np.random.RandomState(0)
out = {}
for bits in (4, 2, 1):
    w = rng.randint(0, 2**bits, size=(16, 128)).astype(np.int8)
    out[f"w_b{bits}"] = w
    packed = ref.general_compress(w, source_bits=bits, storage_dtype=np.int8)
    out[f"compress_b{bits}"] = packed
    for tgt in ("float16", "int8"):
        key = f"interleave_b{bits}_{tgt}"
        try:
            out[key] = ref.interleave_weight(packed.copy(), nbits=bits, target_dtype=tgt)
        except OverflowError as e:  # NumPy 2 + np.int32(0xFF0000FF)
            print(f"reference cannot run {key}: {e!r}")

# reference C++ host functions (compiled from the sources where they lie by oracle/build_ref.py)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import build_ref  # noqa: E402

so = build_ref.build()
lib = ctypes.CDLL(so)
for bits in (4, 2, 1):
    packed = out[f"compress_b{bits}"]
    flat = np.ascontiguousarray(packed).reshape(-1)
    for tgt, fn in (("float16", lib.ref_general_interleave_fp16), ("int8", lib.ref_general_interleave_int8)):
        dst = np.zeros_like(flat)
        fn(flat.ctypes.data_as(ctypes.c_void_p), dst.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(bits),
           ctypes.c_size_t(flat.nbytes))
        out[f"ref_cpp_interleave_b{bits}_{tgt}"] = dst.reshape(packed.shape)
    # C++ general_compress (unsigned)
    w = out[f"w_b{bits}"].reshape(-1)
    dst = np.zeros(w.size * bits // 8, dtype=np.int8)
    lib.ref_general_compress(w.ctypes.data_as(ctypes.c_void_p), dst.ctypes.data_as(ctypes.c_void_p),
                             ctypes.c_int(bits), ctypes.c_int(w.size), ctypes.c_int(0))
    out[f"ref_cpp_compress_b{bits}"] = dst.reshape(packed.shape)

np.savez_compressed(os.path.join(HERE, "quant_golden.npz"), **out)
print("wrote", sorted(out))
