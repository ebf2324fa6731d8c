"""ctypes binding of the C ABI declared in include/bitblas_b200.h.

The reference dlopens one generated .so per operator with ctypes (bitblas/ops/operator.py:226-235); here a
single prebuilt in-tree library is loaded once.  There is NO fallback: if the library is missing the import
of the compute path fails loudly.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libbitblas_b200.so")

# enums (include/bitblas_b200.h)
BB_F16, BB_BF16, BB_F32, BB_I8, BB_I32, BB_E4M3 = 0, 1, 2, 3, 4, 5
BB_W_UINT, BB_W_INT, BB_W_NF, BB_W_FP4, BB_W_FP8_E4M3, BB_W_FP8_E5M2 = 0, 1, 2, 3, 4, 5
BB_ZEROS_ORIGINAL, BB_ZEROS_RESCALE, BB_ZEROS_QUANTIZED = 0, 1, 2
BB_LAYOUT_COMPRESSED, BB_LAYOUT_INTERLEAVED_16, BB_LAYOUT_INTERLEAVED_8 = 0, 1, 2
BB_TILE_ROW_MAJOR, BB_TILE_SLAB = 0, 1
BB_TILE_ROWS, BB_TILE_ROW_BYTES = 32, 512
BB_PEER_FLAG_BYTES = 128
BB_GROUPED_MAX_GROUPS = 256
(BB_KERNEL_AUTO, BB_KERNEL_GENERIC, BB_KERNEL_GEMV_MMA, BB_KERNEL_GEMV_I8, BB_KERNEL_GEMM_TS,
 BB_KERNEL_GEMM_TS_I8, BB_KERNEL_GEMV_SLAB) = 0, 1, 2, 3, 4, 5, 7
BB_KERNEL_GEMM_FP8 = 8   # bb_matmul_fp8 only

DTYPE_IDS = {"float16": BB_F16, "bfloat16": BB_BF16, "float32": BB_F32, "int8": BB_I8, "int32": BB_I32}
WFMT_IDS = {"uint": BB_W_UINT, "int": BB_W_INT, "nf": BB_W_NF, "fp": BB_W_FP4, "fp_e4m3": BB_W_FP8_E4M3,
            "fp_e5m2": BB_W_FP8_E5M2}
ZEROS_IDS = {"original": BB_ZEROS_ORIGINAL, "rescale": BB_ZEROS_RESCALE, "quantized": BB_ZEROS_QUANTIZED}

EXPORTS = [
    "bb_init", "bb_matmul", "bb_matmul_swiglu", "bb_matmul_scaled", "bb_matmul_w4a8", "bb_select_kernel_w4a8", "bb_quantize_act_int8",
    "bb_quantize_act_fp8", "bb_matmul_fp8", "bb_select_kernel_fp8", "bb_workspace_bytes_fp8", "bb_matmul_grouped_fp8",
    "bb_matmul_grouped_fp8_swiglu", "bb_matmul_scatter", "bb_matmul_grouped", "bb_matmul_grouped_gemm", "bb_matmul_grouped_swiglu",
    "bb_matmul_grouped_gemm_swiglu", "bb_matmul_grouped_gemm_swiglu_gather", "bb_moe_route", "bb_moe_route_index",
    "bb_moe_combine", "bb_moe_topk", "bb_permute_cols", "bb_peer_barrier", "bb_workspace_bytes", "bb_select_kernel", "bb_kernel_name", "bb_set_kernel_override",
    "bb_set_sm_count_cap", "bb_launch_count", "bb_last_error", "bb_version", "bb_compress_host", "bb_interleave_host",
    "bb_transform_weight_device", "bb_repack_gptq_qweight_device", "bb_repack_gptq_qzeros_device",
    "bb_retile_weight_device", "bb_debug_decode", "bb_debug_dequant",
]


class MatmulDesc(ctypes.Structure):
    _fields_ = [
        ("N", ctypes.c_int32), ("K", ctypes.c_int32), ("a_dtype", ctypes.c_int32), ("w_fmt", ctypes.c_int32),
        ("w_bits", ctypes.c_int32), ("accum_dtype", ctypes.c_int32), ("out_dtype", ctypes.c_int32),
        ("group_size", ctypes.c_int32), ("with_scaling", ctypes.c_int32), ("with_zeros", ctypes.c_int32),
        ("zeros_mode", ctypes.c_int32), ("with_bias", ctypes.c_int32), ("w_layout", ctypes.c_int32),
        ("w_tile", ctypes.c_int32), ("reserved", ctypes.c_int32 * 2),
    ]


_lib = None
OVERRIDE_GEN = 0   # bumped by every bb_set_kernel_override and bb_set_sm_count_cap call (testing hooks)


def load() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"bitblas_b200: CUDA library not built ({LIB_PATH}). Run `python -c 'import __graft_entry__ as g; "
            f"g.build()'` or `python bitblas_b200/csrc/build.py`. There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
    dp = ctypes.POINTER(MatmulDesc)
    lib.bb_init.argtypes = [i32]; lib.bb_init.restype = i32
    for f in (lib.bb_matmul, lib.bb_matmul_swiglu):
        f.argtypes = [dp, vp, vp, vp, vp, vp, vp, vp, i32, vp, sz, vp]; f.restype = i32
    lib.bb_matmul_scaled.argtypes = [dp, vp, vp, vp, vp, vp, vp, i32, vp, sz, vp]; lib.bb_matmul_scaled.restype = i32
    lib.bb_matmul_w4a8.argtypes = [dp, vp, vp, vp, vp, vp, vp, vp, i32, vp, sz, vp]; lib.bb_matmul_w4a8.restype = i32
    lib.bb_select_kernel_w4a8.argtypes = [dp, i32]; lib.bb_select_kernel_w4a8.restype = i32
    lib.bb_quantize_act_int8.argtypes = [vp, i32, i32, i32, vp, vp, vp]; lib.bb_quantize_act_int8.restype = i32
    lib.bb_quantize_act_fp8.argtypes = [vp, i32, i32, i32, vp, vp, i32, vp]; lib.bb_quantize_act_fp8.restype = i32
    lib.bb_matmul_fp8.argtypes = [dp, vp, vp, i32, vp, vp, vp, vp, i32, vp, sz, vp]; lib.bb_matmul_fp8.restype = i32
    lib.bb_select_kernel_fp8.argtypes = [dp, i32]; lib.bb_select_kernel_fp8.restype = i32
    lib.bb_workspace_bytes_fp8.argtypes = [dp, i32]; lib.bb_workspace_bytes_fp8.restype = sz
    for f in (lib.bb_matmul_grouped_fp8, lib.bb_matmul_grouped_fp8_swiglu):
        f.argtypes = [dp, i32, vp, vp, vp, i32, vp, vp, vp, i32, vp]; f.restype = i32
    lib.bb_matmul_scatter.argtypes = [dp, vp, vp, vp, vp, vp, vp, ctypes.POINTER(vp), i32, i64, i64, i32, vp, sz, vp]
    lib.bb_matmul_scatter.restype = i32
    lib.bb_matmul_grouped.argtypes = [dp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp]; lib.bb_matmul_grouped.restype = i32
    lib.bb_matmul_grouped_gemm.argtypes = [dp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp]; lib.bb_matmul_grouped_gemm.restype = i32
    for f in (lib.bb_matmul_grouped_swiglu, lib.bb_matmul_grouped_gemm_swiglu):
        f.argtypes = [dp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp]; f.restype = i32
    lib.bb_matmul_grouped_gemm_swiglu_gather.argtypes = [dp, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp, i32, vp]
    lib.bb_matmul_grouped_gemm_swiglu_gather.restype = i32
    lib.bb_moe_route.argtypes = [vp, i32, i32, i32, vp, i32, i32, vp, vp, vp, vp]; lib.bb_moe_route.restype = i32
    lib.bb_moe_route_index.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]; lib.bb_moe_route_index.restype = i32
    lib.bb_moe_combine.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, vp]; lib.bb_moe_combine.restype = i32
    lib.bb_moe_topk.argtypes = [vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, i32, ctypes.c_float, vp, vp, vp]
    lib.bb_moe_topk.restype = i32
    lib.bb_permute_cols.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp]; lib.bb_permute_cols.restype = i32
    lib.bb_peer_barrier.argtypes = [ctypes.POINTER(vp), i32, i32, vp]; lib.bb_peer_barrier.restype = i32
    lib.bb_workspace_bytes.argtypes = [dp, i32]; lib.bb_workspace_bytes.restype = sz
    lib.bb_select_kernel.argtypes = [dp, i32]; lib.bb_select_kernel.restype = i32
    lib.bb_kernel_name.argtypes = [i32]; lib.bb_kernel_name.restype = ctypes.c_char_p
    def _bumps_generation(c_fn):   # operators cache bb_workspace_bytes per (m, override generation); both hooks change it
        c_fn.argtypes = [i32]; c_fn.restype = i32

        def call(value):
            global OVERRIDE_GEN
            OVERRIDE_GEN += 1
            return c_fn(int(value))
        return call
    lib.bb_set_kernel_override = _bumps_generation(lib.bb_set_kernel_override)
    lib.bb_set_sm_count_cap = _bumps_generation(lib.bb_set_sm_count_cap)
    lib.bb_launch_count.argtypes = []; lib.bb_launch_count.restype = ctypes.c_uint64
    lib.bb_last_error.argtypes = []; lib.bb_last_error.restype = ctypes.c_char_p
    lib.bb_version.argtypes = []; lib.bb_version.restype = i32
    lib.bb_compress_host.argtypes = [vp, vp, i64, i64, i32]; lib.bb_compress_host.restype = i32
    lib.bb_interleave_host.argtypes = [vp, vp, i64, i32, i32]; lib.bb_interleave_host.restype = i32
    lib.bb_transform_weight_device.argtypes = [vp, vp, i64, i64, i32, i32, vp]; lib.bb_transform_weight_device.restype = i32
    lib.bb_repack_gptq_qweight_device.argtypes = [vp, vp, i64, i64, i32, i32, vp]; lib.bb_repack_gptq_qweight_device.restype = i32
    lib.bb_repack_gptq_qzeros_device.argtypes = [vp, vp, vp, i64, i64, i32, i32, i32, i32, vp]; lib.bb_repack_gptq_qzeros_device.restype = i32
    lib.bb_retile_weight_device.argtypes = [vp, vp, i64, i64, i32, vp]; lib.bb_retile_weight_device.restype = i32
    lib.bb_debug_decode.argtypes = [i32, i32, i32, i32, vp, vp, i32, vp]; lib.bb_debug_decode.restype = i32
    lib.bb_debug_dequant.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp]; lib.bb_debug_dequant.restype = i32
    _lib = lib
    return lib


def last_error() -> str:
    return load().bb_last_error().decode()


def check(rc: int, what: str = "bitblas_b200") -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {last_error()}")


_inited = set()


def ensure_init(device_index: int) -> None:
    if device_index in _inited:
        return
    check(load().bb_init(int(device_index)), "bb_init")
    _inited.add(device_index)


def device_stream(t: torch.Tensor):
    """(device, ordinal, raw current stream) of a CUDA tensor; the library is initialised on that device on first use"""
    dev = t.device
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if idx not in _inited:
        ensure_init(idx)
    return dev, idx, torch.cuda.current_stream(idx).cuda_stream


def call(name: str, device: int, *args) -> None:
    """the library entry point `name` with the device of ordinal `device` current (the kernels launch on the calling thread's
    current device); raises RuntimeError with the library's message when it fails"""
    fn = getattr(_lib or load(), name)
    if device != torch.cuda.current_device():
        with torch.cuda.device(device):
            rc = fn(*args)
    else:
        rc = fn(*args)
    if rc != 0:   # tested here too: every decode step comes through this function, and the success path calls nothing more
        check(rc, name)


_TORCH_DTYPE_IDS = {getattr(torch, name): i for name, i in DTYPE_IDS.items()}


def dtype_id(dtype: torch.dtype) -> int:
    return _TORCH_DTYPE_IDS[dtype]


def check_tensor(t, name: str, dtype: torch.dtype, dim: int = None, numel: int = None) -> None:
    """a tensor argument of a library call: a contiguous CUDA torch.Tensor of `dtype`, `dim`-D and of `numel` elements where
    given.  The type is checked before the device, so a CPU tensor of the wrong type reports its type."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if dim is not None and (t.dtype != dtype or t.dim() != dim):
        raise TypeError(f"{name} must be a {dim}-D {dtype} tensor (got {t.dim()}-D {t.dtype})")
    if t.dtype != dtype:
        raise TypeError(f"{name} has dtype {t.dtype}, expected {dtype}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor: bitblas_b200 has no CPU path")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if numel is not None and t.numel() != numel:
        raise ValueError(f"{name} has {t.numel()} elements, expected {numel}")


def kernel_name(kernel_id: int) -> str:
    return load().bb_kernel_name(int(kernel_id)).decode()
