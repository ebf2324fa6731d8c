"""CPU: MatmulConfig legalisation, Matmul/Linear surface and the C-ABI exports (no compute calls)."""
import ctypes
import os
import re

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.ops.operator import OptimizeStrategy, TransformKind

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "bitblas_b200.h")).read()
    declared = set(re.findall(r"\b(bb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = _lib.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/bitblas_b200.h but not exported"
    assert declared == set(_lib.EXPORTS)
    assert lib.bb_version() == 100
    assert ctypes.sizeof(_lib.MatmulDesc) == 16 * 4


def test_config_defaults_match_reference():
    # bitblas/ops/general_matmul/__init__.py:58-95
    c = bitblas.MatmulConfig(M=1, N=16, K=16)
    assert (c.A_dtype, c.W_dtype, c.out_dtype, c.accum_dtype, c.layout) == ("float16",) * 4 + ("nt",)
    assert (c.with_bias, c.group_size, c.with_scaling, c.with_zeros, c.zeros_mode, c.storage_dtype) == (
        False, -1, False, False, "original", "float16")
    assert c.optimize_stratety == OptimizeStrategy.SingleBatchDecodeOnly
    assert c.propagate_a == TransformKind.NonTransform and c.propagate_b == TransformKind.NonTransform


def test_config_legalisation():
    # M list -> tuple (hashable) :97-98,200 ; None -> default dynamic range :188-192
    assert bitblas.MatmulConfig(M=[1, 16], N=16, K=16).M == (1, 16)
    assert bitblas.MatmulConfig(N=16, K=16).M == (1, 16, 32, 64, 128, 256, 512, 1024)
    assert bitblas.MatmulConfig(N=16, K=16, optimize_stratety=1).M == (16, 32, 64, 128, 256, 512, 1024)
    with pytest.raises(ValueError):
        bitblas.MatmulConfig(M=1, K=16)
    with pytest.raises(ValueError):
        bitblas.MatmulConfig(M=1, N=16)
    # None -> defaults :218-228
    c = bitblas.MatmulConfig(M=1, N=16, K=16, with_bias=None, group_size=None, with_scaling=None, with_zeros=None, zeros_mode=None)
    assert (c.with_bias, c.group_size, c.with_scaling, c.with_zeros, c.zeros_mode) == (False, -1, False, False, "original")
    hash(c)
    # storage dtype :230-237
    assert bitblas.MatmulConfig(M=1, N=16, K=16, A_dtype="int8", W_dtype="int8").storage_dtype == "int8"
    assert bitblas.MatmulConfig(M=1, N=16, K=16, W_dtype="uint4").storage_dtype == "int8"


@pytest.mark.parametrize("A,W,expected", [
    ("float16", "uint4", True), ("float16", "int4", True), ("float16", "int2", True), ("float16", "int1", True),
    ("float16", "nf4", False), ("float16", "fp4_e2m1", False), ("float16", "e4m3_float8", False),
    ("float16", "float16", False), ("float16", "int8", False), ("int8", "int4", False), ("int8", "uint4", False),
    ("int8", "int2", True), ("bfloat16", "uint4", False),
])
def test_fast_decoding_rule(A, W, expected):
    # :163-184
    assert bitblas.MatmulConfig(M=1, N=16, K=64, A_dtype=A, W_dtype=W, accum_dtype="int32" if A == "int8" else "float16").fast_decoding is expected
    assert bitblas.MatmulConfig(M=1, N=16, K=64, A_dtype=A, W_dtype=W, fast_decoding=not expected).fast_decoding is (not expected)


def test_matmul_surface_and_dispatch():
    cfg = bitblas.MatmulConfig(M=[1, 16, 4096], N=12288, K=12288, A_dtype="float16", W_dtype="uint4", group_size=128,
                               with_scaling=True, with_zeros=True, zeros_mode="quantized")
    op = bitblas.Matmul(cfg, enable_tuning=False)
    assert (op.bit, op.source_format) == (4, "uint")
    assert op.dynamic_range == {"m": (1, 16, 4096)}
    assert op.retrieve_weight_shape() == [12288, 6144]
    assert op.weight_transform is not None and op.weight_transform.size == 2 and op.input_transform is None
    assert op.lut is None and op.lib is not None and hasattr(op.lib, "init") and hasattr(op.lib, "call")
    for name in ("M", "N", "K", "A_dtype", "W_dtype", "out_dtype", "accum_dtype", "storage_dtype", "with_scaling", "with_zeros",
                 "group_size", "fast_decoding", "with_bias", "propagate_a", "propagate_b", "layout", "zeros_mode"):
        assert getattr(op, name) == getattr(cfg, name)
    assert op.hardware_aware_finetune(topk=20) is None
    assert [op.kernel_for(m) for m in (1, 8, 9, 32, 128, 4096)] == ["gemv_slab", "gemv_mma"] + ["gemm_ts_wgmma"] * 4
    assert "gemm_ts_wgmma" in op.get_source()
    # W2A8 (integration/BitNet/utils_quant.py:55-69)
    op8 = bitblas.Matmul(bitblas.MatmulConfig(M=[1, 128], N=12288, K=12288, A_dtype="int8", W_dtype="int2", accum_dtype="int32",
                                              out_dtype="float32"), enable_tuning=False)
    assert [op8.kernel_for(m) for m in (1, 128)] == ["gemv_i8", "gemm_ts_wgmma_i8"]
    # formats without a fast kernel fall to the generic CUDA kernel, never to the CPU
    opn = bitblas.Matmul(bitblas.MatmulConfig(M=1, N=64, K=256, W_dtype="nf4", with_scaling=True, group_size=64), enable_tuning=False)
    assert opn.kernel_for(1) == "generic_simt" and opn.lut is not None and opn.lut.numel() == 16
    with pytest.raises(ValueError):
        bitblas.Matmul(bitblas.MatmulConfig(M=1, N=16, K=64, W_dtype="uint4", layout="nn"), enable_tuning=False)


def test_c_abi_validation_without_gpu():
    lib = _lib.load()
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 64, 100, _lib.BB_F16, _lib.BB_W_UINT, 4
    d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.BB_F16, 32
    assert lib.bb_select_kernel(ctypes.byref(d), 1) == -1
    assert b"not divisible" in lib.bb_last_error()
    d.K, d.group_size = 96, -1     # K not a multiple of 128: only the generic kernel covers it
    assert lib.bb_select_kernel(ctypes.byref(d), 1) == _lib.BB_KERNEL_GENERIC
    d.K = 128                      # both storage layouts are consumed by the streaming kernel
    assert lib.bb_select_kernel(ctypes.byref(d), 1) == _lib.BB_KERNEL_GEMV_MMA
    d.w_layout = _lib.BB_LAYOUT_INTERLEAVED_16
    assert lib.bb_select_kernel(ctypes.byref(d), 1) == _lib.BB_KERNEL_GEMV_MMA
    # m == 0 returns before touching the device (builder/wrapper/tl.py:156-157)
    assert lib.bb_matmul(ctypes.byref(d), 1, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0) == 0
    # missing operand -> error code + message, no launch
    d.with_scaling = 1
    assert lib.bb_matmul(ctypes.byref(d), 1, 1, 0, 0, 0, 0, 1, 4, 0, 0, 0) == 1
    assert b"scale is null" in lib.bb_last_error()
    if not torch.cuda.is_available():
        assert lib.bb_init(0) != 0 and b"CUDA" in lib.bb_last_error()


def test_forward_refuses_cpu_tensors():
    op = bitblas.Matmul(bitblas.MatmulConfig(M=1, N=16, K=128, W_dtype="uint4"), enable_tuning=False)
    with pytest.raises(RuntimeError, match="no CPU path"):
        op(torch.zeros(1, 128, dtype=torch.float16), torch.zeros(16, 64, dtype=torch.int8))


def test_linear_buffers_match_reference_shapes():
    # bitblas/module/__init__.py:164-205
    lin = bitblas.Linear(1024, 512, bias=True, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                         zeros_mode="quantized", enable_tuning=False)
    sd = lin.state_dict()
    assert {k: (tuple(v.shape), v.dtype) for k, v in sd.items()} == {
        "qweight": ((512, 512), torch.int8), "scales": ((512, 8), torch.float16),
        "zeros": ((8, 256), torch.int8), "bias": ((512,), torch.float16)}
    lin2 = bitblas.Linear(1024, 512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                          zeros_mode="original", enable_tuning=False)
    assert tuple(lin2.zeros.shape) == (512, 8) and lin2.zeros.dtype == torch.float16 and lin2.bias is None
    with pytest.raises(ValueError):
        bitblas.Linear(1000, 512, W_dtype="uint4")
    with pytest.raises(ValueError):
        bitblas.Linear(1024, 512, W_dtype="uint4", group_size=100)
    assert bitblas.Linear.opt_M == [16, 32, 64, 128, 256, 512]


def test_bitblas_alias_package():
    import bitblas as bb
    from bitblas import Matmul, MatmulConfig, Linear, auto_detect_nvidia_target  # noqa: F401
    from bitblas.cache import global_operator_cache, get_database_path
    from bitblas.quantization.utils import general_compress, interleave_weight  # noqa: F401
    from bitblas.testing import torch_assert_close  # noqa: F401
    assert bb.Matmul is bitblas.Matmul and bb.__version__ == "0.1.0"
    assert global_operator_cache.size() >= 0 and isinstance(get_database_path(), str)
    bb.set_log_level("INFO")


def test_propagate_b_selects_slab_tiling():
    """MatmulConfig(propagate_b=True): the H100 meaning of weight propagation is the slab tiling (include/bitblas_b200.h,
    enum bb_wtile); shapes / formats it does not cover legalise back to the row-major storage like the reference's
    __initialize_propagate does for its own unsupported cases (general_matmul/__init__.py:113-157)."""
    import numpy as np
    import torch
    import bitblas_oracle as O
    from bitblas_b200 import Matmul, MatmulConfig
    from bitblas_b200.ops.operator import TransformKind
    c = MatmulConfig(M=1, N=256, K=2048, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, propagate_b=True)
    assert c.propagate_b == TransformKind.LDMatrixTransform and c.propagate_a == TransformKind.NonTransform
    assert MatmulConfig(M=1, N=256, K=2048, A_dtype="float16", W_dtype="uint4").propagate_b == TransformKind.NonTransform
    assert MatmulConfig(M=1, N=48, K=2048, A_dtype="float16", W_dtype="uint4", propagate_b=True).propagate_b == TransformKind.NonTransform
    assert MatmulConfig(M=1, N=256, K=512, A_dtype="float16", W_dtype="uint4", propagate_b=True).propagate_b == TransformKind.NonTransform
    assert MatmulConfig(M=1, N=256, K=2048, A_dtype="float16", W_dtype="nf4", propagate_b=True).propagate_b == TransformKind.NonTransform
    op, op0 = Matmul(c, enable_tuning=False), Matmul(MatmulConfig(M=1, N=256, K=2048, A_dtype="float16", W_dtype="uint4", group_size=128,
                                                                  with_scaling=True), enable_tuning=False)
    assert op.weight_tiled and not op0.weight_tiled and op._desc.w_tile == 1 and op0._desc.w_tile == 0
    assert op.retrieve_weight_shape() == op0.retrieve_weight_shape()
    g = torch.Generator().manual_seed(0)
    fields = torch.randint(0, 16, (256, 2048), generator=g, dtype=torch.int8)
    plain, tiled = op0.transform_weight(fields), op.transform_weight(fields)
    assert np.array_equal(tiled.numpy(), O.slab_tile(plain.numpy()))
    assert torch.equal(op.tile_weight(tiled, inverse=True), plain)
    # dispatch: the decode kernel and the wgmma kernel take the tiled storage, the register-streaming kernels do not
    assert op.kernel_for(1) == "gemv_slab" and op.kernel_for(4) == "gemm_ts_wgmma" and op.kernel_for(512) == "gemm_ts_wgmma"
