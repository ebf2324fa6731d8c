"""CPU: the grouped wgmma GEMM's C ABI validation (bb_matmul_grouped_gemm) and the `capturable` flag of
Matmul.forward_grouped / GroupedLinear (no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib


def _desc(**kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 256, 512, _lib.BB_F16, _lib.BB_W_UINT, 4
    d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.BB_F16, 128
    d.with_scaling, d.with_zeros, d.zeros_mode = 1, 1, _lib.BB_ZEROS_QUANTIZED
    d.w_layout = _lib.BB_LAYOUT_INTERLEAVED_16
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _grouped_gemm(d, E=8, offsets=0, T=0):
    # fake non-null operand addresses: every call below is refused (or returns) before anything is dereferenced
    return _lib.load().bb_matmul_grouped_gemm(ctypes.byref(d), E, offsets, 16, 16, 16, 16, 16, 16, T, 0)


def test_grouped_gemm_symbol_exported_and_zero_rows_return():
    lib = _lib.load()
    assert "bb_matmul_grouped_gemm" in _lib.EXPORTS and hasattr(lib, "bb_matmul_grouped_gemm")
    assert _grouped_gemm(_desc(), E=8, T=0) == 0
    assert _grouped_gemm(_desc(), E=256, T=0) == 0
    assert _grouped_gemm(_desc(a_dtype=_lib.BB_BF16, out_dtype=_lib.BB_F32, w_fmt=_lib.BB_W_INT, w_bits=2, with_zeros=0,
                               w_layout=_lib.BB_LAYOUT_COMPRESSED, group_size=-1, with_bias=1), E=1, T=0) == 0


@pytest.mark.parametrize("what,kw,E,msg", [
    ("N % 128", dict(N=144), 8, b"N % 128"),
    ("int8 A", dict(a_dtype=_lib.BB_I8, accum_dtype=_lib.BB_I32, out_dtype=_lib.BB_I32, with_scaling=0, with_zeros=0,
                    w_layout=_lib.BB_LAYOUT_INTERLEAVED_8), 8, b"float16 or bfloat16"),
    ("nf4", dict(w_fmt=_lib.BB_W_NF, with_zeros=0, w_layout=_lib.BB_LAYOUT_COMPRESSED), 8, b"uint / int"),
    ("slab tile", dict(w_tile=_lib.BB_TILE_SLAB, K=1024), 8, b"slab-tiled"),
    ("K % 128", dict(K=192, group_size=-1), 8, b"K % 128"),
    ("g = 64", dict(group_size=64), 8, b"group_size"),
    ("no groups", {}, 0, b"num_groups"),
    ("too many groups", {}, 257, b"num_groups"),
])
def test_grouped_gemm_rejects(what, kw, E, msg):
    assert _grouped_gemm(_desc(**kw), E=E, T=4) == 1, what
    assert msg in _lib.last_error().encode(), (what, _lib.last_error())
    assert _grouped_gemm(_desc(**kw), E=E, T=0) == 1, what    # the configuration check does not depend on the rows


def test_grouped_gemm_rejects_null_offsets():
    assert _grouped_gemm(_desc(), E=8, offsets=0, T=4) == 1
    assert "offsets" in _lib.last_error()


def test_grouped_gemm_n144_is_left_to_the_grouped_gemv():
    """N % 16 == 0 but not % 128: the grouped GEMV ABI covers it, the grouped GEMM refuses it"""
    lib = _lib.load()
    assert lib.bb_matmul_grouped(ctypes.byref(_desc(N=144)), 8, 0, 16, 16, 16, 16, 16, 16, 0, 0) == 0
    assert _grouped_gemm(_desc(N=144), E=8, T=0) == 1


def test_capturable_passes_through_grouped_linear(monkeypatch):
    gl = bitblas.GroupedLinear(4, 512, 256, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
                               with_zeros=True, zeros_mode="quantized")
    seen = []
    monkeypatch.setattr(gl.bitblas_matmul, "forward_grouped", lambda *a, **kw: seen.append(kw.get("capturable")))
    A, off = torch.zeros(8, 512, dtype=torch.float16), torch.tensor([0, 2, 4, 6, 8], dtype=torch.int32)
    gl(A, off)
    gl(A, off, capturable=True)
    gl(A, off, output=None, capturable=False)
    assert seen == [False, True, False]


def test_forward_grouped_capturable_keeps_the_argument_checks():
    op = bitblas.Matmul(bitblas.MatmulConfig(M=[1, 16], N=256, K=512, A_dtype="float16", W_dtype="uint4", group_size=128,
                                             with_scaling=True, with_zeros=True, zeros_mode="quantized"), enable_tuning=False)
    W = torch.zeros(4, 256, 256, dtype=torch.int8)
    scale, zeros = torch.ones(4, 256, 4, dtype=torch.float16), torch.zeros(4, 4, 128, dtype=torch.int8)
    A, off = torch.zeros(64, 512, dtype=torch.float16), torch.tensor([0, 16, 32, 48, 64], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        op.forward_grouped(A, W, off, scale=scale, zeros=zeros, capturable=True)
    with pytest.raises(ValueError, match="scale has shape"):
        op.forward_grouped(A, W, off, scale=scale[:, :, :2], zeros=zeros, capturable=True)
