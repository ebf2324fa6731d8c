"""CPU: the dense SwiGLU MLP's C ABI validation (bb_matmul_swiglu), Matmul.forward_swiglu's and SwiGLUMLP's argument errors, and
the interleave-then-tile order of a slab-tiled gate/up weight (no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.moe import deinterleave_gate_up, interleave_gate_up

CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")


def _desc(N=256, K=256, a_dtype=_lib.BB_F16, w_layout=_lib.BB_LAYOUT_COMPRESSED):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = N, K, a_dtype, _lib.BB_W_UINT, 4
    d.accum_dtype = _lib.BB_I32 if a_dtype == _lib.BB_I8 else _lib.BB_F32
    d.out_dtype = _lib.BB_I32 if a_dtype == _lib.BB_I8 else _lib.BB_F16
    d.group_size, d.w_layout = -1, w_layout
    return d


# fake non-null, aligned device addresses: every call below is refused (or returns) before anything is dereferenced
def _call(d, m=1, A=16, W=16, C=16):
    return _lib.load().bb_matmul_swiglu(ctypes.byref(d), A, W, 0, 0, 0, 0, C, m, 0, 0, 0)


def test_export_and_argtypes():
    lib = _lib.load()
    assert "bb_matmul_swiglu" in _lib.EXPORTS and hasattr(lib, "bb_matmul_swiglu")
    assert lib.bb_matmul_swiglu.restype is ctypes.c_int
    assert lib.bb_matmul_swiglu.argtypes == lib.bb_matmul.argtypes


@pytest.mark.parametrize("what,d,kw,msg", [
    ("int8 activations", _desc(a_dtype=_lib.BB_I8, w_layout=_lib.BB_LAYOUT_INTERLEAVED_8), {}, "int8 activations"),
    ("N % 16", _desc(N=264), {}, "I % 8 == 0"),
    ("null C", _desc(), dict(C=0), "must be non-null"),
    ("null A", _desc(), dict(A=0), "must be non-null"),
    ("m < 0", _desc(), dict(m=-1), "m must be >= 0"),
    ("bad descriptor first", _desc(K=0), dict(C=0), "N and K must be positive"),
])
def test_rejects(what, d, kw, msg):
    assert _call(d, **kw) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def test_desc_rejections_do_not_depend_on_m():
    # the int8 and shape checks come before m (bb_matmul's order: descriptor, then m, then pointers)
    assert _call(_desc(N=264), m=0) == 1 and "I % 8 == 0" in _lib.last_error()


def test_zero_rows_return_without_launch():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(_desc(), m=0, A=0, W=0, C=0) == 0
    assert lib.bb_launch_count() == n0


def _op(**kw):
    return bitblas.Matmul(bitblas.MatmulConfig(**dict(dict(M=[1, 16], N=256, K=256), **kw)), enable_tuning=False)


def test_forward_swiglu_argument_errors():
    with pytest.raises(NotImplementedError, match="low-bit"):
        _op(A_dtype="float16", W_dtype="float16").forward_swiglu(None, None)
    with pytest.raises(ValueError, match="int8"):
        _op(A_dtype="int8", W_dtype="int4", accum_dtype="int32", out_dtype="int32").forward_swiglu(None, None)
    with pytest.raises(ValueError, match="I % 8 == 0"):
        _op(N=264, **CFG).forward_swiglu(None, None)
    op = _op(**CFG)
    with pytest.raises(RuntimeError, match="CUDA tensor"):   # the checks of forward() follow
        op.forward_swiglu(torch.zeros(1, 256, dtype=torch.float16), torch.zeros(256, 128, dtype=torch.int8))


def test_mlp_constructor_errors():
    with pytest.raises(ValueError, match="multiple of 8"):
        bitblas.SwiGLUMLP(256, 260, **CFG)
    with pytest.raises(ValueError, match="out_dtype == A_dtype"):
        bitblas.SwiGLUMLP(256, 256, out_dtype="float32", **CFG)
    with pytest.raises(NotImplementedError, match="low-bit"):
        bitblas.SwiGLUMLP(256, 256, A_dtype="float16", W_dtype="float16")
    mlp = bitblas.SwiGLUMLP(256, 512, bias=True, **CFG)
    assert mlp.gate_up.out_features == 1024 and mlp.gate_up.in_features == 256
    assert mlp.down.in_features == 512 and mlp.down.out_features == 256
    assert mlp.gate_up.perm is None and mlp.down.perm is None
    assert bitblas.SwiGLUMLP is __import__("bitblas").SwiGLUMLP


def test_interleave_then_tile_order():
    """propagate_b: the fused weight is interleaved in row-major packed form, then slab-tiled; tile_weight(inverse=True) and
    deinterleave_gate_up undo it in the opposite order, and the two orders differ (the interleave does not commute with tiling)"""
    mlp = bitblas.SwiGLUMLP(2048, 256, propagate_b=True, **CFG)   # two 512-byte segments per packed row
    op = mlp.gate_up.bitblas_matmul
    assert op.weight_tiled
    g = torch.randint(-128, 128, (256, 1024), dtype=torch.int8)   # packed [I, K * bits / 8] rows
    u = torch.randint(-128, 128, (256, 1024), dtype=torch.int8)
    stored = op.tile_weight(interleave_gate_up(g, u, "weight"))
    g2, u2 = deinterleave_gate_up(op.tile_weight(stored, inverse=True), "weight")
    assert torch.equal(g2, g) and torch.equal(u2, u)
    assert not torch.equal(stored, interleave_gate_up(op.tile_weight(g), op.tile_weight(u), "weight"))
