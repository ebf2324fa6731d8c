"""CPU: validation of the copy-free routing (bb_moe_route_index) and the gathering grouped GEMM
(bb_matmul_grouped_gemm_swiglu_gather), and the Python argument checks around them (no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.moe import moe_route_index

CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
GATHER = "bb_matmul_grouped_gemm_swiglu_gather"


def test_exports_and_argtypes():
    lib = _lib.load()
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    for name in (GATHER, "bb_moe_route_index"):
        assert name in _lib.EXPORTS and hasattr(lib, name), name
        assert getattr(lib, name).restype is ctypes.c_int
    assert lib.bb_moe_route_index.argtypes == [vp, i32, i32, i32, vp, vp, vp, vp]
    # desc, num_groups, offsets, row_index, A, a_rows, W, scale, zeros, bias, C, total_rows, stream
    assert lib.bb_matmul_grouped_gemm_swiglu_gather.argtypes == [ctypes.POINTER(_lib.MatmulDesc), i32, vp, vp, vp, i32, vp, vp,
                                                                 vp, vp, vp, i32, vp]


# ---- routing --------------------------------------------------------------------------------------------------------------------
# fake non-null, aligned device addresses: every call below is refused (or returns) before anything is dereferenced
def _route_index(T=4, k=2, E=8, ids=16, offsets=16, rows=16, tokens=16):
    return _lib.load().bb_moe_route_index(ids, T, k, E, offsets, rows, tokens, 0)


@pytest.mark.parametrize("what,kw,msg", [
    ("E = 0", dict(E=0), "num_experts"), ("E = 257", dict(E=257), "num_experts"), ("top_k = 0", dict(k=0), "top_k"),
    ("T * k >= 2^31", dict(T=1 << 28, k=8), "2^31"), ("T < 0", dict(T=-1), "num_tokens"),
])
def test_route_index_rejects(what, kw, msg):
    assert _route_index(**kw) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


@pytest.mark.parametrize("ptr", ["ids", "offsets", "rows", "tokens"])
def test_route_index_rejects_null_and_unaligned(ptr):
    assert _route_index(**{ptr: 0}) == 1
    assert "non-null" in _lib.last_error()
    assert _route_index(**{ptr: 18}) == 5
    assert "4-byte aligned" in _lib.last_error()


def test_route_index_zero_tokens_validates_only():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert lib.bb_moe_route_index(0, 0, 8, 256, 0, 0, 0, 0) == 0
    assert lib.bb_launch_count() == n0
    assert lib.bb_moe_route_index(0, 0, 8, 257, 0, 0, 0, 0) == 1      # still validated
    assert "num_experts" in _lib.last_error()


def test_route_index_python_checks():
    with pytest.raises(TypeError, match="int32"):
        moe_route_index(torch.zeros((4, 2), dtype=torch.int64), 8)
    with pytest.raises(TypeError, match="2-D"):
        moe_route_index(torch.zeros(8, dtype=torch.int32), 8)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        moe_route_index(torch.zeros((4, 2), dtype=torch.int32), 8)


# ---- gathering grouped GEMM -----------------------------------------------------------------------------------------------------
def _desc(**kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 256, 512, _lib.BB_F16, _lib.BB_W_UINT, 4
    d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.BB_F16, 128
    d.with_scaling, d.with_zeros, d.zeros_mode = 1, 1, _lib.BB_ZEROS_QUANTIZED
    d.w_layout = _lib.BB_LAYOUT_INTERLEAVED_16
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _gather(d, E=8, T=4, row_index=16, a_rows=4, offsets=16, A=16):
    return _lib.load().bb_matmul_grouped_gemm_swiglu_gather(ctypes.byref(d), E, offsets, row_index, A, a_rows, 16, 16, 16, 16, 16,
                                                            T, 0)


def _plain(d, E=8, T=4):
    return _lib.load().bb_matmul_grouped_gemm_swiglu(ctypes.byref(d), E, 16, 16, 16, 16, 16, 16, 16, T, 0)


def test_gather_zero_rows_validates_only():
    n0 = _lib.load().bb_launch_count()
    assert _gather(_desc(), T=0, row_index=0, a_rows=0) == 0
    assert _gather(_desc(N=512, a_dtype=_lib.BB_BF16, out_dtype=_lib.BB_F32, with_bias=1), E=256, T=0, row_index=0, a_rows=0) == 0
    assert _lib.load().bb_launch_count() == n0


@pytest.mark.parametrize("what,kw,code,msg", [
    ("null row_index", dict(row_index=0), 1, "row_index"),
    ("a_rows = 0", dict(a_rows=0), 1, "a_rows"),
    ("a_rows < 0", dict(a_rows=-3), 1, "a_rows"),
    ("row_index misaligned", dict(row_index=18), 5, "4-byte aligned"),
    ("A misaligned", dict(A=24), 5, "16-byte aligned"),
    ("offsets misaligned", dict(offsets=18), 5, "aligned"),
    ("null offsets", dict(offsets=0), 1, "offsets"),
])
def test_gather_rejects_arguments(what, kw, code, msg):
    assert _gather(_desc(), **kw) == code, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


@pytest.mark.parametrize("what,kw,E", [
    ("N % 128", dict(N=144), 8),
    ("I % 8", dict(N=2 * 108), 8),
    ("int8 A", dict(a_dtype=_lib.BB_I8, accum_dtype=_lib.BB_I32, out_dtype=_lib.BB_I32, with_scaling=0, with_zeros=0,
                    w_layout=_lib.BB_LAYOUT_INTERLEAVED_8), 8),
    ("nf4", dict(w_fmt=_lib.BB_W_NF, with_zeros=0), 8),
    ("too many groups", {}, 257),
    ("no groups", {}, 0),
    ("bad zeros mode", dict(zeros_mode=7), 8),
])
def test_gather_rejects_what_the_plain_call_rejects(what, kw, E):
    """the configurations bb_matmul_grouped_gemm_swiglu refuses are refused with its code and message, at T = 0 too"""
    for T in (0, 4):
        rc_plain = _plain(_desc(**kw), E=E, T=T)
        msg_plain = _lib.last_error()
        assert rc_plain != 0, what
        assert _gather(_desc(**kw), E=E, T=T) == rc_plain, what
        assert _lib.last_error() == msg_plain, what


def test_gather_checks_the_config_before_the_index():
    assert _gather(_desc(N=144), row_index=0, a_rows=0) == 1
    assert "N % 128" in _lib.last_error()


# ---- Python -------------------------------------------------------------------------------------------------------------------
def _op(**kw):
    return bitblas.MoEExperts(8, 512, 128, **dict(CFG, **kw)).gate_up


def test_forward_grouped_swiglu_row_index_python_checks():
    gl = _op()
    mm = gl.bitblas_matmul
    A = torch.zeros((4, 512), dtype=torch.float16)
    off = torch.zeros(9, dtype=torch.int32)
    args = (A, gl.qweight, off, gl.scales, gl.zeros)
    with pytest.raises(TypeError, match="row_index"):
        mm.forward_grouped_swiglu(*args, row_index=torch.zeros(4, dtype=torch.int64))
    with pytest.raises(TypeError, match="row_index"):
        mm.forward_grouped_swiglu(*args, row_index=torch.zeros((4, 1), dtype=torch.int32))
    with pytest.raises(TypeError, match="row_index"):
        mm.forward_grouped_swiglu(*args, row_index=[0, 1, 2])
    with pytest.raises(RuntimeError, match="CUDA tensor"):        # the stacked parameters are checked before A and the output
        mm.forward_grouped_swiglu(*args, row_index=torch.zeros(6, dtype=torch.int32))

