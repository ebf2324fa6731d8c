"""CPU: the BitNet entry points' C ABI validation (bb_quantize_act_int8, bb_matmul_scaled), the argument errors of
quantize_act_int8, Matmul.forward_scaled and BitLinear, and BitLinear's weight loading on the CPU transform path (no compute
calls: every call below is refused, or returns, before the device is touched)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.bitnet import absmean_ternary


def _desc(N=256, K=256, a_dtype=_lib.BB_I8, out_dtype=_lib.BB_F16, bits=2, layout=_lib.BB_LAYOUT_INTERLEAVED_8, **kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = N, K, a_dtype, _lib.BB_W_INT, bits
    d.accum_dtype = _lib.BB_I32 if a_dtype == _lib.BB_I8 else _lib.BB_F32
    d.out_dtype, d.group_size, d.w_layout = out_dtype, -1, layout
    for k, v in kw.items():
        setattr(d, k, v)
    return d


# fake non-null, aligned device addresses
def _scaled(d, m=1, A=16, W=16, a_scale=16, w_scale=16, bias=0, C=16):
    return _lib.load().bb_matmul_scaled(ctypes.byref(d), A, W, a_scale, w_scale, bias, C, m, 0, 0, 0)


def _quant(x=16, a_dtype=_lib.BB_F16, rows=1, K=256, q=16, scale=16):
    return _lib.load().bb_quantize_act_int8(x, a_dtype, rows, K, q, scale, 0)


def test_exports_and_argtypes():
    lib = _lib.load()
    for name in ("bb_matmul_scaled", "bb_quantize_act_int8"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert getattr(lib, name).restype is ctypes.c_int
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    assert lib.bb_matmul_scaled.argtypes == [ctypes.POINTER(_lib.MatmulDesc), vp, vp, vp, vp, vp, vp, i32, vp, ctypes.c_size_t, vp]
    assert lib.bb_quantize_act_int8.argtypes == [vp, i32, i32, i32, vp, vp, vp]
    assert bitblas.quantize_act_int8 is __import__("bitblas").quantize_act_int8
    assert bitblas.BitLinear is __import__("bitblas").BitLinear


@pytest.mark.parametrize("what,d,kw,code,msg", [
    ("16-bit activations", _desc(a_dtype=_lib.BB_F16, layout=_lib.BB_LAYOUT_COMPRESSED), {}, 1, "needs int8 activations"),
    ("int32 out", _desc(out_dtype=_lib.BB_I32), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    ("int8 out", _desc(out_dtype=_lib.BB_I8), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    ("group scales", _desc(with_scaling=1), {}, 1, "group scales are not supported"),
    ("zeros", _desc(w_fmt=_lib.BB_W_UINT, with_zeros=1), {}, 1, "zero points are not supported"),
    ("null A", _desc(), dict(A=0), 1, "A, W and C must be non-null"),
    ("null C", _desc(), dict(C=0), 1, "A, W and C must be non-null"),
    ("null a_scale", _desc(), dict(a_scale=0), 1, "a_scale must be non-null"),
    ("null w_scale", _desc(), dict(w_scale=0), 1, "w_scale must be non-null"),
    ("misaligned a_scale", _desc(), dict(a_scale=18), 5, "4-byte aligned"),
    ("misaligned w_scale", _desc(), dict(w_scale=17), 5, "4-byte aligned"),
    ("bias missing", _desc(with_bias=1), {}, 1, "with_bias is set but bias is null"),
    ("m < 0", _desc(), dict(m=-1), 1, "m must be >= 0"),
    ("bad descriptor first", _desc(K=0), dict(A=0, a_scale=0), 1, "N and K must be positive"),
    ("descriptor before scaled checks", _desc(w_bits=3), dict(a_scale=0), 1, "unsupported weight bit width"),
])
def test_scaled_rejects(what, d, kw, code, msg):
    assert _scaled(d, **kw) == code, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def test_scaled_check_order():
    # descriptor checks come before m: refused at m = 0 too; m before pointers: m = 0 with null pointers returns 0
    assert _scaled(_desc(out_dtype=_lib.BB_I32), m=0) == 1 and "out_dtype" in _lib.last_error()
    assert _scaled(_desc(a_dtype=_lib.BB_BF16, layout=_lib.BB_LAYOUT_COMPRESSED), m=0) == 1
    assert _scaled(_desc(), m=-1, A=0, a_scale=0) == 1 and "m must be >= 0" in _lib.last_error()
    # pointers in order: A / W / C, then a_scale, then w_scale, then bias
    assert _scaled(_desc(with_bias=1), A=0, a_scale=0, w_scale=0) == 1 and "A, W and C" in _lib.last_error()
    assert _scaled(_desc(with_bias=1), a_scale=0, w_scale=0) == 1 and "a_scale" in _lib.last_error()
    assert _scaled(_desc(with_bias=1), w_scale=0) == 1 and "w_scale" in _lib.last_error()


@pytest.mark.parametrize("out", [_lib.BB_F16, _lib.BB_BF16, _lib.BB_F32])
@pytest.mark.parametrize("bits,layout", [(2, _lib.BB_LAYOUT_INTERLEAVED_8), (4, _lib.BB_LAYOUT_COMPRESSED), (1, _lib.BB_LAYOUT_COMPRESSED)])
def test_scaled_zero_rows_launch_nothing(out, bits, layout):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _scaled(_desc(out_dtype=out, bits=bits, layout=layout, with_bias=1), m=0, A=0, W=0, a_scale=0, w_scale=0, C=0) == 0
    assert lib.bb_launch_count() == n0


@pytest.mark.parametrize("what,kw,code,msg", [
    ("int8 x", dict(a_dtype=_lib.BB_I8), 1, "float16 or bfloat16"),
    ("fp32 x", dict(a_dtype=_lib.BB_F32), 1, "float16 or bfloat16"),
    ("K % 8", dict(K=260), 1, "K % 8 == 0"),
    ("K = 0", dict(K=0), 1, "K > 0"),
    ("rows < 0", dict(rows=-1), 1, "rows must be >= 0"),
    ("null x", dict(x=0), 1, "x must be non-null"),
    ("null q", dict(q=0), 1, "q must be non-null"),
    ("null scale", dict(scale=0), 1, "scale must be non-null"),
    ("misaligned x", dict(x=24), 5, "x must be 16-byte aligned"),
    ("misaligned q", dict(q=8), 5, "q must be 16-byte aligned"),
    ("misaligned scale", dict(scale=18), 5, "scale must be 4-byte aligned"),
    ("dtype before K", dict(a_dtype=7, K=3), 1, "float16 or bfloat16"),
    ("K before rows", dict(K=3, rows=-1), 1, "K % 8 == 0"),
])
def test_quantize_rejects(what, kw, code, msg):
    assert _quant(**kw) == code, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def test_quantize_zero_rows_launch_nothing():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _quant(x=0, rows=0, q=0, scale=0) == 0
    assert _quant(x=0, a_dtype=_lib.BB_BF16, rows=0, K=65536, q=0, scale=0) == 0
    assert lib.bb_launch_count() == n0


def _op(**kw):
    base = dict(M=[1, 16], N=256, K=256, A_dtype="int8", W_dtype="int2", accum_dtype="int32", out_dtype="float16")
    return bitblas.Matmul(bitblas.MatmulConfig(**dict(base, **kw)), enable_tuning=False)


def test_forward_scaled_argument_errors():
    with pytest.raises(NotImplementedError, match="low-bit"):
        _op(A_dtype="float16", W_dtype="float16", accum_dtype="float32").forward_scaled(None, None, None, None)
    with pytest.raises(ValueError, match="int8 activations"):
        _op(A_dtype="float16", W_dtype="uint4", accum_dtype="float32").forward_scaled(None, None, None, None)
    for out in ("int32", "int8"):
        with pytest.raises(ValueError, match="out_dtype"):
            _op(out_dtype=out).forward_scaled(None, None, None, None)
    with pytest.raises(ValueError, match="with_scaling=False"):
        _op(W_dtype="uint4", with_scaling=True).forward_scaled(None, None, None, None)
    op = _op()
    op.check_scaled()
    A = torch.zeros(1, 256, dtype=torch.int8)
    with pytest.raises(RuntimeError, match="CUDA tensor"):   # the checks of forward() follow
        op.forward_scaled(A, torch.zeros(256, 64, dtype=torch.int8), torch.ones(1), torch.ones(256))
    with pytest.raises(TypeError, match="A has dtype"):
        op.forward_scaled(torch.zeros(1, 256, dtype=torch.float16), None, None, None)


def test_quantize_act_int8_argument_errors():
    with pytest.raises(TypeError, match="float16 or bfloat16"):
        bitblas.quantize_act_int8(torch.zeros(2, 64))
    with pytest.raises(TypeError, match="float16 or bfloat16"):
        bitblas.quantize_act_int8([1.0] * 8)
    with pytest.raises(ValueError, match="multiple of 8"):
        bitblas.quantize_act_int8(torch.zeros(2, 60, dtype=torch.float16))
    with pytest.raises(ValueError, match="multiple of 8"):
        bitblas.quantize_act_int8(torch.zeros((), dtype=torch.float16))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        bitblas.quantize_act_int8(torch.zeros(2, 64, dtype=torch.bfloat16))


def test_bitlinear_constructor_and_loading_errors():
    with pytest.raises(ValueError, match="float16 or bfloat16"):
        bitblas.BitLinear(256, 256, A_dtype="float32")
    with pytest.raises(ValueError, match="multiple of 16"):
        bitblas.BitLinear(264, 256)
    with pytest.raises(ValueError, match="out_features"):
        bitblas.BitLinear(256, 0)
    lin = bitblas.BitLinear(256, 128, bias=True, A_dtype="bfloat16")
    assert tuple(lin.qweight.shape) == (128, 64) and lin.qweight.dtype == torch.int8
    assert lin.weight_scale.dtype == torch.float32 and lin.bias.dtype == torch.bfloat16
    cfg = lin.bitblas_matmul.config
    assert (cfg.A_dtype, cfg.W_dtype, cfg.accum_dtype, cfg.out_dtype, cfg.with_bias) == ("int8", "int2", "int32", "bfloat16", True)
    assert lin.bitblas_matmul._desc.w_layout == _lib.BB_LAYOUT_INTERLEAVED_8
    q = torch.zeros(128, 256)
    with pytest.raises(ValueError, match=r"q must be \[128, 256\]"):
        lin.load_quantized(q[:, :128], 1.0, torch.zeros(128))
    with pytest.raises(ValueError, match="ternary"):
        lin.load_quantized(q + 2, 1.0, torch.zeros(128))
    with pytest.raises(ValueError, match="ternary"):
        lin.load_quantized(q + 0.5, 1.0, torch.zeros(128))
    with pytest.raises(ValueError, match="weight_scale"):
        lin.load_quantized(q, torch.ones(7), torch.zeros(128))
    with pytest.raises(ValueError, match="bias"):
        lin.load_quantized(q, 1.0)
    with pytest.raises(ValueError, match="bias"):
        bitblas.BitLinear(256, 128).load_quantized(q, 1.0, torch.zeros(128))
    with pytest.raises(TypeError, match="bfloat16"):
        lin(torch.zeros(1, 256, dtype=torch.float16))
    with pytest.raises(ValueError, match=r"\[\.\., 256\]"):
        lin(torch.zeros(1, 128, dtype=torch.bfloat16))


@pytest.mark.parametrize("bias", [False, True])
def test_load_float_weight_matches_absmean_restatement(bias):
    g = torch.Generator().manual_seed(3)
    N, K = 96, 512
    W = torch.randn(N, K, generator=g) * 0.02
    b = torch.randn(N, generator=g) if bias else None
    lin = bitblas.BitLinear(K, N, bias=bias)
    lin.load_float_weight(W, b)
    # BitNet's weight_quant, restated
    sw = 1.0 / W.float().abs().mean().clamp(min=1e-5)
    q = (W.float() * sw).round().clamp(-1, 1)
    assert torch.equal(absmean_ternary(W)[0], q)
    assert torch.equal(lin.weight_scale, sw.expand(N))
    assert set(q.unique().tolist()) == {-1.0, 0.0, 1.0}
    # the int2 storage holds q + 2 in the interleaved-8 layout of the int8 kernels
    op = lin.bitblas_matmul
    assert torch.equal(lin.qweight, op.weight_transform((q + 2).to(torch.int8)))
    if bias:
        assert torch.equal(lin.bias, b.to(torch.float16))
    sd = lin.state_dict()
    assert set(sd) == ({"qweight", "weight_scale", "bias"} if bias else {"qweight", "weight_scale"})
    lin2 = bitblas.BitLinear(K, N, bias=bias)
    lin2.load_state_dict(sd)
    assert torch.equal(lin2.qweight, lin.qweight) and torch.equal(lin2.weight_scale, lin.weight_scale)


def test_load_quantized_per_row_scale_and_per_tensor_scale():
    lin = bitblas.BitLinear(256, 64)
    q = torch.randint(-1, 2, (64, 256), generator=torch.Generator().manual_seed(1))
    s = torch.rand(64, generator=torch.Generator().manual_seed(2)) + 0.5
    lin.load_quantized(q, s)
    assert torch.equal(lin.weight_scale, s)
    lin.load_quantized(q.to(torch.int8), torch.tensor(3.0))
    assert torch.equal(lin.weight_scale, torch.full((64,), 3.0))
    lin.load_quantized(q.float(), 2.5)
    assert torch.equal(lin.weight_scale, torch.full((64,), 2.5))
