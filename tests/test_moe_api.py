"""CPU: the mixture-of-experts block's C ABI validation (bb_moe_route, bb_moe_combine, the SwiGLU grouped calls), the gate/up
interleave against its definition, and MoEExperts construction (no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.moe import deinterleave_gate_up, interleave_gate_up

NEW = ["bb_moe_route", "bb_moe_combine", "bb_matmul_grouped_swiglu", "bb_matmul_grouped_gemm_swiglu"]
CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")


def test_exports_and_argtypes():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name), name
        assert getattr(lib, name).restype is ctypes.c_int
    assert len(lib.bb_moe_route.argtypes) == 11 and len(lib.bb_moe_combine.argtypes) == 9
    assert lib.bb_matmul_grouped_swiglu.argtypes == lib.bb_matmul_grouped.argtypes
    assert lib.bb_matmul_grouped_gemm_swiglu.argtypes == lib.bb_matmul_grouped_gemm.argtypes


# fake non-null, aligned device addresses: every call below is refused (or returns) before anything is dereferenced
def _route(T=4, k=2, E=8, a_dtype=_lib.BB_F16, K=256):
    return _lib.load().bb_moe_route(16, T, k, E, 16, a_dtype, K, 16, 16, 16, 0)


def _combine(T=4, k=2, out=_lib.BB_F16, N=256):
    return _lib.load().bb_moe_combine(16, 16, 16, out, 16, T, k, N, 0)


@pytest.mark.parametrize("what,kw,msg", [
    ("E = 0", dict(E=0), "num_experts"), ("E = 257", dict(E=257), "num_experts"), ("top_k = 0", dict(k=0), "top_k"),
    ("K % 8", dict(K=260), "K % 8"), ("int8 x", dict(a_dtype=_lib.BB_I8), "float16 or bfloat16"),
    ("T * k >= 2^31", dict(T=1 << 28, k=8), "2^31"), ("T < 0", dict(T=-1), "num_tokens"),
])
def test_route_rejects(what, kw, msg):
    assert _route(**kw) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())
    assert _route(**dict(kw, T=0 if "T" not in kw else kw["T"])) == 1, what   # the checks do not depend on the tokens


def test_route_and_combine_zero_tokens_return_without_launch():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert lib.bb_moe_route(0, 0, 8, 256, 0, _lib.BB_BF16, 2048, 0, 0, 0, 0) == 0
    assert lib.bb_moe_combine(0, 0, 0, _lib.BB_F32, 0, 0, 8, 2048, 0) == 0
    assert lib.bb_launch_count() == n0


def test_route_rejects_null_and_unaligned():
    assert _lib.load().bb_moe_route(16, 4, 2, 8, 0, _lib.BB_F16, 256, 16, 16, 16, 0) == 1
    assert "non-null" in _lib.last_error()
    assert _lib.load().bb_moe_route(16, 4, 2, 8, 24, _lib.BB_F16, 256, 16, 16, 16, 0) == 5
    assert "aligned" in _lib.last_error()


@pytest.mark.parametrize("what,kw,msg", [
    ("top_k = 0", dict(k=0), "top_k"), ("N % 8", dict(N=260), "N % 8"), ("int8 out", dict(out=_lib.BB_I8), "out_dtype"),
    ("T * k >= 2^31", dict(T=1 << 30, k=2), "2^31"),
])
def test_combine_rejects(what, kw, msg):
    assert _combine(**kw) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def _desc(**kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 256, 512, _lib.BB_F16, _lib.BB_W_UINT, 4
    d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.BB_F16, 128
    d.with_scaling, d.with_zeros, d.zeros_mode = 1, 1, _lib.BB_ZEROS_QUANTIZED
    d.w_layout = _lib.BB_LAYOUT_INTERLEAVED_16
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _swiglu(name, d, E=8, T=0, offsets=16):
    return getattr(_lib.load(), name)(ctypes.byref(d), E, offsets, 16, 16, 16, 16, 16, 16, T, 0)


@pytest.mark.parametrize("name", ["bb_matmul_grouped_swiglu", "bb_matmul_grouped_gemm_swiglu"])
def test_swiglu_calls_validate_without_launch(name):
    n0 = _lib.load().bb_launch_count()
    assert _swiglu(name, _desc(), E=8, T=0) == 0
    assert _swiglu(name, _desc(N=512, a_dtype=_lib.BB_BF16, out_dtype=_lib.BB_F32, with_bias=1), E=256, T=0) == 0
    assert _lib.load().bb_launch_count() == n0


@pytest.mark.parametrize("name", ["bb_matmul_grouped_swiglu", "bb_matmul_grouped_gemm_swiglu"])
@pytest.mark.parametrize("what,kw,E,msg", [
    ("I % 8", dict(N=2 * 108), 8, "I % 8"),
    ("int8 A", dict(a_dtype=_lib.BB_I8, accum_dtype=_lib.BB_I32, out_dtype=_lib.BB_I32, with_scaling=0, with_zeros=0,
                    w_layout=_lib.BB_LAYOUT_INTERLEAVED_8), 8, "float16 or bfloat16"),
    ("too many groups", {}, 257, "num_groups"),
])
def test_swiglu_rejects(name, what, kw, E, msg):
    assert _swiglu(name, _desc(**kw), E=E, T=4) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def test_swiglu_gemm_needs_2i_multiple_of_128():
    assert _swiglu("bb_matmul_grouped_swiglu", _desc(N=144), T=0) == 0       # I = 72: the GEMV form covers it
    assert _swiglu("bb_matmul_grouped_gemm_swiglu", _desc(N=144), T=0) == 1
    assert "N % 128" in _lib.last_error()


# ---- gate/up interleave -------------------------------------------------------------------------------------------------------
def _stored_row(n):
    """stored row n of the interleave -> ("gate" | "up", source row), from the definition"""
    b, i = divmod(n, 16)
    return ("gate", 8 * b + i) if i < 8 else ("up", 8 * b + i - 8)


@pytest.mark.parametrize("kind,shape", [("weight", (3, 48, 64)), ("scale", (3, 48, 4)), ("zeros", (2, 48, 5)),
                                        ("bias", (3, 48)), ("weight", (24, 7))])
def test_interleave_rows_match_the_definition(kind, shape):
    g = torch.Generator().manual_seed(len(shape) * 100 + shape[-1])
    gate = torch.randint(-100, 100, shape, generator=g).to(torch.int16)
    up = torch.randint(-100, 100, shape, generator=g).to(torch.int16)
    fused = interleave_gate_up(gate, up, kind)
    dim = -1 if kind == "bias" else -2
    I = shape[dim]
    assert fused.shape[dim] == 2 * I
    for n in range(2 * I):
        which, src = _stored_row(n)
        ref = (gate if which == "gate" else up).select(dim, src)
        assert torch.equal(fused.select(dim, n), ref), (kind, n)
    g2, u2 = deinterleave_gate_up(fused, kind)
    assert torch.equal(g2, gate) and torch.equal(u2, up)


@pytest.mark.parametrize("bits", [4, 2])
def test_interleave_packed_quantized_zeros(bits):
    """quantized zeros [E, G, I*bits/8] packed along the rows: the unpacked zero point of stored row n is that of its source row"""
    E, G, I = 2, 3, 40
    epb = 8 // bits
    g = torch.Generator().manual_seed(bits)
    zg = torch.randint(0, 2 ** bits, (E, G, I), generator=g)
    zu = torch.randint(0, 2 ** bits, (E, G, I), generator=g)

    def pack(z):   # element n of a row in bits (n % epb) of byte n // epb (general_compress along the last axis)
        z = z.reshape(*z.shape[:-1], -1, epb)
        return sum(z[..., j] << (bits * j) for j in range(epb)).to(torch.uint8).view(torch.int8)

    def unpack(p):
        u = p.view(torch.uint8).to(torch.int64)
        return torch.stack([(u >> (bits * j)) & (2 ** bits - 1) for j in range(epb)], dim=-1).reshape(*p.shape[:-1], -1)

    fused = interleave_gate_up(pack(zg), pack(zu), "qzeros", bits)
    assert fused.shape == (E, G, 2 * I * bits // 8) and fused.dtype == torch.int8
    zf = unpack(fused)
    for n in range(2 * I):
        which, src = _stored_row(n)
        assert torch.equal(zf[..., n], (zg if which == "gate" else zu)[..., src]), n
    g2, u2 = deinterleave_gate_up(fused, "qzeros", bits)
    assert torch.equal(g2, pack(zg)) and torch.equal(u2, pack(zu))


def test_interleave_rejects():
    with pytest.raises(ValueError, match="multiple of 8"):
        interleave_gate_up(torch.zeros(12, 4), torch.zeros(12, 4), "weight")
    with pytest.raises(ValueError, match="same shape"):
        interleave_gate_up(torch.zeros(16, 4), torch.zeros(8, 4), "weight")
    with pytest.raises(ValueError, match="kind"):
        interleave_gate_up(torch.zeros(16, 4), torch.zeros(16, 4), "rows")
    with pytest.raises(ValueError, match="bits"):
        interleave_gate_up(torch.zeros(2, 8, dtype=torch.int8), torch.zeros(2, 8, dtype=torch.int8), "qzeros")


# ---- MoEExperts ---------------------------------------------------------------------------------------------------------------
def test_moe_experts_builds_both_projections():
    m = bitblas.MoEExperts(8, 512, 384, **CFG)
    assert m.gate_up.qweight.shape == (8, 768, 512 // 2) and m.down.qweight.shape == (8, 512, 384 // 2)
    assert m.gate_up.bias is None and m.down.bias is None


@pytest.mark.parametrize("args,kw,err,msg", [
    ((8, 512, 100), CFG, ValueError, "multiple of 8"),
    ((8, 512, 208), dict(CFG, group_size=-1), ValueError, "K % 128"),      # down: K = I = 208
    ((0, 512, 384), CFG, ValueError, "num_groups"),
    ((257, 512, 384), CFG, ValueError, "num_groups"),
    ((8, 512, 384), dict(CFG, out_dtype="float32"), ValueError, "out_dtype == A_dtype"),
    ((8, 512, 384), dict(CFG, W_dtype="nf4", with_zeros=False), ValueError, "uint / int"),
])
def test_moe_experts_rejects(args, kw, err, msg):
    with pytest.raises(err, match=msg):
        bitblas.MoEExperts(*args, **kw)
