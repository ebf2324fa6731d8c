"""CPU: the grouped (mixture-of-experts) matmul's C ABI validation and the checks of Matmul.forward_grouped / GroupedLinear
(no compute calls)."""
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


def _grouped(d, E=8, offsets=0, T=0):
    # fake non-null operand addresses: every call below is refused (or returns) before anything is dereferenced
    return _lib.load().bb_matmul_grouped(ctypes.byref(d), E, offsets, 16, 16, 16, 16, 16, 16, T, 0)


def test_grouped_symbol_exported_and_zero_rows_return():
    lib = _lib.load()
    assert "bb_matmul_grouped" in _lib.EXPORTS and hasattr(lib, "bb_matmul_grouped")
    assert _lib.BB_GROUPED_MAX_GROUPS == 256
    assert _grouped(_desc(), E=8, T=0) == 0
    assert _grouped(_desc(), E=256, T=0) == 0
    assert _grouped(_desc(a_dtype=_lib.BB_BF16, out_dtype=_lib.BB_F32, w_fmt=_lib.BB_W_INT, w_bits=2, with_zeros=0,
                          w_layout=_lib.BB_LAYOUT_COMPRESSED, group_size=-1), E=1, T=0) == 0


@pytest.mark.parametrize("what,kw,E,msg", [
    ("int8 A", dict(a_dtype=_lib.BB_I8, accum_dtype=_lib.BB_I32, out_dtype=_lib.BB_I32, with_scaling=0, with_zeros=0,
                    w_layout=_lib.BB_LAYOUT_INTERLEAVED_8), 8, b"float16 or bfloat16"),
    ("nf4", dict(w_fmt=_lib.BB_W_NF, with_zeros=0, w_layout=_lib.BB_LAYOUT_COMPRESSED), 8, b"uint / int"),
    ("slab tile", dict(w_tile=_lib.BB_TILE_SLAB, K=1024), 8, b"slab-tiled"),
    ("K % 128", dict(K=192, group_size=-1), 8, b"K % 128"),
    ("g = 64", dict(group_size=64), 8, b"group_size"),
    ("no groups", {}, 0, b"num_groups"),
    ("negative groups", {}, -3, b"num_groups"),
    ("too many groups", {}, 257, b"num_groups"),
])
def test_grouped_rejects(what, kw, E, msg):
    assert _grouped(_desc(**kw), E=E, T=4) == 1, what
    assert msg in _lib.last_error().encode(), (what, _lib.last_error())
    assert _grouped(_desc(**kw), E=E, T=0) == 1, what    # the configuration check does not depend on the rows


def test_grouped_rejects_null_offsets():
    assert _grouped(_desc(), E=8, offsets=0, T=4) == 1
    assert "offsets" in _lib.last_error()


def _op(**kw):
    cfg = dict(M=[1, 16], N=256, K=512, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
               with_zeros=True, zeros_mode="quantized")
    cfg.update(kw)
    return bitblas.Matmul(bitblas.MatmulConfig(**cfg), enable_tuning=False)


def _stacked(E=4, N=256, K=512, G=4, bits=4, device="cpu"):
    return dict(W=torch.zeros(E, N, K * bits // 8, dtype=torch.int8, device=device),
                scale=torch.ones(E, N, G, dtype=torch.float16, device=device),
                zeros=torch.zeros(E, G, N * bits // 8, dtype=torch.int8, device=device))


def test_forward_grouped_argument_checks():
    op = _op()
    p = _stacked()
    A = torch.zeros(8, 512, dtype=torch.float16)
    off = torch.tensor([0, 2, 4, 6, 8], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="no CPU path"):
        op.forward_grouped(A, p["W"], off, scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(TypeError, match="int32"):
        op.forward_grouped(A, p["W"], off.long(), scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(ValueError, match="stacked shape"):          # offsets of length E + 2 against W of E groups
        op.forward_grouped(A, p["W"], torch.tensor([0, 2, 4, 6, 8, 8], dtype=torch.int32), scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(ValueError, match="num_groups"):
        op.forward_grouped(A, p["W"], torch.tensor([0], dtype=torch.int32), scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(ValueError, match="num_groups"):
        op.forward_grouped(A, p["W"], torch.zeros(2, 5, dtype=torch.int32), scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(ValueError, match="W has shape"):
        op.forward_grouped(A, p["W"][:, :128], off, scale=p["scale"], zeros=p["zeros"])
    with pytest.raises(ValueError, match="scale has shape"):
        op.forward_grouped(A, p["W"], off, scale=p["scale"][:, :, :2], zeros=p["zeros"])
    with pytest.raises(ValueError, match="zeros has shape"):
        op.forward_grouped(A, p["W"], off, scale=p["scale"], zeros=torch.zeros(4, 256, 4, dtype=torch.float16))
    with pytest.raises(ValueError, match="needs zeros"):
        op.forward_grouped(A, p["W"], off, scale=p["scale"])
    with pytest.raises(NotImplementedError):
        bitblas.Matmul(bitblas.MatmulConfig(M=1, N=16, K=128, A_dtype="float16", W_dtype="float16"),
                       enable_tuning=False).forward_grouped(A, p["W"], off)
    # configurations the grouped kernel does not cover are refused before anything runs
    with pytest.raises(ValueError, match="group_size"):
        _op(group_size=64).check_grouped(4)
    _op().check_grouped(256)
    with pytest.raises(ValueError, match="num_groups"):
        _op().check_grouped(257)


def test_grouped_linear_buffers_and_construction_checks():
    gl = bitblas.GroupedLinear(8, 1024, 512, bias=True, A_dtype="float16", W_dtype="uint4", group_size=128,
                               with_scaling=True, with_zeros=True, zeros_mode="quantized")
    lin = bitblas.Linear(1024, 512, bias=True, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
                         with_zeros=True, zeros_mode="quantized")
    per = {k: (tuple(v.shape), v.dtype) for k, v in lin.state_dict().items()}
    assert {k: (tuple(v.shape), v.dtype) for k, v in gl.state_dict().items()} == {k: ((8, *s), d) for k, (s, d) in per.items()}
    assert gl.bitblas_matmul is lin.bitblas_matmul   # the process-wide operator cache serves both
    g2 = bitblas.GroupedLinear(4, 1024, 512, W_dtype="uint2", group_size=-1, with_scaling=True)
    assert g2.bias is None and tuple(g2.qweight.shape) == (4, 512, 256)
    import bitblas as alias
    assert alias.GroupedLinear is bitblas.GroupedLinear
    for kw in (dict(W_dtype="nf4", with_scaling=True, group_size=128), dict(W_dtype="uint4", with_scaling=True, group_size=64),
               dict(A_dtype="int8", W_dtype="int2", accum_dtype="int32", out_dtype="int32"), dict(W_dtype="float16"),
               dict(W_dtype="uint4", propagate_b=True)):
        with pytest.raises(ValueError):
            bitblas.GroupedLinear(8, 1024, 512, **kw)
    with pytest.raises(ValueError):
        bitblas.GroupedLinear(0, 1024, 512, W_dtype="uint4")
    with pytest.raises(ValueError):
        bitblas.GroupedLinear(300, 1024, 512, W_dtype="uint4")
    with pytest.raises(RuntimeError, match="no CPU path"):
        gl(torch.zeros(4, 1024, dtype=torch.float16), torch.tensor([0, 1, 1, 2, 2, 3, 3, 4, 4], dtype=torch.int32))
    with pytest.raises(ValueError):
        gl(torch.zeros(4, 1024, dtype=torch.float16), torch.tensor([0, 4], dtype=torch.int32))
    with pytest.raises(ValueError, match="E=8"):
        gl.load_and_transform_weight(torch.zeros(4, 512, 1024, dtype=torch.int8))
