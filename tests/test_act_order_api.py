"""CPU: GPTQ act-order loading helpers (act_order.py), the validation of bb_permute_cols, and the state_dict of act-order layers
(no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.act_order import perm_from_g_idx, permute_cols, permute_gptq_qweight, permute_gptq_rows


# ---- perm_from_g_idx ----------------------------------------------------------------------------------------------------------
def _act_order_g_idx(K, g, seed):
    """how GPTQ builds it: columns quantized in the order `order` go to groups in that order, g_idx[order[i]] = i // g"""
    order = torch.randperm(K, generator=torch.Generator().manual_seed(seed))
    g_idx = torch.empty(K, dtype=torch.int32)
    g_idx[order] = torch.arange(K, dtype=torch.int32) // g
    return g_idx


def test_trivial_g_idx_gives_none():
    assert perm_from_g_idx(torch.arange(512, dtype=torch.int32) // 128, 512, 128) is None
    assert perm_from_g_idx(torch.zeros(512, dtype=torch.int32), 512, 512) is None       # group_size = K: one group
    assert perm_from_g_idx(None, 512, 128) is None


@pytest.mark.parametrize("K,g", [(512, 128), (256, 32), (1024, 1024)])
def test_act_order_g_idx_gives_stable_argsort(K, g):
    g_idx = _act_order_g_idx(K, g, seed=K + g)
    perm = perm_from_g_idx(g_idx, K, g)
    if g == K:
        assert perm is None
        return
    assert perm.dtype == torch.int32 and perm.shape == (K,)
    assert torch.equal(perm.long(), torch.sort(g_idx.long(), stable=True).indices)
    assert torch.equal(g_idx[perm.long()].long(), torch.arange(K) // g)     # sorted column j is in group j // g


def test_rejects_bad_g_idx():
    K, g = 512, 128
    with pytest.raises(ValueError, match="has 511 entries"):
        perm_from_g_idx(torch.zeros(511, dtype=torch.int32), K, g)
    bad = torch.arange(K, dtype=torch.int32) // g
    bad[7] = 4
    with pytest.raises(ValueError, match=r"g_idx\[7\] = 4 names group 4"):
        perm_from_g_idx(bad, K, g)
    bad[7] = -1
    with pytest.raises(ValueError, match="names group -1"):
        perm_from_g_idx(bad, K, g)
    bad[7] = 2                                # group 0 loses a column, group 2 gains one
    with pytest.raises(ValueError, match="group 0 has 127 columns"):
        perm_from_g_idx(bad, K, g)


# ---- GPTQ tensor helpers, against unpack -> index -> pack written out element by element --------------------------------------
def _unpack_rows(q, bits):
    per = 32 // bits
    out = torch.empty((q.shape[0] * per, q.shape[1]), dtype=torch.int64)
    for r in range(out.shape[0]):
        out[r] = (q[r // per].long() >> (bits * (r % per))) & (2**bits - 1)
    return out


def _pack_rows(v, bits):
    per = 32 // bits
    out = torch.zeros((v.shape[0] // per, v.shape[1]), dtype=torch.int64)
    for r in range(v.shape[0]):
        out[r // per] |= v[r] << (bits * (r % per))
    return torch.where(out >= 2**31, out - 2**32, out).to(torch.int32)


def _random_words(shape, seed):
    return torch.randint(-2**31, 2**31, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.int64).to(torch.int32)


@pytest.mark.parametrize("bits", [4, 2])
def test_permute_gptq_qweight(bits):
    K, N = 256, 48
    qw = _random_words((K * bits // 32, N), seed=bits)
    perm = torch.randperm(K, generator=torch.Generator().manual_seed(1)).to(torch.int32)
    got = permute_gptq_qweight(qw, perm, bits)
    assert got.dtype == torch.int32 and got.shape == qw.shape
    assert torch.equal(got, _pack_rows(_unpack_rows(qw, bits)[perm.long()], bits))


@pytest.mark.parametrize("bits", [4, 2])
def test_permute_gptq_rows(bits):
    K, N, g = 256, 64, 64
    per = 32 // bits

    class G:
        pass
    m = G()
    m.qweight = _random_words((K * bits // 32, N), seed=3)
    m.qzeros = _random_words((K // g, N // per), seed=4)
    m.scales = torch.rand((K // g, N), generator=torch.Generator().manual_seed(5)).half()
    m.bias = torch.nn.Parameter(torch.rand(N).half(), requires_grad=False)
    m.g_idx = torch.arange(K, dtype=torch.int32) // g
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(6)).to(torch.int32)
    got = permute_gptq_rows(m, perm, bits)
    p = perm.long()
    assert torch.equal(got.qweight, m.qweight[:, p])
    assert torch.equal(got.scales, m.scales[:, p])
    assert torch.equal(got.bias, m.bias.data[p])
    assert got.g_idx is m.g_idx
    zeros = _unpack_rows(m.qzeros.T.contiguous(), bits).T          # [K/g, N]: qzeros is packed along N
    assert torch.equal(got.qzeros, _pack_rows(zeros[:, p].T.contiguous(), bits).T)
    m.bias = None
    assert permute_gptq_rows(m, perm, bits).bias is None


# ---- bb_permute_cols ----------------------------------------------------------------------------------------------------------
def test_exports_and_argtypes():
    lib = _lib.load()
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    assert "bb_permute_cols" in _lib.EXPORTS and hasattr(lib, "bb_permute_cols")
    # A, out, perm, rows, K, a_dtype, num_groups, offsets, stream
    assert lib.bb_permute_cols.argtypes == [vp, vp, vp, i32, i32, i32, i32, vp, vp]
    assert lib.bb_permute_cols.restype is ctypes.c_int
    assert bitblas.permute_cols is permute_cols


# fake non-null, aligned device addresses: every call below is refused (or returns) before anything is dereferenced
def _call(A=16, out=16, perm=16, rows=4, K=512, dtype=_lib.BB_F16, E=1, offsets=None):
    return _lib.load().bb_permute_cols(A, out, perm, rows, K, dtype, E, offsets, 0)


@pytest.mark.parametrize("what,kw,code,msg", [
    ("fp32 A", dict(dtype=_lib.BB_F32), 1, "float16 or bfloat16"),
    ("int8 A", dict(dtype=_lib.BB_I8), 1, "float16 or bfloat16"),
    ("K = 0", dict(K=0), 1, "K > 0 and K % 8 == 0"),
    ("K % 8", dict(K=516), 1, "K > 0 and K % 8 == 0"),
    ("K too large", dict(K=112648), 1, "exceeds 112640"),
    ("no groups", dict(E=0), 1, "num_groups must be in [1, 256]"),
    ("too many groups", dict(E=257, offsets=16), 1, "num_groups must be in [1, 256]"),
    ("groups without offsets", dict(E=4), 1, "needs offsets"),
    ("rows < 0", dict(rows=-1), 1, "rows must be >= 0"),
    ("null A", dict(A=0), 1, "non-null"),
    ("null out", dict(out=0), 1, "non-null"),
    ("null perm", dict(perm=0), 1, "non-null"),
    ("A misaligned", dict(A=24), 5, "16-byte aligned"),
    ("out misaligned", dict(out=40), 5, "16-byte aligned"),
    ("perm misaligned", dict(perm=18), 5, "4-byte aligned"),
    ("offsets misaligned", dict(E=4, offsets=18), 5, "4-byte aligned"),
])
def test_permute_cols_rejects(what, kw, code, msg):
    assert _call(**kw) == code, what
    assert msg in _lib.last_error(), (what, _lib.last_error())


def test_permute_cols_zero_rows_validates_only():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(A=0, out=0, perm=0, rows=0) == 0
    assert _call(A=0, out=0, perm=0, rows=0, E=256, offsets=16, dtype=_lib.BB_BF16) == 0
    assert lib.bb_launch_count() == n0
    assert _call(rows=0, K=12) == 1                      # still validated
    assert "K % 8" in _lib.last_error()
    assert _call(rows=0, E=2) == 1
    assert "needs offsets" in _lib.last_error()


def test_permute_cols_python_checks():
    A = torch.zeros((4, 64), dtype=torch.float16)
    perm = torch.arange(64, dtype=torch.int32)
    with pytest.raises(TypeError, match="float16 or bfloat16"):
        permute_cols(A.float(), perm)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        permute_cols(A, perm)


# ---- Linear state_dict ----------------------------------------------------------------------------------------------------------
KW = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")


def test_linear_state_dict_without_perm_is_unchanged():
    lin = bitblas.Linear(512, 256, bias=True, **KW)
    assert lin.perm is None
    assert list(lin.state_dict()) == ["qweight", "scales", "zeros", "bias"]
    gl = bitblas.GroupedLinear(4, 512, 256, **KW)
    assert list(gl.state_dict()) == ["qweight", "scales", "zeros"]


def test_linear_state_dict_round_trip_with_perm():
    lin = bitblas.Linear(512, 256, bias=True, **KW)
    gen = torch.Generator().manual_seed(0)
    for name in ("qweight", "zeros"):
        getattr(lin, name).copy_(torch.randint(-128, 128, getattr(lin, name).shape, generator=gen, dtype=torch.int8))
    lin.scales.copy_(torch.rand(lin.scales.shape, generator=gen).half())
    lin.perm = torch.randperm(512, generator=gen).to(torch.int32)
    sd = lin.state_dict()
    assert list(sd) == ["qweight", "scales", "zeros", "bias", "perm"]
    fresh = bitblas.Linear(512, 256, bias=True, **KW)
    fresh.load_state_dict(sd, strict=True)
    for name, t in sd.items():
        assert torch.equal(getattr(fresh, name), t), name
    # and back: a checkpoint without act-order clears the order
    fresh.load_state_dict(bitblas.Linear(512, 256, bias=True, **KW).state_dict(), strict=True)
    assert fresh.perm is None and "perm" not in fresh.state_dict()


def test_grouped_linear_state_dict_round_trip_with_perm():
    gl = bitblas.GroupedLinear(4, 512, 256, **KW)
    gl.perm = torch.stack([torch.randperm(512) for _ in range(4)]).to(torch.int32)
    fresh = bitblas.GroupedLinear(4, 512, 256, **KW)
    fresh.load_state_dict(gl.state_dict(), strict=True)
    assert torch.equal(fresh.perm, gl.perm)
