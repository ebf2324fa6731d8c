"""CPU: the W4A8 entry points (bb_matmul_w4a8, bb_select_kernel_w4a8): exports, every rejection with its message, m = 0, the
kernel-choice rule against a mirror built on dispatch_table's clauses, the workspace rule, and W4A8Linear's construction,
state_dict round trip and host-side loading (no compute calls: every call below is refused, or returns, before the device is
touched)."""
import ctypes
import itertools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import bitblas_b200 as bitblas
import dispatch_table as DT
from bitblas_b200 import _lib
from bitblas_b200.w4a8 import W4A8Linear, pack_zeros


def _desc(N=256, K=1024, fmt=_lib.BB_W_UINT, bits=4, g=128, zeros=1, out=_lib.BB_F16, layout=_lib.BB_LAYOUT_INTERLEAVED_8, **kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = N, K, _lib.BB_I8, fmt, bits
    d.accum_dtype, d.out_dtype, d.group_size, d.w_layout = _lib.BB_I32, out, g, layout
    d.with_scaling, d.with_zeros, d.zeros_mode = 1, zeros, _lib.BB_ZEROS_QUANTIZED
    for k, v in kw.items():
        setattr(d, k, v)
    return d


# fake non-null, aligned device addresses
def _call(d, m=1, A=16, W=16, a_scale=16, scale=16, zeros=16, bias=0, C=16):
    return _lib.load().bb_matmul_w4a8(ctypes.byref(d), A, W, a_scale, scale, zeros, bias, C, m, 0, 0, 0)


def test_exports():
    lib = _lib.load()
    for name in ("bb_matmul_w4a8", "bb_select_kernel_w4a8"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert bitblas.W4A8Linear is W4A8Linear
    import bitblas as alias
    assert alias.W4A8Linear is W4A8Linear


REJECTIONS = [
    (dict(a_dtype=_lib.BB_F16, accum_dtype=_lib.BB_F32), {}, 1, "needs int8 activations"),
    (dict(out=_lib.BB_I32), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    (dict(with_scaling=0, zeros=0), {}, 1, "needs with_scaling = 1"),
    (dict(zeros_mode=_lib.BB_ZEROS_ORIGINAL), {}, 1, "zero points must be BB_ZEROS_QUANTIZED"),
    (dict(zeros_mode=_lib.BB_ZEROS_RESCALE), {}, 1, "zero points must be BB_ZEROS_QUANTIZED"),
    (dict(bits=2), {}, 1, "needs 4-bit uint or int weights"),
    (dict(bits=8, layout=_lib.BB_LAYOUT_COMPRESSED), {}, 1, "needs 4-bit uint or int weights"),
    (dict(fmt=_lib.BB_W_NF, zeros=0), {}, 1, "configuration not supported"),   # validate(): no int8 kernel reads nf4
    (dict(fmt=_lib.BB_W_INT), {}, 1, "int weights take no zero points"),
    ({}, dict(m=-1), 1, "m must be >= 0"),
    ({}, dict(A=0), 1, "A, W and C must be non-null"),
    ({}, dict(a_scale=0), 1, "a_scale must be non-null"),
    ({}, dict(scale=0), 1, "scale must be non-null"),
    ({}, dict(a_scale=18), 5, "must be 4-byte aligned"),
    ({}, dict(scale=18), 5, "must be 4-byte aligned"),
    ({}, dict(zeros=0), 1, "with_zeros is set but zeros is null"),
    (dict(with_bias=1), {}, 1, "with_bias is set but bias is null"),
    (dict(g=100), {}, 1, "not divisible by group_size"),
]


@pytest.mark.parametrize("dkw,ckw,code,msg", REJECTIONS, ids=[f"{i}-{r[3][:24]}" for i, r in enumerate(REJECTIONS)])
def test_rejections(dkw, ckw, code, msg):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(_desc(**dkw), **ckw) == code
    assert msg in _lib.last_error()
    assert lib.bb_launch_count() == n0
    if code == 1 and not ckw and "null" not in msg:   # a descriptor bb_matmul_w4a8 refuses has no kernel
        assert lib.bb_select_kernel_w4a8(ctypes.byref(_desc(**dkw)), 1) == -1


def test_rejection_order():
    """16-bit activations are reported before the output type, the output type before the scales, and so on"""
    _call(_desc(a_dtype=_lib.BB_BF16, accum_dtype=_lib.BB_F32, bits=2, with_scaling=0))
    assert "int8 activations" in _lib.last_error()
    _call(_desc(out=_lib.BB_I8, with_scaling=0, bits=2))
    assert "out_dtype" in _lib.last_error()
    _call(_desc(with_scaling=0, zeros=1, zeros_mode=_lib.BB_ZEROS_ORIGINAL, bits=2))
    assert "with_scaling" in _lib.last_error()
    _call(_desc(zeros_mode=_lib.BB_ZEROS_ORIGINAL, bits=2), m=-1)
    assert "BB_ZEROS_QUANTIZED" in _lib.last_error()


def test_m0_launches_nothing():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(_desc(), m=0, A=0, C=0, a_scale=0, scale=0) == 0
    assert lib.bb_launch_count() == n0


# ---- the kernel-choice rule ----------------------------------------------------------------------------------------------------
def _w4a8_ok(d):
    return ((d.a_dtype == DT.I8) & np.isin(d.out_dtype, (DT.F16, DT.BF16, DT.F32)) & (d.with_scaling != 0)
            & ((d.with_zeros == 0) | (d.zeros_mode == 2)) & (d.w_bits == 4) & np.isin(d.w_fmt, (DT.W_UINT, DT.W_INT))
            & ~((d.with_zeros != 0) & (d.w_fmt == DT.W_INT)))


def _cleared(d):
    return SimpleNamespace(**{**vars(d), "with_scaling": d.with_scaling * 0, "with_zeros": d.with_zeros * 0})


def select_w4a8(d, m, override=DT.AUTO):
    """bb_select_kernel_w4a8: select() of the descriptor without group scales and zeros; gemv_i8 and gemm_ts_i8 become generic
    (under an override: -1) when g % 128 != 0; -1 for a descriptor bb_matmul_w4a8 refuses"""
    k = DT.select(_cleared(d), m, override)
    g = np.where(d.group_size <= 0, d.K, d.group_size)
    fast = np.isin(k, (DT.GEMV_I8, DT.GEMM_TS_I8)) & (g % 128 != 0)
    k = np.where(fast, DT.GENERIC if override == DT.AUTO else -1, k)
    return np.where(_w4a8_ok(d) & (DT.select(d, m) != -1), k, -1)


OVERRIDES = (DT.AUTO, DT.GENERIC, DT.GEMV_MMA, DT.GEMV_I8, DT.GEMM_TS, DT.GEMM_TS_I8, DT.GEMV_SLAB)


def _grid():
    rows = []
    for N, K, g, fmt, zeros, zmode, layout, out, scaling, tile in itertools.product(
            (16, 48, 128, 256, 384), (256, 384, 1024, 1536, 4096), (-1, 32, 64, 128, 192, 256, 384, 512), (DT.W_UINT, DT.W_INT), (0, 1),
            (0, 2), (0, 1, 2), (DT.F16, DT.I32), (0, 1), (0, 1)):
        if g > 0 and K % g:
            continue
        rows.append((N, K, DT.I8, fmt, 4, DT.I32, out, g, scaling, zeros, zmode, 0, layout, tile, 0, 0))
    for bits in (2, 8):
        rows.append((256, 1024, DT.I8, DT.W_UINT, bits, DT.I32, DT.F16, 128, 1, 0, 0, 0, 0, 0, 0, 0))
    rows.append((256, 1024, DT.F16, DT.W_UINT, 4, DT.F32, DT.F16, 128, 1, 1, 2, 0, 1, 0, 0, 0))
    return np.array(rows, dtype=DT.record_dtype())


def test_select_and_workspace_match_mirror():
    """bb_select_kernel_w4a8 against the mirror over a descriptor x m x override grid, and bb_workspace_bytes of the cleared
    descriptor (the workspace bb_matmul_w4a8 takes) against dispatch_table's workspace rule"""
    lib = _lib.load()
    sms = 132   # no device here: the library's fallback count
    ms = (1, 2, 8, 9, 16, 32, 33, 64, 65, 128, 129, 300, 4096)
    rec = _grid()
    d = DT.grid_view(rec)
    structs = [_lib.MatmulDesc(*[int(v) for v in r[:14]], (ctypes.c_int32 * 2)(0, 0)) for r in rec.tolist()]
    cleared = []
    for c in structs:
        cc = _lib.MatmulDesc.from_buffer_copy(c)
        cc.with_scaling = cc.with_zeros = 0
        cleared.append(cc)
    mismatches, checked = [], 0
    prev = lib.bb_set_kernel_override(DT.AUTO)
    try:
        for override in OVERRIDES:
            lib.bb_set_kernel_override(override)
            for m in ms:
                want = select_w4a8(d, m, override)
                ws_want = DT.workspace_bytes(_cleared(d), m, sms)
                for i, c in enumerate(structs):
                    got = lib.bb_select_kernel_w4a8(ctypes.byref(c), m)
                    checked += 1
                    if got != int(want[i]):
                        mismatches.append((rec[i].tolist(), m, override, got, int(want[i])))
                    if override == DT.AUTO and want[i] != -1 and lib.bb_workspace_bytes(ctypes.byref(cleared[i]), m) != ws_want[i]:
                        mismatches.append((rec[i].tolist(), m, "workspace", int(ws_want[i])))
    finally:
        lib.bb_set_kernel_override(prev)
    assert checked > 500000
    assert not mismatches, f"{len(mismatches)} mismatches, first: {mismatches[:5]}"


def test_select_examples():
    lib = _lib.load()
    pick = lambda d, m: _lib.kernel_name(lib.bb_select_kernel_w4a8(ctypes.byref(d), m))
    assert pick(_desc(), 1) == "gemv_i8"
    assert pick(_desc(), 33) == "gemm_ts_wgmma_i8"
    assert pick(_desc(g=64), 1) == "generic_simt"
    assert pick(_desc(g=64), 4096) == "generic_simt"
    assert pick(_desc(layout=_lib.BB_LAYOUT_COMPRESSED), 4) == "gemm_ts_wgmma_i8"
    assert pick(_desc(N=48), 4096) == "generic_simt"
    assert pick(_desc(K=1536, g=384), 4) == "gemv_i8"
    assert pick(_desc(K=1536, g=384), 100) == "gemm_ts_wgmma_i8"
    assert pick(_desc(K=1536, g=512), 100) == "gemm_ts_wgmma_i8"


# ---- the layer --------------------------------------------------------------------------------------------------------------
def test_layer_construction():
    lin = W4A8Linear(1024, 256, bias=True, A_dtype="bfloat16")
    assert tuple(lin.qweight.shape) == (256, 512) and lin.qweight.dtype == torch.int8
    assert tuple(lin.scales.shape) == (256, 8) and lin.scales.dtype == torch.float32
    assert tuple(lin.zeros.shape) == (8, 128) and lin.zeros.dtype == torch.int8
    assert lin.bias.dtype == torch.bfloat16 and lin.perm is None
    assert lin.bitblas_matmul.kernel_for_w4a8(1) == "gemv_i8"
    lin2 = W4A8Linear(512, 128, W_dtype="int4", group_size=-1, with_zeros=False)
    assert lin2.zeros is None and tuple(lin2.scales.shape) == (128, 1)
    for kw, msg in [(dict(A_dtype="int8"), "A_dtype"), (dict(W_dtype="uint2"), "W_dtype"), (dict(W_dtype="int4"), "zero points"),
                    (dict(group_size=100), "group_size"), (dict(in_features=8), "multiples of 16")]:
        args = dict(in_features=256, out_features=128)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            W4A8Linear(**args)


def test_pack_zeros():
    z = torch.randint(0, 16, (64, 3))
    p = pack_zeros(z).view(torch.uint8).to(torch.int32)
    assert tuple(p.shape) == (3, 32)
    for n in range(64):
        for g in range(3):
            assert int((p[g, n // 2] >> (4 * (n % 2))) & 15) == int(z[n, g])


def _loaded(seed=0, bias=True, W_dtype="uint4", zeros=True):
    g = torch.Generator().manual_seed(seed)
    lin = W4A8Linear(512, 64, bias=bias, W_dtype=W_dtype, group_size=128, with_zeros=zeros)
    q = torch.randint(0, 16, (64, 512), generator=g)
    s = torch.rand(64, 4, generator=g) + 0.5
    z = torch.randint(0, 16, (64, 4), generator=g) if zeros else None
    b = torch.randn(64, generator=g) if bias else None
    lin.load_quantized(q, s, z, b)
    return lin, q, s, z, b


def test_load_quantized_and_state_dict_round_trip():
    lin, q, s, z, b = _loaded()
    ref = lin.bitblas_matmul.weight_transform(q.to(torch.int8))
    assert torch.equal(lin.qweight, ref)
    assert torch.equal(lin.scales, s.float())
    assert torch.equal(lin.zeros, pack_zeros(z))
    sd = lin.state_dict()
    assert set(sd) == {"qweight", "scales", "zeros", "bias"}
    other = W4A8Linear(512, 64, bias=True)
    other.load_state_dict(sd)
    for k in sd:
        assert torch.equal(getattr(other, k), sd[k])
    # an act-order layer keeps its perm through the state dict
    sd["perm"] = torch.arange(512, dtype=torch.int32).flip(0)
    third = W4A8Linear(512, 64, bias=True)
    third.load_state_dict(sd)
    assert torch.equal(third.perm, sd["perm"])
    lin4, q4, *_ = _loaded(1, bias=False, W_dtype="int4", zeros=False)
    assert torch.equal(lin4.qweight, lin4.bitblas_matmul.weight_transform(q4.to(torch.int8)))


def test_load_quantized_rejections():
    lin = W4A8Linear(512, 64)
    q = torch.zeros(64, 512, dtype=torch.int32)
    s = torch.ones(64, 4)
    z = torch.zeros(64, 4, dtype=torch.int32)
    with pytest.raises(ValueError, match="q must be"):
        lin.load_quantized(q[:, :256], s, z)
    with pytest.raises(ValueError, match="4-bit values"):
        lin.load_quantized(q + 16, s, z)
    with pytest.raises(ValueError, match="scales must be"):
        lin.load_quantized(q, s[:, :2], z)
    with pytest.raises(ValueError, match="zeros must be given"):
        lin.load_quantized(q, s)
    with pytest.raises(ValueError, match="zeros must hold"):
        lin.load_quantized(q, s, z - 1)
    with pytest.raises(ValueError, match="bias must be given"):
        lin.load_quantized(q, s, z, torch.zeros(64))


def test_gptq_repack_needs_cuda_and_uint4():
    lin = W4A8Linear(512, 64)
    mod = SimpleNamespace(qweight=torch.zeros(64, 64, dtype=torch.int32), qzeros=torch.zeros(4, 8, dtype=torch.int32),
                          scales=torch.ones(4, 64, dtype=torch.float16))
    with pytest.raises(RuntimeError, match="CUDA"):
        lin.repack_from_gptq(mod, device="cpu")
    with pytest.raises(ValueError, match="uint4"):
        W4A8Linear(512, 64, W_dtype="int4", with_zeros=False).repack_from_gptq_v2(mod)


def test_forward_argument_errors():
    lin = W4A8Linear(512, 64)
    with pytest.raises(TypeError, match="float16"):
        lin(torch.zeros(2, 512, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match=r"\[\.\., 512\]"):
        lin(torch.zeros(2, 256, dtype=torch.float16))
    op = bitblas.Matmul(bitblas.MatmulConfig(N=64, K=512, A_dtype="int8", W_dtype="int2", accum_dtype="int32", out_dtype="float16"),
                        enable_tuning=False)
    with pytest.raises(ValueError, match="with_scaling"):
        op.check_w4a8()
    op16 = bitblas.Matmul(bitblas.MatmulConfig(N=64, K=512, A_dtype="float16", W_dtype="uint4", with_scaling=True,
                                               group_size=128), enable_tuning=False)
    with pytest.raises(ValueError, match="int8 activations"):
        op16.check_w4a8()
