"""CPU: the block-scaled FP8 entry points (bb_quantize_act_fp8, bb_matmul_fp8, bb_select_kernel_fp8, bb_workspace_bytes_fp8):
exports, every rejection with its message, m = 0 / rows = 0, that no other entry point accepts e4m3 activations, the kernel
choice, split factor and workspace against a mirror, and FP8Linear's buffers, state_dict loading and load_fp8 checks (no compute
calls: every call below is refused, or returns, before the device is touched)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.fp8 import FP8Linear, quantize_act_fp8


def _desc(N=576, K=7168, out=_lib.BB_BF16, **kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = N, K, _lib.BB_E4M3, _lib.BB_W_FP8_E4M3, 8
    d.accum_dtype, d.out_dtype, d.group_size, d.with_scaling = _lib.BB_F32, out, 128, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return d


# fake non-null, aligned device addresses
def _call(d, m=1, A=16, a_scale=16, ld=4, W=16, w_scale=16, bias=0, C=16):
    return _lib.load().bb_matmul_fp8(ctypes.byref(d) if d is not None else None, A, a_scale, ld, W, w_scale, bias, C, m, 0, 0, 0)


def test_exports():
    lib = _lib.load()
    for name in ("bb_quantize_act_fp8", "bb_matmul_fp8", "bb_select_kernel_fp8", "bb_workspace_bytes_fp8"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert bitblas.FP8Linear is FP8Linear and bitblas.quantize_act_fp8 is quantize_act_fp8
    import bitblas as alias
    assert alias.FP8Linear is FP8Linear
    assert _lib.kernel_name(_lib.BB_KERNEL_GEMM_FP8) == "gemm_fp8_wgmma"


REJECTIONS = [
    (dict(a_dtype=_lib.BB_BF16), {}, 1, "needs e4m3 activations"),
    (dict(a_dtype=_lib.BB_I8), {}, 1, "needs e4m3 activations"),
    (dict(w_fmt=_lib.BB_W_FP8_E5M2), {}, 1, "needs e4m3 weights"),
    (dict(w_bits=4), {}, 1, "needs e4m3 weights"),
    (dict(accum_dtype=_lib.BB_F16), {}, 1, "accum_dtype must be float32"),
    (dict(out=_lib.BB_I32), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    (dict(out=_lib.BB_E4M3), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    (dict(group_size=-1), {}, 1, "group_size must be 128"),
    (dict(group_size=64), {}, 1, "group_size must be 128"),
    (dict(with_scaling=0), {}, 1, "needs with_scaling = 1"),
    (dict(with_zeros=1), {}, 1, "zero points are not supported"),
    (dict(w_layout=_lib.BB_LAYOUT_INTERLEAVED_16), {}, 1, "row-major compressed storage"),
    (dict(w_tile=_lib.BB_TILE_SLAB), {}, 1, "row-major compressed storage"),
    (dict(reserved=(ctypes.c_int32 * 2)(1, 0)), {}, 1, "reserved fields must be zero"),
    (dict(N=568), {}, 1, "N % 16 == 0"),
    (dict(N=0), {}, 1, "N % 16 == 0"),
    (dict(K=7104), {}, 1, "K % 128 == 0"),
    ({}, dict(m=-1), 1, "m must be >= 0"),
    ({}, dict(m=5, ld=4), 1, "a_scale_ld must be >= m"),
    ({}, dict(m=5, ld=10), 1, "a_scale_ld must be >= m and a multiple of 4"),
    ({}, dict(A=0), 1, "A, W and C must be non-null"),
    ({}, dict(W=0), 1, "A, W and C must be non-null"),
    ({}, dict(C=0), 1, "A, W and C must be non-null"),
    ({}, dict(a_scale=0), 1, "a_scale must be non-null"),
    ({}, dict(w_scale=0), 1, "w_scale must be non-null"),
    (dict(with_bias=1), {}, 1, "with_bias is set but bias is null"),
    ({}, dict(A=24), 5, "A and W must be 16-byte aligned"),
    ({}, dict(W=8), 5, "A and W must be 16-byte aligned"),
    ({}, dict(a_scale=20), 5, "a_scale must be 16-byte aligned"),
    ({}, dict(w_scale=18), 5, "w_scale must be 4-byte aligned"),
]


@pytest.mark.parametrize("dkw,ckw,code,msg", REJECTIONS, ids=[f"{i}-{r[3][:24]}" for i, r in enumerate(REJECTIONS)])
def test_rejections(dkw, ckw, code, msg):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(_desc(**dkw), **ckw) == code
    assert msg in _lib.last_error()
    assert lib.bb_launch_count() == n0
    if not ckw and "null" not in msg:   # a descriptor bb_matmul_fp8 refuses has no kernel and no workspace
        assert lib.bb_select_kernel_fp8(ctypes.byref(_desc(**dkw)), 1) == -1
        assert lib.bb_workspace_bytes_fp8(ctypes.byref(_desc(**dkw)), 1) == 0


def test_null_descriptor():
    assert _call(None) == 1 and "null descriptor" in _lib.last_error()


def test_rejection_order():
    """the descriptor before m, m before a_scale_ld, a_scale_ld before null pointers, null pointers before alignment"""
    _call(_desc(accum_dtype=_lib.BB_F16, out=_lib.BB_I32), m=-1)
    assert "accum_dtype" in _lib.last_error()
    _call(_desc(), m=-1, ld=2, A=0)
    assert "m must be >= 0" in _lib.last_error()
    _call(_desc(), m=8, ld=4, A=0)
    assert "a_scale_ld" in _lib.last_error()
    assert _call(_desc(), A=0, W=8) == 1
    assert "non-null" in _lib.last_error()
    assert _call(_desc(), a_scale=0, A=24) == 1


def test_m_zero_launches_nothing():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(_desc(), m=0, A=0, W=0, C=0, a_scale=0, w_scale=0) == 0
    assert lib.bb_launch_count() == n0


def test_override_refused():
    lib = _lib.load()
    try:
        for ov in (_lib.BB_KERNEL_GENERIC, _lib.BB_KERNEL_GEMM_TS, _lib.BB_KERNEL_GEMM_TS_I8, _lib.BB_KERNEL_GEMV_SLAB):
            lib.bb_set_kernel_override(ov)
            assert lib.bb_select_kernel_fp8(ctypes.byref(_desc()), 4) == -1
            assert lib.bb_workspace_bytes_fp8(ctypes.byref(_desc()), 4) == 0
            assert _call(_desc(), m=4) == 1 and "does not support this entry" in _lib.last_error()
        lib.bb_set_kernel_override(_lib.BB_KERNEL_GEMM_FP8)
        assert lib.bb_select_kernel_fp8(ctypes.byref(_desc()), 4) == _lib.BB_KERNEL_GEMM_FP8
    finally:
        lib.bb_set_kernel_override(_lib.BB_KERNEL_AUTO)


def _plain_desc(a_dtype):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 256, 1024, a_dtype, _lib.BB_W_FP8_E4M3, 8
    d.accum_dtype, d.out_dtype, d.group_size, d.with_scaling = _lib.BB_F32, _lib.BB_F16, 128, 1
    return d


def test_other_entry_points_reject_e4m3():
    """a_dtype = BB_E4M3 is refused by every other entry point with validate()'s message, as before it had a name"""
    lib = _lib.load()
    d = _plain_desc(_lib.BB_E4M3)
    r = ctypes.byref(d)
    msg = "unsupported A_dtype id 5"
    calls = [
        lambda: lib.bb_matmul(r, 16, 16, 0, 16, 0, 0, 16, 1, 0, 0, 0),
        lambda: lib.bb_matmul_swiglu(r, 16, 16, 0, 16, 0, 0, 16, 1, 0, 0, 0),
        lambda: lib.bb_matmul_scaled(r, 16, 16, 16, 16, 0, 16, 1, 0, 0, 0),
        lambda: lib.bb_matmul_w4a8(r, 16, 16, 16, 16, 0, 0, 16, 1, 0, 0, 0),
        lambda: lib.bb_matmul_scatter(r, 16, 16, 0, 16, 0, 0, (ctypes.c_void_p * 1)(16), 1, 256, 0, 1, 0, 0, 0),
        lambda: lib.bb_matmul_grouped(r, 1, 16, 16, 16, 16, 0, 0, 16, 1, 0),
        lambda: lib.bb_matmul_grouped_gemm(r, 1, 16, 16, 16, 16, 0, 0, 16, 1, 0),
        lambda: lib.bb_matmul_grouped_swiglu(r, 1, 16, 16, 16, 16, 0, 0, 16, 1, 0),
        lambda: lib.bb_matmul_grouped_gemm_swiglu(r, 1, 16, 16, 16, 16, 0, 0, 16, 1, 0),
        lambda: lib.bb_matmul_grouped_gemm_swiglu_gather(r, 1, 16, 16, 16, 1, 16, 16, 0, 0, 16, 1, 0),
    ]
    n0 = lib.bb_launch_count()
    for c in calls:
        assert c() == 1
        assert msg in _lib.last_error()
    assert lib.bb_select_kernel(r, 1) == -1 and lib.bb_workspace_bytes(r, 1) == 0
    assert lib.bb_select_kernel_w4a8(r, 1) == -1
    assert lib.bb_quantize_act_int8(16, _lib.BB_E4M3, 1, 128, 16, 16, 0) == 1
    assert lib.bb_quantize_act_fp8(16, _lib.BB_E4M3, 1, 128, 16, 16, 4, 0) == 1
    assert lib.bb_launch_count() == n0


# ---- bb_quantize_act_fp8 rejections ------------------------------------------------------------------------------------------
def _quant(x=16, a_dtype=_lib.BB_BF16, rows=1, K=128, q=16, scale=16, ld=4):
    return _lib.load().bb_quantize_act_fp8(x, a_dtype, rows, K, q, scale, ld, 0)


QUANT_REJECTIONS = [
    (dict(a_dtype=_lib.BB_F32), 1, "x must be float16 or bfloat16"),
    (dict(a_dtype=_lib.BB_E4M3), 1, "x must be float16 or bfloat16"),
    (dict(K=0), 1, "K % 128 == 0"),
    (dict(K=136), 1, "K % 128 == 0"),
    (dict(rows=-1), 1, "rows must be >= 0"),
    (dict(rows=5, ld=4), 1, "scale_ld must be >= rows"),
    (dict(rows=3, ld=6), 1, "scale_ld must be >= rows and a multiple of 4"),
    (dict(x=0), 1, "x must be non-null"),
    (dict(q=0), 1, "q must be non-null"),
    (dict(scale=0), 1, "scale must be non-null"),
    (dict(x=8), 5, "x must be 16-byte aligned"),
    (dict(q=4), 5, "q must be 16-byte aligned"),
    (dict(scale=4), 5, "scale must be 16-byte aligned"),
]


@pytest.mark.parametrize("kw,code,msg", QUANT_REJECTIONS, ids=[f"{i}-{r[2][:24]}" for i, r in enumerate(QUANT_REJECTIONS)])
def test_quantize_rejections(kw, code, msg):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _quant(**kw) == code
    assert msg.replace("%%", "%") in _lib.last_error()
    assert lib.bb_launch_count() == n0


def test_quantize_rows_zero():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _quant(rows=0, x=0, q=0, scale=0, ld=0) == 0
    assert lib.bb_launch_count() == n0


def test_quantize_python_checks():
    with pytest.raises(TypeError):
        quantize_act_fp8(torch.zeros(2, 128, dtype=torch.float32))
    with pytest.raises(ValueError):
        quantize_act_fp8(torch.zeros(2, 96, dtype=torch.bfloat16))


# ---- kernel choice, split factor, workspace -------------------------------------------------------------------------------
def fp8_splits(N, K, m, sms):
    """gemm_ts's choose_splits on the FP8 kernel's tiles: BM = 32 / 64 / 128 activation rows, ceil(N / 128) weight tiles"""
    if m > 128:
        return 1
    bm = 32 if m <= 32 else (64 if m <= 64 else 128)
    tiles = -(-m // bm) * -(-N // 128)
    num_kb = K // 128
    if tiles >= sms:
        return 1
    best = 1
    for sp in range(2, 9):
        if num_kb % sp or num_kb // sp < 8:
            continue
        if tiles * sp <= sms:
            best = sp
    return best


def fp8_workspace(N, K, m, sms):
    sp = fp8_splits(N, K, m, sms)
    return sp * m * N * 4 if sp > 1 else 0


SHAPES = [(576, 7168), (1536, 7168), (24576, 1536), (32768, 512), (7168, 16384), (18432, 7168), (7168, 18432), (8192, 8192),
          (10240, 8192), (57344, 8192), (8192, 28672), (256, 1024), (144, 1024), (16, 128), (1040, 2048)]
MS = [1, 2, 4, 8, 16, 31, 32, 33, 64, 65, 100, 128, 129, 512, 4096]


@pytest.mark.parametrize("cap", [0, 132, 114, 78, 16, 1])
def test_choice_splits_and_workspace(cap):
    lib = _lib.load()
    real = 132 if not torch.cuda.is_available() else torch.cuda.get_device_properties(0).multi_processor_count
    if cap > real:
        pytest.skip("cap above this device's SM count")
    lib.bb_set_sm_count_cap(cap)
    try:
        sms = cap or real
        for N, K in SHAPES:
            d = _desc(N=N, K=K)
            for m in MS:
                assert lib.bb_select_kernel_fp8(ctypes.byref(d), m) == _lib.BB_KERNEL_GEMM_FP8
                assert lib.bb_workspace_bytes_fp8(ctypes.byref(d), m) == fp8_workspace(N, K, m, sms), (N, K, m, sms)
        assert lib.bb_select_kernel_fp8(ctypes.byref(_desc()), 0) == -1
    finally:
        lib.bb_set_sm_count_cap(0)


def test_mirror_splits_somewhere():
    """the mirror is not vacuous: the decode shapes split, K = 512 never does"""
    assert fp8_splits(8192, 8192, 1, 132) == 2
    assert fp8_splits(576, 7168, 1, 132) == 7
    assert fp8_splits(32768, 512, 1, 132) == 1
    assert fp8_splits(8192, 8192, 129, 132) == 1


# ---- Matmul trio ------------------------------------------------------------------------------------------------------------
def _op(out="bfloat16", bias=False, N=576, K=7168, A="e4m3_float8", W="e4m3_float8", accum="float32"):
    return bitblas.Matmul(bitblas.MatmulConfig(N=N, K=K, A_dtype=A, W_dtype=W, accum_dtype=accum, out_dtype=out, with_bias=bias),
                          enable_tuning=False)


def test_matmul_check_fp8():
    _op().check_fp8()
    for kw, msg in [(dict(A="float16", W="float16", accum="float32"), "e4m3_float8"),
                    (dict(A="e4m3_float8", W="e5m2_float8"), "e4m3_float8"),
                    (dict(accum="float16"), "accum_dtype"),
                    (dict(out="int32"), "out_dtype"),
                    (dict(N=568), "N % 16"),
                    (dict(K=1000), "K % 128")]:
        with pytest.raises(ValueError, match=msg):
            _op(**kw).check_fp8()
    assert _op().kernel_for_fp8(4) == "gemm_fp8_wgmma"


def test_forward_fp8_checks_before_launch():
    op = _op()
    with pytest.raises(TypeError):
        op.forward_fp8(torch.zeros(4, 7168, dtype=torch.bfloat16), None, None, None)


# ---- FP8Linear --------------------------------------------------------------------------------------------------------------
def test_linear_buffers():
    lin = FP8Linear(7168, 576, bias=True)
    assert lin.weight.dtype == torch.float8_e4m3fn and tuple(lin.weight.shape) == (576, 7168)
    assert lin.weight_scale_inv.dtype == torch.float32 and tuple(lin.weight_scale_inv.shape) == (5, 56)
    assert lin.bias.dtype == torch.bfloat16 and tuple(lin.bias.shape) == (576,)
    assert set(lin.state_dict()) == {"weight", "weight_scale_inv", "bias"}
    lin = FP8Linear(1536, 24576, A_dtype="float16")
    assert lin.bias is None and set(lin.state_dict()) == {"weight", "weight_scale_inv"}
    assert tuple(lin.weight_scale_inv.shape) == (192, 12)
    assert lin.bitblas_matmul.kernel_for_fp8(1) == "gemm_fp8_wgmma"


@pytest.mark.parametrize("kw", [dict(in_features=100, out_features=128), dict(in_features=128, out_features=24),
                                dict(in_features=128, out_features=128, A_dtype="float32")])
def test_linear_rejects(kw):
    with pytest.raises(ValueError):
        FP8Linear(**kw)


def _checkpoint(N, K, bias, seed=0):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = torch.rand((N + 127) // 128, K // 128, generator=g) + 0.5
    sd = {"weight": w, "weight_scale_inv": s}
    if bias:
        sd["bias"] = torch.randn(N, generator=g).to(torch.bfloat16)
    return sd


def test_load_state_dict_checkpoint_names():
    sd = _checkpoint(576, 1024, True)
    lin = FP8Linear(1024, 576, bias=True)
    lin.load_state_dict(sd)
    assert torch.equal(lin.weight.view(torch.uint8), sd["weight"].view(torch.uint8))
    assert torch.equal(lin.weight_scale_inv, sd["weight_scale_inv"]) and torch.equal(lin.bias, sd["bias"])
    with pytest.raises(RuntimeError):
        FP8Linear(1024, 576).load_state_dict(sd)   # unexpected bias


def test_load_fp8_validation():
    sd = _checkpoint(576, 1024, False)
    lin = FP8Linear(1024, 576)
    lin.load_fp8(sd["weight"], sd["weight_scale_inv"].to(torch.bfloat16))
    assert torch.equal(lin.weight_scale_inv, sd["weight_scale_inv"].to(torch.bfloat16).float())
    with pytest.raises(TypeError):
        lin.load_fp8(sd["weight"].float(), sd["weight_scale_inv"])
    with pytest.raises(ValueError):
        lin.load_fp8(sd["weight"][:560], sd["weight_scale_inv"])
    with pytest.raises(ValueError):
        lin.load_fp8(sd["weight"], sd["weight_scale_inv"][:4])
    with pytest.raises(TypeError):
        lin.load_fp8(sd["weight"], sd["weight_scale_inv"].to(torch.int32))
    with pytest.raises(ValueError):
        lin.load_fp8(sd["weight"], sd["weight_scale_inv"], bias=torch.zeros(576))
    with pytest.raises(ValueError):
        FP8Linear(1024, 576, bias=True).load_fp8(sd["weight"], sd["weight_scale_inv"])
    with pytest.raises(ValueError):
        FP8Linear(1024, 576, bias=True).load_fp8(sd["weight"], sd["weight_scale_inv"], bias=torch.zeros(512))


def test_load_float_weight_cpu_rule():
    """the host restatement of the block rule (the layer's own load_float_weight runs the same torch code on its device)"""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(144, 256, generator=g)
    w[:128, :128] = 0   # an all-zero block
    lin = FP8Linear(256, 144)
    lin.load_float_weight(w)
    s = lin.weight_scale_inv
    assert s[0, 0] == torch.tensor(1e-10) / 448
    assert torch.all(lin.weight[:128, :128].float() == 0)
    amax = w[128:, 128:].abs().max()
    assert s[1, 1] == amax / torch.tensor(448.0)
    deq = lin.weight.float() * s.repeat_interleave(128, 0)[:144].repeat_interleave(128, 1)
    assert torch.allclose(deq, w, rtol=2 ** -4, atol=float(s.max()) * 2 ** -10)   # half an e4m3 step, normal or subnormal
