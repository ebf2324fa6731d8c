"""CPU: the grouped block-scaled FP8 entry points (bb_matmul_grouped_fp8, bb_matmul_grouped_fp8_swiglu): exports, every rejection
with its code and message in order, total_rows = 0, the block-scale interleave and its agreement with the weight interleave, and
FP8MoEExperts' constructor, buffers and loader checks (no compute calls: every call below is refused, or returns, before the device
is touched)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.fp8_moe import FP8MoEExperts
from bitblas_b200.moe import deinterleave_gate_up, interleave_gate_up

NAMES = ("bb_matmul_grouped_fp8", "bb_matmul_grouped_fp8_swiglu")


def _desc(N=4096, K=7168, out=_lib.BB_BF16, **kw):
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = N, K, _lib.BB_E4M3, _lib.BB_W_FP8_E4M3, 8
    d.accum_dtype, d.out_dtype, d.group_size, d.with_scaling = _lib.BB_F32, out, 128, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return d


# fake non-null, aligned device addresses
def _call(name, d, E=8, offsets=16, A=16, a_scale=16, ld=64, W=16, w_scale=16, C=16, T=64):
    fn = getattr(_lib.load(), name)
    return fn(ctypes.byref(d) if d is not None else None, E, offsets, A, a_scale, ld, W, w_scale, C, T, 0)


def test_exports():
    lib = _lib.load()
    for name in NAMES:
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert bitblas.FP8MoEExperts is FP8MoEExperts
    import bitblas as alias
    assert alias.FP8MoEExperts is FP8MoEExperts


REJECTIONS = [
    (dict(a_dtype=_lib.BB_BF16), {}, 1, "needs e4m3 activations"),
    (dict(w_fmt=_lib.BB_W_FP8_E5M2), {}, 1, "needs e4m3 weights"),
    (dict(accum_dtype=_lib.BB_F16), {}, 1, "accum_dtype must be float32"),
    (dict(out=_lib.BB_I32), {}, 1, "out_dtype must be float16, bfloat16 or float32"),
    (dict(group_size=-1), {}, 1, "group_size must be 128"),
    (dict(with_scaling=0), {}, 1, "needs with_scaling = 1"),
    (dict(with_zeros=1), {}, 1, "zero points are not supported"),
    (dict(w_layout=_lib.BB_LAYOUT_INTERLEAVED_16), {}, 1, "row-major compressed storage"),
    (dict(reserved=(ctypes.c_int32 * 2)(0, 1)), {}, 1, "reserved fields must be zero"),
    (dict(N=568), {}, 1, "N % 16 == 0"),
    (dict(K=7104), {}, 1, "K % 128 == 0"),
    (dict(N=576), {}, 1, "N % 128 == 0"),
    (dict(with_bias=1), {}, 1, "with_bias must be 0"),
    ({}, dict(E=0), 1, "num_groups must be in [1, 256]"),
    ({}, dict(E=257), 1, "num_groups must be in [1, 256]"),
    ({}, dict(T=-1), 1, "total_rows must be >= 0"),
    ({}, dict(T=65, ld=64), 1, "a_scale_ld must be >= total_rows"),
    ({}, dict(T=5, ld=6), 1, "a_scale_ld must be >= total_rows and a multiple of 4"),
    ({}, dict(offsets=0), 1, "offsets must be a device pointer"),
    ({}, dict(A=0), 1, "A, W and C must be non-null"),
    ({}, dict(W=0), 1, "A, W and C must be non-null"),
    ({}, dict(C=0), 1, "A, W and C must be non-null"),
    ({}, dict(a_scale=0), 1, "a_scale must be non-null"),
    ({}, dict(w_scale=0), 1, "w_scale must be non-null"),
    ({}, dict(A=24), 5, "A and W must be 16-byte aligned"),
    ({}, dict(W=8), 5, "A and W must be 16-byte aligned"),
    ({}, dict(a_scale=20), 5, "a_scale must be 16-byte aligned"),
    ({}, dict(w_scale=18), 5, "w_scale and offsets must be 4-byte aligned"),
    ({}, dict(offsets=18), 5, "w_scale and offsets must be 4-byte aligned"),
]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dkw,ckw,code,msg", REJECTIONS, ids=[f"{i}-{r[3][:24]}" for i, r in enumerate(REJECTIONS)])
def test_rejections(name, dkw, ckw, code, msg):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(name, _desc(**dkw), **ckw) == code
    if name.endswith("swiglu") and "N % 128" in msg:
        msg = "2I % 128 == 0"
    assert msg in _lib.last_error()
    assert lib.bb_launch_count() == n0


@pytest.mark.parametrize("name", NAMES)
def test_null_descriptor(name):
    assert _call(name, None) == 1 and "null descriptor" in _lib.last_error()


@pytest.mark.parametrize("name", NAMES)
def test_rejection_order(name):
    """descriptor, N % 128, bias, num_groups, total_rows, then (past total_rows = 0) a_scale_ld, null pointers, alignment, override:
    each call breaks two rules and must report the earlier one"""
    cases = [
        (dict(d=_desc(accum_dtype=_lib.BB_F16, N=576)), "accum_dtype"),
        (dict(d=_desc(N=576, with_bias=1)), "128 == 0"),
        (dict(d=_desc(with_bias=1), E=0), "with_bias"),
        (dict(E=0, T=-1), "num_groups"),
        (dict(T=-1, ld=3), "total_rows must be >= 0"),
        (dict(T=8, ld=4, offsets=0), "a_scale_ld"),
        (dict(offsets=0, A=0), "offsets must be"),
        (dict(A=0, a_scale=0), "A, W and C"),
        (dict(a_scale=0, w_scale=0), "a_scale must be non-null"),
        (dict(w_scale=0, A=8), "w_scale must be non-null"),
        (dict(A=8, a_scale=4), "A and W must be 16-byte aligned"),
        (dict(a_scale=4, w_scale=2), "a_scale must be 16-byte aligned"),
    ]
    for kw, msg in cases:
        d = kw.pop("d", _desc())
        assert _call(name, d, **kw) != 0
        assert msg in _lib.last_error(), (kw, msg, _lib.last_error())


@pytest.mark.parametrize("name", NAMES)
def test_total_rows_zero_launches_nothing(name):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _call(name, _desc(), T=0, offsets=0, A=0, a_scale=0, ld=0, W=0, w_scale=0, C=0) == 0
    assert _call(name, _desc(), E=256, T=0, offsets=0, A=0, a_scale=0, ld=0, W=0, w_scale=0, C=0) == 0
    assert lib.bb_launch_count() == n0


@pytest.mark.parametrize("name", NAMES)
def test_override_refused(name):
    lib = _lib.load()
    try:
        for ov in (_lib.BB_KERNEL_GENERIC, _lib.BB_KERNEL_GEMM_TS, _lib.BB_KERNEL_GEMV_SLAB):
            lib.bb_set_kernel_override(ov)
            assert _call(name, _desc()) == 1 and "does not support this entry" in _lib.last_error()
            assert _call(name, _desc(), T=0) == 0   # validation does not depend on the override
    finally:
        lib.bb_set_kernel_override(_lib.BB_KERNEL_AUTO)


def test_grouped_low_bit_calls_still_reject_e4m3():
    lib = _lib.load()
    d = _desc(N=256, K=1024, out=_lib.BB_F16)
    r = ctypes.byref(d)
    for fn in (lib.bb_matmul_grouped, lib.bb_matmul_grouped_gemm, lib.bb_matmul_grouped_swiglu, lib.bb_matmul_grouped_gemm_swiglu):
        assert fn(r, 1, 16, 16, 16, 16, 0, 0, 16, 1, 0) == 1
        assert "unsupported A_dtype id 5" in _lib.last_error()


# ---- the block-scale interleave ----------------------------------------------------------------------------------------------
def test_block_scale_interleave_round_trip():
    g = torch.Generator().manual_seed(0)
    gate, up = torch.rand(3, 5, 7, generator=g), torch.rand(3, 5, 7, generator=g)
    fused = interleave_gate_up(gate, up, "block_scale")
    assert tuple(fused.shape) == (3, 10, 7)
    assert torch.equal(fused[:, 0::2], gate) and torch.equal(fused[:, 1::2], up)
    g2, u2 = deinterleave_gate_up(fused, "block_scale")
    assert torch.equal(g2, gate) and torch.equal(u2, up)


@pytest.mark.parametrize("I", [128, 192, 768, 2048])
def test_block_scales_follow_the_weight_tiles(I):
    """stored weight tile t (128 rows of the gate/up interleave) holds gate and up rows whose 128-row scale blocks are exactly the
    stored scale rows 2(t >> 1) (gate) and 2(t >> 1) + 1 (up), the rows the kernel reads"""
    H = 256
    nb = -(-I // 128)
    gate_rows = torch.arange(I).view(I, 1).expand(I, H)
    up_rows = gate_rows + 100000
    fused = interleave_gate_up(gate_rows, up_rows, "weight")                      # [2I, H]: each stored row's source row
    gs = torch.arange(nb).view(nb, 1).float().expand(nb, H // 128)                # scale block c of gate holds c
    us = gs + 1000
    fs = interleave_gate_up(gs, us, "block_scale")                                 # [2 nb, H / 128]
    assert tuple(fs.shape) == (2 * nb, H // 128)
    for t in range(2 * I // 128):
        tile = fused[128 * t:128 * (t + 1), 0]
        for r in range(128):
            src = int(tile[r])
            is_gate = (r % 16) < 8
            assert is_gate == (src < 100000)
            row = src if is_gate else src - 100000
            assert 64 * t <= row < 64 * t + 64
            srow = 2 * (t >> 1) + (0 if is_gate else 1)
            assert float(fs[srow, 0]) == (row // 128) + (0 if is_gate else 1000)


# ---- FP8MoEExperts --------------------------------------------------------------------------------------------------------------
def test_experts_buffers_and_state_dict():
    m = FP8MoEExperts(8, 1024, 384)
    sd = m.state_dict()
    assert set(sd) == {"gate_up_weight", "gate_up_weight_scale_inv", "down_weight", "down_weight_scale_inv"}
    assert m.gate_up_weight.dtype == torch.float8_e4m3fn and tuple(m.gate_up_weight.shape) == (8, 768, 1024)
    assert m.gate_up_weight_scale_inv.dtype == torch.float32 and tuple(m.gate_up_weight_scale_inv.shape) == (8, 6, 8)
    assert m.down_weight.dtype == torch.float8_e4m3fn and tuple(m.down_weight.shape) == (8, 1024, 384)
    assert tuple(m.down_weight_scale_inv.shape) == (8, 8, 3)
    g = torch.Generator().manual_seed(1)
    sd = {k: (torch.randn(v.shape, generator=g) * 50).clamp(-448, 448).to(v.dtype) if v.dtype == torch.float8_e4m3fn
          else torch.rand(v.shape, generator=g) for k, v in sd.items()}
    m2 = FP8MoEExperts(8, 1024, 384)
    m2.load_state_dict(sd)
    for k, v in m2.state_dict().items():
        assert torch.equal(v.view(torch.uint8) if v.dtype == torch.float8_e4m3fn else v,
                           sd[k].view(torch.uint8) if v.dtype == torch.float8_e4m3fn else sd[k])


@pytest.mark.parametrize("kw", [dict(hidden_size=1000), dict(intermediate_size=192), dict(intermediate_size=0),
                                dict(A_dtype="float32"), dict(num_experts=0), dict(num_experts=257)])
def test_experts_constructor_rejects(kw):
    args = dict(num_experts=4, hidden_size=1024, intermediate_size=256)
    args.update(kw)
    with pytest.raises(ValueError):
        FP8MoEExperts(**args)


def _ckpt(E, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(E, N, K, generator=g) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)
    s = torch.rand(E, -(-N // 128), K // 128, generator=g) + 0.5
    return w, s


def test_load_fp8_stacked_and_per_expert():
    E, H, I = 4, 512, 256
    gate, up, down = _ckpt(E, I, H, 1), _ckpt(E, I, H, 2), _ckpt(E, H, I, 3)
    a, b = FP8MoEExperts(E, H, I), FP8MoEExperts(E, H, I, A_dtype="float16")
    a.load_fp8(gate, up, down)
    b.load_fp8(*[([w[e] for e in range(E)], [s[e].to(torch.bfloat16) for e in range(E)]) for w, s in (gate, up, down)])
    u8 = torch.uint8
    assert torch.equal(a.gate_up_weight.view(u8), interleave_gate_up(gate[0].view(u8), up[0].view(u8), "weight"))
    assert torch.equal(a.gate_up_weight_scale_inv, interleave_gate_up(gate[1], up[1], "block_scale"))
    assert torch.equal(a.down_weight.view(u8), down[0].view(u8)) and torch.equal(a.down_weight_scale_inv, down[1])
    assert torch.equal(a.gate_up_weight.view(u8), b.gate_up_weight.view(u8))
    assert torch.equal(b.gate_up_weight_scale_inv,
                       interleave_gate_up(gate[1].to(torch.bfloat16).float(), up[1].to(torch.bfloat16).float(), "block_scale"))


def test_load_fp8_validation():
    E, H, I = 4, 512, 256
    gate, up, down = _ckpt(E, I, H, 1), _ckpt(E, I, H, 2), _ckpt(E, H, I, 3)
    m = FP8MoEExperts(E, H, I)
    bad = [
        ((gate[0].float(), gate[1]), up, down, TypeError),               # weight not e4m3
        ((gate[0][:, :128], gate[1]), up, down, ValueError),             # weight shape
        (gate, (up[0], up[1][:, :1]), down, ValueError),                 # scale shape
        (gate, up, (down[0], down[1].to(torch.int32)), TypeError),       # scale dtype
        (gate, up, (down[0][:3], down[1][:3]), ValueError),              # expert count
        (([gate[0][e] for e in range(3)], gate[1]), up, down, ValueError),   # per-expert list of the wrong length
        (gate[0], up, down, TypeError),                                   # not a pair
    ]
    for g_, u_, d_, exc in bad:
        with pytest.raises(exc):
            m.load_fp8(g_, u_, d_)


def test_load_float_weight_validation():
    m = FP8MoEExperts(2, 256, 128)
    with pytest.raises(ValueError):
        m.load_float_weight(torch.randn(2, 128, 256), torch.randn(2, 128, 256), torch.randn(2, 128, 256))
    with pytest.raises(ValueError):
        m.load_float_weight([torch.randn(128, 256)], torch.randn(2, 128, 256), torch.randn(2, 256, 128))
    with pytest.raises(TypeError):
        m.load_float_weight("w", torch.randn(2, 128, 256), torch.randn(2, 256, 128))


def test_load_float_weight_cpu():
    """quantize_weight_blocks per expert, then the interleave (the layer's own device is the CPU here)"""
    from bitblas_b200.fp8 import quantize_weight_blocks
    E, H, I = 2, 256, 128
    g = torch.Generator().manual_seed(4)
    gw, uw, dw = torch.randn(E, I, H, generator=g), torch.randn(E, I, H, generator=g), torch.randn(E, H, I, generator=g)
    m = FP8MoEExperts(E, H, I)
    m.load_float_weight(gw, uw, [dw[e] for e in range(E)])
    for e in range(E):
        qg, sg = quantize_weight_blocks(gw[e])
        qu, su = quantize_weight_blocks(uw[e])
        qd, sd = quantize_weight_blocks(dw[e])
        u8 = torch.uint8
        assert torch.equal(m.gate_up_weight[e].view(u8), interleave_gate_up(qg.view(u8), qu.view(u8), "weight"))
        assert torch.equal(m.gate_up_weight_scale_inv[e], interleave_gate_up(sg, su, "block_scale"))
        assert torch.equal(m.down_weight[e].view(u8), qd.view(u8)) and torch.equal(m.down_weight_scale_inv[e], sd)


def test_matmul_grouped_fp8_checks():
    op = bitblas.Matmul(bitblas.MatmulConfig(N=1024, K=512, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32",
                                             out_dtype="bfloat16"), enable_tuning=False)
    op.check_grouped_fp8(256)
    op.check_grouped_fp8(8, swiglu=True)
    with pytest.raises(ValueError, match="num_groups"):
        op.check_grouped_fp8(257)
    op576 = bitblas.Matmul(bitblas.MatmulConfig(N=576, K=512, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32",
                                                out_dtype="bfloat16"), enable_tuning=False)
    with pytest.raises(ValueError, match="128 == 0"):
        op576.check_grouped_fp8(8)
    with pytest.raises(TypeError):
        op.forward_grouped_fp8(torch.zeros(4, 512, dtype=torch.bfloat16), None, torch.zeros(9, dtype=torch.int32), None, None)
    with pytest.raises(TypeError):
        op.forward_grouped_fp8(torch.zeros(4, 512).to(torch.float8_e4m3fn), None, torch.zeros(9), None, None)
