"""GPU: BitNet b1.58 layers from 16-bit activations, bit for bit.

quantize_act_int8 (bb_quantize_act_int8) against BitNet's activation_quant restated in torch on the CPU; Matmul.forward_scaled
(bb_matmul_scaled) on every int8 kernel family and instance, forced with bb_set_kernel_override, against the exact int32 sum
divided by the two scales in fp32 on the CPU; the production shapes of a 2B BitNet model and the 12288^2 layer under the
dispatcher's own choice; capped SM counts; PDL chains that would expose an early read of the activation scales; and BitLinear
end to end.  The int32 accumulator is exact and every fp32 step is correctly rounded, so every comparison is torch.equal.
"""
import ctypes

import pytest
import torch

import helpers as H
from test_gpu_exact_shapes import _split_shape
from test_gpu_kernel_grid import (K_GEMM_TS_I8, K_GEMV_I8, K_GENERIC, KERNEL_NAME, OUTS, TS_ROWS_FOR_BM, _check_split, _decoded,
                                  forced, make_case, mma_nt, ts_bm, ts_splits)
from test_gpu_moe import _launches
from test_gpu_sm_counts import sm_cap

import bitblas_b200 as bitblas
from bitblas_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = "cuda"
TORCH = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- CPU restatements ------------------------------------------------------------------------------------------------------------
def quant_ref(x):
    """BitNet's activation_quant on the CPU: (q int8, scale float32 [rows]); torch evaluates `127.0 / t` as t.reciprocal() * 127"""
    xf = x.cpu().float().reshape(-1, x.shape[-1])
    s = 127.0 / xf.abs().amax(-1, keepdim=True).clamp(min=1e-5)
    q = (xf * s).round().clamp(-128, 127).to(torch.int8)
    return q, s.reshape(-1)


def exact_acc(q, w):
    """the int32 sum q [m, K] x w [N, K]^T on the CPU.  In fp32 it is exact: every partial sum is an integer below 2^24"""
    assert q.shape[1] * 128 * int(w.abs().max()) < 2 ** 24
    return q.float() @ w.float().T


def scaled_ref(acc, s_a, s_w, out, bias=None):
    """round_out((float(acc) / s_a) / s_w) (+ bias in out_dtype), fp32 on the CPU"""
    y = (acc.float() / s_a.cpu().reshape(-1, 1)) / s_w.cpu().reshape(1, -1)
    if out == "float32":
        return y + bias.cpu() if bias is not None else y
    r = y.to(TORCH[out])
    return r + bias.cpu() if bias is not None else r


def _equal(got, ref, what):
    got = got.cpu()
    if not torch.equal(got, ref):
        bad = (got.double() != ref.double()) & ~(got.double().isnan() & ref.double().isnan())
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements differ; first at {idx}: "
                             f"got {[got[tuple(i)].item() for i in idx]} ref {[ref[tuple(i)].item() for i in idx]}")


# ---- quantization ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("K", [2560, 6912, 12288, 65536])
@pytest.mark.parametrize("rows", [1, 7, 128, 4096])
def test_quantize_matches_activation_quant(rows, K, dtype):
    g = torch.Generator().manual_seed(rows * 131 + K)
    mag = torch.exp2(torch.randint(-6, 7, (rows, 1), generator=g).float())   # a different absmax per row
    x = (torch.randn(rows, K, generator=g) * mag).to(TORCH[dtype])
    q, s = bitblas.quantize_act_int8(x.to(DEV))
    torch.cuda.synchronize()
    qr, sr = quant_ref(x)
    _equal(s, sr, f"scale rows={rows} K={K} {dtype}")
    _equal(q, qr, f"q rows={rows} K={K} {dtype}")
    assert q.shape == x.shape and q.dtype == torch.int8 and s.shape == (rows,) and s.dtype == torch.float32


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_quantize_edge_rows(dtype):
    """an all-zero row, one large outlier, the maximum at either sign and at both, a row below the 1e-5 clamp, and dyadic rows
    that land exactly on .5 after scaling (round half to even)"""
    K = 2560
    dt = TORCH[dtype]
    g = torch.Generator().manual_seed(5)
    base = (torch.rand(K, generator=g) - 0.5)
    rows = [torch.zeros(K)]
    r = base.clone(); r[1234] = 1000.0; rows.append(r)                  # one outlier
    r = base.clone(); r[7] = -3.0; rows.append(r)                       # maximum negative
    r = base.clone(); r[9] = 3.0; r[2000] = -3.0; rows.append(r)        # maximum at both signs
    rows.append(torch.full((K,), 2.0 ** -20))                           # amax below the clamp
    halves = torch.arange(K) % 16 - 8 + 0.5                             # -7.5 .. 7.5
    r = halves.clone(); r[0] = 127.0; rows.append(r)                    # scale 1: x itself is on .5
    r = halves / 2; r[0] = 63.5; rows.append(r)                         # scale 2: x * 2 is on .5 again
    x = torch.stack(rows).to(dt)
    q, s = bitblas.quantize_act_int8(x.to(DEV))
    torch.cuda.synchronize()
    qr, sr = quant_ref(x)
    _equal(s, sr, f"edge scales {dtype}")
    _equal(q, qr, f"edge q {dtype}")
    q, s = q.cpu(), s.cpu()
    assert s[0] == 127.0 / torch.tensor(1e-5) and not q[0].any()
    assert q[1, 1234] == 127 and q[2, 7] == -127 and q[3, 9] == 127 and q[3, 2000] == -127
    assert s[5] == 1.0 and s[6] == 2.0
    expect = torch.tensor([-8, -6, -6, -4, -4, -2, -2, 0, 0, 2, 2, 4, 4, 6, 6, 8])   # rint(k + 0.5), k = -8 .. 7, half to even
    assert torch.equal(q[5, 16:32].long(), expect) and torch.equal(q[6, 16:32].long(), expect)


def test_quantize_rows_with_inf_and_nan_do_not_disturb_the_others():
    """the values of a row holding Inf or NaN are unspecified; the call completes and every other row is exact"""
    g = torch.Generator().manual_seed(9)
    x = torch.randn(5, 4096, generator=g).to(torch.float16)
    x[1, 17] = float("inf")
    x[3, 100] = float("nan")
    q, s = bitblas.quantize_act_int8(x.to(DEV))
    torch.cuda.synchronize()
    qr, sr = quant_ref(x)
    for r in (0, 2, 4):
        _equal(q[r], qr[r], f"row {r}")
        _equal(s[r], sr[r], f"scale {r}")


def test_quantize_output_buffers_and_3d():
    x = torch.randn(2, 3, 1024, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16)
    q = torch.full((2, 3, 1024), 99, dtype=torch.int8, device=DEV)
    s = torch.zeros(6, dtype=torch.float32, device=DEV)
    q2, s2 = bitblas.quantize_act_int8(x.to(DEV), q=q, scale=s)
    assert q2 is q and s2 is s
    qr, sr = quant_ref(x)
    _equal(q.reshape(6, 1024), qr, "q out")
    _equal(s, sr, "scale out")
    _, n = _launches(lambda: bitblas.quantize_act_int8(x.to(DEV), q=q, scale=s))
    assert n == 1


# ---- the scaled matmul on every int8 kernel instance -----------------------------------------------------------------------------
def scaled_case(m, N, K, W, il, out, bias, per_row, seed, a_range=128):
    """make_case's int8 inputs with out_dtype `out`, fp32 a_scale [m] and w_scale [N] (N copies of one value unless per_row) and
    a bias [N] in out_dtype"""
    case = make_case(m, N, K, A_dtype="int8", W_dtype=W, out_dtype="int32", fast_decoding=il, seed=seed, a_range=a_range)
    case["cfg"] = dict(case["cfg"], out_dtype=out, with_bias=bias)
    g = torch.Generator().manual_seed(seed + 1)
    case["a_scale"] = torch.rand(m, generator=g) * 100 + 20
    case["w_scale"] = (torch.rand(N if per_row else 1, generator=g) * 4 + 1).expand(N).contiguous()
    case["obias"] = ((torch.rand(N, generator=g) - 0.5) * 8).to(TORCH[out]) if bias else None
    return case


def case_ref(case, rows=None):
    A = case["A"] if rows is None else case["A"][rows]
    acc = exact_acc(A, _decoded(case))
    s_a = case["a_scale"] if rows is None else case["a_scale"][rows]
    return scaled_ref(acc, s_a, case["w_scale"], case["cfg"]["out_dtype"], case["obias"])


def _dev(case):
    b = case["obias"]
    return (case["A"].to(DEV), case["a_scale"].to(DEV), case["w_scale"].to(DEV), None if b is None else b.to(DEV))


def run_scaled(case, kernel_id, m=None):
    """forward_scaled of the case (kernel_id: forced, asserted through kernel_for; None: the dispatcher's choice); (op, W, output)"""
    m = case["M"] if m is None else m
    op = H.product_operator(case, M=[1, m])
    W = H.product_weight(op, case, DEV)
    A, sa, sw, b = _dev(case)
    if kernel_id is None:
        got = op.forward_scaled(A, W, sa, sw, b)
    else:
        with forced(kernel_id):
            assert op.kernel_for(m) == KERNEL_NAME[kernel_id], (op.kernel_for(m), case["cfg"])
            got = op.forward_scaled(A, W, sa, sw, b)
    torch.cuda.synchronize()
    return op, W, got


def _id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


# gemv_i8: NT = 1 (m <= 8, the dispatcher's range), 2 and 4 (m <= 32, the fallback), 2- and 4-bit, signed and unsigned
GEMV_CELLS = [dict(m=m, W=("int" if m % 3 else "uint") + str((2, 4)[m % 2]), out=OUTS[m % 3], bias=m % 2 == 0, per_row=m % 4 < 2)
              for m in range(1, 33)]


@pytest.mark.parametrize("c", GEMV_CELLS, ids=[_id(c) for c in GEMV_CELLS])
def test_gemv_i8_scaled(c):
    case = scaled_case(c["m"], 256, 1024, c["W"], True, c["out"], c["bias"], c["per_row"], seed=c["m"] * 17)
    assert mma_nt(c["m"]) in (1, 2, 4)
    _, _, got = run_scaled(case, K_GEMV_I8)
    _equal(got, case_ref(case), f"gemv_i8 {c}")


# gemm_ts_wgmma_i8: bits x storage x BM x split-K, each with an output type, bias and scale kind
TS_CELLS = []
for _i, (_bits, _il, _bm, _split) in enumerate([(b, il, bm, sp) for b in (2, 4) for il in (True, False) for bm in (32, 64, 128)
                                                for sp in (True, False)]):
    _rows = TS_ROWS_FOR_BM[_bm]
    TS_CELLS.append(dict(W=("int" if _i % 2 else "uint") + str(_bits), il=_il, bm=_bm, split=_split, m=_rows[_i % len(_rows)],
                         out=OUTS[_i % 3], bias=_i % 4 < 2, per_row=_i % 3 != 0))


@pytest.mark.parametrize("c", TS_CELLS, ids=[_id(c) for c in TS_CELLS])
def test_gemm_ts_i8_scaled(c):
    assert ts_bm(c["m"]) == c["bm"]
    K = 2048 if c["split"] else 1024   # 16 / 8 k-blocks of 128
    case = scaled_case(c["m"], 256, K, c["W"], c["il"], c["out"], c["bias"], c["per_row"], seed=len(_id(c)) * 31 + c["m"])
    op, _, got = run_scaled(case, K_GEMM_TS_I8)
    assert op._desc.w_layout == (_lib.BB_LAYOUT_INTERLEAVED_8 if c["il"] else _lib.BB_LAYOUT_COMPRESSED)
    with forced(K_GEMM_TS_I8):
        _check_split(op, c["m"], c["split"] and c["m"] <= 128, 128)
    _equal(got, case_ref(case), f"gemm_ts_i8 {c}")


# every split-K factor f: K = 1024 f gives 8 f k-blocks of 128, which split f ways while the 2 tiles leave SMs idle
SPLITS = [(2, 16), (3, 40), (4, 100), (5, 128), (6, 20), (7, 60), (8, 127)]


@pytest.mark.parametrize("f,m", SPLITS, ids=[f"split{f}-m{m}" for f, m in SPLITS])
def test_gemm_ts_i8_every_split_factor_and_no_workspace(f, m):
    """the split output (factor read from bb_workspace_bytes) and the same call through the C ABI without a workspace (no split) are
    both exact, hence bit-identical"""
    out = OUTS[f % 3]
    case = scaled_case(m, 256, 1024 * f, "int2", f % 2 == 0, out, f % 2 == 1, f % 3 != 0, seed=f * 101 + m)
    assert ts_splits(m, 256, 1024 * f, 128, _sms()) == f
    op, W, got = run_scaled(case, K_GEMM_TS_I8)
    ref = case_ref(case)
    _equal(got, ref, f"split {f}")
    lib = _lib.load()
    A, sa, sw, b = _dev(case)
    C = torch.empty((m, 256), dtype=TORCH[out], device=DEV)
    with forced(K_GEMM_TS_I8):
        _check_split(op, m, True, 128)
        _, n = _launches(lambda: _lib.check(lib.bb_matmul_scaled(ctypes.byref(op._desc), A.data_ptr(), W.data_ptr(), sa.data_ptr(),
                                                                 sw.data_ptr(), 0 if b is None else b.data_ptr(), C.data_ptr(), m,
                                                                 None, 0, None), "bb_matmul_scaled"))
    assert n == 1   # no workspace: no split, no reduce launch
    _equal(C, ref, f"unsplit {f}")


# generic_simt: 1-bit weights, K % 128 != 0, N % 16 != 0 and the 4-bit formats, at several m
GENERIC_CELLS = [dict(W=W, K=K, m=m, out=OUTS[i % 3], bias=i % 2 == 0, per_row=i % 4 < 2, il=i % 2 == 1)
                 for i, (W, K, m) in enumerate([(W, K, m) for W, K in (("uint1", 768), ("int1", 544), ("int2", 272), ("uint4", 1024),
                                                                        ("int4", 400))
                                                for m in (1, 5, 40)])]


@pytest.mark.parametrize("c", GENERIC_CELLS, ids=[_id(c) for c in GENERIC_CELLS])
def test_generic_scaled(c):
    il = c["il"] and c["W"] not in ("uint4", "int4")   # the int8 kernels' 4-bit storage is compressed
    case = scaled_case(c["m"], 72, c["K"], c["W"], il, c["out"], c["bias"], c["per_row"], seed=c["K"] + c["m"])
    _, _, got = run_scaled(case, K_GENERIC)
    _equal(got, case_ref(case), f"generic {c}")


def test_generic_only_desc_dispatches_to_generic():
    """K % 128 != 0 and N % 16 != 0: the dispatcher's own choice is the generic kernel for every m"""
    for m in (1, 9, 200):
        case = scaled_case(m, 72, 272, "int2", True, "float16", True, True, seed=m)
        op, _, got = run_scaled(case, None, m)
        assert op.kernel_for(m) == "generic_simt"
        _equal(got, case_ref(case), f"auto generic m={m}")


# ---- production shapes -----------------------------------------------------------------------------------------------------------
# (N, K): the linears of a 2B BitNet b1.58 model (hidden 2560, intermediate 6912: q/o, k/v, gate/up, down) and 12288^2
PROD = [(2560, 2560), (640, 2560), (6912, 2560), (2560, 6912), (12288, 12288)]


def _ternary_layer(N, K, bias, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randint(-1, 2, (N, K), generator=g, dtype=torch.int8)
    sw = torch.rand(N, generator=g) * 2 + 0.5
    b = ((torch.rand(N, generator=g) - 0.5) * 4).to(TORCH[dtype]) if bias else None
    lin = bitblas.BitLinear(K, N, bias=bias, A_dtype=dtype).to(DEV)
    lin.load_quantized(w, sw, b)
    return lin, w, sw, b


def layer_ref(x, w, sw, b, dtype):
    q, s = quant_ref(x)
    return scaled_ref(exact_acc(q, w), s, sw, dtype, b)


@pytest.mark.parametrize("N,K", PROD, ids=[f"{n}x{k}" for n, k in PROD])
def test_production_shapes(N, K):
    lin, w, sw, b = _ternary_layer(N, K, N == 640, "float16", N + K)
    x = torch.randn(4096, K, generator=torch.Generator().manual_seed(K)).to(torch.float16)
    ref = layer_ref(x, w, sw, b, "float16")
    xd = x.to(DEV)
    for m in (1, 16, 128, 4096):
        assert lin.bitblas_matmul.kernel_for(m) == ("gemv_i8" if m <= 8 else "gemm_ts_wgmma_i8"), m
        got = lin(xd[:m])
        torch.cuda.synchronize()
        _equal(got, ref[:m], f"{N}x{K} m={m}")


# ---- capped SM counts ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 8, 33, 66, 114])
def test_scaled_at_sm_caps(cap):
    """gemv_i8's K split (pick_ks) and every wgmma split-K factor at `cap` SMs: each output exact, hence bit-identical across caps"""
    if cap > _sms():
        pytest.skip(f"{cap} SMs is above this device's {_sms()}")
    with sm_cap(cap):
        for m in (1, 12):
            case = scaled_case(m, 2048, 8192, "int2", True, "float16", m == 1, True, seed=m + cap)
            _, _, got = run_scaled(case, K_GEMV_I8)
            _equal(got, case_ref(case), f"gemv_i8 m={m} on {cap} SMs")
        for f in range(2, 9) if cap >= 8 else ():   # on fewer SMs no shape splits 8 ways at 16 rows
            N, K, _ = _split_shape(f, 16, 128, cap)
            case = scaled_case(16, N, K, "int2", True, OUTS[(f + cap) % 3], f % 2 == 0, True, seed=f * 7 + cap)
            op, _, got = run_scaled(case, K_GEMM_TS_I8)
            with forced(K_GEMM_TS_I8):
                _check_split(op, 16, True, 128, sms=cap)
            _equal(got, case_ref(case), f"gemm_ts_i8 split {f} ({N}x{K}) on {cap} SMs")


# ---- PDL: the matmul reads a_scale only after the quantization that wrote it has completed -----------------------------------------
def _chain_inputs(steps, m, K, seed):
    """activations whose absmax changes from step to step by a power of two: a scale read early would be off by that factor"""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(m, K, generator=g) * 2.0 ** ((i * 3) % 7 - 3)).to(torch.float16) for i in range(steps)]


@pytest.mark.parametrize("m", [1, 16, 200])
def test_pdl_chain_reads_each_calls_scales(m):
    """quantize -> scaled matmul, 12 times back to back on one stream without synchronisation, every quantization into the SAME
    q and scale buffers: each output must be exact for its own activations"""
    N, K = 2560, 2560
    lin, w, sw, _ = _ternary_layer(N, K, False, "float16", 77)
    xs = _chain_inputs(12, m, K, m)
    xd = [x.to(DEV) for x in xs]
    qbuf = torch.empty((m, K), dtype=torch.int8, device=DEV)
    sbuf = torch.empty(m, dtype=torch.float32, device=DEV)
    op = lin.bitblas_matmul
    torch.cuda.synchronize()
    outs = []
    for x in xd:
        q, s = bitblas.quantize_act_int8(x, q=qbuf, scale=sbuf)
        outs.append(op.forward_scaled(q, lin.qweight, s, lin.weight_scale))
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(xs, outs)):
        _equal(y, layer_ref(x, w, sw, None, "float16"), f"step {i} m={m}")


def test_pdl_chain_captured_replay():
    """the same chain (m = 1 and m = 16 interleaved) captured once and replayed with new activations"""
    N, K = 2560, 2560
    lin, w, sw, _ = _ternary_layer(N, K, False, "float16", 78)
    op = lin.bitblas_matmul
    rows = [1, 16, 1, 16, 1, 16]
    x_d = [torch.zeros((m, K), dtype=torch.float16, device=DEV) for m in rows]
    y_d = [torch.empty((m, N), dtype=torch.float16, device=DEV) for m in rows]
    q_d = [torch.empty((m, K), dtype=torch.int8, device=DEV) for m in (1, 16)]
    s_d = [torch.empty(m, dtype=torch.float32, device=DEV) for m in (1, 16)]

    def chain():
        for i, m in enumerate(rows):
            j = 0 if m == 1 else 1
            q, s = bitblas.quantize_act_int8(x_d[i], q=q_d[j], scale=s_d[j])
            op.forward_scaled(q, lin.qweight, s, lin.weight_scale, output=y_d[i])

    step = bitblas.CapturedStep(chain)
    for trial in range(3):
        xs = [x[0] for x in (_chain_inputs(1, m, K, 1000 * trial + i) for i, m in enumerate(rows))]
        for d, x in zip(x_d, xs):
            d.copy_(x)
        step()
        for i, x in enumerate(xs):
            _equal(y_d[i], layer_ref(x, w, sw, None, "float16"), f"replay {trial} step {i}")


# ---- BitLinear -------------------------------------------------------------------------------------------------------------------
def torch_composition(lin, x):
    """the integration's glue around the int32 matmul: activation_quant, Matmul.forward with int32 output, / s_a / s_w, cast, bias"""
    xf = x.float()
    s = 127.0 / xf.abs().amax(-1, keepdim=True).clamp(min=1e-5)
    q = (xf * s).round().clamp(-128, 127).to(torch.int8)
    op32 = bitblas.Matmul(bitblas.MatmulConfig(N=lin.out_features, K=lin.in_features, A_dtype="int8", W_dtype="int2",
                                               accum_dtype="int32", out_dtype="int32"), enable_tuning=False)
    acc = op32.forward(q, lin.qweight)
    y = (acc.float() / s / lin.weight_scale).to(x.dtype)
    return y + lin.bias if lin.bias is not None else y


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("m", [1, 5, 16, 300])
def test_bitlinear_matches_torch_composition(m, bias, dtype):
    lin, w, sw, b = _ternary_layer(640, 2560, bias, dtype, m + 3 * bias)
    x = torch.randn(m, 2560, generator=torch.Generator().manual_seed(m)).to(TORCH[dtype]).to(DEV)
    got = lin(x)
    _equal(got, torch_composition(lin, x).cpu(), f"BitLinear m={m} bias={bias} {dtype}")
    _equal(got, layer_ref(x.cpu(), w, sw, b, dtype), f"BitLinear vs restatement m={m}")


def test_load_float_weight_matches_absmean_on_device():
    W = (torch.randn(640, 2560, generator=torch.Generator().manual_seed(4)) * 0.03).to(DEV)
    lin = bitblas.BitLinear(2560, 640).to(DEV)
    lin.load_float_weight(W)
    sw = 1.0 / W.float().abs().mean().clamp(min=1e-5)
    q = (W.float() * sw).round().clamp(-1, 1)
    assert torch.equal(lin.weight_scale, sw.expand(640))
    assert torch.equal(lin.qweight, lin.bitblas_matmul.weight_transform((q + 2).to(torch.int8)))
    x = torch.randn(3, 2560, generator=torch.Generator().manual_seed(5)).to(torch.float16)
    _equal(lin(x.to(DEV)), layer_ref(x, q.cpu(), sw.cpu().expand(640), None, "float16"), "float-loaded layer")


def test_bitlinear_3d_bf16_and_launch_counts():
    lin, w, sw, b = _ternary_layer(256, 4096, True, "bfloat16", 6)
    x = torch.randn(2, 3, 4096, generator=torch.Generator().manual_seed(6)).to(torch.bfloat16).to(DEV)
    y, n = _launches(lambda: lin(x))
    assert y.shape == (2, 3, 256) and y.dtype == torch.bfloat16 and n == 2   # m = 6: gemv_i8
    _equal(y.reshape(6, 256), layer_ref(x.reshape(6, 4096).cpu(), w, sw, b, "bfloat16"), "3-D")
    x16 = torch.randn(16, 4096, generator=torch.Generator().manual_seed(7)).to(torch.bfloat16).to(DEV)
    f = ts_splits(16, 256, 4096, 128, _sms())
    assert f > 1
    y, n = _launches(lambda: lin(x16))
    assert n == 3   # quantization, the split wgmma GEMM, its reduce
    _equal(y, layer_ref(x16.cpu(), w, sw, b, "bfloat16"), "split-K layer")


def test_bitlinear_graph_replay_and_state_dict():
    lin, w, sw, b = _ternary_layer(2560, 2560, True, "float16", 8)
    x_d = torch.zeros((4, 2560), dtype=torch.float16, device=DEV)
    y_d = torch.empty((4, 2560), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: lin(x_d, output=y_d))
    for trial in range(3):
        x = torch.randn(4, 2560, generator=torch.Generator().manual_seed(trial)).to(torch.float16)
        x_d.copy_(x)
        step()
        _equal(y_d, layer_ref(x, w, sw, b, "float16"), f"replay {trial}")
        eager = lin(x.to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(eager, y_d)
    lin2 = bitblas.BitLinear(2560, 2560, bias=True).to(DEV)
    lin2.load_state_dict(lin.state_dict())
    assert torch.equal(lin2(x_d), y_d)
