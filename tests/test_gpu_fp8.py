"""GPU: block-scaled FP8 (bb_quantize_act_fp8, bb_matmul_fp8, FP8Linear).

  * quantization bit for bit against the torch restatement of the rule (include/bitblas_b200.h), edge values included, and
    every finite float16 and bfloat16 encoding as a block's amax and beneath nine others;
  * the GEMM bit for bit on exactly representable inputs: every BM instance, split and unsplit (asserted), every output type,
    with and without bias, N % 128 != 0, K = 128 and 512, at capped SM counts;
  * the GEMM bit for bit on exact block sums with inexact scales against the header's fp32 order (fp8_restate): every BM
    instance, every output type, with and without bias, a_scale_ld > m, every split factor 2 .. 8 and the unsplit C call;
  * random inputs against float64 with a per-element bound (the accumulation assumption is stated at ACC_REL);
  * determinism, graph replay, launch counts and a PDL chain through reused buffers;
  * FP8Linear end to end and its float-weight loader.
"""
import ctypes

import pytest
import torch

from bitblas_b200 import _lib
from bitblas_b200.fp8 import FP8Linear, quantize_act_fp8, quantize_weight_blocks
import fp8_restate as R
from fp8_restate import OUT, round_out
from test_fp8_api import fp8_splits

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
# How the tensor core sums the 128 products of one k-block is not specified.  Measured on an H100 (tools/fp8_accum_probe.py,
# DESIGN.md §3.2.6): each k32 step aligns its 32 products and the running sum to the largest of them and drops what lies more
# than 13 binades below it.  So each of the 4 steps loses less than 33 * 2^-13 of a value no larger than sum_k |a_k w_k|, and the
# assumption is |P - exact| <= ACC_REL * sum_k |a_k w_k| with ACC_REL = 4 * 33 * 2^-13 < 2^-5.9.
ACC_REL = 4 * 33 * 2.0 ** -13


def quant_ref(x):
    """the torch restatement of bb_quantize_act_fp8: (q float8 [rows, K], s float32 [rows, K / 128]); torch.to(e4m3) alone
    turns values above 464 into NaN, so the clamp is part of the rule"""
    rows, K = x.shape
    xf = x.float().view(rows, K // 128, 128)
    amax = xf.abs().amax(-1).clamp(min=1e-10)
    s = amax / torch.full_like(amax, 448.0)   # a tensor divisor: torch turns division by a Python scalar into a reciprocal product
    q = (xf / s[..., None]).clamp(-448.0, 448.0).to(E4M3)
    return q.view(rows, K), s


def _bytes(q):
    return q.view(torch.uint8)


def _check_quant(x):
    q, s = quantize_act_fp8(x)
    qr, sr = quant_ref(x)
    assert torch.equal(_bytes(q), _bytes(qr))
    assert torch.equal(s, sr)
    assert s.stride(0) == 1 or s.shape[0] == 1


QUANT_SHAPES = [(1, 128), (1, 28672), (3, 256), (17, 7168), (64, 1536), (129, 512), (1000, 2048), (4096, 7168), (4096, 128),
                (2, 28672), (4096, 28672)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("rows,K", QUANT_SHAPES, ids=lambda v: str(v))
def test_quant_random(rows, K, dtype):
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + K)
    x = (torch.randn(rows, K, device="cuda", generator=g) * torch.rand(rows, 1, device="cuda", generator=g) * 50).to(dtype)
    _check_quant(x)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
def test_quant_edges(dtype):
    """an all-zero block, quotients exactly on 448 and just past it before the clamp, round-half-to-even ties, e4m3 subnormals"""
    K = 1024
    x = torch.zeros(6, K, dtype=torch.float32)
    # row 0: block 0 all zero, block 1 one tiny value, the rest random
    x[0, 128] = 1e-3
    x[0, 256:] = torch.randn(K - 256)
    # row 1: amax 448 so s = 1 exactly: ties of the e4m3 grid (1.0625 -> 1, 1.1875 -> 1.25, 17 -> 16, 19 -> 20, 304 -> 288 ...)
    ties = torch.tensor([448.0, 1.0625, 1.1875, -1.0625, 17.0, 19.0, -19.0, 304.0, 336.0, 0.5 + 1 / 32, 3.0 / 1024])
    x[1, :ties.numel()] = ties
    # row 2: e4m3 subnormals at s = 1: multiples of 2^-9 and the ties between them
    sub = torch.tensor([448.0] + [k * 2.0 ** -10 for k in range(1, 16)] + [-(2.0 ** -10), 2.0 ** -11])
    x[2, 128:128 + sub.numel()] = sub
    # rows 3-5: amax values whose quotient rounds to just above / below 448 before the clamp
    for r, a in ((3, 1000.0), (4, 3.14159), (5, 0.1)):
        for b in range(K // 128):
            blk = torch.linspace(-a, a, 128) * (1 + b / 7)
            x[r, b * 128:(b + 1) * 128] = blk
    xd = x.to(dtype).cuda()
    _check_quant(xd)
    q, s = quantize_act_fp8(xd)
    assert torch.all(_bytes(q)[0, :128] == 0) and s[0, 0] == torch.tensor(1e-10, dtype=torch.float32) / 448
    qf = q.float()
    assert qf.abs().max() <= 448 and not torch.isnan(qf).any()


def _every_finite(dtype):
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    return v[torch.isfinite(v)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
def test_quant_every_encoding(dtype):
    """every finite bit pattern of the input type, once as its block's amax (with 127 smaller values of either sign beside it)
    and once as a smaller element of blocks whose amax is 448 * 2^j (the scale a power of two: quotients land exactly on every
    e4m3 value, the ties between them and the subnormals), 1, 0.1, 1000, the type's largest and smallest normal value and, in
    bfloat16, amax values below the 1e-10 floor -- byte for byte against the CPU restatement"""
    g = torch.Generator().manual_seed(5)
    v = _every_finite(dtype)
    # 1. each value as the amax of its block, at a position that moves with the value
    frac = torch.rand(127, generator=g) * 2 - 1
    blk = torch.cat([v[:, None], (v.float()[:, None] * frac[None, :]).to(dtype)], 1)
    shift = (torch.arange(128)[None, :] + torch.arange(v.numel())[:, None]) % 128
    blocks = [torch.gather(blk, 1, shift)]
    assert torch.equal(blocks[0].float().abs().amax(1), v.float().abs())
    # 2. each value under larger amax values
    fi = torch.finfo(dtype)
    amaxes = [448.0 * 2.0 ** j for j in (-24, -8, 0, 7)] + [1.0, 0.1, 1000.0, fi.max, fi.tiny]
    if dtype == torch.bfloat16:
        amaxes += [448.0 * 2.0 ** 100, 448.0 * 2.0 ** -120, 1e-12]
    for a in torch.tensor(amaxes).to(dtype):
        x = v[v.float().abs() <= a.float()]
        x = torch.cat([x, torch.zeros((-x.numel()) % 127, dtype=dtype)]).view(-1, 127)
        blocks.append(torch.cat([a.expand(x.shape[0], 1), x], 1))
    blocks = torch.cat(blocks)
    blocks = torch.cat([blocks, torch.zeros((-blocks.shape[0]) % 64, 128, dtype=dtype)])
    x = blocks.view(-1, 64 * 128)
    q, s = quantize_act_fp8(x.cuda())
    qr, sr = quant_ref(x)
    bad = (_bytes(q).cpu() != _bytes(qr)).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} bytes differ, first at {bad[:4].tolist()}: x = {x[tuple(bad[0])].item()!r}"
    assert torch.equal(s.cpu(), sr)
    assert torch.equal(torch.unique(_bytes(qr)), torch.tensor([b for b in range(256) if b & 0x7f != 0x7f], dtype=torch.uint8))


def test_quant_scale_ld_and_pdl_order():
    """scale_ld > rows through the C entry: the gap between the rows' scales is not written"""
    lib = _lib.load()
    rows, K, ld = 5, 512, 12
    x = torch.randn(rows, K, device="cuda").to(torch.bfloat16)
    q = torch.empty(rows, K, dtype=torch.uint8, device="cuda")
    buf = torch.full((K // 128, ld), -7.0, device="cuda")
    n0 = lib.bb_launch_count()
    rc = lib.bb_quantize_act_fp8(x.data_ptr(), _lib.BB_BF16, rows, K, q.data_ptr(), buf.data_ptr(), ld,
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0 and lib.bb_launch_count() == n0 + 1
    torch.cuda.synchronize()
    qr, sr = quant_ref(x)
    assert torch.equal(q, _bytes(qr)) and torch.equal(buf[:, :rows].t(), sr)
    assert torch.all(buf[:, rows:] == -7.0)


# ---- the GEMM on exact inputs ------------------------------------------------------------------------------------------------
def exact_case(m, N, K, seed):
    """e4m3 operands in {0, +-1/2, +-1, +-2} (activations) and {0, +-1/2, +-1} (weights), power-of-two scales 2^-2 .. 2^2: every
    product is a multiple of 2^-2, a block sum is at most 256 in magnitude (exact in any fp32 order, even with 14 kept bits), each
    promoted term a multiple of 2^-6, and the whole sum stays below 2^17 -- S is exact and only the output rounding remains"""
    g = torch.Generator().manual_seed(seed)
    av = torch.tensor([0.0, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0])
    wv = torch.tensor([0.0, 0.5, -0.5, 1.0, -1.0])
    qa = av[torch.randint(0, av.numel(), (m, K), generator=g)]
    qw = wv[torch.randint(0, wv.numel(), (N, K), generator=g)]
    KB = K // 128
    sa = 2.0 ** torch.randint(-2, 3, (m, KB), generator=g).float()
    sw = 2.0 ** torch.randint(-2, 3, ((N + 127) // 128, KB), generator=g).float()
    return qa, qw, sa, sw


def exact_S(qa, qw, sa, sw):
    """S in float64 (exact for exact_case's inputs)"""
    m, K = qa.shape
    N = qw.shape[0]
    KB = K // 128
    P = torch.einsum("mbk,nbk->mnb", qa.double().view(m, KB, 128), qw.double().view(N, KB, 128))
    swn = sw.double().repeat_interleave(128, 0)[:N]          # [N, KB]
    terms = P * sa.double()[:, None, :] * swn[None, :, :]
    assert float(terms.abs().sum(-1).max()) < 2.0 ** 17      # every fp32 partial sum of S is a multiple of 2^-6 below 2^17
    return terms.sum(-1)


def _dev(qa, qw, sa, sw):
    A = qa.to(E4M3).cuda()
    W = qw.to(E4M3).cuda()
    m, KB = sa.shape
    ld = (m + 3) // 4 * 4
    buf = torch.zeros(KB, ld)
    buf[:, :m] = sa.t()
    a_scale = buf.cuda().t()[:m]
    return A, W, a_scale, sw.cuda().contiguous()


def _op(N, K, out, bias):
    from bitblas_b200 import Matmul, MatmulConfig
    return Matmul(MatmulConfig(N=N, K=K, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32", out_dtype=out,
                               with_bias=bias), enable_tuning=False)


def _run_counted(op, A, W, a_scale, w_scale, bias):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    y = op.forward_fp8(A, W, a_scale, w_scale, bias)
    torch.cuda.synchronize()
    return y, lib.bb_launch_count() - n0


EXACT = []
for m in (1, 20, 32, 40, 64, 100, 128, 300):            # BM 32, 64 and 128, one or several m tiles
    for N, K in ((576, 2048), (144, 512), (1040, 128), (256, 4096)):
        EXACT.append((m, N, K))


@pytest.mark.parametrize("out", ["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("m,N,K", EXACT, ids=lambda v: str(v))
def test_exact(m, N, K, out):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for bias in (False, True):
        qa, qw, sa, sw = exact_case(m, N, K, seed=m * 31 + N + K)
        A, W, a_scale, w_scale = _dev(qa, qw, sa, sw)
        b = (torch.randn(N) * 4).to(OUT[out]).cuda() if bias else None
        op = _op(N, K, out, bias)
        y, launches = _run_counted(op, A, W, a_scale, w_scale, b)
        sp = fp8_splits(N, K, m, sms)
        assert launches == (2 if sp > 1 else 1)
        ref = round_out(exact_S(qa, qw, sa, sw).cuda(), out, b)
        assert torch.equal(y, ref)


@pytest.mark.parametrize("cap", [114, 78, 16, 1])
def test_exact_capped(cap):
    """split factors of smaller parts, asserted through the launch count, bit for bit"""
    lib = _lib.load()
    prev = lib.bb_set_sm_count_cap(cap)
    try:
        for m, N, K in ((1, 576, 7168), (4, 1536, 2048), (16, 256, 4096), (33, 1040, 2048), (128, 144, 1024), (200, 576, 512)):
            qa, qw, sa, sw = exact_case(m, N, K, seed=cap + m)
            A, W, a_scale, w_scale = _dev(qa, qw, sa, sw)
            op = _op(N, K, "bfloat16", False)
            y, launches = _run_counted(op, A, W, a_scale, w_scale, None)
            assert launches == (2 if fp8_splits(N, K, m, cap) > 1 else 1)
            assert torch.equal(y, round_out(exact_S(qa, qw, sa, sw).cuda(), "bfloat16", None))
    finally:
        lib.bb_set_sm_count_cap(prev)


def test_split_and_unsplit_forced():
    """the same exact problem with a workspace (split 7 ways at 132 SMs) and without one (unsplit): identical bits"""
    m, N, K = 2, 576, 7168
    qa, qw, sa, sw = exact_case(m, N, K, seed=5)
    A, W, a_scale, w_scale = _dev(qa, qw, sa, sw)
    op = _op(N, K, "float32", False)
    lib = _lib.load()
    y_split, n_split = _run_counted(op, A, W, a_scale, w_scale, None)
    y = torch.empty_like(y_split)
    n0 = lib.bb_launch_count()
    rc = lib.bb_matmul_fp8(ctypes.byref(op._fp8_desc()), A.data_ptr(), a_scale.data_ptr(), a_scale.stride(1), W.data_ptr(),
                           w_scale.data_ptr(), 0, y.data_ptr(), m, 0, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0 and lib.bb_launch_count() - n0 == 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert n_split == (2 if fp8_splits(N, K, m, sms) > 1 else 1)
    assert torch.equal(y, y_split) and torch.equal(y, exact_S(qa, qw, sa, sw).float().cuda())


# ---- inexact scales: the header's fp32 order, bit for bit (fp8_restate) ----------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("m,N,K", R.FP8_CASES, ids=lambda v: str(v))
def test_inexact_scales_restated(m, N, K):
    """integer operands (the block sums exact) with inexact scales, so the promotion, block order, split reduce and output
    rounding decide every bit: every output type, with and without a bias, the latter with a_scale_ld > m and NaN in the gap"""
    qa, qw, sa, sw = R.fp8_case(m, N, K)
    sp = fp8_splits(N, K, m, _sms())
    S = R.restate(qa.cuda(), qw.cuda(), sa.cuda(), sw.cuda(), sp)
    A, W, w_scale = qa.to(E4M3).cuda(), qw.to(E4M3).cuda(), sw.cuda()
    for out in OUT:
        for bias in (False, True):
            b = R.bias_for(N, out, m + N).cuda() if bias else None
            a_scale = R.a_scale_view(sa, 8 if bias else 0, "cuda")
            y, launches = _run_counted(_op(N, K, out, bias), A, W, a_scale, w_scale, b)
            assert launches == (2 if sp > 1 else 1)
            assert torch.equal(y, round_out(S, out, b)), (out, bias, int((y != round_out(S, out, b)).sum()))


@pytest.mark.parametrize("f,m,N,K,cap", R.SPLIT_CASES, ids=lambda v: str(v))
def test_split_factors_restated(f, m, N, K, cap):
    """every split factor 2 .. 8, asserted through bb_workspace_bytes_fp8, against the restated per-split sums and ordered
    reduce; the same call through the C ABI without a workspace runs unsplit and matches the unsplit restatement"""
    lib = _lib.load()
    cap = cap or 132
    if cap > _sms():
        pytest.skip("the split factors are those of 132 SMs")
    qa, qw, sa, sw = R.split_case(f, m, N, K, cap)
    P, swn = R.block_sums(qa.cuda(), qw.cuda()), R.scale_rows(sw.cuda(), N)
    R.prove_exact(qa, qw)
    S_split, S_one = R.promote(P, sa.cuda(), swn, f), R.promote(P, sa.cuda(), swn, 1)
    A, W, w_scale = qa.to(E4M3).cuda(), qw.to(E4M3).cuda(), sw.cuda()
    a_scale = R.a_scale_view(sa, 4, "cuda")
    stream = torch.cuda.current_stream().cuda_stream
    prev = lib.bb_set_sm_count_cap(cap)
    try:
        for out in OUT:
            for bias in (False, True):
                op = _op(N, K, out, bias)
                assert lib.bb_workspace_bytes_fp8(ctypes.byref(op._fp8_desc()), m) == f * m * N * 4
                b = R.bias_for(N, out, f).cuda() if bias else None
                y, launches = _run_counted(op, A, W, a_scale, w_scale, b)
                assert launches == 2 and torch.equal(y, round_out(S_split, out, b)), (out, bias)
                y1 = torch.empty_like(y)
                n0 = lib.bb_launch_count()
                rc = lib.bb_matmul_fp8(ctypes.byref(op._fp8_desc()), A.data_ptr(), a_scale.data_ptr(), a_scale.stride(1),
                                       W.data_ptr(), w_scale.data_ptr(), b.data_ptr() if bias else 0, y1.data_ptr(), m, 0, 0,
                                       stream)
                torch.cuda.synchronize()
                assert rc == 0 and lib.bb_launch_count() - n0 == 1
                assert torch.equal(y1, round_out(S_one, out, b)), (out, bias)
                if out == "float32":
                    assert not torch.equal(y, y1)   # the split order shows in the bits
    finally:
        lib.bb_set_sm_count_cap(prev)


# ---- random inputs against float64 ---------------------------------------------------------------------------------------------
LLAMA70B = [(10240, 8192), (8192, 8192), (57344, 8192), (8192, 28672)]
DEEPSEEK = [(1536, 7168), (24576, 1536), (576, 7168), (32768, 512), (7168, 16384), (18432, 7168), (7168, 18432)]


def float64_bound(A, a_scale, W, w_scale, y, out):
    """(reference S in float64, per-element bound): the block sums within ACC_REL of exact, fp32 promotion (KB + 1 roundings of
    at most 2^-24 of the running magnitude), then one rounding to the output type"""
    m, K = A.shape
    N = W.shape[0]
    KB = K // 128
    swn = w_scale.double().repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)     # [N, K]
    sak = a_scale.double().repeat_interleave(128, 1)                                   # [m, K]
    Ad, Wd = A.double() * sak, W.double() * swn
    ref = Ad @ Wd.t()
    T = Ad.abs() @ Wd.abs().t()
    ulp = {"float16": 2.0 ** -11, "bfloat16": 2.0 ** -8, "float32": 2.0 ** -24}[out]
    err = T * (ACC_REL + (KB + 1) * 2.0 ** -24)
    return ref, err + ulp * (ref.abs() + err) + 1e-30


@pytest.mark.parametrize("m", [1, 4, 16, 128, 1024, 4096])
@pytest.mark.parametrize("N,K", LLAMA70B + DEEPSEEK, ids=lambda v: str(v))
def test_random_float64(N, K, m):
    torch.manual_seed(N + K + m)
    x = torch.randn(m, K, device="cuda").to(torch.bfloat16)
    A, a_scale = quantize_act_fp8(x)
    w = torch.randn(N, K, device="cuda") * 0.02
    W, w_scale = quantize_weight_blocks(w)
    op = _op(N, K, "bfloat16", False)
    y = op.forward_fp8(A, W, a_scale, w_scale)
    ref, bound = float64_bound(A, a_scale, W, w_scale, y, "bfloat16")
    err = (y.double() - ref).abs()
    assert bool((err <= bound).all()), f"max excess {(err - bound).max().item():.3g}"


# ---- determinism, graphs, launch counts, PDL chain --------------------------------------------------------------------------
def _layer(K, N, bias, seed):
    torch.manual_seed(seed)
    lin = FP8Linear(K, N, bias=bias).cuda()
    lin.load_float_weight(torch.randn(N, K, device="cuda") * 0.05, torch.randn(N, device="cuda") if bias else None)
    return lin


@pytest.mark.parametrize("m", [1, 4, 100, 512])
def test_repeat_graph_and_launches(m):
    lin = _layer(2048, 576, True, m)
    lib = _lib.load()
    x = torch.randn(m, 2048, device="cuda").to(torch.bfloat16)
    n0 = lib.bb_launch_count()
    a = lin(x)
    torch.cuda.synchronize()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert lib.bb_launch_count() - n0 == (3 if fp8_splits(576, 2048, m, sms) > 1 else 2)
    b = lin(x)
    out = torch.empty_like(a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lin(x, output=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lin(x, output=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, out)


def test_pdl_chain_reused_buffers():
    """four layer calls through one layer's workspace and two ping-pong outputs, eager and replayed, against separate calls with
    synchronisation in between"""
    K = 2048
    lin = _layer(K, K, True, 0)
    for m in (1, 4, 64, 300):
        x = torch.randn(m, K, device="cuda").to(torch.bfloat16)
        ref = x
        for _ in range(4):
            ref = lin(ref).clone()
            torch.cuda.synchronize()
        bufs = [torch.empty(m, K, device="cuda", dtype=torch.bfloat16) for _ in range(2)]

        def chain():
            y = x
            for i in range(4):
                y = lin(y, output=bufs[i % 2])
            return y
        assert torch.equal(chain(), ref)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = chain()
        bufs[0].zero_(); bufs[1].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, ref)


# ---- FP8Linear end to end ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K,m,dtype", [(576, 7168, 3, "bfloat16"), (1536, 7168, 64, "float16"), (2048, 1024, 257, "bfloat16")])
def test_linear_vs_float64(N, K, m, dtype):
    lin = FP8Linear(K, N, bias=True, A_dtype=dtype).cuda()
    torch.manual_seed(N + m)
    lin.load_float_weight(torch.randn(N, K, device="cuda") * 0.03, torch.randn(N, device="cuda"))
    x = torch.randn(m, K, device="cuda").to(OUT[dtype])
    y = lin(x)
    q, s = quantize_act_fp8(x)
    ref, bound = float64_bound(q, s, lin.weight, lin.weight_scale_inv, y, dtype)
    bias = lin.bias.double()
    # the bias is added after the rounding, in the output type: one more half ulp
    ulp = {"float16": 2.0 ** -11, "bfloat16": 2.0 ** -8}[dtype]
    err = (y.double() - (ref + bias)).abs()
    assert bool((err <= bound + ulp * (ref + bias).abs() * 2).all())
    # the same through F.linear on the dequantized operands in float64
    xd = q.double() * s.double().repeat_interleave(128, 1)
    wd = lin.weight.double() * lin.weight_scale_inv.double().repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)
    assert torch.allclose(torch.nn.functional.linear(xd, wd), ref, rtol=1e-12, atol=1e-12)


def test_load_float_weight_round_trip():
    N, K = 576, 1024
    w = torch.randn(N, K, device="cuda") * 0.1
    w[:128, 256:384] = 0
    lin = FP8Linear(K, N).cuda()
    lin.load_float_weight(w)
    s = lin.weight_scale_inv
    wb = torch.zeros(640, K, device="cuda")
    wb[:N] = w
    amax = wb.view(5, 128, 8, 128).abs().amax(dim=(1, 3)).clamp(min=1e-10)
    assert torch.equal(s, amax / torch.full_like(amax, 448.0))
    assert torch.all(_bytes(lin.weight)[:128, 256:384] == 0)
    sk = s.repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)
    assert torch.all((lin.weight.float() * sk - w).abs() <= w.abs() * 2 ** -4 + sk * 2 ** -10)
    # a saved state_dict loads into a fresh layer bit for bit
    lin2 = FP8Linear(K, N).cuda()
    lin2.load_state_dict(lin.state_dict())
    x = torch.randn(5, K, device="cuda").to(torch.bfloat16)
    assert torch.equal(lin(x), lin2(x))
