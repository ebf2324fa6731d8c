"""GPU: the grouped block-scaled FP8 GEMM (bb_matmul_grouped_fp8[_swiglu]) and FP8MoEExperts.

  * exact inputs (test_gpu_fp8.exact_case per expert: S is exact, only the output rounding remains), bit for bit against float64:
    every BM instance (asserted through the mirror grouped_bm), both forms, every output type, empty experts, all rows in one
    expert, descending and out-of-range offsets with unclaimed rows left untouched, E = 1 and E = 256, N = 128 and K = 128, T not
    a multiple of BM, and capped SM counts;
  * exact block sums with inexact scales (fp8_restate), bit for bit against the header's fp32 order restated per expert: every
    BM bucket, both forms, every output type, experts starting at rows not = 0 mod 4, E = 1 and 256, capped SM counts;
  * random inputs: bit-identical to per-expert bb_matmul_fp8 run unsplit where every expert is in the instance's BM bucket,
    within test_gpu_fp8's float64 bound elsewhere; the SwiGLU form bit-identical to torch silu * mul on the plain call's output
    for the de-interleaved weights;
  * two runs, graph replay, launch counts and a PDL chain through reused buffers;
  * FP8MoEExperts end to end at the DeepSeek-V3, Qwen3-235B-A22B and Qwen3-30B-A3B hidden / intermediate sizes: bit-identical to
    the six steps composed from existing calls, within a float64 bound of the dequantized model, and its two loaders agree.
"""
import ctypes
import itertools

import pytest
import torch

from bitblas_b200 import _lib
from bitblas_b200.fp8 import quantize_act_fp8, quantize_weight_blocks
from bitblas_b200.fp8_moe import FP8MoEExperts
from bitblas_b200.moe import deinterleave_gate_up, interleave_gate_up, moe_combine, moe_route
import fp8_restate as R
from fp8_restate import silu_mul
from test_gpu_fp8 import ACC_REL, OUT, exact_case, exact_S, float64_bound

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
DEV = "cuda"


def grouped_bm(T, E):
    """launch_grouped_fp8_bm: rows of A per tile from the mean rows per active expert"""
    active = min(E, T)
    mean = -(-T // active)
    return 32 if mean <= 32 else (64 if mean <= 64 else 128)


def _op(N, K, out="bfloat16"):
    from bitblas_b200 import Matmul, MatmulConfig
    return Matmul(MatmulConfig(N=N, K=K, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32", out_dtype=out),
                  enable_tuning=False)


def _a_scale(sa):
    """host [T, KB] -> quantize_act_fp8's device layout: the [T, KB] view of a k-block-major [KB, ld] buffer"""
    T, KB = sa.shape
    ld = max((T + 3) // 4 * 4, 4)
    buf = torch.zeros(KB, ld)
    buf[:, :T] = sa.t()
    return buf.to(DEV).t()[:T]


def _launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bb_launch_count() - n0


def _clamped(offsets, T):
    return [(min(max(offsets[e], 0), T), max(min(max(offsets[e + 1], 0), T), min(max(offsets[e], 0), T)))
            for e in range(len(offsets) - 1)]


def exact_grouped(counts_or_offsets, T, N, K, seed, swiglu=False):
    """exact operands for E experts: (A, a_scale, W, w_scale, offsets) on the device and the host pieces (qa, sa, per-expert qw and
    sw, de-interleaved for the SwiGLU form: gate and up [E, N/2, K] with their [E, ceil(N/256), KB] scales)"""
    offsets = counts_or_offsets
    E = len(offsets) - 1
    qa, _, sa, _ = exact_case(T, 128, K, seed)
    if swiglu:
        I = N // 2
        parts = [exact_case(1, I, K, seed * 1000 + 2 * e + h) for e in range(E) for h in range(2)]
        gate = torch.stack([p[1] for p in parts[0::2]]); up = torch.stack([p[1] for p in parts[1::2]])
        sg = torch.stack([p[3] for p in parts[0::2]]); su = torch.stack([p[3] for p in parts[1::2]])
        W = interleave_gate_up(gate, up, "weight")
        ws = interleave_gate_up(sg, su, "block_scale")
        host = (gate, up, sg, su)
    else:
        parts = [exact_case(1, N, K, seed * 1000 + e) for e in range(E)]
        W = torch.stack([p[1] for p in parts]); ws = torch.stack([p[3] for p in parts])
        host = (W, ws)
    dev = (qa.to(E4M3).to(DEV), _a_scale(sa), W.to(E4M3).to(DEV), ws.to(DEV).contiguous(),
           torch.tensor(offsets, dtype=torch.int32, device=DEV))
    return dev, qa, sa, host


def exact_reference(qa, sa, host, offsets, T, N, out, swiglu, sentinel):
    cols = N // 2 if swiglu else N
    ref = torch.full((T, cols), sentinel, dtype=OUT[out], device=DEV)
    for e, (r0, r1) in enumerate(_clamped(offsets, T)):
        if r1 <= r0:
            continue
        if swiglu:
            gate, up, sg, su = host
            g = exact_S(qa[r0:r1], gate[e], sa[r0:r1], sg[e]).to(DEV).to(OUT[out])
            u = exact_S(qa[r0:r1], up[e], sa[r0:r1], su[e]).to(DEV).to(OUT[out])
            ref[r0:r1] = silu_mul(g, u, out)
        else:
            W, ws = host
            ref[r0:r1] = exact_S(qa[r0:r1], W[e], sa[r0:r1], ws[e]).to(DEV).to(OUT[out])
    return ref


def run_exact(offsets, T, N, K, out, swiglu, seed, sentinel=-3.0):
    (A, a_scale, W, ws, off), qa, sa, host = exact_grouped(offsets, T, N, K, seed, swiglu)
    op = _op(N, K, out)
    cols = N // 2 if swiglu else N
    y = torch.full((T, cols), sentinel, dtype=OUT[out], device=DEV)
    fwd = op.forward_grouped_fp8_swiglu if swiglu else op.forward_grouped_fp8
    _, n = _launches(lambda: fwd(A, W, off, a_scale, ws, output=y))
    assert n == 1
    ref = exact_reference(qa, sa, host, offsets, T, N, out, swiglu, sentinel)
    assert torch.equal(y, ref)
    return y


def _offsets(counts):
    return [0] + list(itertools.accumulate(counts))


# routings per BM bucket: an empty expert, counts that are no multiple of BM, an expert with several m-tiles
ROUTINGS = {32: [5, 0, 32, 17, 1, 40], 64: [50, 0, 64, 100, 33], 128: [300, 0, 129, 1, 200]}


@pytest.mark.parametrize("out", ["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("swiglu", [False, True], ids=["plain", "swiglu"])
@pytest.mark.parametrize("bm", [32, 64, 128])
def test_exact_instance(bm, swiglu, out):
    counts = ROUTINGS[bm]
    T = sum(counts)
    assert grouped_bm(T, len(counts)) == bm
    # N = 384: three n-tiles, so the SwiGLU form's odd tile reads the second half of its scale block pair (I = 192)
    run_exact(_offsets(counts), T, 384, 512, out, swiglu, seed=bm + 7 * swiglu + len(out))


@pytest.mark.parametrize("swiglu", [False, True], ids=["plain", "swiglu"])
@pytest.mark.parametrize("case", ["one_expert", "empty_experts", "descending", "out_of_range", "negative", "unclaimed_tail"])
def test_exact_offsets(case, swiglu):
    T = 100
    offsets = {"one_expert": [0, 0, 100, 100, 100],
               "empty_experts": [0, 0, 0, 37, 37, 100],
               "descending": [10, 5, 40, 60, 100],          # expert 0 ends before it starts: empty; rows 0-4 unclaimed
               "out_of_range": [0, 30, 70, 150, 300],        # clamped to T: expert 3 is empty
               "negative": [-50, 20, 20, 64, 90],            # rows 90-99 unclaimed
               "unclaimed_tail": [0, 33, 61]}[case]          # rows 61-99 unclaimed
    run_exact(offsets, T, 256, 384, "bfloat16", swiglu, seed=len(case) + swiglu)


@pytest.mark.parametrize("swiglu", [False, True], ids=["plain", "swiglu"])
def test_exact_one_and_256_experts(swiglu):
    run_exact([0, 77], 77, 256, 256, "float32", swiglu, seed=1)                 # E = 1
    g = torch.Generator().manual_seed(2)
    counts = torch.randint(0, 6, (256,), generator=g).tolist()
    counts[17] = 0
    counts[255] = 3
    run_exact(_offsets(counts), sum(counts), 128, 128, "bfloat16", swiglu, seed=3)   # E = 256, N = 128, K = 128


def test_exact_k128_n128_each_bm():
    for bm, counts in ROUTINGS.items():
        T = sum(counts)
        run_exact(_offsets(counts), T, 128, 128, "float16", False, seed=bm)
        run_exact(_offsets(counts), T + 5, 128, 128, "float16", True, seed=bm + 1)   # 5 unclaimed tail rows


@pytest.mark.parametrize("cap", [1, 7, 114, 0])
def test_exact_capped_sm_counts(cap):
    """the persistent grid at 1, a prime count, 114 (H100 PCIe) SMs and the full device: identical bits"""
    lib = _lib.load()
    prev = lib.bb_set_sm_count_cap(cap)
    try:
        for bm, counts in ROUTINGS.items():
            for swiglu in (False, True):
                run_exact(_offsets(counts), sum(counts), 384, 1024, "bfloat16", swiglu, seed=bm * 3 + swiglu)
    finally:
        lib.bb_set_sm_count_cap(prev)


# ---- inexact scales: the header's fp32 order, bit for bit (fp8_restate) ----------------------------------------------------------
@pytest.mark.parametrize("swiglu", [False, True], ids=["plain", "swiglu"])
@pytest.mark.parametrize("case", list(R.GROUPED_CASES))
def test_inexact_scales_restated(case, swiglu):
    """integer operands (the block sums exact) with inexact scales, every output type, a_scale_ld > T with NaN in the gap:
    each expert's rows equal the restated order on those rows (the SwiGLU form: g and u restated on the de-interleaved gate
    and up rows, rounded to out_dtype, then silu(g) * u on the device)"""
    counts, N, K, cap, bm = R.GROUPED_CASES[case]
    off = R.offsets_of(counts)
    T, E = off[-1], len(counts)
    assert grouped_bm(T, E) == bm
    qa, sa, experts = R.grouped_case(counts, N, K, swiglu)
    stack = lambda i, j: torch.stack([halves[i][j] for halves in experts])
    if swiglu:
        W = interleave_gate_up(stack(0, 0), stack(1, 0), "weight")
        ws = interleave_gate_up(stack(0, 1), stack(1, 1), "block_scale")
    else:
        W, ws = stack(0, 0), stack(0, 1)
    A, a_scale = qa.to(E4M3).to(DEV), R.a_scale_view(sa, 8, DEV)
    W, ws, offsets = W.to(E4M3).to(DEV), ws.to(DEV), torch.tensor(off, dtype=torch.int32, device=DEV)
    qa, sa = qa.to(DEV), sa.to(DEV)
    S = [[R.restate(qa[off[e]:off[e + 1]], qw.to(DEV), sa[off[e]:off[e + 1]], sw.to(DEV)) for qw, sw in halves]
         if off[e + 1] > off[e] else None for e, halves in enumerate(experts)]
    lib = _lib.load()
    prev = lib.bb_set_sm_count_cap(cap)
    try:
        for out in OUT:
            op = _op(N, K, out)
            fwd = op.forward_grouped_fp8_swiglu if swiglu else op.forward_grouped_fp8
            y, n = _launches(lambda: fwd(A, W, offsets, a_scale, ws))
            assert n == 1
            for e, Se in enumerate(S):
                if Se is None:
                    continue
                Ye = [R.round_out(s, out) for s in Se]
                ref = silu_mul(*Ye, out) if swiglu else Ye[0]
                assert torch.equal(y[off[e]:off[e + 1]], ref), (out, e, int((y[off[e]:off[e + 1]] != ref).sum()))
    finally:
        lib.bb_set_sm_count_cap(prev)


# ---- random inputs ---------------------------------------------------------------------------------------------------------------
def fp8_unsplit(op, q, s, W, ws, out=None):
    """bb_matmul_fp8 without a workspace (never split) on rows q with quantize_act_fp8's scales s"""
    m = q.shape[0]
    y = torch.empty(m, op.config.N, dtype=op.torch_output_dtype, device=DEV) if out is None else out
    rc = _lib.load().bb_matmul_fp8(ctypes.byref(op._fp8_desc()), q.data_ptr(), s.data_ptr(), op._fp8_a_scale_ld(s, m),
                                   W.data_ptr(), ws.data_ptr(), 0, y.data_ptr(), m, 0, 0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    return y


def _random(E, N, K, counts, seed):
    torch.manual_seed(seed)
    T = sum(counts)
    x = torch.randn(T, K, device=DEV).to(torch.bfloat16)
    q, s = quantize_act_fp8(x)
    Ws, Ss = zip(*[quantize_weight_blocks(torch.randn(N, K, device=DEV) * 0.02) for _ in range(E)])
    return x, q, s, torch.stack(Ws), torch.stack(Ss)


RANDOM = [  # (E, N, K, counts): DeepSeek-V3's gate/up and down, Qwen3-235B-A22B's, Qwen3-30B-A3B's
    (8, 4096, 7168, [3, 1, 0, 7, 2, 9, 4, 1]),
    (8, 7168, 2048, [40, 33, 64, 0, 50, 61, 45, 36]),
    (6, 3072, 4096, [200, 129, 300, 0, 170, 250]),
    (6, 4096, 1536, [1, 100, 3, 0, 250, 64]),          # mixed buckets: the float64 bound
    (16, 1536, 2048, [20] * 8 + [0] * 4 + [200, 1, 2, 90]),
]


@pytest.mark.parametrize("E,N,K,counts", RANDOM, ids=lambda v: str(v) if not isinstance(v, list) else f"T{sum(v)}")
def test_random_against_unsplit_fp8(E, N, K, counts):
    x, q, s, W, ws = _random(E, N, K, counts, seed=E + N + K)
    T = sum(counts)
    op = _op(N, K)
    off = _offsets(counts)
    y = op.forward_grouped_fp8(q, W, torch.tensor(off, dtype=torch.int32, device=DEV), s, ws)
    bm = grouped_bm(T, E)
    same_bucket = all(grouped_bm(c, 1) == bm for c in counts if c)
    for e in range(E):
        r0, r1 = off[e], off[e + 1]
        if r1 == r0:
            continue
        qe, se = quantize_act_fp8(x[r0:r1])   # per-row quantization: the same bytes and scales as the rows of q, s
        if same_bucket:
            assert torch.equal(y[r0:r1], fp8_unsplit(op, qe, se, W[e], ws[e])), f"expert {e}"
        else:
            ref, bound = float64_bound(qe, se, W[e], ws[e], y[r0:r1], "bfloat16")
            assert bool(((y[r0:r1].double() - ref).abs() <= bound).all()), f"expert {e}"


@pytest.mark.parametrize("E,I,K,counts", [(8, 2048, 7168, [3, 1, 0, 7, 2, 9, 4, 1]), (6, 1536, 4096, [200, 129, 0, 300, 170, 1]),
                                          (16, 768, 2048, [40] * 12 + [0, 50, 61, 33])])
def test_random_swiglu_against_plain(E, I, K, counts):
    """the SwiGLU form on the interleaved weights and scales equals silu(g) * u from the plain call on gate and on up"""
    torch.manual_seed(E + I)
    T = sum(counts)
    x = torch.randn(T, K, device=DEV).to(torch.bfloat16)
    q, s = quantize_act_fp8(x)
    gate, sg = zip(*[quantize_weight_blocks(torch.randn(I, K, device=DEV) * 0.02) for _ in range(E)])
    up, su = zip(*[quantize_weight_blocks(torch.randn(I, K, device=DEV) * 0.02) for _ in range(E)])
    gate, up, sg, su = (torch.stack(t) for t in (gate, up, sg, su))
    u8 = torch.uint8
    W = interleave_gate_up(gate.view(u8), up.view(u8), "weight").view(E4M3)
    ws = interleave_gate_up(sg, su, "block_scale")
    off = torch.tensor(_offsets(counts), dtype=torch.int32, device=DEV)
    h = _op(2 * I, K).forward_grouped_fp8_swiglu(q, W, off, s, ws)
    plain = _op(I, K)
    g = plain.forward_grouped_fp8(q, gate, off, s, sg)
    u = plain.forward_grouped_fp8(q, up, off, s, su)
    assert torch.equal(h, silu_mul(g, u, "bfloat16"))
    # and the de-interleave of the stored weight gives the plain operands back
    g2, u2 = deinterleave_gate_up(W.view(u8), "weight")
    assert torch.equal(g2, gate.view(u8)) and torch.equal(u2, up.view(u8))


# ---- run behaviour -------------------------------------------------------------------------------------------------------------
def test_repeat_graph_and_launch_count():
    E, N, K = 8, 1024, 2048
    counts = [30, 0, 5, 100, 1, 64, 7, 2]
    x, q, s, W, ws = _random(E, N, K, counts, seed=11)
    off = torch.tensor(_offsets(counts), dtype=torch.int32, device=DEV)
    for swiglu in (False, True):
        op = _op(N, K)
        fwd = op.forward_grouped_fp8_swiglu if swiglu else op.forward_grouped_fp8
        a, n = _launches(lambda: fwd(q, W, off, s, ws))   # 2 ceil(I/128) = N/128 scale rows either way
        assert n == 1
        b = fwd(q, W, off, s, ws)
        out = torch.empty_like(a)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            fwd(q, W, off, s, ws, output=out)
        torch.cuda.current_stream().wait_stream(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fwd(q, W, off, s, ws, output=out)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, out)


def _experts(E, H, I, seed, A_dtype="bfloat16"):
    torch.manual_seed(seed)
    with torch.device(DEV):
        m = FP8MoEExperts(E, H, I, A_dtype=A_dtype)
    m.load_float_weight(torch.randn(E, I, H, device=DEV) * 0.03, torch.randn(E, I, H, device=DEV) * 0.03,
                        torch.randn(E, H, I, device=DEV) * 0.03)
    return m


def _routing(T, E, k, seed, drop=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.argsort(torch.rand(T, E, device=DEV, generator=g), dim=1)[:, :k].to(torch.int32)
    if drop and T > 1:
        ids[0, 0] = -1
        ids[T - 1, k - 1] = E
    w = torch.rand(T, k, device=DEV, generator=g)
    return ids, w / w.sum(1, keepdim=True)


def test_pdl_chain_reused_buffers():
    """four expert blocks through two ping-pong outputs, eager and replayed, against separate calls with synchronisation"""
    E, H, I, k = 16, 1024, 512, 4
    m = _experts(E, H, I, 5)
    for T in (1, 8, 200):
        ids, w = _routing(T, E, k, T)
        x = torch.randn(T, H, device=DEV).to(torch.bfloat16)
        ref = x
        for _ in range(4):
            ref = m(ref, ids, w).clone()
            torch.cuda.synchronize()
        bufs = [torch.empty(T, H, device=DEV, dtype=torch.bfloat16) for _ in range(2)]

        def chain():
            y = x
            for i in range(4):
                y = m(y, ids, w, output=bufs[i % 2])
            return y
        y, n = _launches(chain)
        assert n == 24 and torch.equal(y, ref)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            chain()
        torch.cuda.current_stream().wait_stream(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = chain()
        bufs[0].zero_(); bufs[1].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, ref)


# ---- FP8MoEExperts end to end --------------------------------------------------------------------------------------------------
def composed(m, x, ids, w):
    """the six steps from existing calls: moe_route, then per expert quantize_act_fp8 + unsplit bb_matmul_fp8 of gate and of up,
    torch silu * mul, quantize_act_fp8 + unsplit bb_matmul_fp8 of down, then moe_combine"""
    E, H, I = m.num_experts, m.hidden_size, m.intermediate_size
    offsets, slot_rows, xs = moe_route(ids, x, E)
    off = offsets.cpu().tolist()
    u8 = torch.uint8
    gw, uw = deinterleave_gate_up(m.gate_up_weight.view(u8), "weight")
    gs, us = deinterleave_gate_up(m.gate_up_weight_scale_inv, "block_scale")
    gop, dop = _op(I, H, m.A_dtype), _op(H, I, m.A_dtype)
    h = torch.zeros(xs.shape[0], I, dtype=x.dtype, device=DEV)
    y = torch.zeros(xs.shape[0], H, dtype=x.dtype, device=DEV)
    for e in range(E):
        r0, r1 = off[e], off[e + 1]
        if r1 == r0:
            continue
        q, s = quantize_act_fp8(xs[r0:r1])
        g = fp8_unsplit(gop, q, s, gw[e].view(E4M3), gs[e])
        u = fp8_unsplit(gop, q, s, uw[e].view(E4M3), us[e])
        h[r0:r1] = silu_mul(g, u, m.A_dtype)
        q, s = quantize_act_fp8(h[r0:r1])
        y[r0:r1] = fp8_unsplit(dop, q, s, m.down_weight[e], m.down_weight_scale_inv[e])
    return moe_combine(y, slot_rows, w)


def dequantized_bound(m, x, ids, w, y):
    """the dequantized model in float64, y_ref[t] = sum_j w[t, j] * Wd_e (silu(Wg_e x_t) * (Wu_e x_t)), and a per-element bound
    on the block's distance from it, propagated to first order: each e4m3 quantization of x and h moves an element by at most
    2^-4 of itself plus 2^-18 of its 128-block's amax (half of e4m3's subnormal step at s = amax / 448), each block sum by ACC_REL
    of the sum of magnitudes plus 2^-17 for the fp32 promotion, each rounding to A_dtype by twice its relative half ulp (2^-8 for
    bfloat16, 2^-11 for float16), and silu is 1.1-Lipschitz"""
    E, H, I = m.num_experts, m.hidden_size, m.intermediate_size
    ulp = 2.0 ** -7 if m.A_dtype == "bfloat16" else 2.0 ** -10
    rq = 2.0 ** -4 + ACC_REL + 2.0 ** -17
    u8 = torch.uint8
    gw, uw = (t.view(E4M3).double() for t in deinterleave_gate_up(m.gate_up_weight.view(u8), "weight"))
    gs, us = deinterleave_gate_up(m.gate_up_weight_scale_inv, "block_scale")

    def deq(q, s):   # [E, N, K] e4m3 with [E, N/128, K/128] scales -> float64
        return q.double() * s.double().repeat_interleave(128, 1).repeat_interleave(128, 2)
    Wg, Wu, Wd = deq(gw, gs), deq(uw, us), deq(m.down_weight, m.down_weight_scale_inv)
    T, k = ids.shape
    xd = x.double()
    amax_x = xd.abs().view(T, H // 128, 128).amax(-1).repeat_interleave(128, 1)
    ref = torch.zeros(T, H, dtype=torch.float64, device=DEV)
    err = torch.zeros(T, H, dtype=torch.float64, device=DEV)
    mag = torch.zeros(T, H, dtype=torch.float64, device=DEV)
    for j in range(k):
        for e in ids[:, j].unique().tolist():
            if not 0 <= e < E:
                continue
            rows = (ids[:, j] == e).nonzero().squeeze(1)
            xe, ae = xd[rows], amax_x[rows]
            g, u = xe @ Wg[e].t(), xe @ Wu[e].t()
            mag_x = xe.abs() * rq + ae * 2.0 ** -18
            eg = mag_x @ Wg[e].abs().t() + ulp * g.abs()
            eu = mag_x @ Wu[e].abs().t() + ulp * u.abs()
            sg = g / (1 + torch.exp(-g))
            h = sg * u
            eh = 1.1 * eg * (u.abs() + eu) + sg.abs() * eu
            eh = eh + ulp * (h.abs() + eh)
            ha = h.abs() + eh
            amax_h = ha.view(-1, I // 128, 128).amax(-1).repeat_interleave(128, 1)
            yd = h @ Wd[e].t()
            ey = (eh + ha * rq + amax_h * 2.0 ** -18) @ Wd[e].abs().t()
            ey = ey + ulp * (yd.abs() + ey)
            wj = w[rows, j].double()[:, None]
            ref[rows] += wj * yd
            err[rows] += wj.abs() * ey
            mag[rows] += wj.abs() * (yd.abs() + ey)
    # the combine: k fp32 sums, then one rounding
    err = err + 2.0 ** -24 * k * mag + ulp * (ref.abs() + err) + 1e-30
    return ref, err


MODELS = {"DeepSeek-V3": (7168, 2048), "Qwen3-235B-A22B": (4096, 1536), "Qwen3-30B-A3B": (2048, 768)}


@pytest.mark.parametrize("T", [1, 4, 16, 128, 512, 2048])
@pytest.mark.parametrize("model", list(MODELS))
def test_block_end_to_end(model, T):
    H, I = MODELS[model]
    E, k = 16, 8
    m = _experts(E, H, I, seed=T + H)
    ids, w = _routing(T, E, k, seed=T, drop=True)
    x = torch.randn(T, H, device=DEV).to(torch.bfloat16)
    y, n = _launches(lambda: m(x, ids, w))
    assert n == 6 and y.shape == (T, H) and y.dtype == torch.bfloat16
    assert torch.equal(y, composed(m, x, ids, w))
    if T <= 512:
        ref, bound = dequantized_bound(m, x, ids, w, y)
        excess = (y.double() - ref).abs() - bound
        assert bool((excess <= 0).all()), f"max excess {excess.max().item():.3g}"


def test_block_256_experts():
    """DeepSeek-V3's expert count at the Qwen3-30B-A3B sizes, float16 activations, with a graph replay"""
    E, H, I, k, T = 256, 2048, 768, 8, 300
    m = _experts(E, H, I, seed=256, A_dtype="float16")
    ids, w = _routing(T, E, k, seed=9, drop=True)
    x = torch.randn(T, H, device=DEV).to(torch.float16)
    y, n = _launches(lambda: m(x, ids, w))
    assert n == 6 and torch.equal(y, composed(m, x, ids, w))
    ref, bound = dequantized_bound(m, x, ids, w, y)
    assert bool(((y.double() - ref).abs() <= bound).all())
    out = torch.empty_like(y)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m(x, ids, w, output=out)
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        m(x, ids, w, output=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, y)


def test_loaders_agree():
    """load_fp8 from per-expert tensors under the checkpoint's names, load_float_weight and load_state_dict give the same block"""
    E, H, I = 8, 2048, 768
    torch.manual_seed(3)
    gate, up, down = (torch.randn(E, a, b, device=DEV) * 0.03 for a, b in ((I, H), (I, H), (H, I)))
    with torch.device(DEV):
        a, b, c = FP8MoEExperts(E, H, I), FP8MoEExperts(E, H, I), FP8MoEExperts(E, H, I)
    a.load_float_weight(gate, up, down)
    shard = {}
    for e in range(E):
        for name, t in (("gate", gate), ("up", up), ("down", down)):
            q, s = quantize_weight_blocks(t[e])
            shard[f"model.layers.3.mlp.experts.{e}.{name}_proj.weight"] = q.cpu()
            shard[f"model.layers.3.mlp.experts.{e}.{name}_proj.weight_scale_inv"] = s.cpu()

    def proj(name):
        pre = "model.layers.3.mlp.experts.{}." + name + "_proj."
        return ([shard[pre.format(e) + "weight"] for e in range(E)], [shard[pre.format(e) + "weight_scale_inv"] for e in range(E)])
    b.load_fp8(proj("gate"), proj("up"), proj("down"))
    c.load_state_dict(a.state_dict())
    ids, w = _routing(64, E, 8, seed=4)
    x = torch.randn(64, H, device=DEV).to(torch.bfloat16)
    ya = a(x, ids, w)
    assert torch.equal(ya, b(x, ids, w)) and torch.equal(ya, c(x, ids, w))
