"""GPU: the grouped wgmma GEMM (bb_matmul_grouped_gemm / Matmul.forward_grouped(capturable=True)) expert by expert against the
float64 gemm_ts contract and per-element bound of test_gpu_kernel_grid.py, bit for bit against per-expert bb_matmul on gemm_ts,
and as one graph-capturable launch."""
import ctypes
import itertools

import pytest
import torch

import helpers as H
from test_gpu_kernel_grid import K_GEMM_TS, MODES, OUTS, check_float, forced, make_case

pytestmark = pytest.mark.gpu

DEV = "cuda"


def grouped_bm(counts):
    """launch_grouped_gemm_bm: rows of A per tile from the mean rows per active group"""
    T = sum(counts)
    mean = -(-T // min(len(counts), T))
    return 32 if mean <= 32 else (64 if mean <= 64 else 128)


def _offsets(counts):
    return [0] + list(itertools.accumulate(counts))


def _build(counts, N, K, seed, *, A_dtype="float16", W="uint4", out="float16", g=128, mode="quantized", bias=False, il=None,
           T=None):
    """E experts of one config sharing the activations A [T, K] (T = sum(counts) unless given)"""
    T = sum(counts) if T is None else T
    kw = dict(A_dtype=A_dtype, W_dtype=W, out_dtype=out, group_size=g, mode=mode, bias=bias, fast_decoding=il)
    A = make_case(T, 8, K, seed=seed, **dict(kw, mode="none", bias=False))["A"]
    cases = [make_case(T, N, K, seed=seed * 31 + e, A=A, **kw) for e in range(len(counts))]
    op = H.product_operator(cases[0], M=[1, 16])
    st = lambda k: torch.stack([x[k] for x in cases]).to(DEV) if cases[0][k] is not None else None   # noqa: E731
    W_ = torch.stack([H.product_weight(op, x, DEV) for x in cases])
    return op, cases, A, W_, st("scale"), st("zeros"), st("bias")


def _launches(fn):
    from bitblas_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bb_launch_count() - n0


def _check(cases, offsets, got, what, rule="gemm_ts"):
    for e, x in enumerate(cases):
        r0, r1 = offsets[e], offsets[e + 1]
        if r1 > r0:
            rows = slice(r0, r1)
            check_float(got[rows], x, rule, f"{what} expert {e}", rows=rows)


# ---- every instance: T x bits x layout x BM (24), each with the 5 modes x 3 output types x +- bias --------------------------------
# routings: one empty expert, counts that are no multiple of BM and straddle tile boundaries, one expert with several m-tiles
ROUTINGS = {32: [3, 0, 40, 20, 17], 64: [70, 0, 50, 33, 90], 128: [200, 0, 130, 77, 300]}
CELLS = [dict(T=T, bits=bits, il=il, bm=bm, mode=mode)
         for T, bits, il, bm, mode in itertools.product(["float16", "bfloat16"], [4, 2], [True, False], [32, 64, 128], MODES)]


@pytest.mark.parametrize("c", CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_grouped_gemm_instance(c):
    counts = ROUTINGS[c["bm"]]
    assert grouped_bm(counts) == c["bm"]
    offsets = _offsets(counts)
    for i, (out, bias) in enumerate(itertools.product(OUTS, [False, True])):
        signed = c["mode"] in ("none", "scale") and bias
        W = ("int" if signed else "uint") + str(c["bits"])
        g = [128, 384, -1][i % 3]
        op, cases, A, Wq, s, z, b = _build(counts, 256, 768, seed=1000 * i + len(c["mode"]) + c["bm"], A_dtype=c["T"], W=W,
                                           out=out, g=g, mode=c["mode"], bias=bias, il=c["il"])
        assert bool(op.fast_decoding) == c["il"]
        off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
        got, n = _launches(lambda: op.forward_grouped(A.to(DEV), Wq, off, scale=s, zeros=z, bias=b, capturable=True))
        assert n == 1
        _check(cases, offsets, got.cpu(), f"{c} out={out} bias={bias} W={W} g={g}")


@pytest.mark.parametrize("K,g", [(384, 128), (384, -1), (4096, 128)])
def test_grouped_gemm_k_blocks(K, g):
    """K = 384: three 128-wide blocks, fewer k-blocks than ring stages, so several tiles share one pass of the ring; K = 4096: the
    ring wraps inside every tile"""
    counts = [70, 0, 33, 150, 9]
    op, cases, A, W, s, z, _ = _build(counts, 256, K, seed=K + g, g=g, mode="original")
    offsets = _offsets(counts)
    got = op.forward_grouped(A.to(DEV), W, torch.tensor(offsets, dtype=torch.int32, device=DEV), scale=s, zeros=z,
                             capturable=True)
    _check(cases, offsets, got.cpu(), f"K={K} g={g}")


# ---- bit-equality with per-expert bb_matmul on gemm_ts, split-K off ---------------------------------------------------------------
@pytest.mark.parametrize("counts", [[20, 0, 30, 25], [40, 50, 0, 60, 33], [100, 200, 0, 129, 300]],
                         ids=lambda c: f"bm{grouped_bm(c)}")
@pytest.mark.parametrize("kw", [dict(mode="quantized", out="float16", bias=True),
                                dict(mode="rescale", out="float32", W="uint2", il=False),
                                dict(mode="original", A_dtype="bfloat16", out="bfloat16", bias=True, il=True)],
                         ids=["q-f16", "r-f32-u2", "o-bf16"])
def test_grouped_gemm_bit_identical_to_gemm_ts(counts, kw):
    bm = grouped_bm(counts)
    assert all(grouped_bm([m]) == bm for m in counts if m), "every expert must land in the grouped BM bucket"
    op, cases, A, W, s, z, b = _build(counts, 256, 1024, seed=len(counts) * 7 + bm, **kw)
    offsets = _offsets(counts)
    Ad = A.to(DEV)
    got = op.forward_grouped(Ad, W, torch.tensor(offsets, dtype=torch.int32, device=DEV), scale=s, zeros=z, bias=b,
                             capturable=True)
    ref = torch.zeros_like(got)
    stream = torch.cuda.current_stream().cuda_stream
    with forced(K_GEMM_TS) as lib:
        for e in range(len(counts)):
            r0, r1 = offsets[e], offsets[e + 1]
            if r1 <= r0:
                continue
            assert op.kernel_for(r1 - r0) == "gemm_ts_wgmma"
            rc = lib.bb_matmul(ctypes.byref(op._desc), Ad[r0:r1].data_ptr(), W[e].data_ptr(), 0,
                               s[e].data_ptr() if s is not None else 0, z[e].data_ptr() if z is not None else 0,
                               b[e].data_ptr() if b is not None else 0, ref[r0:r1].data_ptr(), r1 - r0, 0, 0, stream)
            assert rc == 0
    torch.cuda.synchronize()
    for e in range(len(counts)):
        r0, r1 = offsets[e], offsets[e + 1]
        assert torch.equal(got[r0:r1], ref[r0:r1]), f"expert {e} rows [{r0}, {r1})"


# ---- routing distributions ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("counts", [
    [0, 0, 300, 0],                                   # one expert takes all rows
    [0, 40, 30, 20, 60], [40, 30, 20, 60, 0], [40, 30, 0, 0, 20, 60],   # empty first / last / middle experts
    [500, 1, 1, 700, 2, 0, 900, 3],                   # very uneven: several m-tiles next to single rows
], ids=lambda c: f"E{len(c)}-T{sum(c)}")
def test_grouped_gemm_distributions(counts):
    op, cases, A, W, s, z, _ = _build(counts, 128, 512, seed=sum(counts))
    offsets = _offsets(counts)
    got, n = _launches(lambda: op.forward_grouped(A.to(DEV), W, torch.tensor(offsets, dtype=torch.int32, device=DEV),
                                                  scale=s, zeros=z, capturable=True))
    assert n == 1
    _check(cases, offsets, got.cpu(), f"counts={counts}")


@pytest.mark.parametrize("E,T", [(256, 3000), (8, 4096), (64, 2048)])   # all above GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E
def test_grouped_gemm_uniform_routing(E, T):
    gen = torch.Generator().manual_seed(E * 7 + T)
    counts = torch.bincount(torch.randint(0, E, (T,), generator=gen), minlength=E).tolist()
    op, cases, A, W, s, z, _ = _build(counts, 128, 256, seed=E + T, mode="scale", W="int4")
    offsets = _offsets(counts)
    got, n = _launches(lambda: op.forward_grouped(A.to(DEV), W, torch.tensor(offsets, dtype=torch.int32, device=DEV),
                                                  scale=s, capturable=True))
    assert n == 1
    _check(cases, offsets, got.cpu(), f"E={E} T={T}")


# ---- malformed offsets ----------------------------------------------------------------------------------------------------------
def test_grouped_gemm_malformed_offsets_stay_in_bounds():
    """offsets clamped to [0, T], a group whose end is below its start is empty: A / C carry 16 guard rows beyond T that keep
    their sentinel, and rows no group claims are not written"""
    E, N, K, T = 4, 256, 512, 80     # T above GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E: the grouped GEMM runs
    op, cases, A_full, W, s, z, _ = _build([0] * E, N, K, seed=5, T=T + 16)
    A_dev = A_full.to(DEV)
    sentinel = -1234.0

    def run(offsets):
        C_full = torch.full((T + 16, N), sentinel, dtype=torch.float16, device=DEV)
        off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
        _, n = _launches(lambda: op.forward_grouped(A_dev[:T], W, off, scale=s, zeros=z, output=C_full[:T], capturable=True))
        assert n == 1
        C = C_full.cpu()
        assert torch.all(C[T:] == sentinel), "a guard row beyond T was written"
        return C

    # negative start, past-the-end stop: groups [0, 30), [30, 50), empty, [50, T)
    C = run([-5, 30, 50, 50, T + 16])
    _check(cases, [0, 30, 50, 50, T], C, "clamped")
    # rows 0..9 and 70..T-1 belong to no group
    C = run([10, 40, 40, 70, 70])
    assert torch.all(C[:10] == sentinel) and torch.all(C[70:] == sentinel)
    _check(cases, [10, 40, 40, 70, 70], C, "unclaimed rows")
    # a decreasing entry: group 1 = [37, 12) is empty; group 2 = [12, 60) overlaps group 0 on rows 12..36
    C = run([0, 37, 12, 60, 60])
    check_float(C[0:12], cases[0], "gemm_ts", "before the overlap", rows=slice(0, 12))
    check_float(C[37:60], cases[2], "gemm_ts", "after the overlap", rows=slice(37, 60))
    assert torch.all(C[60:T] == sentinel)


# ---- launch count of forward_grouped(capturable=True) above the threshold ----------------------------------------------------------
@pytest.mark.parametrize("N", [256, 144])
def test_capturable_is_one_launch(N):
    """N % 128 == 0 runs the grouped GEMM, N = 144 (N % 16 == 0 only) the grouped GEMV; both in one launch at T above the
    threshold, where capturable=False issues one bb_matmul per expert"""
    from bitblas_b200.ops.general_matmul import GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP as R
    counts = [3 * R, 0, 5 * R + 40, 7, R + 1]
    assert sum(counts) > R * len(counts)
    op, cases, A, W, s, z, _ = _build(counts, N, 512, seed=N)
    offsets = _offsets(counts)
    off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
    got, n = _launches(lambda: op.forward_grouped(A.to(DEV), W, off, scale=s, zeros=z, capturable=True))
    assert n == 1
    _check(cases, offsets, got.cpu(), f"N={N}", rule="gemm_ts" if N % 128 == 0 else "exact")
    _, n = _launches(lambda: op.forward_grouped(A.to(DEV), W, off, scale=s, zeros=z))
    assert n >= 3


# ---- CUDA graph --------------------------------------------------------------------------------------------------------------------
def test_grouped_gemm_graph_replay_with_changing_routing():
    """one CUDA graph at prefill size; every replay refreshes the device offsets and the activations through pinned h2d copies"""
    import bitblas_b200 as bitblas
    E, N, K, T = 8, 256, 512, 512
    op, cases, _, W, s, z, _ = _build([0] * E, N, K, seed=6, T=T)
    host_off = torch.zeros(E + 1, dtype=torch.int32).pin_memory()
    host_A = torch.zeros((T, K), dtype=torch.float16).pin_memory()
    host_C = torch.zeros((T, N), dtype=torch.float16).pin_memory()
    dev_off = torch.zeros(E + 1, dtype=torch.int32, device=DEV)
    dev_off[-1] = T
    dev_A = torch.zeros((T, K), dtype=torch.float16, device=DEV)
    dev_C = torch.zeros((T, N), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: op.forward_grouped(dev_A, W, dev_off, scale=s, zeros=z, output=dev_C, capturable=True),
                                h2d=[(dev_off, host_off), (dev_A, host_A)], d2h=[(host_C, dev_C)])
    for trial in range(4):
        g = torch.Generator().manual_seed(100 + trial)
        counts = torch.bincount(torch.randint(0, E if trial else 3, (T,), generator=g), minlength=E).tolist()
        offsets = _offsets(counts)
        host_off.copy_(torch.tensor(offsets, dtype=torch.int32))
        A = (torch.rand((T, K), generator=g) - 0.5).half()
        host_A.copy_(A)
        step()
        for x in cases:
            x["A"] = A
        _check(cases, offsets, host_C.clone(), f"replay {trial}")


# ---- programmatic dependent launch chain -------------------------------------------------------------------------------------------
def test_grouped_gemm_pdl_dependent_chain():
    """offsets computed on the device (bincount + cumsum) right before each call, then a gate/up -> down chain of two capturable
    calls, 16 times back to back without synchronisation: bit-identical to the same calls with a synchronisation after each"""
    E, T, K, N1, N2 = 8, 256, 512, 1024, 512
    op1, c1, _, W1, s1, z1, _ = _build([0] * E, N1, K, seed=7, T=1)
    op2, c2, _, W2, s2, z2, _ = _build([0] * E, N2, N1, seed=8, T=1)
    gen = torch.Generator(device=DEV).manual_seed(9)
    ids = [torch.randint(0, E, (T,), device=DEV, generator=gen) for _ in range(16)]
    xs = [((torch.rand((T, K), device=DEV, generator=gen) - 0.5) * 0.5).half() for _ in range(16)]
    mid = torch.empty((T, N1), dtype=torch.float16, device=DEV)
    outs = [torch.empty((T, N2), dtype=torch.float16, device=DEV) for _ in range(16)]
    offs = [torch.empty(E + 1, dtype=torch.int32, device=DEV) for _ in range(16)]

    def route(i, off):   # bincount + cumsum; scatter_add_ counts without torch.bincount's host read of max(ids)
        counts = torch.zeros(E, dtype=torch.int64, device=DEV).scatter_add_(0, ids[i], torch.ones_like(ids[i]))
        off[0] = 0
        off[1:] = torch.cumsum(counts, 0).to(torch.int32)

    torch.cuda.synchronize()
    for i in range(16):                 # no synchronisation anywhere in this loop
        route(i, offs[i])
        op1.forward_grouped(xs[i], W1, offs[i], scale=s1, zeros=z1, output=mid, capturable=True)
        op2.forward_grouped(mid, W2, offs[i], scale=s2, zeros=z2, output=outs[i], capturable=True)
    torch.cuda.synchronize()
    got = [o.cpu() for o in outs]
    off_ref = torch.empty(E + 1, dtype=torch.int32, device=DEV)
    for i in range(16):
        route(i, off_ref)
        torch.cuda.synchronize()
        op1.forward_grouped(xs[i], W1, off_ref, scale=s1, zeros=z1, output=mid, capturable=True)
        torch.cuda.synchronize()
        ref = op2.forward_grouped(mid, W2, off_ref, scale=s2, zeros=z2, capturable=True)
        torch.cuda.synchronize()
        assert torch.equal(got[i], ref.cpu()), f"chain step {i}"
        assert torch.equal(offs[i].cpu(), off_ref.cpu())
    offsets = offs[-1].cpu().tolist()
    assert offsets[-1] == T
    x = xs[-1].cpu()
    for c in c1:
        c["A"] = x
    _check(c1, offsets, op1.forward_grouped(xs[-1], W1, offs[-1], scale=s1, zeros=z1, capturable=True).cpu(), "gate/up")
