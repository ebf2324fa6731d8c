"""GPU parity of the m = 1 decode kernel (bb_gemv_slab.cu: per-CTA TMA slabs + CTA-level stream-K), through the C ABI
(Matmul.forward -> bb_matmul), against the CPU oracle on the same seeded inputs -- small shapes that exercise every
zero-point mode / layout / ragged-K path, and the BASELINE.json shapes (C1: Llama-2-70B linears + the
12288^2 target) with the FULL output compared.  Mirrors the reference's
testing/python/operators/test_general_matmul_ops_backend_tl.py:127-283 (tolerance rtol = atol = 1e-2)."""
import ctypes

import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

Q = dict(W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")

SLAB_CASES = [
    dict(N=256, K=256, W_dtype="uint4"),                                   # no scale, no zeros, one partial unit
    dict(N=256, K=256, W_dtype="uint4", fast_decoding=False),              # plain compressed storage
    dict(N=256, K=256, W_dtype="int4", group_size=-1, with_scaling=True),   # constant zero point 8, per-channel scale
    dict(N=256, K=512, W_dtype="int4", group_size=128, with_scaling=True),
    dict(N=256, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(N=256, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(N=256, K=512, **Q),
    dict(N=1024, K=1024, **Q),                                              # BASELINE C0 shape
    dict(N=512, K=2048, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", with_bias=True),
    dict(N=512, K=1024, W_dtype="uint4", group_size=256, with_scaling=True, with_zeros=True, zeros_mode="original", int_zeros=False),
    dict(N=16, K=4096, **Q),                                                # one row block split over many CTAs
    dict(N=48, K=2304, **Q),                                                # K = 2048 + 256: ragged last unit (1 valid slice)
    dict(N=2064, K=3840, **Q),                                              # ragged last unit (7 valid slices), N/16 odd
    dict(N=4096, K=4096, **Q),
    dict(N=4112, K=6144, with_bias=True, **Q),                              # ranges start and end inside row blocks
    dict(N=96, K=11264, with_bias=True, **Q),                               # tiny N, long K: few row blocks over many CTAs
    dict(N=512, K=8192, W_dtype="uint4", group_size=1024, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(N=512, K=3072, W_dtype="uint4", group_size=384, with_scaling=True, with_zeros=True, zeros_mode="original"),   # 128 | g, g not a power of 2
    dict(N=1024, K=2048, W_dtype="uint4", fast_decoding=False, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(N=1024, K=2048, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(N=1024, K=2048, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", fast_decoding=True, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(N=1024, K=2048, W_dtype="uint4", out_dtype="float32", accum_dtype="float32", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
]


def _ids(k):
    return "-".join(f"{a}{b}" for a, b in k.items())


def _slab(case):
    op = H.product_operator(case)
    assert op.kernel_for(1) == "gemv_slab", op.kernel_for(1)
    return op, H.run_product(op, case)


@pytest.mark.parametrize("kw", SLAB_CASES, ids=_ids)
def test_gemv_slab_parity(kw):
    kw = dict(kw)
    case = H.make_case(1, kw.pop("N"), kw.pop("K"), **kw)
    op, got = _slab(case)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    H.assert_fp_close(got, ref, "gemv_slab", max_mismatched_ratio=2e-3 if case["cfg"]["out_dtype"] == "bfloat16" else 0.0)
    # the summation order is fixed (CTA reduction + ordered stream-K fix-up): a second run is bit-identical
    got2 = H.run_product(op, case)
    assert torch.equal(got, got2)


# BASELINE.json configs[1] (C1: W4A16 GEMV M=1 on the Llama-2-70B linears) + the 12288^2 target shape, full output vs the oracle
BASELINE_SHAPES = [(8192, 8192), (28672, 8192), (8192, 28672), (12288, 12288)]


@pytest.mark.parametrize("N,K", BASELINE_SHAPES, ids=lambda v: str(v))
def test_gemv_slab_baseline_shapes(N, K):
    case = H.make_case(1, N, K, **Q)
    op, got = _slab(case)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    H.assert_fp_close(got, ref, f"gemv_slab {N}x{K}")


@pytest.mark.parametrize("N,K", [(12288, 12288), (8192, 28672)], ids=lambda v: str(v))
@pytest.mark.parametrize("zeros_mode", ["original", "rescale"])
def test_gemv_slab_baseline_shapes_fp_zeros(N, K, zeros_mode):
    case = H.make_case(1, N, K, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode=zeros_mode,
                       int_zeros=False, with_bias=True)
    op, got = _slab(case)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    H.assert_fp_close(got, ref, f"gemv_slab {N}x{K} {zeros_mode}")


@pytest.mark.parametrize("M", [2, 8])
@pytest.mark.parametrize("N,K", BASELINE_SHAPES, ids=lambda v: str(v))
def test_gemv_mma_baseline_shapes(M, N, K):
    """m = 2..8 still run the register-queue kernel: full output at the BASELINE shapes (multi-wave grids, ks = 2 / 3 / 4)."""
    case = H.make_case(M, N, K, **Q)
    op = H.product_operator(case)
    assert op.kernel_for(M) == "gemv_mma"
    got = H.run_product(op, case)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    H.assert_fp_close(got, ref, f"gemv_mma M={M} {N}x{K}")


def test_gemv_slab_adversarial_activation_ranges():
    """the decode magic (1024 + u / 64 + u) is removed through per-step activation sums, not per element: check it on
    activations whose sums cancel badly, are all of one sign, are tiny, and are close to the fp16 maximum."""
    N, K = 512, 4096
    base = H.make_case(1, N, K, **Q)
    g = torch.Generator().manual_seed(7)
    variants = {
        "one_sign_large": (torch.rand((1, K), generator=g) * 8 + 2).half(),
        "tiny": ((torch.rand((1, K), generator=g) - 0.5) * 2e-4).half(),
        "wide_range": (torch.randn((1, K), generator=g) * torch.pow(10.0, torch.randint(-4, 2, (1, K), generator=g).float())).half(),
        "alternating": (torch.tensor([1.0, -1.0]).repeat(K // 2).reshape(1, K) * 300).half(),
    }
    for name, A in variants.items():
        case = dict(base, A=A)
        op, got = _slab(case)
        ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
        assert torch.isfinite(ref.float()).all(), name
        H.assert_fp_close(got, ref, f"gemv_slab activations={name}")


def test_gemv_slab_graph_replay_and_errors():
    """CUDA-graph replay (the per-call nonce is frozen in the graph; the owner CTAs reset the exchange slots, so every replay is
    still correct) and the loud failure without a workspace."""
    from bitblas_b200 import _lib
    case = H.make_case(1, 2064, 6144, **Q)
    op = H.product_operator(case)
    dev = "cuda"
    A = case["A"].to(dev)
    Wd = H.product_weight(op, case, dev)
    sc, zr = case["scale"].to(dev), case["zeros"].to(dev)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    got = H.run_product(op, case)
    H.assert_fp_close(got, ref, "slab")
    out = torch.empty(1, 2064, dtype=torch.float16, device=dev)
    rc = op.lib._c.bb_matmul(ctypes.byref(op._desc), A.data_ptr(), Wd.data_ptr(), 0, sc.data_ptr(), zr.data_ptr(), 0,
                             out.data_ptr(), 1, 0, 0, torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and "workspace" in _lib.last_error()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        op.forward(A, Wd, scale=sc, zeros=zr, output=out)   # warm-up outside capture (occupancy query, attributes, tensor map)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            op.forward(A, Wd, scale=sc, zeros=zr, output=out)
        for _ in range(3):
            out.zero_()
            g.replay()
            s.synchronize()
            assert torch.equal(out.cpu(), got.reshape(1, -1)), "graph replay differs"


def test_captured_step_matches_eager():
    """bitblas_b200.CapturedStep: pinned H2D + two dependent-free projections + pinned D2H replayed as one CUDA graph give the
    eager results bit for bit, for fresh host inputs on every replay."""
    import bitblas_b200 as bitblas
    dev = torch.device("cuda")
    shapes = [(512, 1024), (256, 2048)]
    ops = []
    for i, (N, K) in enumerate(shapes):
        case = H.make_case(1, N, K, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", seed=40 + i)
        op = H.product_operator(case)
        ops.append((op, H.product_weight(op, case, dev), case["scale"].to(dev), case["zeros"].to(dev), N, K))
    Ks, Ns = [K for _, K in shapes], [N for N, _ in shapes]
    hostA = torch.empty((sum(Ks),), dtype=torch.float16).pin_memory()
    hostC = torch.empty((sum(Ns),), dtype=torch.float16).pin_memory()
    devA = torch.empty((sum(Ks),), dtype=torch.float16, device=dev)
    devC = torch.empty((sum(Ns),), dtype=torch.float16, device=dev)
    av = [devA[:Ks[0]].view(1, -1), devA[Ks[0]:].view(1, -1)]
    cv = [devC[:Ns[0]].view(1, -1), devC[Ns[0]:].view(1, -1)]

    def fn():
        for (op, W, s, z, N, K), a, c in zip(ops, av, cv):
            op.forward(a, W, scale=s, zeros=z, output=c)

    step = bitblas.CapturedStep(fn, h2d=[(devA, hostA)], d2h=[(hostC, devC)])
    for trial in range(3):
        hostA.copy_((torch.rand(sum(Ks), generator=torch.Generator().manual_seed(trial)) - 0.5).half())
        step()
        got = hostC.clone()
        devA.copy_(hostA); fn(); torch.cuda.synchronize()
        assert torch.equal(got, devC.cpu()), f"replay {trial}"
    with pytest.raises(ValueError):
        bitblas.CapturedStep(fn, h2d=[(devA, torch.empty(8))])       # unpinned host buffer
