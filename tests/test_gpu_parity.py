"""GPU parity: every kernel family, through the C ABI (Matmul.forward -> bb_matmul), against the CPU oracle on
the same seeded inputs.  Bit-exact for INT accumulate, <= 1e-2 relative for FP accumulate (north_star)."""
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu


def _run(case, expect_kernel=None, force=None):
    """force: kernel family id to pin with bb_set_kernel_override (the dispatcher prefers the wgmma kernel above m = 8,
    the streaming kernels still cover m <= 32 and are tested there through the override)."""
    from bitblas_b200 import _lib
    op = H.product_operator(case)
    lib = _lib.load()
    prev = lib.bb_set_kernel_override(force) if force is not None else None
    try:
        if expect_kernel is not None:
            assert op.kernel_for(case["M"]) == expect_kernel, (op.kernel_for(case["M"]), expect_kernel)
        got = H.run_product(op, case)
    finally:
        if force is not None:
            lib.bb_set_kernel_override(prev)
    ref = H.oracle_output(case, fast_decoding=bool(op.fast_decoding))
    return op, got, ref


GEMV_CASES = [
    # reference GEMV cases (test_general_matmul_ops_backend_tl.py:327-334) at a 128-aligned size
    dict(M=1, N=256, K=256, W_dtype="uint4"),
    dict(M=1, N=256, K=256, W_dtype="uint4", fast_decoding=False),
    dict(M=1, N=256, K=256, W_dtype="int4", group_size=-1, with_scaling=True),
    dict(M=1, N=256, K=512, W_dtype="int4", group_size=128, with_scaling=True),
    dict(M=1, N=256, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=1, N=256, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=1, N=256, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    # C0 / C1 style
    dict(M=1, N=1024, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=1, N=512, K=2048, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", with_bias=True),
    dict(M=1, N=512, K=1024, W_dtype="uint4", group_size=256, with_scaling=True, with_zeros=True, zeros_mode="original", int_zeros=False),
    dict(M=3, N=512, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", with_bias=True),
    dict(M=8, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=16, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=27, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=32, N=256, K=512, W_dtype="uint4", group_size=-1, with_scaling=True),
    dict(M=1, N=256, K=1024, W_dtype="uint2", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=5, N=256, K=1024, W_dtype="uint2", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=1, N=256, K=1024, W_dtype="int2", group_size=128, with_scaling=True),
    dict(M=2, N=256, K=512, W_dtype="uint2", fast_decoding=False, group_size=128, with_scaling=True),
    dict(M=1, N=256, K=1024, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=4, N=256, K=1024, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", fast_decoding=True, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=1, N=256, K=1024, W_dtype="uint4", out_dtype="float32", accum_dtype="float32", group_size=128, with_scaling=True),
]


@pytest.mark.parametrize("kw", GEMV_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_gemv_mma_parity(kw):
    kw = dict(kw)
    case = H.make_case(kw.pop("M"), kw.pop("N"), kw.pop("K"), **kw)
    from bitblas_b200 import _lib
    op, got, ref = _run(case, "gemv_mma", force=_lib.BB_KERNEL_GEMV_MMA)
    H.assert_fp_close(got, ref, "gemv_mma")


def test_gemv_pdl_dependent_chain():
    """Programmatic dependent launch: kernel i+1 starts (and prefetches weights) before kernel i has finished, and must
    still see kernel i's output as its activations and never overwrite a buffer kernel i is still reading.  A chain
    y = W2 (W1 x) is launched 24 times back to back without any synchronisation, re-using the intermediate buffer, then
    every result is compared bit-for-bit with the same chain run with a device synchronisation after every launch."""
    torch.manual_seed(3)
    dev = "cuda"
    c1 = H.make_case(1, 2048, 1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", seed=1)
    c2 = H.make_case(1, 512, 2048, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", seed=2)
    op1, op2 = H.product_operator(c1), H.product_operator(c2)
    assert op1.kernel_for(1) == "gemv_slab" and op2.kernel_for(1) == "gemv_slab"
    W1, W2 = H.product_weight(op1, c1, dev), H.product_weight(op2, c2, dev)
    s1, z1, s2, z2 = c1["scale"].to(dev), c1["zeros"].to(dev), c2["scale"].to(dev), c2["zeros"].to(dev)
    xs = [((torch.rand(1, 1024) - 0.5) * 0.5).half().to(dev) for _ in range(24)]
    mid = torch.empty(1, 2048, dtype=torch.float16, device=dev)
    outs = [torch.empty(1, 512, dtype=torch.float16, device=dev) for _ in xs]
    torch.cuda.synchronize()
    for x, o in zip(xs, outs):          # no synchronisation anywhere in this loop
        op1.forward(x, W1, scale=s1, zeros=z1, output=mid)
        op2.forward(mid, W2, scale=s2, zeros=z2, output=o)
    torch.cuda.synchronize()
    got = [o.cpu() for o in outs]
    for x, g in zip(xs, got):
        op1.forward(x, W1, scale=s1, zeros=z1, output=mid)
        torch.cuda.synchronize()
        ref = op2.forward(mid, W2, scale=s2, zeros=z2)
        torch.cuda.synchronize()
        assert torch.equal(g, ref.cpu())
    # and the chain is numerically the oracle's
    mid_ref = H.oracle_output(dict(c1, A=xs[-1].cpu()), fast_decoding=bool(op1.fast_decoding))
    out_ref = H.oracle_output(dict(c2, A=mid_ref.to(torch.float16)), fast_decoding=bool(op2.fast_decoding))
    H.assert_fp_close(got[-1], out_ref, "pdl chain")


GEMM_CASES = [
    # reference GEMM cases (test_general_matmul_ops_backend_tl.py:337-343), M=256 N=K=256
    dict(M=256, N=256, K=256, W_dtype="uint4"),
    dict(M=256, N=256, K=256, W_dtype="int4", group_size=-1, with_scaling=True),
    dict(M=256, N=256, K=256, W_dtype="int4", group_size=64, with_scaling=True),
    dict(M=256, N=256, K=256, W_dtype="uint4", group_size=64, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=256, N=256, K=256, W_dtype="uint4", group_size=64, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=256, N=256, K=256, W_dtype="uint4", group_size=64, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    # tile-shape coverage: BM = 32 / 64 / 128 / 256, ragged M, several n tiles, long K (pipeline wrap-around)
    dict(M=33, N=128, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=64, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", with_bias=True),
    dict(M=100, N=256, K=2048, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", with_bias=True),
    dict(M=128, N=384, K=4096, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=300, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", int_zeros=False),
    dict(M=512, N=512, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=128, N=256, K=1024, W_dtype="uint2", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=128, N=256, K=1024, W_dtype="int2", group_size=-1, with_scaling=True),
    dict(M=128, N=256, K=1024, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", fast_decoding=True, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=128, N=256, K=1024, W_dtype="uint4", out_dtype="float32", accum_dtype="float32", group_size=128, with_scaling=True),
    dict(M=9, N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=16, N=128, K=2048, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", with_bias=True),
    dict(M=32, N=256, K=1024, W_dtype="uint2", group_size=128, with_scaling=True),
    # more CTAs than SMs at BM = 128: several waves of tiles over the SMs
    dict(M=100, N=19200, K=512, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    # split-K (few output tiles, long K): fp32 partials in the workspace + reduce kernel
    dict(M=64, N=128, K=4096, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", with_bias=True),
    dict(M=40, N=256, K=8192, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=128, N=128, K=2048, W_dtype="uint2", group_size=64, with_scaling=True),
    # plain compressed storage (fast_decoding=False; the default for bfloat16 activations, general_matmul/__init__.py:174-176)
    dict(M=128, N=256, K=1024, W_dtype="uint4", fast_decoding=False, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=64, N=128, K=512, W_dtype="uint2", fast_decoding=False, group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=96, N=256, K=1024, W_dtype="int4", fast_decoding=False, group_size=-1, with_scaling=True),
    dict(M=128, N=256, K=1024, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=128, N=128, K=512, W_dtype="uint2", A_dtype="bfloat16", out_dtype="bfloat16", group_size=128, with_scaling=True),
    # group length of 3 k-blocks, not a power of two: the one-group-ahead parameter prefetch must name the right group
    dict(M=16, N=128, K=1536, W_dtype="uint4", group_size=192, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=100, N=256, K=1536, W_dtype="uint4", group_size=192, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=300, N=256, K=3072, W_dtype="uint4", group_size=192, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=64, N=128, K=1920, W_dtype="uint2", group_size=320, with_scaling=True),
]


@pytest.mark.parametrize("kw", GEMM_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
# (the name is kept from the Blackwell build so that test ids stay stable; the kernel under test is gemm_ts_wgmma)
def test_gemm_tcgen05_parity(kw):
    kw = dict(kw)
    case = H.make_case(kw.pop("M"), kw.pop("N"), kw.pop("K"), **kw)
    op, got, ref = _run(case, "gemm_ts_wgmma")
    H.assert_fp_close(got, ref, "gemm_ts")


W2A8_CASES = [
    dict(M=1, N=256, K=512, W_dtype="int2", out_dtype="int32"),
    dict(M=1, N=256, K=1024, W_dtype="int2", out_dtype="float32"),
    dict(M=7, N=256, K=1024, W_dtype="uint2", out_dtype="int32"),
    dict(M=32, N=256, K=512, W_dtype="int2", out_dtype="int32"),
    dict(M=16, N=256, K=512, W_dtype="int4", out_dtype="int32", fast_decoding=True),
    dict(M=128, N=256, K=1024, W_dtype="int2", out_dtype="int32"),
    dict(M=200, N=384, K=2048, W_dtype="int2", out_dtype="int32"),
    dict(M=128, N=256, K=1024, W_dtype="uint2", out_dtype="int32"),
    dict(M=64, N=128, K=512, W_dtype="int4", out_dtype="int32", fast_decoding=True),
    dict(M=128, N=256, K=1024, W_dtype="int2", out_dtype="int8"),
    dict(M=64, N=128, K=4096, W_dtype="int2", out_dtype="int32"),     # split-K, int32 partials
    dict(M=128, N=256, K=8192, W_dtype="int2", out_dtype="float32"),
    # W4A8 default is the plain compressed storage (general_matmul/__init__.py:171-173)
    dict(M=128, N=256, K=1024, W_dtype="int4", out_dtype="int32"),
    dict(M=64, N=128, K=512, W_dtype="uint4", out_dtype="int32"),
    dict(M=100, N=128, K=512, W_dtype="int2", out_dtype="int32", fast_decoding=False),
    dict(M=48, N=128, K=512, W_dtype="uint2", out_dtype="int32", fast_decoding=False),
]


@pytest.mark.parametrize("kw", W2A8_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_int8_activation_bit_exact(kw):
    kw = dict(kw)
    M = kw["M"]
    case = H.make_case(kw.pop("M"), kw.pop("N"), kw.pop("K"), A_dtype="int8", accum_dtype="int32", **kw)
    from bitblas_b200 import _lib
    il8 = case["cfg"]["fast_decoding"] is not False and not (case["cfg"]["W_dtype"] in ("int4", "uint4") and case["cfg"]["fast_decoding"] is None)
    if M <= 32 and il8:
        op, got, ref = _run(case, "gemv_i8", force=_lib.BB_KERNEL_GEMV_I8)
    else:
        op, got, ref = _run(case, "gemm_ts_wgmma_i8")
    assert torch.equal(got, ref)


GENERIC_CASES = [
    dict(M=1, N=64, K=256, W_dtype="nf4", group_size=64, with_scaling=True),
    dict(M=5, N=64, K=256, W_dtype="fp4_e2m1", group_size=-1, with_scaling=True),
    dict(M=2, N=64, K=256, W_dtype="e4m3_float8"),
    dict(M=1, N=64, K=256, W_dtype="int1"),
    dict(M=3, N=64, K=256, W_dtype="uint1", group_size=32, with_scaling=True, with_zeros=True, zeros_mode="original"),
    dict(M=1, N=256, K=256, W_dtype="int4", group_size=32, with_scaling=True),   # reference GEMV case, g=32
    dict(M=1, N=256, K=256, W_dtype="uint4", group_size=32, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(M=40, N=48, K=96, W_dtype="uint4", group_size=32, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(M=9, N=64, K=256, W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", group_size=64, with_scaling=True),
    dict(M=6, N=64, K=256, W_dtype="int8", A_dtype="float16"),
]


@pytest.mark.parametrize("kw", GENERIC_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_generic_kernel_parity(kw):
    kw = dict(kw)
    case = H.make_case(kw.pop("M"), kw.pop("N"), kw.pop("K"), **kw)
    if case["fmt"] == "fp_e4m3":  # keep to normal e4m3 codes (the reference's bit trick is wrong for 0/subnormals)
        f = case["fields"]
        case["fields"] = torch.where((f & 0x78) == 0, f | 0x08, f)
        case["fields"] = torch.where((case["fields"] & 0x7F) == 0x7F, case["fields"] & 0xF7, case["fields"])
    op, got, ref = _run(case, "generic_simt")
    H.assert_fp_close(got, ref, "generic")


# 16-entry table formats (NF4 / "fp4") on the fast kernels: PRMT table decode in the decode GEMV (m = 1) and in the wgmma dequant
# warps (m > 1); reference semantics matmul_dequantize_impl.py:424-430 (nf: LUT[w]) and quantization.py:141-156 (fp4), support
# matrix README.md:61-88.  Same oracle, same tolerance as every other float case.
TABLE_CASES = [
    dict(M=1, N=256, K=2048, W_dtype="nf4", group_size=128, with_scaling=True),
    dict(M=1, N=4096, K=4096, W_dtype="nf4", group_size=128, with_scaling=True),
    dict(M=1, N=512, K=1024, W_dtype="nf4", A_dtype="bfloat16", out_dtype="bfloat16", accum_dtype="float32", group_size=128, with_scaling=True),
    dict(M=1, N=256, K=2048, W_dtype="fp4_e2m1", group_size=-1, with_scaling=True),
    dict(M=1, N=256, K=1024, W_dtype="fp4_e2m1"),
    dict(M=16, N=256, K=2048, W_dtype="nf4", group_size=128, with_scaling=True, with_bias=True),
    dict(M=64, N=128, K=8192, W_dtype="fp4_e2m1", group_size=128, with_scaling=True),        # split-K
    dict(M=300, N=256, K=2048, W_dtype="nf4", group_size=64, with_scaling=True),
    dict(M=128, N=256, K=1024, W_dtype="nf4", A_dtype="bfloat16", out_dtype="bfloat16", accum_dtype="float32", group_size=128, with_scaling=True),
    dict(M=200, N=384, K=1024, W_dtype="fp4_e2m1", A_dtype="bfloat16", out_dtype="bfloat16", accum_dtype="float32"),
]


@pytest.mark.parametrize("kw", TABLE_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_table_formats_fast_kernels(kw):
    kw = dict(kw)
    M = kw["M"]
    case = H.make_case(kw.pop("M"), kw.pop("N"), kw.pop("K"), **kw)
    bf = kw.get("A_dtype") == "bfloat16"
    op, got, ref = _run(case, "gemv_slab" if M == 1 else "gemm_ts_wgmma")
    H.assert_fp_close(got, ref, f"table format {kw['W_dtype']} M={M}", max_mismatched_ratio=2e-3 if bf else 0.0)
    # and the generic kernel on the same inputs (the spec-order implementation these formats used before)
    from bitblas_b200 import _lib
    op2, got2, _ = _run(case, "generic_simt", force=_lib.BB_KERNEL_GENERIC)
    H.assert_fp_close(got, got2, "fast vs generic", max_mismatched_ratio=2e-3 if bf else 0.0)


@pytest.mark.parametrize("wd", ["e4m3_float8", "e5m2_float8"])
@pytest.mark.parametrize("M,N,K,adt", [(1, 256, 1024, "float16"), (16, 256, 2048, "float16"), (300, 384, 1024, "float16"),
                                       (64, 128, 8192, "float16"), (128, 256, 1024, "bfloat16")])
def test_fp8_weights_tcgen05(wd, M, N, K, adt):
    """8-bit float weights x 16-bit activations on the wgmma kernel (README.md:61-88 support matrix; decode formulas
    quantization.py:169-182).  e4m3 codes are kept to normal numbers like in the generic-kernel test: the reference's bit trick
    maps the zero / subnormal codes to large garbage values, and sums of those overflow fp16."""
    bf = adt == "bfloat16"
    case = H.make_case(M, N, K, A_dtype=adt, W_dtype=wd, out_dtype=adt, accum_dtype="float32" if bf else "float16", seed=M + K)
    f = case["fields"]
    if wd == "e4m3_float8":
        f = torch.where((f & 0x78) == 0, f | 0x08, f)
        f = torch.where((f & 0x7F) == 0x7F, f & 0xF7, f)
        f = torch.where((f & 0x78) >= 0x50, f & 0xCF, f)       # |w| < 8: keeps K-long sums inside fp16
    else:
        f = torch.where((f & 0x7C) == 0x7C, f & 0xBF, f)       # no inf / nan codes
        f = torch.where((f & 0x7C) >= 0x48, f & 0xB7 | 0x20, f)  # moderate magnitudes
    case["fields"] = f
    op, got, ref = _run(case, "gemm_ts_wgmma")
    H.assert_fp_close(got, ref, f"{wd} M={M}", max_mismatched_ratio=2e-3 if bf else 0.0)
    from bitblas_b200 import _lib
    _, got2, _ = _run(case, "generic_simt", force=_lib.BB_KERNEL_GENERIC)
    H.assert_fp_close(got, got2, "fast vs generic", max_mismatched_ratio=2e-3 if bf else 0.0)


def test_fast_kernels_agree_with_generic_on_device():
    """on-device cross check: same inputs through the forced generic kernel and the auto-dispatched one."""
    from bitblas_b200 import _lib
    lib = _lib.load()
    for M in (1, 16, 128):
        case = H.make_case(M, 256, 1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                           zeros_mode="quantized", with_bias=True, seed=M)
        op = H.product_operator(case)
        fast = H.run_product(op, case)
        prev = lib.bb_set_kernel_override(_lib.BB_KERNEL_GENERIC)
        try:
            slow = H.run_product(op, case)
        finally:
            lib.bb_set_kernel_override(prev)
        H.assert_fp_close(fast, slow, f"fast-vs-generic M={M}")


def test_empty_and_error_paths():
    case = H.make_case(4, 256, 512, W_dtype="uint4", group_size=128, with_scaling=True)
    op = H.product_operator(case, M=[1, 16])
    W = H.product_weight(op, case)
    s = case["scale"].cuda()
    out = op(torch.empty((0, 512), dtype=torch.float16, device="cuda"), W, scale=s)
    assert out.shape == (0, 256)
    with pytest.raises(RuntimeError):
        op(case["A"], W, scale=s)                     # CPU activations: no CPU path
    with pytest.raises(ValueError):
        op(case["A"].cuda()[:, :256].contiguous(), W, scale=s)   # wrong K
    with pytest.raises(ValueError):
        op(case["A"].cuda(), W)                        # missing scale
    with pytest.raises(TypeError):
        op(case["A"].cuda().float(), W, scale=s)       # wrong dtype


def test_linear_module_and_state_dict_roundtrip():
    import bitblas_b200 as bitblas
    case = H.make_case(8, 256, 1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                       zeros_mode="quantized", with_bias=True)
    lin = bitblas.Linear(1024, 256, bias=True, A_dtype="float16", W_dtype="uint4", accum_dtype="float16", out_dtype="float16",
                         group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", enable_tuning=False).cuda()
    lin.load_and_transform_weight(case["fields"].to(torch.int8).cuda(), scales=case["scale"].cuda(),
                                  zeros=case["zeros"].cuda(), bias=case["bias"].cuda())
    ref = H.oracle_output(case)
    got = lin(case["A"].cuda()).cpu()
    H.assert_fp_close(got, ref, "Linear")
    # 3-d input (batch, seq, K) -> m = batch*seq (module/__init__.py:282-284)
    got3 = lin(case["A"].cuda().reshape(2, 4, 1024)).cpu().reshape(8, 256)
    assert torch.equal(got3, got)
    lin2 = bitblas.Linear(1024, 256, bias=True, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
                          with_zeros=True, zeros_mode="quantized", enable_tuning=False)
    lin2.load_state_dict(lin.state_dict())
    assert torch.equal(lin2.cuda()(case["A"].cuda()).cpu(), got)


def test_gptq_repack_device_matches_reference_loops():
    """bb_repack_gptq_*_device vs the reference's python unpack (module/__init__.py:24-74) restated in the oracle."""
    import bitblas_oracle as O
    import numpy as np
    import bitblas_b200 as bitblas
    torch.manual_seed(0)
    K, N, g, bits = 512, 256, 128, 4
    intw = torch.randint(0, 16, (K, N), dtype=torch.int32)     # GPTQ: [K, N]
    qweight = torch.zeros((K * bits // 32, N), dtype=torch.int32)
    for k in range(K):
        qweight[k // 8] |= intw[k] << (4 * (k % 8))
    zint = torch.randint(0, 15, (K // g, N), dtype=torch.int32)
    qzeros = torch.zeros((K // g, N * bits // 32), dtype=torch.int32)
    for n in range(N):
        qzeros[:, n // 8] |= zint[:, n] << (4 * (n % 8))
    scales = (torch.rand(K // g, N) * 0.1 + 0.01).half()

    class G:  # minimal stand-in for an auto_gptq QuantLinear
        pass
    gm = G(); gm.qweight = qweight; gm.qzeros = qzeros; gm.scales = scales; gm.bias = None
    for mode in ("original", "rescale", "quantized"):
        lin = bitblas.Linear(K, N, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True,
                             zeros_mode=mode, enable_tuning=False).cuda()
        lin.repack_from_gptq(gm)
        fields = intw.T.contiguous()                              # [N, K]
        exp_w = O.transform_weight(fields.to(torch.int8), "uint4", "float16", fast_decoding=True)
        assert torch.equal(lin.qweight.cpu(), exp_w)
        zi = O.unpack_qzeros(qzeros, bits).T.contiguous()        # [N, G], +1 applied
        if mode == "original":
            assert torch.equal(lin.zeros.cpu(), zi.half())
        elif mode == "rescale":
            assert torch.equal(lin.zeros.cpu(), zi.half() * scales.T.contiguous())
        else:
            assert torch.equal(lin.zeros.cpu(), torch.from_numpy(O.general_compress(zi.T.contiguous().numpy(), bits)))
        A = (torch.rand(4, K) - 0.5).half()
        ref = O.matmul_dequant(A, fields, W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True,
                               zeros_mode=mode, scale=scales.T.contiguous(), zeros=lin.zeros.cpu())
        H.assert_fp_close(lin(A.cuda()).cpu(), ref, f"gptq-{mode}")


@pytest.mark.parametrize("bits", [4, 2])
@pytest.mark.parametrize("m", [1, 16])
def test_gptq_repack_v2_module(bits, m):
    """Linear.repack_from_gptq_v2 (bitblas/module/__init__.py:340-363; testing/python/module/test_repack_from_gptq_v2.py): the
    v2 checkpoint format stores the zero point itself (no +1, unpack_qzeros_v2 :43-58).  A synthetic GPTQ module (int32-packed
    qweight [K*bits/32, N], qzeros [K/g, N*bits/32], scales [K/g, N], bias) is repacked on the device for every zeros mode and
    the module output is compared with the dequantised dense layer, m = 1 (GEMV) and m = 16 (tensor-core path)."""
    import bitblas_oracle as O
    import bitblas_b200 as bitblas
    torch.manual_seed(1)
    K, N, g = 1024, 512, 128
    per = 32 // bits
    intw = torch.randint(0, 2**bits, (K, N), dtype=torch.int32)
    qweight = torch.zeros((K // per, N), dtype=torch.int32)
    for k in range(K):
        qweight[k // per] |= intw[k] << (bits * (k % per))
    zint = torch.randint(0, 2**bits, (K // g, N), dtype=torch.int32)   # v2: the full range is representable
    qzeros = torch.zeros((K // g, N // per), dtype=torch.int32)
    for n in range(N):
        qzeros[:, n // per] |= zint[:, n] << (bits * (n % per))
    scales = (torch.rand(K // g, N) * 0.1 + 0.01).half()
    bias = torch.rand(N).half()

    class G:
        pass
    gm = G(); gm.qweight = qweight; gm.qzeros = qzeros; gm.scales = scales
    gm.bias = torch.nn.Parameter(bias.clone(), requires_grad=False)
    dense = ((intw.T.float() - zint.T.repeat_interleave(g, dim=1).float()) * scales.T.repeat_interleave(g, dim=1).float())   # [N, K]
    A = (torch.rand(m, K) - 0.5).half()
    ref = (A.float() @ dense.t() + bias.float()).half()
    assert torch.equal(O.unpack_qzeros(qzeros, bits, v2=True).T.contiguous(), zint.T.contiguous().to(torch.int8))
    for mode in ("original", "rescale", "quantized"):
        lin = bitblas.Linear(K, N, bias=True, A_dtype="float16", W_dtype=f"uint{bits}", group_size=g, with_scaling=True,
                             with_zeros=True, zeros_mode=mode, enable_tuning=False).cuda()
        lin.repack_from_gptq_v2(gm)
        fields = intw.T.contiguous()
        assert torch.equal(lin.qweight.cpu(), O.transform_weight(fields.to(torch.int8), f"uint{bits}", "float16", fast_decoding=True))
        if mode == "original":
            assert torch.equal(lin.zeros.cpu(), zint.T.contiguous().half())
        elif mode == "quantized":
            assert torch.equal(lin.zeros.cpu(), torch.from_numpy(O.general_compress(zint.to(torch.int8).numpy(), bits)))
        got = lin(A.cuda()).cpu()
        H.assert_fp_close(got, ref, f"gptq-v2 {mode} bits={bits} m={m}")


# ---- BASELINE.json configs[2] / [3] at their real shapes: W4A16 GEMM M in {16, 128, 4096} on the Llama-2-70B linears and the
# 12288^2 target, W2A8 INT32 at 12288^2 (mirrors testing/python/operators/test_general_matmul_ops_backend_tl.py:127-283) --------
_BASELINE_NK = [(8192, 8192), (28672, 8192), (8192, 28672), (12288, 12288)]


@pytest.mark.parametrize("N,K", _BASELINE_NK, ids=lambda v: str(v))
def test_gemm_ts_baseline_shapes(N, K):
    """one weight matrix per shape, M = 16 / 128 (every output row) and M = 4096 (64 sampled rows x all N columns: the oracle's
    CPU matmul on all 4096 rows would take minutes); GPTQ-style quantized zeros, group 128."""
    import bitblas_oracle as O
    import bitblas_b200 as bitblas
    g = torch.Generator().manual_seed(N + K)
    fields = torch.randint(0, 16, (N, K), generator=g, dtype=torch.int8)
    scale = (torch.rand((N, K // 128), generator=g) * 0.125 + 0.01).half()
    zq = torch.randint(0, 16, (K // 128, N), generator=g, dtype=torch.int8)
    qz = torch.from_numpy(O.general_compress(zq.numpy(), 4))
    cfg = bitblas.MatmulConfig(M=[16, 128, 4096], N=N, K=K, A_dtype="float16", W_dtype="uint4", accum_dtype="float16",
                               out_dtype="float16", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
    op = bitblas.Matmul(cfg, enable_tuning=False)
    W = op.transform_weight(fields.cuda())
    sc, zz = scale.cuda(), qz.cuda()
    Wd = O.dequantize_weight(fields.to(torch.int32), W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                             zeros_mode="quantized", scale=scale, zeros=qz).float()
    for M in (16, 128, 4096):
        assert op.kernel_for(M) == "gemm_ts_wgmma"
        A = (torch.rand((M, K), generator=g) - 0.5).half()
        got = op.forward(A.cuda(), W, scale=sc, zeros=zz).cpu()
        rows = torch.arange(M) if M <= 128 else torch.randperm(M, generator=g)[:64].sort().values
        ref = (A[rows].float() @ Wd.t()).half()
        H.assert_fp_close(got[rows], ref, f"gemm_ts M={M} {N}x{K}")


@pytest.mark.parametrize("M", [1, 128])
def test_w2a8_baseline_shape(M):
    """BASELINE configs[3]: W2A8 (BitNet b1.58: int8 activations x ternary int2 weights), int32 accumulate, N = K = 12288: exact."""
    import bitblas_b200 as bitblas
    N = K = 12288
    g = torch.Generator().manual_seed(5)
    Wt = torch.randint(-1, 2, (N, K), generator=g, dtype=torch.int8)
    A = torch.randint(-128, 128, (M, K), generator=g, dtype=torch.int8)
    cfg = bitblas.MatmulConfig(M=M, N=N, K=K, A_dtype="int8", W_dtype="int2", accum_dtype="int32", out_dtype="int32")
    op = bitblas.Matmul(cfg, enable_tuning=False)
    W = op.transform_weight(Wt.cuda())
    got = op.forward(A.cuda(), W).cpu()
    ref = (A.double() @ Wt.double().t()).to(torch.int32)   # |sum| <= 12288 * 128: exact in float64
    assert torch.equal(got, ref)
