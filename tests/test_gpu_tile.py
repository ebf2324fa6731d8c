"""MatmulConfig(propagate_b=True): BB_TILE_SLAB weight storage (include/bitblas_b200.h) through every kernel that consumes it --
the decode GEMV (one contiguous 16 KB bulk copy per unit), the wgmma GEMM (4-D TMA box over the tiled tensor) and the generic
kernel (tiled addressing) -- against the CPU oracle, and bit for bit against the same operator on the row-major storage.
Mirrors the role of the reference's propagate_b cases in testing/python/operators/test_general_matmul_ops.py (weight propagation
must not change the result)."""
import numpy as np
import pytest
import torch

import bitblas_oracle as O
import helpers as H

pytestmark = pytest.mark.gpu


def _ops(case, M):
    import bitblas_b200 as bitblas
    c = case["cfg"]
    mk = lambda pb: bitblas.Matmul(bitblas.MatmulConfig(  # noqa: E731
        M=M, N=case["N"], K=case["K"], A_dtype=c["A_dtype"], W_dtype=c["W_dtype"], accum_dtype=c["accum_dtype"], out_dtype=c["out_dtype"],
        with_bias=c["with_bias"], group_size=c["group_size"], with_scaling=c["with_scaling"], with_zeros=c["with_zeros"],
        zeros_mode=c["zeros_mode"], propagate_b=pb), enable_tuning=False)
    return mk(False), mk(True)


def test_device_retile_matches_definition():
    g = torch.Generator().manual_seed(1)
    w = torch.randint(-128, 128, (160, 1536), generator=g, dtype=torch.int8)
    case = H.make_case(1, 256, 2048, W_dtype="uint4")
    _, opt = _ops(case, 1)
    t = opt.tile_weight(w.cuda())
    assert np.array_equal(t.cpu().numpy(), O.slab_tile(w.numpy()))
    assert torch.equal(opt.tile_weight(t, inverse=True).cpu(), w)
    assert torch.equal(opt.tile_weight(w), t.cpu())          # host permute == device kernel


TILE_CASES = [
    # M, N, K, A_dtype, W_dtype, zeros_mode, bias, group
    (1, 256, 2048, "float16", "uint4", "quantized", True, 128),      # gemv_slab, bulk-copy units
    (1, 4096, 4096, "float16", "uint4", "original", False, 128),     # gemv_slab, stream-K over many CTAs
    (1, 1024, 8192, "bfloat16", "uint4", "rescale", False, 128),
    (1, 256, 2048, "float16", "int4", None, False, -1),
    (4, 256, 2048, "float16", "uint4", "quantized", False, 128),     # small m on the tiled storage: wgmma BM=32
    (16, 128, 8192, "float16", "uint4", "quantized", True, 128),     # split-K
    (100, 384, 2048, "float16", "uint4", "original", False, 128),
    (300, 256, 4096, "float16", "uint4", "quantized", True, 128),    # BM=128, three m-tiles
    (64, 256, 4096, "float16", "uint2", "quantized", False, 128),    # 2-bit: 16-byte box rows
    (1, 256, 4096, "float16", "uint2", "original", False, 128),
    (1, 256, 4096, "int8", "int2", None, False, -1),                 # W2A8 on the tiled storage (wgmma int8)
    (128, 256, 4096, "int8", "int2", None, False, -1),
]


@pytest.mark.parametrize("M,N,K,adt,wdt,zm,bias,g", TILE_CASES)
def test_tiled_matches_row_major_and_oracle(M, N, K, adt, wdt, zm, bias, g):
    int_path = adt == "int8"
    signed = wdt.startswith("int")
    case = H.make_case(M, N, K, A_dtype=adt, W_dtype=wdt, accum_dtype="int32" if int_path else ("float32" if adt == "bfloat16" else "float16"),
                       out_dtype="int32" if int_path else adt, group_size=g, with_scaling=not signed, with_zeros=zm is not None,
                       zeros_mode=zm or "original", with_bias=bias and not int_path, seed=M + N + K)
    op0, opt = _ops(case, M)
    assert opt.weight_tiled, "legalisation dropped the tiling for a supported shape"
    dev = torch.device("cuda")
    W0 = H.product_weight(op0, case, dev)          # the reference tests' weight_transform(intweight) on the row-major operator
    Wt = opt.tile_weight(W0)                         # (Matmul.transform_weight applies exactly this after the same transform)
    assert np.array_equal(Wt.cpu().numpy(), O.slab_tile(W0.cpu().numpy()))
    kw = {k: (case[k].to(dev) if case[k] is not None else None) for k in ("scale", "zeros", "bias")}
    A = case["A"].to(dev)
    out0 = op0.forward(A, W0, **kw)
    outt = opt.forward(A, Wt, **kw)
    torch.cuda.synchronize()
    ref = H.oracle_output(case)
    if int_path:
        assert torch.equal(outt.cpu(), ref), f"tiled {opt.kernel_for(M)} != oracle"
        assert torch.equal(out0.cpu(), ref)
    else:
        H.assert_fp_close(outt.cpu(), ref, f"tiled M={M} kernel={opt.kernel_for(M)}", max_mismatched_ratio=2e-3 if adt == "bfloat16" else 0.0)
        if op0.kernel_for(M) == opt.kernel_for(M):
            assert torch.equal(outt, out0), "same kernel, same arithmetic: tiled and row-major results must be identical"
    # the generic kernel reads the tiled storage through its own addressing
    from bitblas_b200 import _lib
    lib = _lib.load()
    prev = lib.bb_set_kernel_override(_lib.BB_KERNEL_GENERIC)
    try:
        assert opt.kernel_for(M) == "generic_simt"
        outg = opt.forward(A, Wt, **kw)
        torch.cuda.synchronize()
    finally:
        lib.bb_set_kernel_override(prev)
    if int_path:
        assert torch.equal(outg.cpu(), ref)
    else:
        H.assert_fp_close(outg.cpu(), ref, "generic on tiled storage", max_mismatched_ratio=2e-3 if adt == "bfloat16" else 0.0)


def test_tiled_baseline_shape_decode():
    """the headline shape on the tiled storage: full output against the oracle on a row sample, identical to row-major"""
    N, K = 12288, 12288
    case = H.make_case(1, N, K, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", seed=77)
    op0, opt = _ops(case, 1)
    dev = torch.device("cuda")
    W0 = op0.transform_weight(case["fields"].to(torch.int8).to(dev))
    Wt = opt.transform_weight(case["fields"].to(torch.int8).to(dev))
    kw = {k: case[k].to(dev) for k in ("scale", "zeros")}
    A = case["A"].to(dev)
    out0, outt = op0.forward(A, W0, **kw), opt.forward(A, Wt, **kw)
    torch.cuda.synchronize()
    assert opt.kernel_for(1) == "gemv_slab" and torch.equal(out0, outt)
    H.assert_fp_close(outt.cpu(), H.oracle_output(case), "12288^2 tiled")


def test_linear_propagate_b_gptq_repack():
    """bitblas.Linear(propagate_b=True).repack_from_gptq: the GPTQ ingest lands in the tiled storage"""
    import bitblas_b200 as bitblas
    N, K, g = 256, 2048, 128
    gen = torch.Generator().manual_seed(3)
    intw = torch.randint(0, 16, (K, N), generator=gen, dtype=torch.int32)
    qweight = torch.zeros((K // 8, N), dtype=torch.int32)
    for k in range(K):
        qweight[k // 8] |= intw[k] << (4 * (k % 8))
    zint = torch.randint(0, 16, (K // g, N), generator=gen, dtype=torch.int32)
    qzeros = torch.zeros((K // g, N // 8), dtype=torch.int32)
    for n in range(N):
        qzeros[:, n // 8] |= zint[:, n] << (4 * (n % 8))

    class G:  # GPTQ v2 checkpoint layout (bitblas/module/__init__.py:340-363)
        pass
    gm = G(); gm.qweight = qweight; gm.qzeros = qzeros
    gm.scales = (torch.rand((K // g, N), generator=gen) * 0.1 + 0.01).half()
    gm.bias = None
    lin_t = bitblas.Linear(K, N, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True,
                           zeros_mode="quantized", enable_tuning=False, propagate_b=True).cuda()
    lin_0 = bitblas.Linear(K, N, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True,
                           zeros_mode="quantized", enable_tuning=False).cuda()
    lin_t.repack_from_gptq_v2(gm)
    lin_0.repack_from_gptq_v2(gm)
    assert lin_t.bitblas_matmul.weight_tiled
    assert np.array_equal(lin_t.qweight.cpu().numpy(), O.slab_tile(lin_0.qweight.cpu().numpy()))
    x = (torch.rand((3, K), generator=gen) - 0.5).half().cuda()
    y_t, y_0 = lin_t(x), lin_0(x)
    x1 = x[:1]
    assert torch.equal(lin_t(x1), lin_0(x1))
    torch.testing.assert_close(y_t.float(), y_0.float(), rtol=1e-2, atol=1e-2)
