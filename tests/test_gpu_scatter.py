"""Column-parallel scatter epilogue (bb_matmul_scatter) on ONE device: two local [m, ldc] buffers stand in for the peers'
symmetric-memory outputs.  The result in every destination must equal the plain bb_matmul output bit for bit (same kernel, same
arithmetic; only the store path differs), in the right column
window, and nothing outside the window may be touched.  The real multi-GPU run is tests/test_gpu_multi.py."""
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu


def _tensors(op, case, dev):
    return dict(W=H.product_weight(op, case, dev), scale=case["scale"].to(dev) if case["scale"] is not None else None,
                zeros=case["zeros"].to(dev) if case["zeros"] is not None else None,
                bias=case["bias"].to(dev) if case["bias"] is not None else None)

CASES = [
    # M, N, K, A_dtype, out_dtype, bias, group
    (1, 256, 1024, "float16", "float16", True, 128),      # gemv_slab
    (4, 256, 1024, "float16", "float16", False, 128),     # gemv_mma
    (16, 128, 8192, "float16", "float16", True, 128),     # wgmma BM=32, split-K + reduce kernel
    (40, 256, 1024, "float16", "float16", True, 128),     # BM=64, ragged rows
    (100, 384, 2048, "float16", "float16", False, 128),   # BM=128, ragged rows
    (300, 256, 1024, "float16", "float16", True, 128),    # BM=128: third m-tile has 44 valid rows
    (512, 512, 2048, "bfloat16", "bfloat16", True, 128),  # bf16 output
    (257, 256, 1024, "float16", "float16", False, -1),    # one valid row in the last tile
]


@pytest.mark.parametrize("M,N,K,adt,odt,bias,g", CASES)
def test_scatter_matches_plain(M, N, K, adt, odt, bias, g):
    case = H.make_case(M, N, K, A_dtype=adt, W_dtype="uint4", accum_dtype="float32" if adt == "bfloat16" else "float16", out_dtype=odt,
                       group_size=g, with_scaling=True, with_zeros=True, zeros_mode="quantized", with_bias=bias, seed=M + N)
    op = H.product_operator(case)
    dev = torch.device("cuda")
    t = _tensors(op, case, dev)
    A = case["A"].to(dev)
    plain = op.forward(A, t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    ldc, off = 2 * N + 64, N + 64 - 8 * (M % 2)        # offsets stay multiples of 8 elements (16-byte row segments)
    odtype = getattr(torch, odt)
    bufs = [torch.full((M, ldc), 7.0, dtype=odtype, device=dev) for _ in range(2)]
    op.forward_scatter(A, t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"],
                       peer_ptrs=[b.data_ptr() for b in bufs], ldc=ldc, col_offset=off)
    torch.cuda.synchronize()
    for b in bufs:
        assert torch.equal(b[:, off:off + N], plain), f"scatter != plain (kernel {op.kernel_for(M)})"
        assert bool((b[:, :off] == 7.0).all()) and bool((b[:, off + N:] == 7.0).all()), "stores outside the column window"
    # and against the oracle (the plain path's own parity tests cover it; this guards the test itself)
    H.assert_fp_close(plain.cpu(), H.oracle_output(case), f"M={M}")


def test_scatter_unaligned_window_falls_back():
    """a column window that is not 16-byte aligned must still be correct (scalar store path)"""
    M, N, K = 300, 256, 1024
    case = H.make_case(M, N, K, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized", seed=5)
    op = H.product_operator(case)
    dev = torch.device("cuda")
    t = _tensors(op, case, dev)
    A = case["A"].to(dev)
    plain = op.forward(A, t["W"], scale=t["scale"], zeros=t["zeros"])
    ldc, off = 2 * N + 3, 5
    bufs = [torch.zeros((M, ldc), dtype=torch.float16, device=dev) for _ in range(2)]
    op.forward_scatter(A, t["W"], scale=t["scale"], zeros=t["zeros"], peer_ptrs=[b.data_ptr() for b in bufs], ldc=ldc, col_offset=off)
    torch.cuda.synchronize()
    for b in bufs:
        assert torch.equal(b[:, off:off + N], plain)
