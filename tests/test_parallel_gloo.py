"""CPU, world_size 2, gloo: the host logic of the column-parallel path (sharding + all-gather re-assembly).

There is no CPU matmul in the product, so each rank's local operator is replaced by a stand-in that evaluates
the ORACLE on that rank's shard (test infrastructure only) -- what is under test is shard_quantized_params,
the chunked all-gather and the [G, rows, N/G] -> [rows, N] re-assembly of ColumnParallelLinear.forward."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, chunks, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import bitblas_oracle as O
        import helpers as H
        from bitblas_b200.parallel import ColumnParallelLinear, shard_quantized_params
        M, N, K, g = 12, 64, 256, 128
        for mode, tiled in (("original", False), ("quantized", False), ("quantized", True)):
            if tiled:
                N, K = 384, 2048  # propagate_b: the full weight is slab-tiled (N % 128 == 0, 1024 bytes per row), the 192-row shard is not
            case = H.make_case(M, N, K, W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True, zeros_mode=mode,
                               with_bias=True, seed=7)
            full_ref = H.oracle_output(case)
            layer = ColumnParallelLinear(K, N, bias=True, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True,
                                         with_zeros=True, zeros_mode=mode, enable_tuning=False, pipeline_chunks=chunks, propagate_b=tiled)
            op = layer.local.bitblas_matmul
            assert not op.weight_tiled
            import bitblas_b200 as bitblas
            full_op = bitblas.Matmul(bitblas.MatmulConfig(M=M, N=N, K=K, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True,
                                                          with_zeros=True, zeros_mode=mode, propagate_b=tiled), enable_tuning=False)
            assert full_op.weight_tiled == tiled
            stored = full_op.transform_weight(case["fields"].to(torch.int8))        # full-size, in the full layer's own storage
            layer.load_full_params(stored, case["scale"], case["zeros"], case["bias"])
            if tiled:
                stored = full_op.tile_weight(stored, inverse=True)
            lo, hi = layer.n_lo, layer.n_hi
            assert (lo, hi) == (rank * N // world, (rank + 1) * N // world)
            assert torch.equal(layer.local.qweight, stored[lo:hi])
            sh = shard_quantized_params(stored, case["scale"], case["zeros"], case["bias"], rank=rank, world=world, bits=4,
                                        zeros_mode=mode)
            shard_fields = torch.from_numpy(O.general_decompress(
                O.deinterleave_weight(sh["qweight"].numpy(), 4, "float16"), 4)).to(torch.int32)
            assert torch.equal(shard_fields, case["fields"][lo:hi])

            def fake_local(x, _sh=sh, _f=shard_fields, _mode=mode):
                return O.matmul_dequant(x, _f, W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True,
                                        zeros_mode=_mode, scale=_sh["scales"], zeros=_sh["zeros"], bias=_sh["bias"])

            layer.local.forward = fake_local
            out = layer(case["A"])
            assert out.shape == (M, N)
            assert torch.equal(out, full_ref), f"rank {rank} mode {mode}"
            out3 = layer(case["A"].reshape(3, 4, K))
            assert torch.equal(out3.reshape(M, N), full_ref)
        ret[rank] = "ok"
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("chunks", [1, 3])
def test_column_parallel_world2(chunks):
    world = 2
    port = 29500 + os.getpid() % 1000 + chunks
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, chunks, ret), nprocs=world, join=True)
    assert dict(ret) == {0: "ok", 1: "ok"}


def _row_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import bitblas_oracle as O
        import helpers as H
        from bitblas_b200.parallel import RowParallelLinear
        M, N, g = 6, 64, 128
        for mode, tiled, K in (("original", False, 2048), ("quantized", False, 2048), ("quantized", True, 2048), ("quantized", True, 3072)):
            if tiled:
                N = 128          # slab tiling needs N % 128 == 0 and (K/world)/2 % 512 == 0
            # K = 3072: the full weight is slab-tiled (1536 bytes per row), the world-2 shard (768 bytes per row) is not
            shard_tiled = tiled and K == 2048
            case = H.make_case(M, N, K, W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True, zeros_mode=mode, with_bias=True,
                               seed=11)
            layer = RowParallelLinear(K, N, bias=True, input_is_parallel=False, A_dtype="float16", W_dtype="uint4", group_size=g,
                                      with_scaling=True, with_zeros=True, zeros_mode=mode, enable_tuning=False, propagate_b=tiled)
            op = layer.local.bitblas_matmul
            assert op.weight_tiled == shard_tiled and op.config.K == K // world and op.config.out_dtype == "float32"
            import bitblas_b200 as bitblas
            full_op = bitblas.Matmul(bitblas.MatmulConfig(M=M, N=N, K=K, A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True,
                                                          with_zeros=True, zeros_mode=mode, propagate_b=tiled), enable_tuning=False)
            assert full_op.weight_tiled == tiled
            stored = full_op.transform_weight(case["fields"].to(torch.int8))        # full-size, in the full layer's own storage
            layer.load_full_params(stored, case["scale"], case["zeros"], case["bias"])
            lo, hi = layer.k_lo, layer.k_hi
            assert (lo, hi) == (rank * K // world, (rank + 1) * K // world)
            # the shard decodes to exactly this rank's K range of the original fields
            w_local = op.tile_weight(layer.local.qweight, inverse=True) if shard_tiled else layer.local.qweight
            shard_fields = torch.from_numpy(O.general_decompress(O.deinterleave_weight(w_local.numpy(), 4, "float16"), 4)).to(torch.int32)
            assert torch.equal(shard_fields, case["fields"][:, lo:hi])
            sc, zz = layer.local.scales, layer.local.zeros

            def fake_local(x, _f=shard_fields, _sc=sc, _zz=zz, _mode=mode):       # oracle partial product in fp32 (no CPU matmul in the product)
                return O.matmul_dequant(x, _f, W_dtype="uint4", accum_dtype="float32", out_dtype="float32", group_size=g, with_scaling=True,
                                        with_zeros=True, zeros_mode=_mode, scale=_sc, zeros=_zz)

            layer.local.forward = fake_local
            out = layer(case["A"])
            ref = O.matmul_dequant(case["A"], case["fields"], W_dtype="uint4", accum_dtype="float32", out_dtype="float32", group_size=g,
                                   with_scaling=True, with_zeros=True, zeros_mode=mode, scale=case["scale"], zeros=case["zeros"])
            ref = (ref.to(torch.float16) + case["bias"])
            assert out.dtype == torch.float16 and out.shape == (M, N)
            torch.testing.assert_close(out.float(), ref.float(), rtol=2e-3, atol=2e-3)
        ret[rank] = "ok"
    finally:
        dist.destroy_process_group()


def test_row_parallel_world2():
    world = 2
    port = 29700 + os.getpid() % 1000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_row_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {0: "ok", 1: "ok"}


def test_shard_k_errors():
    from bitblas_b200.parallel import shard_quantized_params_k
    w = torch.zeros((16, 512), dtype=torch.int8)
    with pytest.raises(ValueError):
        shard_quantized_params_k(w, None, None, rank=0, world=3, K=1024, bits=4, group_size=128)
    with pytest.raises(ValueError):
        shard_quantized_params_k(w, None, None, rank=0, world=2, K=1024, bits=4, group_size=1024)
    sh = shard_quantized_params_k(w, torch.zeros((16, 8)), torch.zeros((8, 8), dtype=torch.int8), rank=1, world=2, K=1024, bits=4,
                                  group_size=128, zeros_mode="quantized")
    assert sh["qweight"].shape == (16, 256) and sh["scales"].shape == (16, 4) and sh["zeros"].shape == (4, 8)


def test_shard_bounds_errors():
    from bitblas_b200.parallel import shard_bounds
    assert shard_bounds(12288, 3, 8) == (4608, 6144)
    with pytest.raises(ValueError):
        shard_bounds(100, 0, 8)
    with pytest.raises(ValueError):
        shard_bounds(8 * 24, 0, 8)
