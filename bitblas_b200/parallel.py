"""Column-parallel (N-sharded) low-bit linear over the GPUs of one node.

The reference has no distributed code at all (SURVEY.md §2a "Collectives: none"); this is the optional multi-GPU
path BASELINE.json's north_star asks for.  The matmul shards naturally along N: output column n depends only on
row n of W / scales / zeros (column n of quantized zeros / bias), the per-int32 pack + interleave runs along K so a
row shard never splits a storage word.  Rank r of G owns rows [r*N/G, (r+1)*N/G); activations are replicated (as
in tensor-parallel inference); one exchange step -- an all-gather of the [m, N/G] partial outputs -- rebuilds C.

One process per GPU, ``torch.distributed`` (NCCL over NVLink5/NVSwitch; gloo on CPU for the host-logic tests).
For large m the all-gather is pipelined against the matmul in row chunks on a side stream so the transfer of
chunk i overlaps the wgmma kernel of chunk i+1.
"""
from __future__ import annotations

from typing import Optional

import ctypes

import torch
import torch.distributed as dist
import torch.nn as nn

from .module import Linear


class PeerBarrier:
    """Device-side barrier across the ranks of a group, one small kernel per call (bb_peer_barrier): ordered after the peer stores
    of the preceding bb_matmul_scatter launches on the same stream, CUDA-graph capturable, and -- being a programmatic dependent
    launch -- overlapped with the next matmul kernel's weight prefetch.  Replaces the symmetric-memory library barrier on the
    fused column-parallel path."""

    def __init__(self, device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        from . import _lib
        self._lib = _lib.load()
        self.group = group if group is not None else dist.group.WORLD
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.flags = symm_mem.empty((_lib.BB_PEER_FLAG_BYTES // 4,), dtype=torch.int32, device=device)
        self.flags.zero_()
        self.handle = symm_mem.rendezvous(self.flags, self.group)
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        self._arr = (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(p) for p in ptrs])
        torch.cuda.synchronize(device)
        self.handle.barrier(channel=0)          # every rank's flag block is zeroed before anyone signals into it
        torch.cuda.synchronize(device)
        self.device = device

    def __call__(self, stream=None):
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        rc = self._lib.bb_peer_barrier(self._arr, self.world, self.rank, st.cuda_stream)
        if rc != 0:
            from . import _lib
            raise RuntimeError(f"bb_peer_barrier failed (code {rc}): {_lib.last_error()}")


def shard_bounds(n: int, rank: int, world: int, multiple: int = 16):
    if n % world:
        raise ValueError(f"N={n} is not divisible by world size {world}")
    per = n // world
    if per % multiple:
        raise ValueError(f"N/world = {per} must be a multiple of {multiple}")
    return rank * per, (rank + 1) * per


def shard_quantized_params(qweight, scales, zeros, bias, *, rank: int, world: int, bits: int, zeros_mode: str = "original"):
    """Slice full-size BitBLAS-layout parameters for one rank (works on CPU or CUDA tensors)."""
    N = qweight.shape[0]
    lo, hi = shard_bounds(N, rank, world)
    out = {"qweight": qweight[lo:hi].contiguous()}
    if scales is not None:
        out["scales"] = scales[lo:hi].contiguous()
    if zeros is not None:
        if zeros_mode == "quantized":
            epb = 8 // bits
            if lo % epb or hi % epb:
                raise ValueError("shard boundary splits a packed zero-point byte")
            out["zeros"] = zeros[:, lo // epb:hi // epb].contiguous()
        else:
            out["zeros"] = zeros[lo:hi].contiguous()
    if bias is not None:
        out["bias"] = bias[lo:hi].contiguous()
    return out


class ColumnParallelLinear(nn.Module):
    """y = gather_N( x @ dequant(W_r)^T (+ b_r) ) with W sharded by rows (output features) across the group."""

    def __init__(self, in_features: int, out_features: int, *, process_group=None, gather_output: bool = True,
                 pipeline_chunks: Optional[int] = None, fused_gather: Optional[bool] = None, fused_ring: int = 2,
                 clone_output: bool = False, **linear_kwargs):
        super().__init__()
        # fused_gather: the matmul kernel's epilogue stores this rank's column slice straight into every rank's output
        # (peer-mapped symmetric memory over NVLink/NVSwitch) -- no separate collective, the transfer overlaps the math
        # tile by tile.  None = decided COLLECTIVELY at the first CUDA forward (every rank must be able to use it, else all
        # ranks take the NCCL all-gather; a rank-local choice would leave peers waiting in a rendezvous / barrier).
        # LIFETIME of the fused result: forward() returns a view into a ring of `fused_ring` symmetric buffers; it stays
        # valid until `fused_ring - 1` further forward() calls of this layer have been issued (the call after that lets the
        # peers overwrite it).  Pass clone_output=True (one extra copy) or a deeper ring to hold results longer.
        if fused_ring < 2:
            raise ValueError("fused_ring must be >= 2 (a rank may only overwrite a buffer after the next call's barrier)")
        self.fused_gather = fused_gather
        self.fused_ring = int(fused_ring)
        self.clone_output = bool(clone_output)
        self._fused_decided = fused_gather is False
        self._symm = {}       # (rows capacity, dtype) -> [ring of (tensor, handle, peer pointer array), next index]
        self._barrier = None  # PeerBarrier, created with the first symmetric buffer
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.in_features = in_features
        self.out_features = out_features
        lo, hi = shard_bounds(out_features, self.rank, self.world)
        self.n_lo, self.n_hi = lo, hi
        self.gather_output = gather_output
        self.pipeline_chunks = pipeline_chunks
        self.local = Linear(in_features, hi - lo, **linear_kwargs)
        self._comm_stream = None

    def load_full_params(self, qweight, scales=None, zeros=None, bias=None):
        """Take full-size (already transformed) parameters and keep this rank's shard."""
        op = self.local.bitblas_matmul
        sh = shard_quantized_params(qweight, scales, zeros, bias, rank=self.rank, world=self.world, bits=op.bit,
                                    zeros_mode=op.config.zeros_mode)
        dev = self.local.qweight.device
        self.local.qweight = sh["qweight"].to(dev)
        if "scales" in sh:
            self.local.scales = sh["scales"].to(dev)
        if "zeros" in sh:
            self.local.zeros = sh["zeros"].to(dev)
        if "bias" in sh:
            self.local.bias = sh["bias"].to(dev)
        self.local.q_params = None

    def _chunks_for(self, m: int) -> int:
        if self.pipeline_chunks is not None:
            return max(1, min(self.pipeline_chunks, m))
        return max(1, min(8, m // 512))

    def _symm_buffers(self, m: int, dtype, device):
        import torch.distributed._symmetric_memory as symm_mem
        cap = 1
        while cap < m:
            cap *= 2
        key = (cap, dtype)
        if key not in self._symm:
            pairs = []
            for _ in range(self.fused_ring):  # ring: one barrier per call is enough (see _forward_fused)
                t = symm_mem.empty((cap, self.out_features), dtype=dtype, device=device)
                h = symm_mem.rendezvous(t, self.group if self.group is not None else dist.group.WORLD)
                ptrs = [int(p) for p in h.buffer_ptrs]
                arr = (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(p) for p in ptrs])   # built once per buffer
                pairs.append((t, h, arr))
            self._symm[key] = [pairs, 0]
        entry = self._symm[key]
        t, h, arr = entry[0][entry[1]]
        entry[1] = (entry[1] + 1) % self.fused_ring
        return t, h, arr

    def _forward_fused(self, x2: torch.Tensor) -> torch.Tensor:
        m = x2.shape[0]
        op = self.local.bitblas_matmul
        out_dtype = getattr(torch, op.out_dtype)
        buf, hdl, peer_arr = self._symm_buffers(m, out_dtype, x2.device)
        lin = self.local
        op.forward_scatter(x2.contiguous(), lin.qweight, scale=lin.scales if op.with_scaling else None,
                           zeros=lin.zeros if op.with_zeros else None, bias=lin.bias if op.with_bias else None,
                           peer_ptrs=peer_arr, ldc=self.out_features, col_offset=self.n_lo)
        # every rank's slice has landed in every buffer once all ranks passed this point.  Buffers alternate between calls:
        # a rank can only overwrite buffer b again after the NEXT call's barrier, which every peer reaches after its
        # (stream-ordered) reads of this call's result.
        if self._barrier is None:
            self._barrier = PeerBarrier(x2.device, self.group)
        self._barrier()
        return buf[:m].clone() if self.clone_output else buf[:m]

    def _fused_supported_here(self, x2: torch.Tensor) -> bool:
        """can THIS rank run the fused path for this call: symmetric memory importable and a kernel family with the scatter
        epilogue (everything but the generic SIMT kernel) dispatched for this m."""
        if not x2.is_cuda or self.local.consistent:
            return False
        try:
            import torch.distributed._symmetric_memory  # noqa: F401
        except Exception:
            return False
        return self.local.bitblas_matmul.kernel_for(int(x2.shape[0])) != "generic_simt"

    def _decide_fused(self, x2: torch.Tensor) -> None:
        """one collective decision per layer (MIN over ranks of the local capability), taken at the first CUDA forward."""
        ok = torch.tensor([1 if self._fused_supported_here(x2) else 0], dtype=torch.int32, device=x2.device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
        agreed = bool(int(ok.item()))
        if self.fused_gather is True and not agreed:
            raise RuntimeError("fused_gather=True was requested but at least one rank cannot use it")
        self.fused_gather = agreed
        self._fused_decided = True

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.world == 1 or not self.gather_output:
            return self.local(x)
        if x.is_cuda and not self._fused_decided:
            self._decide_fused(x.reshape(-1, x.shape[-1]))
        if x.is_cuda and self.fused_gather:
            x2 = x.reshape(-1, x.shape[-1])
            # per-call probe (the dispatcher's choice depends on m): an m that lands on the generic kernel takes the NCCL path
            # for this call only -- identically on every rank, since all ranks see the same m and the same shard shape
            if self.local.bitblas_matmul.kernel_for(int(x2.shape[0])) != "generic_simt":
                return self._forward_fused(x2).reshape(*x.shape[:-1], self.out_features)
        lead = x.shape[:-1]
        x2 = x.reshape(-1, x.shape[-1])
        m = x2.shape[0]
        per = self.n_hi - self.n_lo
        out_dtype = getattr(torch, self.local.bitblas_matmul.out_dtype)
        full = torch.empty((m, self.out_features), dtype=out_dtype, device=x.device)
        nchunks = self._chunks_for(m)
        if x.is_cuda and self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=x.device)
        bounds = [(i * m) // nchunks for i in range(nchunks + 1)]
        staged = []
        for i in range(nchunks):
            r0, r1 = bounds[i], bounds[i + 1]
            if r1 == r0:
                continue
            part = self.local(x2[r0:r1]).contiguous()         # [rows, N/G] on the compute stream
            gathered = torch.empty((self.world * (r1 - r0), per), dtype=out_dtype, device=x.device)
            if x.is_cuda:
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(x.device))
                with torch.cuda.stream(self._comm_stream):
                    self._comm_stream.wait_event(ev)
                    dist.all_gather_into_tensor(gathered, part, group=self.group)
                    part.record_stream(self._comm_stream)
            else:
                dist.all_gather_into_tensor(gathered, part, group=self.group)
            staged.append((r0, r1, gathered))
        if x.is_cuda:
            torch.cuda.current_stream(x.device).wait_stream(self._comm_stream)
        for r0, r1, gathered in staged:
            # [G, rows, N/G] -> [rows, G, N/G] == rows of the full output
            full[r0:r1].view(r1 - r0, self.world, per).copy_(gathered.view(self.world, r1 - r0, per).permute(1, 0, 2))
        return full.reshape(*lead, self.out_features)


def shard_quantized_params_k(qweight, scales, zeros, *, rank: int, world: int, K: int, bits: int, group_size: int,
                             zeros_mode: str = "original"):
    """Slice full-size BitBLAS-layout parameters along K (input features) for one rank of a row-parallel layer.  The shard
    boundary must fall on a group boundary and on a 32-bit storage word (the LOP3 interleave permutes inside one word only, so a
    word-aligned K range of an interleaved row is the interleaved row of that K range).  Row-major storage only: slab-tiled
    weights are un-tiled by the caller first (RowParallelLinear.load_full_params does)."""
    if K % world:
        raise ValueError(f"K={K} is not divisible by world size {world}")
    per = K // world
    g = K if group_size in (-1, None) else group_size
    if per % g:
        raise ValueError(f"K/world = {per} must be a multiple of the group size {g}")
    if (per * bits) % 32:
        raise ValueError(f"K/world = {per} must cover whole 32-bit storage words at {bits} bits")
    lo, hi = rank * per, (rank + 1) * per
    out = {"qweight": qweight[:, lo * bits // 8:hi * bits // 8].contiguous()}
    if scales is not None:
        out["scales"] = scales[:, lo // g:hi // g].contiguous()
    if zeros is not None:
        out["zeros"] = (zeros[lo // g:hi // g] if zeros_mode == "quantized" else zeros[:, lo // g:hi // g]).contiguous()
    return out


class RowParallelLinear(nn.Module):
    """y = sum_r x[:, K_r] @ dequant(W[:, K_r])^T (+ b): W sharded along K (input features) across the group -- the second half
    of a tensor-parallel MLP / attention block (column-parallel up-projection, row-parallel down-projection: the activations arrive
    already sharded, only the output is exchanged).  The reference has no distributed code (SURVEY.md 2a); this is SURVEY.md 8(f)'s
    "row-parallel" item.  Each rank runs the ordinary low-bit matmul on its K slice with fp32 output, the partial sums meet in ONE
    all-reduce (NCCL: in-switch NVLS reduction on NVSwitch systems), bias is added once, the result is cast to out_dtype.
    Unlike the column-parallel layer the exchange moves REDUCED data: it cannot be expressed as peer stores from the epilogue
    without atomics, so it stays a collective (a reduce-scatter epilogue over multimem.red is the follow-up, DESIGN.md 3.4)."""

    def __init__(self, in_features: int, out_features: int, *, process_group=None, input_is_parallel: bool = True,
                 bias: bool = False, out_dtype: str = "float16", **linear_kwargs):
        super().__init__()
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        if in_features % self.world:
            raise ValueError(f"in_features={in_features} is not divisible by world size {self.world}")
        self.in_features, self.out_features = in_features, out_features
        self.k_per = in_features // self.world
        self.k_lo, self.k_hi = self.rank * self.k_per, (self.rank + 1) * self.k_per
        self.input_is_parallel = input_is_parallel
        self.final_dtype = getattr(torch, out_dtype)
        gs = linear_kwargs.get("group_size", -1)
        if gs in (-1, None):
            linear_kwargs["group_size"] = in_features      # "whole row" groups stay whole-row groups of the FULL K: one scale per
            if self.world > 1:                            # row cannot be split -- each shard then uses the same scale column
                linear_kwargs["group_size"] = self.k_per
        # partial sums leave the kernel in fp32 (the all-reduce must not round per rank); bias is added after the reduction
        self.local = Linear(self.k_per, out_features, bias=False, out_dtype="float32" if self.world > 1 else out_dtype, **linear_kwargs)
        self._whole_row_groups = gs in (-1, None)
        self.register_buffer("bias", torch.zeros((out_features,), dtype=self.final_dtype) if bias else None)

    def load_full_params(self, qweight, scales=None, zeros=None, bias=None):
        """full-size parameters in the operator's own storage (as produced by Matmul.transform_weight of the FULL layer, row-major
        or slab-tiled per this layer's propagate_b) -> this rank's K shard."""
        op = self.local.bitblas_matmul
        if op.weight_tiled:
            qweight = op.tile_weight(qweight, inverse=True)
        g = self.in_features if self._whole_row_groups else op.config.group_size
        if self._whole_row_groups and scales is not None and self.world > 1:
            # one group spanning the full K: every shard multiplies by the same per-row scale (and zero point)
            sh = {"qweight": qweight[:, self.k_lo * op.bit // 8:self.k_hi * op.bit // 8].contiguous(), "scales": scales.contiguous()}
            if zeros is not None:
                sh["zeros"] = zeros.contiguous()
        else:
            sh = shard_quantized_params_k(qweight, scales, zeros, rank=self.rank, world=self.world, K=self.in_features, bits=op.bit,
                                          group_size=g, zeros_mode=op.config.zeros_mode)
        dev = self.local.qweight.device
        w = sh["qweight"].to(dev)
        self.local.qweight = op.tile_weight(w) if op.weight_tiled else w
        if "scales" in sh:
            self.local.scales = sh["scales"].to(dev)
        if "zeros" in sh:
            self.local.zeros = sh["zeros"].to(dev)
        if bias is not None and self.bias is not None:
            self.bias = bias.to(dev).to(self.final_dtype)
        self.local.q_params = None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xs = x if self.input_is_parallel else x[..., self.k_lo:self.k_hi]
        if xs.shape[-1] != self.k_per:
            raise ValueError(f"expected the K shard of width {self.k_per}, got {xs.shape[-1]}")
        part = self.local(xs.contiguous())
        if self.world > 1:
            dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.group)
        out = part if part.dtype == self.final_dtype else part.to(self.final_dtype)
        if self.bias is not None:
            out = out + self.bias
        return out


__all__ = ["PeerBarrier", "ColumnParallelLinear", "RowParallelLinear", "shard_quantized_params", "shard_quantized_params_k", "shard_bounds"]
