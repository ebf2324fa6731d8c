"""GPTQ act-order (``desc_act=True``) checkpoints: the permutation that makes their groups contiguous, and the activation gather.

An act-order checkpoint assigns input column k to quantization group ``g_idx[k]`` instead of ``k // group_size``.  GPTQ gives every
group exactly ``group_size`` columns, so with ``perm = stable_argsort(g_idx)`` sorted column j is in group ``j // group_size``: the
contiguous layout every kernel reads.  The loaders therefore sort the weight's K axis by ``perm`` (scales and zeros are indexed by
group and do not move) and the layers compute ``y = A[:, perm] x W_sorted^T``, the gather being one ``bb_permute_cols`` launch.

``perm_from_g_idx`` is the one place that decides whether a layer is act-order; ``Linear``, ``GroupedLinear`` and ``MoEExperts``
call it from their GPTQ repack paths.  A checkpoint without act-order (``g_idx = arange(K) // group_size``, or no ``g_idx``) gets
``None`` and loads and runs exactly as before.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from . import _lib


def perm_from_g_idx(g_idx, K: int, group_size: int):
    """The column order of an act-order layer: int32 [K] ``stable_argsort(g_idx)`` on g_idx's device, or None when that is the
    identity (g_idx None, or every column in group k // group_size).  Raises ValueError when g_idx is not a GPTQ group assignment:
    a length other than K, a value outside [0, K / group_size), or a group without exactly group_size columns."""
    if g_idx is None:
        return None
    g = torch.as_tensor(g_idx).reshape(-1).to(torch.int64)
    if g.numel() != K:
        raise ValueError(f"g_idx has {g.numel()} entries, expected K = {K}")
    G = K // group_size
    bad = ((g < 0) | (g >= G)).nonzero()
    if bad.numel():
        k = int(bad[0])
        raise ValueError(f"g_idx[{k}] = {int(g[k])} names group {int(g[k])}, outside [0, {G})")
    counts = torch.bincount(g, minlength=G)
    wrong = (counts != group_size).nonzero()
    if wrong.numel():
        e = int(wrong[0])
        raise ValueError(f"group {e} has {int(counts[e])} columns in g_idx, expected group_size = {group_size}")
    perm = torch.sort(g, stable=True).indices
    if torch.equal(perm, torch.arange(K, device=perm.device)):
        return None
    return perm.to(torch.int32)


def _unpack(packed: torch.Tensor, bits: int, dim: int) -> torch.Tensor:
    """int32 words packed along `dim` (element i of a word at bits * i) -> int64 values, 32 / bits per word along `dim`"""
    per = 32 // bits
    p = packed.view(torch.int32).movedim(dim, -1).to(torch.int64)
    shifts = torch.arange(per, device=p.device, dtype=torch.int64) * bits
    v = (p.unsqueeze(-1) >> shifts) & (2**bits - 1)
    return v.reshape(*p.shape[:-1], p.shape[-1] * per).movedim(-1, dim)


def _pack(vals: torch.Tensor, bits: int, dim: int) -> torch.Tensor:
    """the inverse of _unpack: int64 values -> int32 words packed along `dim`"""
    per = 32 // bits
    v = vals.movedim(dim, -1)
    v = v.reshape(*v.shape[:-1], v.shape[-1] // per, per)
    word = torch.zeros(v.shape[:-1], dtype=torch.int64, device=v.device)
    for i in range(per):
        word |= v[..., i] << (bits * i)
    word = torch.where(word >= 2**31, word - 2**32, word)   # the same 32 bits as an int32
    return word.to(torch.int32).movedim(-1, dim).contiguous()


def permute_gptq_qweight(qweight: torch.Tensor, perm: torch.Tensor, bits: int) -> torch.Tensor:
    """GPTQ qweight int32 [K * bits / 32, N] -> the same weight with its K axis sorted: row j of the result's unpacked [K, N] is
    row perm[j] of qweight's.  Runs in torch on qweight's device; the result goes to bb_repack_gptq_qweight_device as before."""
    return _pack(_unpack(qweight, bits, 0)[perm.to(device=qweight.device, dtype=torch.long)], bits, 0)


def permute_gptq_rows(module, perm: torch.Tensor, bits: int):
    """A GPTQ module whose output rows (its N axis) are reordered: output n of the result is output perm[n] of `module`.  qweight
    [K * bits / 32, N] and scales [K / g, N] move by column, qzeros [K / g, N * bits / 32] is unpacked along N, indexed and
    repacked, and bias [N] moves with the rows; g_idx (the K axis) is kept.  Returns a stand-in with those attributes."""
    idx = perm.to(device=module.qweight.device, dtype=torch.long)
    qzeros = module.qzeros.view(torch.int32)
    bias = getattr(module, "bias", None)
    return SimpleNamespace(
        qweight=module.qweight.view(torch.int32)[:, idx].contiguous(),
        scales=module.scales[:, idx.to(module.scales.device)].contiguous(),
        qzeros=_pack(_unpack(qzeros, bits, 1)[:, idx.to(qzeros.device)], bits, 1),
        bias=None if bias is None else bias.data[idx.to(bias.device)].contiguous(),
        g_idx=getattr(module, "g_idx", None))


def permute_cols(A: torch.Tensor, perm: torch.Tensor, offsets: torch.Tensor = None, output: torch.Tensor = None) -> torch.Tensor:
    """out[r, j] = A[r, perm[j]] in one launch (bb_permute_cols).  A [rows, K] float16 / bfloat16, perm int32 [K] on A's device.
    With offsets (int32 [E + 1], the offsets of the grouped matmuls) perm is [E, K] and row r of group e reads perm[e]; rows that no
    group claims are left unwritten.  Perm values are clamped to [0, K), offsets to [0, rows].  Returns output ([rows, K])."""
    if not isinstance(A, torch.Tensor) or A.dtype not in (torch.float16, torch.bfloat16):
        raise TypeError("A must be a float16 or bfloat16 torch.Tensor")
    _lib.check_tensor(A, "A", A.dtype, 2)
    rows, K = A.shape
    if offsets is None:
        _lib.check_tensor(perm, "perm", torch.int32, 1)
        if perm.numel() != K:
            raise ValueError(f"perm must be [K={K}] without offsets (got {tuple(perm.shape)})")
        E = 1
    else:
        _lib.check_tensor(offsets, "offsets", torch.int32, 1)
        _lib.check_tensor(perm, "perm", torch.int32, 2)
        E = offsets.numel() - 1
        if tuple(perm.shape) != (E, K):
            raise ValueError(f"perm must be [E={E}, K={K}] for {E + 1} offsets (got {tuple(perm.shape)})")
    if perm.device != A.device or (offsets is not None and offsets.device != A.device):
        raise ValueError("A, perm and offsets must be on the same device")
    dev, idx, stream = _lib.device_stream(A)
    if output is None:
        output = torch.empty_like(A)
    else:
        _lib.check_tensor(output, "output", A.dtype, 2)
        if tuple(output.shape) != (rows, K) or output.device != dev:
            raise ValueError(f"output must be [{rows}, {K}] on {dev}")
    _lib.call("bb_permute_cols", idx, A.data_ptr(), output.data_ptr(), perm.data_ptr(), rows, K, _lib.dtype_id(A.dtype), E,
              None if offsets is None else offsets.data_ptr(), stream)
    return output


def stack_perms(perms, K: int, device):
    """per-expert perms (None = identity) -> int32 [E, K] on `device`, or None when every expert is the identity"""
    if all(p is None for p in perms):
        return None
    ident = torch.arange(K, dtype=torch.int32, device=device)
    return torch.stack([ident if p is None else p.to(device) for p in perms])


__all__ = ["perm_from_g_idx", "permute_gptq_qweight", "permute_gptq_rows", "permute_cols", "stack_perms"]
