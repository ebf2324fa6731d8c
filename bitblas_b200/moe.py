"""Mixture-of-experts expert block: top-k gating from router logits (bb_moe_topk), device routing (bb_moe_route;
bb_moe_route_index without the copy), the gate/up interleave that the SwiGLU grouped calls read, the weighted top-k combine
(bb_moe_combine), and ``MoEExperts``, which runs router output to layer output in four library launches.

Above 8 rows per expert, moe_route_index -> forward_grouped_swiglu(x, ..., row_index=row_token) -> down -> moe_combine computes
MoEExperts' bits without the [T*k, H] routed copy of x (T*k*H*2 bytes: 64 MiB per layer at 2048 tokens, top-8, H = 2048).
MoEExperts keeps the copy: the gathering GEMM measured 1.06-1.55x the time of the plain one (H100 80GB HBM3, 700 W, 64-2048
tokens), more than the copy costs, at every measured point.

Gate/up interleave (include/bitblas_b200.h): the fused gate/up projection of I rows each is stored as 2I rows in which stored row
16b + i is gate row 8b + i for i < 8 and up row 8b + i - 8 for i >= 8.  Every per-row buffer follows the same permutation:
the weight, scales and zeros ([.., 2I, *]) and the bias ([.., 2I]) along their row axis; quantized zeros ([.., G, 2I*bits/8],
packed along the rows) in whole bytes, 8 rows being `bits` bytes.  The 128 x 128 block scales of a block-scaled FP8 weight
([.., ceil(I/128), K/128], kind "block_scale") alternate by block: stored scale row 2c is gate block c and row 2c + 1 up block c.
A 128-row tile t of the stored weight holds gate rows 64t .. 64t + 63 and up rows 64t .. 64t + 63, so its scales are stored
rows 2(t >> 1) and 2(t >> 1) + 1.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .act_order import perm_from_g_idx, permute_cols, permute_gptq_rows

INTERLEAVE_ROWS = 8
# kind -> (axis holding the rows, rows per element along it: None = 1, "bits" = 8 / bits packed rows per byte, "block" = one
# element per 128 rows)
_KINDS = {"weight": (-2, None), "scale": (-2, None), "zeros": (-2, None), "bias": (-1, None), "qzeros": (-1, "bits"),
          "block_scale": (-2, "block")}


def _block(kind, bits):
    if kind not in _KINDS:
        raise ValueError(f"kind must be one of {sorted(_KINDS)} (got {kind!r})")
    dim, packed = _KINDS[kind]
    if packed is None:
        return dim, INTERLEAVE_ROWS
    if packed == "block":
        return dim, 1
    if bits not in (2, 4):
        raise ValueError("quantized zeros need bits = 4 or 2 (8 rows are `bits` whole bytes)")
    return dim, INTERLEAVE_ROWS * bits // 8


def interleave_gate_up(gate: torch.Tensor, up: torch.Tensor, kind: str, bits: int = None) -> torch.Tensor:
    """gate, up [.., I, ..] (the rows on the axis of `kind`) -> the stored [.., 2I, ..] of the gate/up interleave.  kind: "weight",
    "scale", "zeros", "bias", "qzeros" (quantized zeros packed along the rows; needs `bits`), or "block_scale" (FP8 128 x 128
    block scales [.., ceil(I/128), K/128] -> [.., 2 ceil(I/128), K/128]).  CPU or CUDA tensors."""
    dim, blk = _block(kind, bits)
    if gate.shape != up.shape:
        raise ValueError(f"gate and up must have the same shape (got {tuple(gate.shape)} and {tuple(up.shape)})")
    n = gate.shape[dim]
    if n % blk:
        raise ValueError(f"the {kind} row axis ({n}) must be a multiple of {blk}: the interleave moves blocks of 8 rows")
    g, u = gate.movedim(dim, -1), up.movedim(dim, -1)
    lead = g.shape[:-1]
    out = torch.stack([g.reshape(*lead, n // blk, blk), u.reshape(*lead, n // blk, blk)], dim=-2).reshape(*lead, 2 * n)
    return out.movedim(-1, dim).contiguous()


def deinterleave_gate_up(fused: torch.Tensor, kind: str, bits: int = None):
    """the inverse of interleave_gate_up: stored [.., 2I, ..] -> (gate, up)"""
    dim, blk = _block(kind, bits)
    n2 = fused.shape[dim]
    if n2 % (2 * blk):
        raise ValueError(f"the {kind} row axis ({n2}) must be a multiple of {2 * blk}")
    f = fused.movedim(dim, -1)
    lead = f.shape[:-1]
    pairs = f.reshape(*lead, n2 // (2 * blk), 2, blk)
    gate = pairs[..., 0, :].reshape(*lead, n2 // 2).movedim(-1, dim).contiguous()
    up = pairs[..., 1, :].reshape(*lead, n2 // 2).movedim(-1, dim).contiguous()
    return gate, up


def gate_up_act_order(gate, up, down, H: int, I: int, gate_up_group_size: int, down_group_size: int, bits: int, where: str = ""):
    """The act-order rule of a SwiGLU gate/up/down triple of GPTQ modules (MoEExperts per expert, SwiGLUMLP): gate and up read
    the same input, so they must carry the same g_idx (ValueError otherwise; `where` prefixes the message) and keep it as the
    gate/up projection's column order.  The down projection's column order is absorbed: gate and up are returned with their
    output rows in down's sorted K order (permute_gptq_rows), so silu(gate) * up arrives in the order down's sorted weight reads and
    down needs no gather.  Returns (gate, up), the modules themselves when down is not act-order."""
    pg, pu = (perm_from_g_idx(getattr(m, "g_idx", None), H, gate_up_group_size) for m in (gate, up))
    if (pg is None) != (pu is None) or (pg is not None and not torch.equal(pg.cpu(), pu.cpu())):
        raise ValueError(f"{where}gate and up have different g_idx; they read the same input, so act-order "
                         "checkpoints must give them the same column order")
    pd = perm_from_g_idx(getattr(down, "g_idx", None), I, down_group_size)
    if pd is None:
        return gate, up
    return permute_gptq_rows(gate, pd, bits), permute_gptq_rows(up, pd, bits)


def moe_route(topk_ids: torch.Tensor, x: torch.Tensor, num_experts: int):
    """Route the tokens of x [T, K] (fp16 / bf16) by topk_ids (int32 [T, k]) on the device, in one launch (bb_moe_route).
    Returns (offsets int32 [E + 1], slot_rows int32 [T*k], x_sorted [T*k, K]): slot t*k + j goes to sorted row slot_rows[t*k + j]
    of expert topk_ids[t, j]; rows are ordered by expert, then by slot.  Ids outside [0, E) are dropped (slot_rows = -1) and
    x_sorted rows offsets[E] .. T*k - 1 are left unwritten."""
    _lib.check_tensor(topk_ids, "topk_ids", torch.int32, 2)
    if not isinstance(x, torch.Tensor) or x.dtype not in (torch.float16, torch.bfloat16):
        raise TypeError("x must be a float16 or bfloat16 torch.Tensor")
    _lib.check_tensor(x, "x", x.dtype, 2)
    T, k = topk_ids.shape
    if x.shape[0] != T:
        raise ValueError(f"x has {x.shape[0]} rows, topk_ids {T}")
    if x.device != topk_ids.device:
        raise ValueError("x and topk_ids must be on the same device")
    dev, idx, stream = _lib.device_stream(x)
    E, K = int(num_experts), x.shape[1]
    offsets = torch.empty(max(E, 0) + 1, dtype=torch.int32, device=dev)
    slot_rows = torch.empty(T * k, dtype=torch.int32, device=dev)
    x_sorted = torch.empty((T * k, K), dtype=x.dtype, device=dev)
    _lib.call("bb_moe_route", idx, topk_ids.data_ptr(), T, k, E, x.data_ptr(), _lib.dtype_id(x.dtype), K,
              offsets.data_ptr(), slot_rows.data_ptr(), x_sorted.data_ptr(), stream)
    return offsets, slot_rows, x_sorted


def moe_route_index(topk_ids: torch.Tensor, num_experts: int):
    """moe_route without the copy, in one launch (bb_moe_route_index).  Returns (offsets int32 [E + 1], slot_rows int32 [T*k],
    row_token int32 [T*k]): offsets and slot_rows are exactly moe_route's, and row_token[slot_rows[s]] = s // k for every kept
    slot s, so x[row_token] is moe_route's x_sorted.  Rows offsets[E] .. T*k - 1 of row_token are left unwritten."""
    _lib.check_tensor(topk_ids, "topk_ids", torch.int32, 2)
    T, k = topk_ids.shape
    dev, idx, stream = _lib.device_stream(topk_ids)
    E = int(num_experts)
    offsets = torch.empty(max(E, 0) + 1, dtype=torch.int32, device=dev)
    slot_rows = torch.empty(T * k, dtype=torch.int32, device=dev)
    row_token = torch.empty(T * k, dtype=torch.int32, device=dev)
    _lib.call("bb_moe_route_index", idx, topk_ids.data_ptr(), T, k, E, offsets.data_ptr(), slot_rows.data_ptr(),
              row_token.data_ptr(), stream)
    return offsets, slot_rows, row_token


def moe_combine(y_sorted: torch.Tensor, slot_rows: torch.Tensor, topk_weights: torch.Tensor, output: torch.Tensor = None):
    """out[t] = sum_j topk_weights[t, j] * y_sorted[slot_rows[t*k + j]] in one launch (bb_moe_combine): fp32 accumulation in j
    order, one rounding to y_sorted's dtype (fp16 / bf16 / fp32); dropped slots add nothing.  y_sorted [T*k, N], slot_rows
    int32 [T*k], topk_weights float32 [T, k]; returns [T, N]."""
    if not isinstance(y_sorted, torch.Tensor) or y_sorted.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        raise TypeError("y_sorted must be a float16, bfloat16 or float32 torch.Tensor")
    _lib.check_tensor(y_sorted, "y_sorted", y_sorted.dtype, 2)
    _lib.check_tensor(topk_weights, "topk_weights", torch.float32, 2)
    _lib.check_tensor(slot_rows, "slot_rows", torch.int32, 1)
    T, k = topk_weights.shape
    N = y_sorted.shape[1]
    if slot_rows.numel() != T * k or y_sorted.shape[0] != T * k:
        raise ValueError(f"slot_rows and y_sorted need T*k = {T * k} rows (got {slot_rows.numel()} and {y_sorted.shape[0]})")
    if not (y_sorted.device == slot_rows.device == topk_weights.device):
        raise ValueError("y_sorted, slot_rows and topk_weights must be on the same device")
    dev, idx, stream = _lib.device_stream(y_sorted)
    if output is None:
        output = torch.empty((T, N), dtype=y_sorted.dtype, device=dev)
    else:
        _lib.check_tensor(output, "output", y_sorted.dtype, 2)
        if tuple(output.shape) != (T, N) or output.device != dev:
            raise ValueError(f"output must be [T={T}, N={N}] on {dev}")
    _lib.call("bb_moe_combine", idx, slot_rows.data_ptr(), topk_weights.data_ptr(), y_sorted.data_ptr(),
              _lib.dtype_id(y_sorted.dtype), output.data_ptr(), T, k, N, stream)
    return output


_SCORING = {"softmax": 0, "sigmoid": 1}
_GROUP_SCORE = {"max": 0, "top2_sum": 1}


def moe_topk(router_logits: torch.Tensor, top_k: int, scoring: str = "softmax", renormalize: bool = False,
             correction_bias: torch.Tensor = None, num_expert_group: int = None, topk_group: int = None,
             group_score: str = "max", routed_scaling_factor: float = 1.0):
    """Top-k gating on the device in one launch (bb_moe_topk): router_logits [T, E] (fp16 / bf16 / fp32) -> (topk_ids int32
    [T, k], topk_weights float32 [T, k]), what ``MoEExperts.forward`` takes.

    Per token: scores s = softmax(logits) or sigmoid(logits) in fp32; selection values v = s + correction_bias (fp32 [E], which
    steers the selection only); with ``num_expert_group`` = n > 1, the experts form n contiguous groups, each scored by the max of
    its v ("max") or the sum of its two largest ("top2_sum"), and only the ``topk_group`` best groups can be chosen; then the k
    largest v in descending order, ties to the lower expert (group) index, NaN below every number.  The weights are the chosen s,
    divided by their fp32 sum in slot order with ``renormalize``, times ``routed_scaling_factor``.  The ids and their order are
    library-defined, so two runs and graph replays are bit-identical.  1 <= E <= 256, 1 <= k <= min(E, 32).

    Presets:

    ================  ==========================================================================================================
    model             arguments
    ================  ==========================================================================================================
    Mixtral-8x7B      ``moe_topk(logits, 2, renormalize=True)``
    Qwen3-30B-A3B     ``moe_topk(logits, 8, renormalize=True)`` (``norm_topk_prob``)
    Qwen1.5/2-MoE     ``moe_topk(logits, 4)``
    DeepSeek-V2-Lite  ``moe_topk(logits, 6)`` (``routed_scaling_factor`` 1.0)
    DeepSeek-V2       ``moe_topk(logits, 6, num_expert_group=8, topk_group=3, group_score="max", routed_scaling_factor=16.0)``
    DeepSeek-V3       ``moe_topk(logits, 8, scoring="sigmoid", correction_bias=e_score_correction_bias, num_expert_group=8,
                      topk_group=4, group_score="top2_sum", renormalize=True, routed_scaling_factor=2.5)``
    ================  ==========================================================================================================
    """
    if not isinstance(router_logits, torch.Tensor) or router_logits.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        raise TypeError("router_logits must be a float16, bfloat16 or float32 torch.Tensor")
    if router_logits.dim() != 2:
        raise TypeError(f"router_logits must be a 2-D [T, E] tensor (got {router_logits.dim()}-D)")
    T, E = router_logits.shape
    if scoring not in _SCORING:
        raise ValueError(f"scoring must be one of {sorted(_SCORING)} (got {scoring!r})")
    if group_score not in _GROUP_SCORE:
        raise ValueError(f"group_score must be one of {sorted(_GROUP_SCORE)} (got {group_score!r})")
    grouped = num_expert_group is not None and int(num_expert_group) > 1
    if grouped and topk_group is None:
        raise ValueError("num_expert_group > 1 needs topk_group")
    if correction_bias is not None:
        if not isinstance(correction_bias, torch.Tensor) or correction_bias.dtype != torch.float32 or \
                tuple(correction_bias.shape) != (E,):
            raise TypeError(f"correction_bias must be a float32 tensor of shape [E={E}]")
        if correction_bias.device != router_logits.device:
            raise ValueError("router_logits and correction_bias must be on the same device")
        _lib.check_tensor(correction_bias, "correction_bias", torch.float32, 1)
    _lib.check_tensor(router_logits, "router_logits", router_logits.dtype, 2)
    dev, idx, stream = _lib.device_stream(router_logits)
    k = int(top_k)
    topk_ids = torch.empty((T, max(k, 0)), dtype=torch.int32, device=dev)
    topk_weights = torch.empty((T, max(k, 0)), dtype=torch.float32, device=dev)
    _lib.call("bb_moe_topk", idx, router_logits.data_ptr(), _lib.dtype_id(router_logits.dtype), T, E, k,
              _SCORING[scoring], None if correction_bias is None else correction_bias.data_ptr(),
              int(num_expert_group) if grouped else 0, int(topk_group) if grouped else 0,
              _GROUP_SCORE[group_score], int(bool(renormalize)), float(routed_scaling_factor),
              topk_ids.data_ptr(), topk_weights.data_ptr(), stream)
    return topk_ids, topk_weights


class MoEExperts(nn.Module):
    """The expert block of a SwiGLU mixture-of-experts layer, from router output to layer output:
    ``y[t] = sum_j w[t, j] * down_e(silu(gate_e(x[t])) * up_e(x[t]))`` with e = topk_ids[t, j], as four library launches with no
    host synchronisation (CUDA-graph capturable): moe_route -> grouped gate/up with SwiGLU in the epilogue -> grouped down ->
    moe_combine.  ``gate_up`` (H -> 2I, gate/up interleaved) and ``down`` (I -> H) are ``GroupedLinear``s built from the
    ``Linear`` keyword arguments; ``out_dtype`` must equal ``A_dtype`` (the gate/up output is the down projection's input).

    GPTQ act-order experts (act_order.py): the gate/up projections' column order is ``gate_up.perm`` [E, H], and ``forward`` gathers
    the routed rows with it (one more launch, five in all).  The down projection's order costs nothing at run time: each expert's
    gate and up output rows are loaded in that order, so the SwiGLU output arrives already sorted for the down projection's K axis.
    The copy-free path (moe_route_index + forward_grouped_swiglu(row_index=)) cannot apply a column order."""

    def __init__(self, num_experts: int, hidden_size: int, intermediate_size: int, bias: bool = False, **linear_kwargs):
        super().__init__()
        from .module import GroupedLinear
        if intermediate_size % INTERLEAVE_ROWS:
            raise ValueError(f"intermediate_size must be a multiple of {INTERLEAVE_ROWS} (gate/up interleave; got {intermediate_size})")
        a_dtype = linear_kwargs.get("A_dtype", "float16")
        if linear_kwargs.get("out_dtype", "float16") != a_dtype:
            raise ValueError("MoEExperts needs out_dtype == A_dtype: the gate/up output is the down projection's input")
        self.num_experts, self.hidden_size, self.intermediate_size = int(num_experts), hidden_size, intermediate_size
        self.gate_up = GroupedLinear(num_experts, hidden_size, 2 * intermediate_size, bias=bias, **linear_kwargs)
        self.down = GroupedLinear(num_experts, intermediate_size, hidden_size, bias=bias, **linear_kwargs)
        self.gate_up.bitblas_matmul.check_grouped(self.num_experts, swiglu=True)
        self._linear_kwargs = dict(linear_kwargs, bias=bias)

    def forward(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor, output: torch.Tensor = None):
        """x [T, H], topk_ids int32 [T, k], topk_weights float32 [T, k] -> [T, H]"""
        if x.dim() != 2 or x.shape[1] != self.hidden_size:
            raise ValueError(f"x must be [T, H={self.hidden_size}], got {tuple(x.shape)}")
        if tuple(topk_weights.shape) != tuple(topk_ids.shape):
            raise ValueError("topk_ids and topk_weights must have the same [T, k] shape")
        offsets, slot_rows, x_sorted = moe_route(topk_ids, x, self.num_experts)
        gu, cfg = self.gate_up, self.gate_up.bitblas_matmul.config
        if gu.perm is not None:
            x_sorted = permute_cols(x_sorted, gu.perm, offsets)
        h = gu.bitblas_matmul.forward_grouped_swiglu(x_sorted, gu.qweight, offsets, gu.scales if cfg.with_scaling else None,
                                                     gu.zeros if cfg.with_zeros else None, gu.bias)
        y = self.down(h, offsets, capturable=True)
        return moe_combine(y, slot_rows, topk_weights, output)

    # ---- loading -----------------------------------------------------------------------------------------------------------
    def _zeros_kind(self):
        return "qzeros" if self.gate_up.bitblas_matmul.config.zeros_mode == "quantized" else "zeros"

    def load_and_transform_weight(self, gate, up, down):
        """gate, up, down: (weight, scales, zeros, bias) per projection, each stacked over the experts as
        GroupedLinear.load_and_transform_weight takes it (None where the config has none; missing trailing entries are None).
        gate / up are interleaved into gate_up before the storage transform (which works row by row)."""
        g, u = (tuple(gate) + (None,) * 4)[:4], (tuple(up) + (None,) * 4)[:4]
        kinds = ("weight", "scale", self._zeros_kind(), "bias")
        fused = [None if a is None else interleave_gate_up(a, b, kind, self.gate_up.bits) for a, b, kind in zip(g, u, kinds)]
        self.gate_up.load_and_transform_weight(*fused)
        self.down.load_and_transform_weight(*down)

    def _repack(self, gate_modules, up_modules, down_modules, device, v2):
        from .module import GroupedLinear
        E, H, I = self.num_experts, self.hidden_size, self.intermediate_size
        if not len(gate_modules) == len(up_modules) == len(down_modules) == E:
            raise ValueError(f"expected {E} GPTQ modules per projection, got {len(gate_modules)}, {len(up_modules)}, {len(down_modules)}")
        gate_modules, up_modules = list(gate_modules), list(up_modules)
        for e in range(E):
            gate_modules[e], up_modules[e] = gate_up_act_order(gate_modules[e], up_modules[e], down_modules[e], H, I,
                                                               self.gate_up.group_size, self.down.group_size,
                                                               self.gate_up.bits, f"expert {e}: ")
        kw = dict(self._linear_kwargs)
        bias = kw.pop("bias")
        halves = []
        for mods in (gate_modules, up_modules):
            half = GroupedLinear(self.num_experts, self.hidden_size, self.intermediate_size, bias=bias, **kw)
            half._repack(mods, device, v2)
            halves.append(half)
        g, u = halves
        gu = self.gate_up
        gu.qweight = interleave_gate_up(g.qweight, u.qweight, "weight")
        gu.scales = interleave_gate_up(g.scales, u.scales, "scale")
        gu.zeros = interleave_gate_up(g.zeros, u.zeros, self._zeros_kind(), gu.bits)
        if gu.bias is not None:
            gu.bias = interleave_gate_up(g.bias, u.bias, "bias")
        gu.perm = g.perm
        self.down._repack(down_modules, device, v2, keep_perm=False)

    def repack_from_gptq(self, gate_modules, up_modules, down_modules, device="cuda"):
        """one GPTQ QuantLinear per expert and projection: GroupedLinear's repack of gate and up, then the interleave.  Act-order
        modules (g_idx) are taken as described in the class documentation; an expert's gate and up must have the same g_idx."""
        self._repack(gate_modules, up_modules, down_modules, device, v2=False)

    def repack_from_gptq_v2(self, gate_modules, up_modules, down_modules, device="cuda"):
        self._repack(gate_modules, up_modules, down_modules, device, v2=True)


__all__ = ["MoEExperts", "moe_topk", "moe_route", "moe_route_index", "moe_combine", "interleave_gate_up", "deinterleave_gate_up",
           "gate_up_act_order"]
