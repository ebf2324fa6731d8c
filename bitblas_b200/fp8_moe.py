"""The expert block of a mixture-of-experts layer whose experts are 128 x 128 block-scaled FP8 (DeepSeek-V3 / R1, the Qwen3 -FP8
releases), from router output to layer output on the FP8 tensor cores:

    moe_route -> quantize_act_fp8(x_sorted) -> forward_grouped_fp8_swiglu -> quantize_act_fp8(h) -> forward_grouped_fp8 -> moe_combine

Six library launches with no host synchronisation (CUDA-graph capturable).  Every step is the rule of its own entry point
(include/bitblas_b200.h), so the block equals, bit for bit, routing, then per expert quantize_act_fp8 + the unsplit bb_matmul_fp8
of gate and of up, silu(g) * u rounded once, quantize_act_fp8 + the unsplit bb_matmul_fp8 of down, then the weighted combine.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .fp8 import _ACT_DTYPES, quantize_act_fp8, quantize_weight_blocks
from .moe import interleave_gate_up, moe_combine, moe_route
from .ops.general_matmul import Matmul, MatmulConfig

E4M3 = torch.float8_e4m3fn


def _stacked(t, name, shape, fp8):
    """a checkpoint tensor stacked over the experts, or a list of per-expert tensors: -> one tensor of `shape` (the weight as
    float8_e4m3fn, a scale as float32, converted exactly from float32 / 16-bit floats)"""
    if isinstance(t, (list, tuple)):
        if len(t) != shape[0]:
            raise ValueError(f"{name}: expected {shape[0]} per-expert tensors (got {len(t)})")
        if not all(isinstance(x, torch.Tensor) for x in t):
            raise TypeError(f"{name}: every per-expert entry must be a torch.Tensor")
        dtypes = {x.dtype for x in t}
        t = torch.stack([x.view(torch.uint8) if x.dtype == E4M3 else x for x in t])
        if dtypes == {E4M3}:
            t = t.view(E4M3)
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor or a list of per-expert tensors")
    if fp8 and t.dtype != E4M3:
        raise TypeError(f"{name} must be float8_e4m3fn (got {t.dtype})")
    if not fp8 and t.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        raise TypeError(f"{name} must be float32 (or float16 / bfloat16) (got {t.dtype})")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must be {list(shape)} stacked over the experts (got {list(t.shape)})")
    return t if fp8 else t.float()


class FP8MoEExperts(nn.Module):
    """``y[t] = sum_j w[t, j] * down_e(silu(gate_e(x[t])) * up_e(x[t]))`` with e = topk_ids[t, j], for experts stored as 128 x 128
    block-scaled e4m3 weights, x and y of A_dtype (float16 | bfloat16).  hidden_size and intermediate_size are multiples of 128.

    Buffers (``state_dict`` round-trips):
      * ``gate_up_weight`` float8_e4m3fn [E, 2I, H]: gate and up in the gate/up interleave (moe.interleave_gate_up "weight");
      * ``gate_up_weight_scale_inv`` float32 [E, 2 ceil(I/128), H/128]: their block scales interleaved by block ("block_scale");
      * ``down_weight`` float8_e4m3fn [E, H, I] and ``down_weight_scale_inv`` float32 [E, H/128, I/128].

    ``forward`` is six launches (see the module documentation).  Ids outside [0, E) are dropped by the routing, so a rank holding a
    slice of the experts passes its local ids."""

    def __init__(self, num_experts: int, hidden_size: int, intermediate_size: int, A_dtype: str = "bfloat16"):
        super().__init__()
        if A_dtype not in _ACT_DTYPES:
            raise ValueError(f"A_dtype must be float16 or bfloat16 (got {A_dtype})")
        for name, v in (("hidden_size", hidden_size), ("intermediate_size", intermediate_size)):
            if v <= 0 or v % 128:
                raise ValueError(f"{name} must be a positive multiple of 128 (got {v})")
        E, H, I = int(num_experts), int(hidden_size), int(intermediate_size)
        self.num_experts, self.hidden_size, self.intermediate_size, self.A_dtype = E, H, I, A_dtype
        self.torch_dtype = _ACT_DTYPES[A_dtype]

        def op(N, K):
            return Matmul(MatmulConfig(N=N, K=K, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32",
                                       out_dtype=A_dtype), enable_tuning=False)
        self.gate_up_matmul, self.down_matmul = op(2 * I, H), op(H, I)
        self.gate_up_matmul.check_grouped_fp8(E, swiglu=True)
        self.down_matmul.check_grouped_fp8(E)
        self.register_buffer("gate_up_weight", torch.zeros(E, 2 * I, H, dtype=E4M3))
        self.register_buffer("gate_up_weight_scale_inv", torch.ones(E, 2 * (I // 128), H // 128, dtype=torch.float32))
        self.register_buffer("down_weight", torch.zeros(E, H, I, dtype=E4M3))
        self.register_buffer("down_weight_scale_inv", torch.ones(E, H // 128, I // 128, dtype=torch.float32))

    def forward(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor, output: torch.Tensor = None):
        """x [T, H] of A_dtype, topk_ids int32 [T, k], topk_weights float32 [T, k] -> [T, H] of A_dtype"""
        if not isinstance(x, torch.Tensor) or x.dtype != self.torch_dtype:
            raise TypeError(f"x must be a {self.torch_dtype} torch.Tensor")
        if x.dim() != 2 or x.shape[1] != self.hidden_size:
            raise ValueError(f"x must be [T, H={self.hidden_size}], got {tuple(x.shape)}")
        if tuple(topk_weights.shape) != tuple(topk_ids.shape):
            raise ValueError("topk_ids and topk_weights must have the same [T, k] shape")
        offsets, slot_rows, x_sorted = moe_route(topk_ids, x, self.num_experts)
        q, s = quantize_act_fp8(x_sorted)
        h = self.gate_up_matmul.forward_grouped_fp8_swiglu(q, self.gate_up_weight, offsets, s, self.gate_up_weight_scale_inv)
        q, s = quantize_act_fp8(h)
        y = self.down_matmul.forward_grouped_fp8(q, self.down_weight, offsets, s, self.down_weight_scale_inv)
        return moe_combine(y, slot_rows, topk_weights, output)

    # ---- loading -----------------------------------------------------------------------------------------------------------
    def load_fp8(self, gate, up, down) -> None:
        """A checkpoint's experts: gate, up and down are each (weight, weight_scale_inv), either stacked over the experts or as
        lists of per-expert tensors.  In a DeepSeek-V3 / R1 or Qwen3 -FP8 shard, expert e of layer l is stored under
        ``model.layers.{l}.mlp.experts.{e}.{gate,up,down}_proj.{weight,weight_scale_inv}``: weight float8_e4m3fn [out, in] and
        weight_scale_inv float32 [ceil(out/128), in/128] (16-bit float scales are converted exactly).  gate and up ([I, H]) are
        interleaved into gate_up_weight and its scales here."""
        E, H, I = self.num_experts, self.hidden_size, self.intermediate_size
        parts = {}
        for pname, pair, (N, K) in (("gate", gate, (I, H)), ("up", up, (I, H)), ("down", down, (H, I))):
            if not isinstance(pair, (list, tuple)) or len(pair) != 2:
                raise TypeError(f"{pname} must be a (weight, weight_scale_inv) pair")
            w = _stacked(pair[0], f"{pname} weight", (E, N, K), True)
            s = _stacked(pair[1], f"{pname} weight_scale_inv", (E, (N + 127) // 128, K // 128), False)
            parts[pname] = (w, s)
        (gw, gs), (uw, us), (dw, ds) = parts["gate"], parts["up"], parts["down"]
        gu = interleave_gate_up(gw.view(torch.uint8), uw.view(torch.uint8), "weight").view(E4M3)
        self.gate_up_weight.copy_(gu.to(self.gate_up_weight.device))
        self.gate_up_weight_scale_inv.copy_(interleave_gate_up(gs, us, "block_scale").to(self.gate_up_weight_scale_inv.device))
        self.down_weight.copy_(dw.to(self.down_weight.device))
        self.down_weight_scale_inv.copy_(ds.to(self.down_weight_scale_inv.device))

    def load_float_weight(self, gate, up, down) -> None:
        """float weights gate, up [E, I, H] and down [E, H, I] (stacked or per-expert lists), each expert quantized in 128 x 128
        blocks on the layer's device (fp8.quantize_weight_blocks), then load_fp8"""
        E, H, I = self.num_experts, self.hidden_size, self.intermediate_size
        dev = self.gate_up_weight.device
        pairs = []
        for pname, w, (N, K) in (("gate", gate, (I, H)), ("up", up, (I, H)), ("down", down, (H, I))):
            if isinstance(w, (list, tuple)):
                if len(w) != E:
                    raise ValueError(f"{pname}: expected {E} per-expert tensors (got {len(w)})")
            elif not isinstance(w, torch.Tensor):
                raise TypeError(f"{pname} must be a torch.Tensor or a list of per-expert tensors")
            elif tuple(w.shape) != (E, N, K):
                raise ValueError(f"{pname} must be [{E}, {N}, {K}] stacked over the experts (got {list(w.shape)})")
            qs = []
            for e in range(E):
                if tuple(w[e].shape) != (N, K):
                    raise ValueError(f"{pname} expert {e} must be [{N}, {K}] (got {list(w[e].shape)})")
                qs.append(quantize_weight_blocks(w[e].to(dev)))
            pairs.append(([q for q, _ in qs], [s for _, s in qs]))
        self.load_fp8(*pairs)

    def extra_repr(self) -> str:
        return (f"num_experts={self.num_experts}, hidden_size={self.hidden_size}, intermediate_size={self.intermediate_size}, "
                f"A_dtype={self.A_dtype}")


__all__ = ["FP8MoEExperts"]
