"""``SwiGLUMLP``: the MLP of a dense SwiGLU model (Llama, Mistral, Qwen), ``down(silu(gate(x)) * up(x))``, as two library
launches.  The gate and up projections are one ``Linear`` of 2I rows in the gate/up interleave of ``bitblas_b200.moe`` (stored row
16b + i is gate row 8b + i for i < 8 and up row 8b + i - 8 for i >= 8), run by ``Matmul.forward_swiglu`` (bb_matmul_swiglu), which
forms silu(gate) * up in its kernel epilogue: the [m, 2I] pre-activations never reach memory and no elementwise kernel runs
between the two projections.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .act_order import permute_cols
from .moe import INTERLEAVE_ROWS, gate_up_act_order, interleave_gate_up
from .module import Linear


class SwiGLUMLP(nn.Module):
    """``y = down(silu(gate(x)) * up(x))`` for x [.., H]: ``gate_up`` (H -> 2I, gate/up interleaved) and ``down`` (I -> H) are
    ``Linear``s built from the ``Linear`` keyword arguments; ``out_dtype`` must equal ``A_dtype`` (the gate/up output is the down
    projection's input) and I a multiple of 8.  ``forward`` is ``gate_up.bitblas_matmul.forward_swiglu`` then ``down``: two
    launches with no host synchronisation (``CapturedStep`` can capture it).

    GPTQ act-order checkpoints (act_order.py): the gate/up projection's column order is ``gate_up.perm``, and ``forward`` gathers
    x with it first (three launches).  The down projection's order costs nothing: the gate and up output rows are loaded in it, so
    silu(gate) * up arrives sorted for the down projection's K axis and ``down.perm`` stays None.

    propagate_b=True (slab tiling): the interleave permutes rows and does not commute with the 32-row tiling, so the gate/up
    weight is interleaved in row-major packed form first and tiled after."""

    def __init__(self, hidden_size: int, intermediate_size: int, bias: bool = False, **linear_kwargs):
        super().__init__()
        if intermediate_size % INTERLEAVE_ROWS:
            raise ValueError(f"intermediate_size must be a multiple of {INTERLEAVE_ROWS} (gate/up interleave; got {intermediate_size})")
        a_dtype = linear_kwargs.get("A_dtype", "float16")
        if linear_kwargs.get("out_dtype", "float16") != a_dtype:
            raise ValueError("SwiGLUMLP needs out_dtype == A_dtype: the gate/up output is the down projection's input")
        self.hidden_size, self.intermediate_size = hidden_size, intermediate_size
        self.gate_up = Linear(hidden_size, 2 * intermediate_size, bias=bias, **linear_kwargs)
        self.down = Linear(intermediate_size, hidden_size, bias=bias, **linear_kwargs)
        self.gate_up.bitblas_matmul.check_swiglu()
        self._linear_kwargs = dict(linear_kwargs, bias=bias)

    def forward(self, x: torch.Tensor, output: torch.Tensor = None) -> torch.Tensor:
        """x [.., H] -> [.., H]; `output` as in Linear.forward"""
        gu = self.gate_up
        op, cfg = gu.bitblas_matmul, gu.bitblas_matmul.config
        if not x.is_contiguous():
            x = x.contiguous()
        # every check passes before the act-order gather: a refused call launches nothing
        h, ptrs = op._check_forward(x, gu.qweight, gu.scales if cfg.with_scaling else None, gu.zeros if cfg.with_zeros else None,
                                    gu.bias if cfg.with_bias else None, None, swiglu=True)
        if gu.perm is not None:
            x = permute_cols(x.view(-1, self.hidden_size), gu.perm).view(x.shape)
        op._launch(x, ptrs, h, swiglu=True)
        return self.down(h, output)

    # ---- loading -----------------------------------------------------------------------------------------------------------
    def _zeros_kind(self):
        return "qzeros" if self.gate_up.bitblas_matmul.config.zeros_mode == "quantized" else "zeros"

    def load_and_transform_weight(self, gate, up, down):
        """gate, up, down: (weight, scales, zeros, bias) per projection as Linear.load_and_transform_weight takes them (None where
        the config has none; missing trailing entries are None).  gate and up are interleaved row by row before the storage
        transform, which packs (and with propagate_b tiles) the fused rows."""
        g, u = (tuple(gate) + (None,) * 4)[:4], (tuple(up) + (None,) * 4)[:4]
        kinds = ("weight", "scale", self._zeros_kind(), "bias")
        fused = [None if a is None else interleave_gate_up(a, b, kind, self.gate_up.bits) for a, b, kind in zip(g, u, kinds)]
        self.gate_up.load_and_transform_weight(*fused)
        self.down.load_and_transform_weight(*down)

    def _repack(self, gate_module, up_module, down_module, device, v2):
        H, I = self.hidden_size, self.intermediate_size
        gu = self.gate_up
        gate_module, up_module = gate_up_act_order(gate_module, up_module, down_module, H, I, gu.group_size, self.down.group_size,
                                                   gu.bits)
        # the halves in row-major storage: the fused rows are tiled after the interleave
        kw = dict(self._linear_kwargs, propagate_b=False)
        bias = kw.pop("bias")
        halves = []
        for mod in (gate_module, up_module):
            half = Linear(H, I, bias=bias, **kw)
            half._repack(mod, device, v2)
            halves.append(half)
        g, u = halves
        op = gu.bitblas_matmul
        qweight = interleave_gate_up(g.qweight, u.qweight, "weight")
        gu.qweight = op.tile_weight(qweight) if op.weight_tiled else qweight
        gu.scales = interleave_gate_up(g.scales, u.scales, "scale")
        gu.zeros = interleave_gate_up(g.zeros, u.zeros, self._zeros_kind(), gu.bits)
        if gu.bias is not None:
            gu.bias = interleave_gate_up(g.bias, u.bias, "bias")
        gu.perm = g.perm
        self.down._repack(down_module, device, v2)
        self.down.perm = None   # absorbed into the gate/up rows: down's input arrives in its sorted K order

    def repack_from_gptq(self, gate_module, up_module, down_module, device="cuda"):
        """one GPTQ QuantLinear per projection: Linear's repack of gate and up, the interleave, then down.  Act-order modules
        (g_idx) are taken as described in the class documentation; gate and up must have the same g_idx (ValueError otherwise)."""
        self._repack(gate_module, up_module, down_module, device, v2=False)

    def repack_from_gptq_v2(self, gate_module, up_module, down_module, device="cuda"):
        self._repack(gate_module, up_module, down_module, device, v2=True)


__all__ = ["SwiGLUMLP"]
