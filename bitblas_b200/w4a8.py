"""GPTQ 4-bit checkpoints with int8 activations (W4A8).

A W4A8 linear quantizes each token of its 16-bit input to int8 (``quantize_act_int8``, BitNet's absmax rule: one fp32 scale
per row, ``q = rint(x * s)``), then multiplies by the 4-bit weight on the int8 tensor cores (``Matmul.forward_w4a8``,
bb_matmul_w4a8): each quantization group's dot product is exact in int32, is promoted to fp32 with the group's scale, and the
sum over groups is divided by the row's activation scale.  The restatement in torch, with w the decoded integer weight
(u - z for uint weights with zero points, u - 8 for int4, u for uint4 without zeros):

    acc[r, n, g] = (q[:, group g] @ w[:, group g].T)                      exact
    S[r, n]      = sum_g float32(acc[r, n, g]) * scales[n, g]             fp32, the kernel's group order
    y[r, n]      = (S[r, n] / s[r]).to(A_dtype) (+ bias)

Activations are quantized per token, so W4A8 output differs from the W4A16 ``Linear`` on the same checkpoint by the int8
rounding of x; it is reproducible bit for bit for a given kernel, split factor and SM count (include/bitblas_b200.h).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib, act_order
from .bitnet import quantize_act_int8
from .module import _load_perm_from_state_dict
from .ops.general_matmul import Matmul, MatmulConfig

_ACT_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def pack_zeros(z: torch.Tensor) -> torch.Tensor:
    """zero points [N, G] (values 0 .. 15) -> the packed quantized layout [G, N / 2] int8: byte j of group g holds row 2j in
    its low nibble and row 2j + 1 in its high nibble"""
    zt = z.to(torch.int32).T.contiguous()
    return ((zt[:, 0::2] & 15) | ((zt[:, 1::2] & 15) << 4)).to(torch.uint8).view(torch.int8).contiguous()


class W4A8Linear(nn.Module):
    """``y = x W^T (+ bias)`` for x [.., in_features] of A_dtype (float16 | bfloat16), the output in the same dtype, with a
    4-bit weight (W_dtype uint4 or int4) in groups of ``group_size`` input columns (-1: one group), one fp32 scale per (row,
    group) and, for uint4 with ``with_zeros``, one 4-bit zero point per (row, group), as GPTQ stores them.

    Buffers: ``qweight`` int8 [out, in / 2] (interleaved for int8 activations), ``scales`` float32 [out, in / g], ``zeros`` int8
    [in / g, out / 2] (packed quantized zero points, with_zeros only), ``bias`` [out] in A_dtype (or None), and ``perm`` int32
    [in] for act-order checkpoints only.  ``forward`` is ``quantize_act_int8`` then ``Matmul.forward_w4a8``: two launches, three
    when the wgmma GEMM splits K or the layer is act-order (the input columns are gathered first), four with both; there is no
    host synchronisation, so ``CapturedStep`` can capture it."""

    def __init__(self, in_features: int, out_features: int, bias: bool = False, A_dtype: str = "float16",
                 W_dtype: str = "uint4", group_size: int = 128, with_zeros: bool = True):
        super().__init__()
        if A_dtype not in _ACT_DTYPES:
            raise ValueError(f"A_dtype must be float16 or bfloat16 (got {A_dtype})")
        if W_dtype not in ("uint4", "int4"):
            raise ValueError(f"W_dtype must be uint4 or int4 (got {W_dtype})")
        if with_zeros and W_dtype == "int4":
            raise ValueError("int4 weights take no zero points (with_zeros=False)")
        if in_features <= 0 or in_features % 16 or out_features <= 0 or out_features % 16:
            raise ValueError(f"in_features and out_features must be positive multiples of 16 (got {in_features}, {out_features})")
        g = in_features if group_size in (-1, None) else int(group_size)
        if g <= 0 or in_features % g:
            raise ValueError(f"group_size must be -1 or a positive divisor of in_features (got {group_size})")
        self.in_features, self.out_features, self.A_dtype, self.W_dtype = in_features, out_features, A_dtype, W_dtype
        self.group_size, self.with_zeros = g, bool(with_zeros)
        self.torch_dtype = _ACT_DTYPES[A_dtype]
        self.bitblas_matmul = Matmul(MatmulConfig(N=out_features, K=in_features, A_dtype="int8", W_dtype=W_dtype,
                                                  accum_dtype="int32", out_dtype=A_dtype, group_size=g, with_scaling=True,
                                                  with_zeros=self.with_zeros, zeros_mode="quantized" if self.with_zeros else None,
                                                  with_bias=bias, fast_decoding=True), enable_tuning=False)
        self.bitblas_matmul.check_w4a8()
        G = in_features // g
        self.register_buffer("qweight", torch.zeros(self.bitblas_matmul.retrieve_weight_shape(), dtype=torch.int8))
        self.register_buffer("scales", torch.ones(out_features, G, dtype=torch.float32))
        if self.with_zeros:
            self.register_buffer("zeros", torch.zeros(G, out_features // 2, dtype=torch.int8))
        else:
            self.zeros = None
        if bias:
            self.register_buffer("bias", torch.zeros(out_features, dtype=self.torch_dtype))
        else:
            self.bias = None
        self.register_buffer("perm", None)

    def load_quantized(self, q: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor = None, bias: torch.Tensor = None) -> None:
        """q [out, in] the stored 4-bit values u (0 .. 15, any integer dtype), scales [out, in / g] (converted to float32),
        zeros [out, in / g] the zero points (0 .. 15) exactly when the layer has them, bias [out] when the layer has one.  The
        weight's value is (u - z) * scale (uint4), (u - 8) * scale (int4)."""
        N, K, G = self.out_features, self.in_features, self.in_features // self.group_size
        q = torch.as_tensor(q)
        if tuple(q.shape) != (N, K):
            raise ValueError(f"q must be [{N}, {K}] (got {tuple(q.shape)})")
        qi = q.to(torch.int32)
        if not torch.equal(qi.to(q.dtype), q) or bool(((qi < 0) | (qi > 15)).any()):
            raise ValueError("q must hold 4-bit values 0 .. 15")
        scales = torch.as_tensor(scales)
        if tuple(scales.shape) != (N, G):
            raise ValueError(f"scales must be [{N}, {G}] (got {tuple(scales.shape)})")
        if (zeros is None) == self.with_zeros:
            raise ValueError("zeros must be given exactly when the layer was built with with_zeros=True")
        if zeros is not None:
            zeros = torch.as_tensor(zeros)
            if tuple(zeros.shape) != (N, G):
                raise ValueError(f"zeros must be [{N}, {G}] (got {tuple(zeros.shape)})")
            zi = zeros.to(torch.int32)
            if bool(((zi < 0) | (zi > 15)).any()):
                raise ValueError("zeros must hold 4-bit values 0 .. 15")
        if (bias is None) != (self.bias is None):
            raise ValueError("bias must be given exactly when the layer was built with bias=True")
        if bias is not None and tuple(bias.shape) != (N,):
            raise ValueError(f"bias must be [{N}] (got {tuple(bias.shape)})")
        # the stored fields are u for both formats (int4 decodes u - 8)
        self.qweight.copy_(self.bitblas_matmul.weight_transform(qi.to(torch.int8)).to(self.qweight.device))
        self.scales.copy_(scales.to(device=self.scales.device, dtype=torch.float32))
        if zeros is not None:
            self.zeros.copy_(pack_zeros(zeros).to(self.zeros.device))
        if bias is not None:
            self.bias.copy_(bias.to(device=self.bias.device, dtype=self.torch_dtype))
        self.perm = None

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        _load_perm_from_state_dict(self, state_dict, prefix)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def _repack(self, gptq_module, device, v2: bool):
        """Linear's GPTQ repack for int8 activations: qweight through bb_repack_gptq_qweight_device (interleaved for 8-bit
        targets), the fp16 / bf16 scales converted exactly to float32, qzeros through bb_repack_gptq_qzeros_device (packed,
        quantized).  An act-order module (g_idx) has its K axis sorted and keeps the order in ``perm``."""
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("repack_from_gptq needs a CUDA device: bitblas_b200 has no CPU path")
        if self.W_dtype != "uint4" or not self.with_zeros:
            raise ValueError("GPTQ checkpoints are uint4 with zero points: build the layer with W_dtype='uint4', with_zeros=True")
        if self.bias is not None and getattr(gptq_module, "bias", None) is None:
            raise ValueError("the layer has bias=True but the GPTQ module has no bias")
        op = self.bitblas_matmul
        K, N, G = self.in_features, self.out_features, self.in_features // self.group_size
        qw = gptq_module.qweight.to(dev).contiguous().view(torch.int32)   # [K / 8, N]
        if tuple(qw.shape) != (K // 8, N):
            raise ValueError(f"unexpected GPTQ qweight shape {tuple(qw.shape)} (expected {(K // 8, N)})")
        _, idx, stream = _lib.device_stream(qw)
        perm = act_order.perm_from_g_idx(getattr(gptq_module, "g_idx", None), K, self.group_size)
        if perm is not None:
            perm = perm.to(dev)
            qw = act_order.permute_gptq_qweight(qw, perm, 4)
        out = torch.empty(op.retrieve_weight_shape(), dtype=torch.int8, device=dev)
        _lib.call("bb_repack_gptq_qweight_device", idx, qw.data_ptr(), out.data_ptr(), K, N, 4, 8, stream)
        self.qweight = out
        self.scales = gptq_module.scales.to(dev).T.to(torch.float32).contiguous()
        qz = gptq_module.qzeros.to(dev).contiguous().view(torch.int32)   # [K / g, N / 8]
        zeros = torch.empty((G, N // 2), dtype=torch.int8, device=dev)
        _lib.call("bb_repack_gptq_qzeros_device", idx, qz.data_ptr(), 0, zeros.data_ptr(), G, N, 4, _lib.BB_ZEROS_QUANTIZED,
                  _lib.BB_F16, int(v2), stream)
        self.zeros = zeros
        if self.bias is not None:
            self.bias = gptq_module.bias.data.to(dev).to(self.torch_dtype).contiguous()
        self.perm = perm

    def repack_from_gptq(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=False)

    def repack_from_gptq_v2(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=True)

    def forward(self, x: torch.Tensor, output: torch.Tensor = None) -> torch.Tensor:
        """x [.., in_features] of A_dtype -> [.., out_features] of A_dtype; `output` may be given (contiguous, m * out elements)"""
        if not isinstance(x, torch.Tensor) or x.dtype != self.torch_dtype:
            raise TypeError(f"x must be a {self.torch_dtype} torch.Tensor")
        if x.dim() < 1 or x.shape[-1] != self.in_features:
            raise ValueError(f"x must be [.., {self.in_features}] (got {tuple(x.shape)})")
        if not x.is_contiguous():
            x = x.contiguous()
        if self.perm is not None:   # act-order: the weight's K axis is sorted, so x's columns are gathered to match
            x = act_order.permute_cols(x.view(-1, self.in_features), self.perm).view(x.shape)
        q, s = quantize_act_int8(x)
        return self.bitblas_matmul.forward_w4a8(q, self.qweight, s, self.scales, self.zeros, self.bias, output)

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"A_dtype={self.A_dtype}, W_dtype={self.W_dtype}, group_size={self.group_size}, with_zeros={self.with_zeros}")


__all__ = ["W4A8Linear", "pack_zeros"]
