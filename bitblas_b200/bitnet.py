"""BitNet b1.58 layers: ternary weights (int2 storage) against int8 activations quantized per token on the device.

A BitNet linear quantizes each token of its 16-bit input to int8 with its own absmax scale (``activation_quant``), multiplies by
the ternary weight in exact int32, and divides the sum by the activation scale and then by the weight scale.  Here that is two
library launches: ``quantize_act_int8`` (bb_quantize_act_int8) and ``Matmul.forward_scaled`` (bb_matmul_scaled), whose kernel
epilogue applies both scales.  Every step is fp32 and correctly rounded, so a layer's output is reproducible bit for bit against
the torch restatement

    s = 127.0 / x.float().abs().amax(-1).clamp(min=1e-5);   q = (x.float() * s).round().clamp(-128, 127).to(int8)
    y = ((q @ w.T).float() / s / w_scale).to(dtype) (+ bias)
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .ops.general_matmul import Matmul, MatmulConfig

_ACT_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def quantize_act_int8(x: torch.Tensor, q: torch.Tensor = None, scale: torch.Tensor = None):
    """Per-token int8 quantization in one launch (bb_quantize_act_int8): x [.., K] float16 / bfloat16 (K % 8 == 0) -> (q int8
    [.., K], scale float32 [m]) with m = x.numel() / K, per row scale = 127 * (1 / max(max|x|, 1e-5)) (torch's evaluation of
    BitNet's `127.0 / t`) and q = clamp(rint(x * scale), -128, 127), all in fp32.  `q` and `scale` may be given as outputs
    (contiguous, on x's device)."""
    if not isinstance(x, torch.Tensor) or x.dtype not in (torch.float16, torch.bfloat16):
        raise TypeError("x must be a float16 or bfloat16 torch.Tensor")
    if x.dim() < 1 or x.shape[-1] == 0 or x.shape[-1] % 8:
        raise ValueError(f"x must be [.., K] with K a positive multiple of 8 (got shape {tuple(x.shape)})")
    _lib.check_tensor(x, "x", x.dtype)
    K = x.shape[-1]
    rows = x.numel() // K
    if q is None:
        q = torch.empty(x.shape, dtype=torch.int8, device=x.device)
    else:
        _lib.check_tensor(q, "q", torch.int8, numel=x.numel())
    if scale is None:
        scale = torch.empty(rows, dtype=torch.float32, device=x.device)
    else:
        _lib.check_tensor(scale, "scale", torch.float32, numel=rows)
    if q.device != x.device or scale.device != x.device:
        raise ValueError(f"q and scale must be on x's device {x.device}")
    _, idx, stream = _lib.device_stream(x)
    _lib.call("bb_quantize_act_int8", idx, x.data_ptr(), _lib.dtype_id(x.dtype), rows, K, q.data_ptr(), scale.data_ptr(), stream)
    return q, scale


def absmean_ternary(weight: torch.Tensor):
    """BitNet b1.58's weight quantization: (ternary values [N, K] as float32, their scale sw = 1 / max(mean|W|, 1e-5)), in fp32
    on weight's device"""
    w = weight.float()
    sw = 1.0 / w.abs().mean().clamp(min=1e-5)
    return (w * sw).round().clamp(-1, 1), sw


class BitLinear(nn.Module):
    """A BitNet b1.58 linear layer, ``y = x W^T (+ bias)`` for x [.., in_features] of A_dtype (float16 | bfloat16), the output in
    the same dtype.  The weight is ternary, stored as int2 (``Matmul`` with A_dtype="int8", W_dtype="int2", interleaved for int8
    activations), with one fp32 quantization scale per output row.

    Buffers: ``qweight`` int8 [out, in / 4], ``weight_scale`` float32 [out], ``bias`` [out] in A_dtype (or None).  ``forward`` is
    ``quantize_act_int8`` then ``Matmul.forward_scaled``: two launches (three when the wgmma GEMM splits K) and no host
    synchronisation, so ``CapturedStep`` can capture it."""

    def __init__(self, in_features: int, out_features: int, bias: bool = False, A_dtype: str = "float16"):
        super().__init__()
        if A_dtype not in _ACT_DTYPES:
            raise ValueError(f"A_dtype must be float16 or bfloat16 (got {A_dtype})")
        if in_features <= 0 or in_features % 16:
            raise ValueError(f"in_features must be a positive multiple of 16 (2-bit weights fill whole 32-bit words; got {in_features})")
        if out_features <= 0:
            raise ValueError(f"out_features must be positive (got {out_features})")
        self.in_features, self.out_features, self.A_dtype = in_features, out_features, A_dtype
        self.torch_dtype = _ACT_DTYPES[A_dtype]
        self.bitblas_matmul = Matmul(MatmulConfig(N=out_features, K=in_features, A_dtype="int8", W_dtype="int2",
                                                  accum_dtype="int32", out_dtype=A_dtype, with_bias=bias), enable_tuning=False)
        self.bitblas_matmul.check_scaled()
        self.register_buffer("qweight", torch.zeros(self.bitblas_matmul.retrieve_weight_shape(), dtype=torch.int8))
        self.register_buffer("weight_scale", torch.ones(out_features, dtype=torch.float32))
        if bias:
            self.register_buffer("bias", torch.zeros(out_features, dtype=self.torch_dtype))
        else:
            self.bias = None

    def load_quantized(self, q: torch.Tensor, weight_scale, bias: torch.Tensor = None) -> None:
        """q [out, in] with values in {-1, 0, 1} (any numeric dtype); weight_scale a number, a one-element tensor or [out]: the
        quantization scale(s), so the weight's value is q / weight_scale; bias [out] when the layer has one"""
        N, K = self.out_features, self.in_features
        q = torch.as_tensor(q)
        if tuple(q.shape) != (N, K):
            raise ValueError(f"q must be [{N}, {K}] (got {tuple(q.shape)})")
        qi = q.to(torch.int32)
        if not torch.equal(qi.to(q.dtype), q) or bool(((qi < -1) | (qi > 1)).any()):
            raise ValueError("q must hold ternary values -1, 0 and 1")
        sw = torch.as_tensor(weight_scale, dtype=torch.float32).reshape(-1)
        if sw.numel() == 1:
            sw = sw.expand(N)
        if sw.numel() != N:
            raise ValueError(f"weight_scale must be one value or [{N}] (got {sw.numel()} values)")
        if (bias is None) != (self.bias is None):
            raise ValueError("bias must be given exactly when the layer was built with bias=True")
        if bias is not None and tuple(bias.shape) != (N,):
            raise ValueError(f"bias must be [{N}] (got {tuple(bias.shape)})")
        packed = self.bitblas_matmul.transform_weight(qi.to(torch.int8))
        self.qweight.copy_(packed.to(self.qweight.device))
        self.weight_scale.copy_(sw.to(self.weight_scale.device))
        if bias is not None:
            self.bias.copy_(bias.to(device=self.bias.device, dtype=self.torch_dtype))

    def load_float_weight(self, weight: torch.Tensor, bias: torch.Tensor = None) -> None:
        """a float weight [out, in] quantized by BitNet's absmean rule (absmean_ternary): one per-tensor scale for every row"""
        q, sw = absmean_ternary(weight)
        self.load_quantized(q, sw, bias)

    def forward(self, x: torch.Tensor, output: torch.Tensor = None) -> torch.Tensor:
        """x [.., in_features] of A_dtype -> [.., out_features] of A_dtype; `output` may be given (contiguous, m * out elements)"""
        if not isinstance(x, torch.Tensor) or x.dtype != self.torch_dtype:
            raise TypeError(f"x must be a {self.torch_dtype} torch.Tensor")
        if x.dim() < 1 or x.shape[-1] != self.in_features:
            raise ValueError(f"x must be [.., {self.in_features}] (got {tuple(x.shape)})")
        if not x.is_contiguous():
            x = x.contiguous()
        q, s = quantize_act_int8(x)
        return self.bitblas_matmul.forward_scaled(q, self.qweight, s, self.weight_scale, self.bias, output)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, A_dtype={self.A_dtype}"


__all__ = ["BitLinear", "absmean_ternary", "quantize_act_int8"]
