"""128 x 128 block-scaled FP8 checkpoints (DeepSeek-V3 / R1, the Qwen3 -FP8 releases) on the H100's FP8 tensor cores.

Such a checkpoint stores each linear's ``weight`` as float8_e4m3fn [out, in] and ``weight_scale_inv`` as float32
[ceil(out / 128), in / 128]: the weight's value is weight[n, k] * weight_scale_inv[n // 128, k // 128].  At run time each token of
the 16-bit input is quantized to e4m3 in groups of 128 columns (vLLM's ``per_token_group_quant_fp8``), and the matmul promotes
each 128-k block's tensor-core sum into fp32 with the product of the two block scales.  Here that is two library launches,
``quantize_act_fp8`` (bb_quantize_act_fp8) and ``Matmul.forward_fp8`` (bb_matmul_fp8), three when the GEMM splits K.  The torch
restatement, with P_b the tensor core's sum over block b (each product exact; include/bitblas_b200.h):

    s[r, b] = max(max_{k in b} |x[r, k]|, 1e-10) / 448;   q = e4m3(clamp(x / s, -448, 448))
    S[r, n] = sum_b P_b[r, n] * (s[r, b] * weight_scale_inv[n // 128, b])       fp32, blocks ascending
    y       = S.to(A_dtype) (+ bias)
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .ops.general_matmul import Matmul, MatmulConfig

_ACT_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16}
E4M3_MAX = 448.0


def quantize_act_fp8(x: torch.Tensor):
    """Per-(token, 128-column block) e4m3 quantization in one launch (bb_quantize_act_fp8): x [.., K] float16 / bfloat16
    (K % 128 == 0) -> (q float8_e4m3fn with x's shape, s float32 [m, K / 128]) with m = x.numel() / K and, in fp32,
    s = max(amax, 1e-10) / 448 and q = e4m3_rn(clamp(x / s, -448, 448)) per block.  s is the transposed view of a k-block-major
    [K / 128, ld] buffer (ld = m rounded up to 4), the layout forward_fp8 reads."""
    if not isinstance(x, torch.Tensor) or x.dtype not in (torch.float16, torch.bfloat16):
        raise TypeError("x must be a float16 or bfloat16 torch.Tensor")
    if x.dim() < 1 or x.shape[-1] == 0 or x.shape[-1] % 128:
        raise ValueError(f"x must be [.., K] with K a positive multiple of 128 (got shape {tuple(x.shape)})")
    _lib.check_tensor(x, "x", x.dtype)
    K = x.shape[-1]
    rows = x.numel() // K
    ld = (rows + 3) // 4 * 4
    q = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    buf = torch.empty((K // 128, ld), dtype=torch.float32, device=x.device)
    _, idx, stream = _lib.device_stream(x)
    _lib.call("bb_quantize_act_fp8", idx, x.data_ptr(), _lib.dtype_id(x.dtype), rows, K, q.data_ptr(), buf.data_ptr(), ld, stream)
    return q, buf.t()[:rows]


def quantize_weight_blocks(w: torch.Tensor):
    """a float weight [N, K] (K % 128 == 0) -> (q float8_e4m3fn [N, K], s float32 [ceil(N / 128), K / 128]), in fp32 on w's
    device: per 128 x 128 block s = max(amax, 1e-10) / 448 and q = e4m3_rn(clamp(w / s, -448, 448)), the activation rule"""
    N, K = w.shape
    nb = (N + 127) // 128
    wf = torch.zeros((nb * 128, K), dtype=torch.float32, device=w.device)
    wf[:N] = w.float()
    blocks = wf.view(nb, 128, K // 128, 128)
    amax = blocks.abs().amax(dim=(1, 3)).clamp(min=1e-10)
    s = amax / torch.full_like(amax, E4M3_MAX)   # IEEE division (torch multiplies by the reciprocal of a Python scalar)
    q = (blocks / s[:, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(nb * 128, K)[:N].contiguous(), s


class FP8Linear(nn.Module):
    """``y = x W^T (+ bias)`` for x [.., in_features] of A_dtype (float16 | bfloat16), the output in the same dtype, with a
    128 x 128 block-scaled e4m3 weight as DeepSeek-V3 and Qwen3-FP8 store it.

    Buffers, under the checkpoint's own names so ``load_state_dict`` takes a shard's tensors unchanged: ``weight``
    float8_e4m3fn [out, in], ``weight_scale_inv`` float32 [ceil(out / 128), in / 128] and ``bias`` [out] in A_dtype (or None).
    ``forward`` is ``quantize_act_fp8`` then ``Matmul.forward_fp8``: two launches, three when the GEMM splits K, with no host
    synchronisation, so ``CapturedStep`` can capture it.  in_features % 128 == 0 and out_features % 16 == 0."""

    def __init__(self, in_features: int, out_features: int, bias: bool = False, A_dtype: str = "bfloat16"):
        super().__init__()
        if A_dtype not in _ACT_DTYPES:
            raise ValueError(f"A_dtype must be float16 or bfloat16 (got {A_dtype})")
        if in_features <= 0 or in_features % 128:
            raise ValueError(f"in_features must be a positive multiple of 128 (got {in_features})")
        if out_features <= 0 or out_features % 16:
            raise ValueError(f"out_features must be a positive multiple of 16 (got {out_features})")
        self.in_features, self.out_features, self.A_dtype = in_features, out_features, A_dtype
        self.torch_dtype = _ACT_DTYPES[A_dtype]
        self.bitblas_matmul = Matmul(MatmulConfig(N=out_features, K=in_features, A_dtype="e4m3_float8", W_dtype="e4m3_float8",
                                                  accum_dtype="float32", out_dtype=A_dtype, with_bias=bias), enable_tuning=False)
        self.bitblas_matmul.check_fp8()
        self.register_buffer("weight", torch.zeros(out_features, in_features, dtype=torch.float8_e4m3fn))
        self.register_buffer("weight_scale_inv", torch.ones((out_features + 127) // 128, in_features // 128, dtype=torch.float32))
        if bias:
            self.register_buffer("bias", torch.zeros(out_features, dtype=self.torch_dtype))
        else:
            self.bias = None

    def load_fp8(self, weight: torch.Tensor, weight_scale_inv: torch.Tensor, bias: torch.Tensor = None) -> None:
        """a checkpoint's tensors: weight float8_e4m3fn [out, in], weight_scale_inv [ceil(out / 128), in / 128] (float32, or
        16-bit floats, converted exactly), bias [out] exactly when the layer has one"""
        N, K = self.out_features, self.in_features
        if not isinstance(weight, torch.Tensor) or weight.dtype != torch.float8_e4m3fn:
            raise TypeError(f"weight must be a float8_e4m3fn tensor (got {getattr(weight, 'dtype', type(weight))})")
        if tuple(weight.shape) != (N, K):
            raise ValueError(f"weight must be [{N}, {K}] (got {tuple(weight.shape)})")
        sshape = ((N + 127) // 128, K // 128)
        if not isinstance(weight_scale_inv, torch.Tensor) or weight_scale_inv.dtype not in (torch.float32, torch.bfloat16,
                                                                                             torch.float16):
            raise TypeError("weight_scale_inv must be a float32 (or float16 / bfloat16) tensor")
        if tuple(weight_scale_inv.shape) != sshape:
            raise ValueError(f"weight_scale_inv must be {list(sshape)} (got {list(weight_scale_inv.shape)})")
        if (bias is None) != (self.bias is None):
            raise ValueError("bias must be given exactly when the layer was built with bias=True")
        if bias is not None and tuple(bias.shape) != (N,):
            raise ValueError(f"bias must be [{N}] (got {tuple(bias.shape)})")
        self.weight.copy_(weight.to(self.weight.device))
        self.weight_scale_inv.copy_(weight_scale_inv.to(device=self.weight_scale_inv.device, dtype=torch.float32))
        if bias is not None:
            self.bias.copy_(bias.to(device=self.bias.device, dtype=self.torch_dtype))

    def load_float_weight(self, weight: torch.Tensor, bias: torch.Tensor = None) -> None:
        """a float weight [out, in], quantized in 128 x 128 blocks on the layer's device (quantize_weight_blocks)"""
        if tuple(weight.shape) != (self.out_features, self.in_features):
            raise ValueError(f"weight must be [{self.out_features}, {self.in_features}] (got {tuple(weight.shape)})")
        q, s = quantize_weight_blocks(weight.to(self.weight.device))
        self.load_fp8(q, s, bias)

    def forward(self, x: torch.Tensor, output: torch.Tensor = None) -> torch.Tensor:
        """x [.., in_features] of A_dtype -> [.., out_features] of A_dtype; `output` may be given (contiguous, m * out elements)"""
        if not isinstance(x, torch.Tensor) or x.dtype != self.torch_dtype:
            raise TypeError(f"x must be a {self.torch_dtype} torch.Tensor")
        if x.dim() < 1 or x.shape[-1] != self.in_features:
            raise ValueError(f"x must be [.., {self.in_features}] (got {tuple(x.shape)})")
        if not x.is_contiguous():
            x = x.contiguous()
        q, s = quantize_act_fp8(x)
        return self.bitblas_matmul.forward_fp8(q, self.weight, s, self.weight_scale_inv, self.bias, output)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, A_dtype={self.A_dtype}"


__all__ = ["FP8Linear", "quantize_act_fp8", "quantize_weight_blocks"]
