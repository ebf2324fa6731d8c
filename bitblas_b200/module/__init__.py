"""``bitblas.Linear`` (bitblas/module/__init__.py:77-370) on the H100 library.

Same constructor, buffers (``qweight`` / ``scales`` / ``zeros`` / ``bias`` or ``weight``; shapes and dtypes as in
module/__init__.py:164-205 so reference checkpoints load), ``forward``, ``load_and_transform_weight`` and the GPTQ
repack entry points.  Differences that matter here: the output is ``torch.empty`` (the reference memsets with
``torch.zeros`` on every call, :277), the pointer list is built once, and the GPTQ repack runs as device kernels
(bb_repack_gptq_*_device) instead of Python column loops (:24-74).
"""
from __future__ import annotations

import ctypes
import operator
from functools import reduce
from logging import getLogger
from typing import List, Optional, Union

import torch
import torch.nn as nn

from .. import _lib
from ..cache import get_database_path, global_operator_cache
from ..ops.general_matmul import Matmul, MatmulConfig
from ..quantization.utils import general_compress
from ..utils import auto_detect_nvidia_target

logger = getLogger(__name__)

BITBLAS_DATABASE_PATH = get_database_path()


def unpack_qzeros(qzeros, bits):
    """module/__init__.py:24-39 (GPTQ v1: stored zero is z-1)."""
    qzeros = qzeros.view(torch.int32)
    epi = 32 // bits
    cols = torch.arange(qzeros.shape[1] * epi, device=qzeros.device)
    un = (qzeros[:, cols // epi] >> (bits * (cols % epi)).to(torch.int32)).to(torch.int8)
    return torch.bitwise_and(un + 1, 2**bits - 1)


def unpack_qzeros_v2(qzeros, bits):
    """module/__init__.py:43-58."""
    qzeros = qzeros.view(torch.int32)
    epi = 32 // bits
    cols = torch.arange(qzeros.shape[1] * epi, device=qzeros.device)
    un = (qzeros[:, cols // epi] >> (bits * (cols % epi)).to(torch.int32)).to(torch.int8)
    return torch.bitwise_and(un, 2**bits - 1)


def unpack_qweight(qweight, bits):
    """module/__init__.py:61-74."""
    qweight = qweight.view(torch.int8)
    epb = 8 // bits
    cols = torch.arange(qweight.shape[1] * epb, device=qweight.device)
    un = qweight[:, cols // epb] >> (bits * (cols % epb)).to(torch.int8)
    return torch.bitwise_and(un, 2**bits - 1)


class Linear(nn.Module):
    """Drop-in for ``bitblas.Linear``.  Public surface kept from the reference (module/__init__.py:77-370): constructor
    signature, the registered buffers and their shapes (so reference state dicts load), ``bitblas_matmul``, ``bits``,
    ``source_format``, ``opt_M``, ``q_params`` / ``init_params()``, ``consistent``, ``forward``, ``warmup``,
    ``load_and_transform_weight``, ``repack_from_gptq[_v2]``.  Everything underneath is this package's own."""

    opt_M = [16, 32, 64, 128, 256, 512]
    STORAGE_DTYPE = "int8"
    TORCH_STORAGE_DTYPE = torch.int8
    BITBLAS_DTYPES = {torch.float32: "float32", torch.float16: "float16", torch.half: "float16", torch.int8: "int8"}

    def __init__(self, in_features: int, out_features: int, bias: bool = False, A_dtype: str = "float16",
                 W_dtype: str = "float16", accum_dtype: str = "float16", out_dtype: str = "float16",
                 group_size: int = -1, with_scaling: bool = None, with_zeros: bool = False, zeros_mode: str = None,
                 opt_M: Union[int, List[int]] = opt_M, enable_tuning: bool = True,
                 fast_decoding: Optional[bool] = None, propagate_b: bool = False):
        super().__init__()
        if in_features % 16 or out_features % 16:
            raise ValueError("`in_features` and `out_features` must be divisible by 16.")
        gsize = in_features if group_size in (-1, None) else int(group_size)
        if gsize <= 0 or in_features % gsize:
            raise ValueError("`in_features` must be divisible by `group_size`.")
        self.in_features, self.out_features = in_features, out_features
        self.opt_M = opt_M
        self.group_size = gsize
        self.zeros_mode = zeros_mode
        self.torch_dtype = getattr(torch, A_dtype)
        self.is_consitent = A_dtype == W_dtype   # (sic) attribute name read by integrations of the reference
        config = MatmulConfig(M=opt_M, N=out_features, K=in_features, A_dtype=A_dtype, W_dtype=W_dtype,
                              accum_dtype=accum_dtype, out_dtype=out_dtype, storage_dtype=self.STORAGE_DTYPE,
                              group_size=gsize, with_scaling=with_scaling, with_zeros=with_zeros, zeros_mode=zeros_mode,
                              with_bias=bias, fast_decoding=fast_decoding, propagate_b=propagate_b)
        self.bitblas_matmul = self._operator_for(config)
        self.bits = self.bitblas_matmul.bit
        self.source_format = self.bitblas_matmul.source_format
        for name, shape, dtype in self._buffer_specs(bias):
            self.register_buffer(name, torch.zeros(shape, dtype=dtype))
        if not bias:
            self.bias = None
        self.q_params = None
        self._q_param_key = None

    # ---- construction helpers ------------------------------------------------------------------------
    def _buffer_specs(self, bias: bool):
        """(name, shape, dtype) of every registered buffer; shapes follow module/__init__.py:164-205."""
        n, groups = self.out_features, self.in_features // self.group_size
        specs = []
        if self.consistent:
            specs.append(("weight", (n, self.in_features), self.torch_dtype))
        else:
            specs.append(("qweight", tuple(self.bitblas_matmul.retrieve_weight_shape()), self.TORCH_STORAGE_DTYPE))
            specs.append(("scales", (n, groups), self.torch_dtype))
            if self.zeros_mode == "quantized":
                specs.append(("zeros", (groups, n * self.bits // 8), self.TORCH_STORAGE_DTYPE))   # `bits`-packed along N
            else:
                specs.append(("zeros", (n, groups), self.torch_dtype))
        if bias:
            specs.append(("bias", (n,), self.torch_dtype))
        return specs

    @staticmethod
    def _operator_for(config: MatmulConfig) -> Matmul:
        """one Matmul per distinct config, shared through the process-wide cache like the reference (:245-256)."""
        target = auto_detect_nvidia_target()
        if global_operator_cache.size() == 0:
            global_operator_cache.load_from_database(BITBLAS_DATABASE_PATH, target)
        op = global_operator_cache.get(config)
        if op is None:
            op = Matmul(config, target=target, enable_tuning=False)
            global_operator_cache.add(config, op)
        return op

    def _live_params(self):
        """tensors `lib.call` needs after the activations, in the reference's positional order."""
        cfg = self.bitblas_matmul.config
        if self.consistent:
            named = [("weight", True), ("bias", cfg.with_bias)]
        else:
            named = [("qweight", True), ("scales", cfg.with_scaling), ("zeros", cfg.with_zeros), ("bias", cfg.with_bias)]
        return [getattr(self, name) for name, used in named if used]

    def init_params(self):
        tensors = self._live_params()
        self.q_params = [ctypes.c_void_p(t.data_ptr()) for t in tensors]
        self._q_param_key = tuple(t.data_ptr() for t in tensors)

    def warmup(self, topk=20):
        self.bitblas_matmul.hardware_aware_finetune(topk=topk)

    def forward(self, A, output=None):
        op = self.bitblas_matmul
        if self.consistent:
            return op.forward(A, self.weight, bias=self.bias, output=output)
        if not A.is_cuda:
            raise RuntimeError("A must be a CUDA tensor: bitblas_b200 has no CPU path")
        if not A.is_contiguous():
            A = A.contiguous()
        if A.dtype != self.torch_dtype:
            raise TypeError(f"A has dtype {A.dtype}, expected {self.torch_dtype}")
        if A.shape[-1] != self.in_features:
            raise ValueError(f"A has inner dimension {A.shape[-1]}, expected {self.in_features}")
        stream = torch.cuda.current_stream(A.device)
        # the reference rebuilds this list on every call (module/__init__.py:274); rebuild only if a buffer moved
        if self.q_params is None or self._q_param_key != tuple(t.data_ptr() for t in self._live_params()):
            self.init_params()
        if output is None:
            output = torch.empty(A.shape[:-1] + (self.out_features,), dtype=getattr(torch, op.out_dtype), device=A.device)
        args = [ctypes.c_void_p(A.data_ptr()), *self.q_params, ctypes.c_void_p(output.data_ptr())]
        if op.dynamic_range is not None:
            args.append(reduce(operator.mul, A.shape[:-1], 1))
        args.append(ctypes.c_void_p(stream.cuda_stream))
        op.lib.call(*args)
        return output

    def load_and_transform_weight(self, weight: torch.Tensor, scales: torch.Tensor = None, zeros: torch.Tensor = None,
                                  bias: torch.Tensor = None):
        if self.consistent:
            assert scales is None, "scales should be None for consistent mode."
            assert zeros is None, "zeros should be None for consistent mode."
            weight = self.bitblas_matmul.transform_weight(weight)
            self.weight = nn.Parameter(weight, requires_grad=False)
            if bias is not None:
                self.bias = bias
        else:
            weight = self.bitblas_matmul.transform_weight(weight)
            self.qweight = weight
            if scales is not None:
                self.scales = scales
            if zeros is not None:
                self.zeros = zeros
            if bias is not None:
                self.bias = bias
        self.q_params = None

    def _repack(self, gptq_module, device, v2: bool):
        """module/__init__.py:315-363 as two device kernels (qweight transpose+permute, qzeros unpack)."""
        lib = _lib.load()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("repack_from_gptq needs a CUDA device: bitblas_b200 has no CPU path")
        _lib.ensure_init(dev.index if dev.index is not None else torch.cuda.current_device())
        op = self.bitblas_matmul
        bits = self.bits
        stream = torch.cuda.current_stream(dev).cuda_stream
        qw = gptq_module.qweight.to(dev).contiguous().view(torch.int32)  # [K*bits/32, N]
        K, N = self.in_features, self.out_features
        assert qw.shape == (K * bits // 32, N), f"unexpected GPTQ qweight shape {tuple(qw.shape)}"
        out = torch.empty(op.retrieve_weight_shape(), dtype=torch.int8, device=dev)
        tgt = op.weight_transform.interleave_target if op.weight_transform is not None else 0
        with torch.cuda.device(dev):
            _lib.check(lib.bb_repack_gptq_qweight_device(qw.data_ptr(), out.data_ptr(), K, N, bits, tgt, stream),
                       "bb_repack_gptq_qweight_device")
            self.qweight = op.tile_weight(out) if op.weight_tiled else out   # propagate_b: slab tiling of the packed rows
            self.scales = gptq_module.scales.to(dev).T.contiguous().view(self.torch_dtype)
            qz = gptq_module.qzeros.to(dev).contiguous().view(torch.int32)  # [K/g, N*bits/32]
            G = K // self.group_size
            mode = op.config.zeros_mode
            if mode == "quantized":
                zeros = torch.empty((G, N * bits // 8), dtype=torch.int8, device=dev)
            else:
                zeros = torch.empty((N, G), dtype=self.torch_dtype, device=dev)
            _lib.check(lib.bb_repack_gptq_qzeros_device(qz.data_ptr(), self.scales.data_ptr(), zeros.data_ptr(), G, N, bits,
                                                        _lib.ZEROS_IDS[mode], _lib.DTYPE_IDS[op.A_dtype], int(v2), stream),
                       "bb_repack_gptq_qzeros_device")
            self.zeros = zeros
        if self.bias is not None:
            self.bias = gptq_module.bias.data.to(dev).to(torch.float16).contiguous()
        self.q_params = None

    def repack_from_gptq(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=False)

    def repack_from_gptq_v2(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=True)

    @property
    def consistent(self):
        return self.is_consitent


__all__ = ["Linear", "unpack_qzeros", "unpack_qzeros_v2", "unpack_qweight"]
