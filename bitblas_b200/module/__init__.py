"""``bitblas.Linear`` (bitblas/module/__init__.py:77-370) on the H100 library.

Same constructor, buffers (``qweight`` / ``scales`` / ``zeros`` / ``bias`` or ``weight``; shapes and dtypes as in
module/__init__.py:164-205 so reference checkpoints load), ``forward``, ``load_and_transform_weight`` and the GPTQ
repack entry points.  Differences that matter here: the output is ``torch.empty`` (the reference memsets with
``torch.zeros`` on every call, :277), ``forward`` is ``Matmul.forward`` on the layer's buffers (checked once per distinct set)
instead of a pointer list handed to ``lib.call``, and the GPTQ repack runs as device kernels (bb_repack_gptq_*_device) instead of
Python column loops (:24-74).
"""
from __future__ import annotations

import ctypes
from logging import getLogger
from typing import List, Optional, Union

import torch
import torch.nn as nn

from .. import _lib, act_order
from ..cache import get_database_path, global_operator_cache
from ..ops.general_matmul import Matmul, MatmulConfig
from ..quantization.utils import general_compress
from ..utils import auto_detect_nvidia_target

logger = getLogger(__name__)

BITBLAS_DATABASE_PATH = get_database_path()


def _load_perm_from_state_dict(layer, state_dict, prefix):
    """`perm` is a buffer only on act-order layers (a layer without it keeps the reference's state_dict): take its presence and
    shape from the state dict being loaded, so that a strict load works in either direction."""
    saved = state_dict.get(prefix + "perm")
    layer.perm = None if saved is None else torch.empty_like(saved, device=layer.scales.device)


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
        # GPTQ act-order: int32 [K], sorted column j of qweight is input column perm[j]; None (and absent from the state_dict)
        # for every other layer
        self.register_buffer("perm", None)
        self.q_params = None

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

    def init_params(self):
        """``q_params``: the buffers' pointers in ``lib.call``'s positional order, for integrations that call it themselves after
        loading (the reference's surface).  ``forward`` does not read them."""
        cfg = self.bitblas_matmul.config
        named = [("weight", True)] if self.consistent else [("qweight", True), ("scales", cfg.with_scaling), ("zeros", cfg.with_zeros)]
        named.append(("bias", cfg.with_bias))
        self.q_params = [ctypes.c_void_p(getattr(self, name).data_ptr()) for name, used in named if used]

    def warmup(self, topk=20):
        self.bitblas_matmul.hardware_aware_finetune(topk=topk)

    def forward(self, A, output=None):
        op = self.bitblas_matmul
        if self.consistent:
            return op.forward(A, self.weight, bias=self.bias, output=output)
        if not A.is_contiguous():
            A = A.contiguous()
        cfg = op.config
        # every check of Matmul.forward passes before the act-order gather: a refused call launches nothing
        output, ptrs = op._check_forward(A, self.qweight, self.scales if cfg.with_scaling else None,
                                         self.zeros if cfg.with_zeros else None, self.bias if cfg.with_bias else None, output)
        if self.perm is not None:   # act-order: the weight's K axis is sorted, so A's columns are gathered to match
            A = act_order.permute_cols(A.view(-1, self.in_features), self.perm).view(A.shape)
        return op._launch(A, ptrs, output)

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
            self.perm = None   # field values come in input-column order

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        if not self.consistent:
            _load_perm_from_state_dict(self, state_dict, prefix)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def _repack(self, gptq_module, device, v2: bool):
        """module/__init__.py:315-363 as two device kernels (qweight transpose+permute, qzeros unpack).  An act-order module
        (g_idx, see act_order.py) has its qweight's K axis sorted first and keeps the order in `perm`."""
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("repack_from_gptq needs a CUDA device: bitblas_b200 has no CPU path")
        op = self.bitblas_matmul
        if self.torch_dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"GPTQ checkpoints need float16 or bfloat16 activations (A_dtype {op.A_dtype}): their scales are "
                             "stored in the activations' type")
        if self.bias is not None and getattr(gptq_module, "bias", None) is None:
            raise ValueError("the layer has bias=True but the GPTQ module has no bias")
        bits = self.bits
        qw = gptq_module.qweight.to(dev).contiguous().view(torch.int32)  # [K*bits/32, N]
        _, idx, stream = _lib.device_stream(qw)
        K, N = self.in_features, self.out_features
        assert qw.shape == (K * bits // 32, N), f"unexpected GPTQ qweight shape {tuple(qw.shape)}"
        perm = act_order.perm_from_g_idx(getattr(gptq_module, "g_idx", None), K, self.group_size)
        if perm is not None:
            perm = perm.to(dev)
            qw = act_order.permute_gptq_qweight(qw, perm, bits)
        out = torch.empty(op.retrieve_weight_shape(), dtype=torch.int8, device=dev)
        tgt = op.weight_transform.interleave_target if op.weight_transform is not None else 0
        _lib.call("bb_repack_gptq_qweight_device", idx, qw.data_ptr(), out.data_ptr(), K, N, bits, tgt, stream)
        self.qweight = op.tile_weight(out) if op.weight_tiled else out   # propagate_b: slab tiling of the packed rows
        # converted, not reinterpreted: checkpoints usually store float16 scales, whatever the layer's type
        self.scales = gptq_module.scales.to(dev).T.to(self.torch_dtype).contiguous()
        qz = gptq_module.qzeros.to(dev).contiguous().view(torch.int32)  # [K/g, N*bits/32]
        G = K // self.group_size
        mode = op.config.zeros_mode
        if mode == "quantized":
            zeros = torch.empty((G, N * bits // 8), dtype=torch.int8, device=dev)
        else:
            zeros = torch.empty((N, G), dtype=self.torch_dtype, device=dev)
        _lib.call("bb_repack_gptq_qzeros_device", idx, qz.data_ptr(), self.scales.data_ptr(), zeros.data_ptr(), G, N, bits,
                  _lib.ZEROS_IDS[mode], _lib.DTYPE_IDS[op.A_dtype], int(v2), stream)
        self.zeros = zeros
        if self.bias is not None:
            self.bias = gptq_module.bias.data.to(dev).to(self.torch_dtype).contiguous()
        self.perm = perm

    def repack_from_gptq(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=False)

    def repack_from_gptq_v2(self, gptq_module, device="cuda"):
        self._repack(gptq_module, device, v2=True)

    @property
    def consistent(self):
        return self.is_consitent


class GroupedLinear(nn.Module):
    """E quantized linear layers of one shape -- the experts of a mixture-of-experts projection -- run as one grouped matmul
    (``Matmul.forward_grouped``).  Constructor arguments after ``num_groups`` are those of ``Linear``; the buffers are
    ``Linear``'s stacked over the experts: ``qweight`` [E, N, K*bits/8], ``scales`` [E, N, K/g], ``zeros`` [E, N, K/g] (or
    [E, K/g, N*bits/8] for ``zeros_mode="quantized"``), ``bias`` [E, N] and, when some expert's GPTQ checkpoint is act-order,
    ``perm`` int32 [E, K] (the identity for the other experts), which ``forward`` gathers the activations with.  ``forward(A, offsets)`` takes the activations sorted
    by expert and the int32 device row offsets [E + 1]; routing, top-k weighting and combining stay with the caller (``MoEExperts``
    runs the whole SwiGLU expert block)."""

    def __init__(self, num_groups: int, in_features: int, out_features: int, bias: bool = False, **linear_kwargs):
        super().__init__()
        num_groups = int(num_groups)
        if not 1 <= num_groups <= _lib.BB_GROUPED_MAX_GROUPS:
            raise ValueError(f"num_groups must be in [1, {_lib.BB_GROUPED_MAX_GROUPS}] (got {num_groups})")
        # one Linear describes an expert (config, operator, per-expert buffer shapes); it owns no storage used here
        expert = Linear(in_features, out_features, bias=bias, **linear_kwargs)
        op = expert.bitblas_matmul
        if expert.consistent:
            raise ValueError("GroupedLinear needs a low-bit weight format (A_dtype != W_dtype)")
        op.check_grouped(num_groups)
        self.num_groups, self.in_features, self.out_features = num_groups, in_features, out_features
        self.bitblas_matmul, self.bits, self.group_size = op, expert.bits, expert.group_size
        self.torch_dtype = expert.torch_dtype
        self._expert_attrs = {k: getattr(expert, k) for k in ("in_features", "out_features", "group_size", "bits",
                                                              "torch_dtype", "bitblas_matmul")}
        for name, shape, dtype in expert._buffer_specs(bias):
            self.register_buffer(name, torch.zeros((num_groups, *shape), dtype=dtype))
        if not bias:
            self.bias = None
        self.register_buffer("perm", None)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        _load_perm_from_state_dict(self, state_dict, prefix)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def forward(self, A, offsets, output=None, capturable=False):
        """capturable=True: one graph-capturable launch at every token count (see Matmul.forward_grouped); an act-order layer
        launches the grouped column gather (act_order.permute_cols) first"""
        op = self.bitblas_matmul
        cfg = op.config
        if self.perm is not None:
            A = act_order.permute_cols(A, self.perm, offsets)
        return op.forward_grouped(A, self.qweight, offsets, scale=self.scales if cfg.with_scaling else None,
                                  zeros=self.zeros if cfg.with_zeros else None, bias=self.bias, output=output,
                                  capturable=capturable)

    def load_and_transform_weight(self, weight: torch.Tensor, scales: torch.Tensor = None, zeros: torch.Tensor = None,
                                  bias: torch.Tensor = None):
        """weight [E, N, K] of unsigned field values (signed for "int" formats), as Linear.load_and_transform_weight takes
        per expert; the storage transform works row by row, so the stacked tensor is transformed in one call."""
        if weight.dim() != 3 or weight.shape[0] != self.num_groups:
            raise ValueError(f"weight must be [E={self.num_groups}, N, K], got {tuple(weight.shape)}")
        self.qweight = self.bitblas_matmul.transform_weight(weight)
        if scales is not None:
            self.scales = scales
        if zeros is not None:
            self.zeros = zeros
        if bias is not None:
            self.bias = bias
        self.perm = None

    def _repack(self, gptq_modules, device, v2: bool, keep_perm: bool = True):
        """Linear's device repack (bb_repack_gptq_*_device) per expert, copied into the expert's slice of the stacked buffers.
        keep_perm=False: the act-order experts' K axes are sorted, but the caller feeds inputs already in that order (MoEExperts'
        down projection, whose perm is absorbed into the gate/up rows), so no perm is kept."""
        from types import SimpleNamespace
        if len(gptq_modules) != self.num_groups:
            raise ValueError(f"expected {self.num_groups} GPTQ modules, got {len(gptq_modules)}")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("repack_from_gptq needs a CUDA device: bitblas_b200 has no CPU path")
        for name in ("qweight", "scales", "zeros", "bias"):
            t = getattr(self, name)
            if t is not None and t.device != dev:
                setattr(self, name, t.to(dev))
        perms = []
        for e, gm in enumerate(gptq_modules):
            one = SimpleNamespace(**self._expert_attrs, bias=None if self.bias is None else self.bias[e])
            Linear._repack(one, gm, dev, v2)
            self.qweight[e].copy_(one.qweight)
            self.scales[e].copy_(one.scales)
            self.zeros[e].copy_(one.zeros)
            if self.bias is not None:
                self.bias[e].copy_(one.bias)
            perms.append(one.perm)
        self.perm = act_order.stack_perms(perms, self.in_features, dev) if keep_perm else None

    def repack_from_gptq(self, gptq_modules, device="cuda"):
        """one GPTQ QuantLinear per expert (how GPTQ mixture-of-experts checkpoints store them)"""
        self._repack(gptq_modules, device, v2=False)

    def repack_from_gptq_v2(self, gptq_modules, device="cuda"):
        self._repack(gptq_modules, device, v2=True)


__all__ = ["Linear", "GroupedLinear", "unpack_qzeros", "unpack_qzeros_v2", "unpack_qweight"]
