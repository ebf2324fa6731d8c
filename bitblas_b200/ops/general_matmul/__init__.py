"""``MatmulConfig`` / ``Matmul``: the operator API of bitblas/ops/general_matmul/__init__.py, re-hosted on the
prebuilt sm_90a library.

Same fields, defaults and legalisation as the reference ``MatmulConfig`` (general_matmul/__init__.py:58-237), same
``Matmul`` surface (``forward/__call__``, ``transform_weight``, ``transform_input``, ``retrieve_weight_shape``,
``weight_transform``, ``lib.init()/lib.call(...)``, config-mirroring properties :761-841).  What changes is what is
underneath: no TVM/TileLang code generation, no tuning, no per-operator compilation -- ``lib.call`` crosses the C ABI
of ``include/bitblas_b200.h`` into hand-written CUDA.
"""
from __future__ import annotations

import ctypes
import logging
import operator as _operator
from dataclasses import dataclass
from functools import reduce
from typing import Any, Literal, Optional, Tuple, Union

import torch

from ... import _lib
from ..operator import Operator, OperatorConfig, OptimizeStrategy, TransformKind

logger = logging.getLogger(__name__)

WORKSPACE_SIZE = 1024 * 1024 * 256

NATIVE_COMPUTE_PATTERNS = [  # general_matmul/__init__.py:33-47
    ("float64", "float64"), ("float32", "float32"), ("float16", "float16"), ("bfloat16", "bfloat16"),
    ("int8", "int8"), ("uint8", "uint8"), ("int4", "int4"), ("uint4", "uint4"),
    ("e4m3_float8", "e4m3_float8"), ("e4m3_float8", "e5m2_float8"), ("e5m2_float8", "e4m3_float8"),
    ("e5m2_float8", "e5m2_float8"),
]


def is_native_compute(A_dtype, W_dtype) -> bool:
    return (A_dtype, W_dtype) in NATIVE_COMPUTE_PATTERNS


@dataclass(frozen=True)
class MatmulConfig(OperatorConfig):
    M: Union[int, Tuple[int]] = None
    N: Optional[int] = None
    K: Optional[int] = None
    A_dtype: str = "float16"
    W_dtype: str = A_dtype
    out_dtype: str = "float16"
    accum_dtype: str = "float16"
    layout: Literal["nn", "nt", "tn", "tt"] = "nt"
    with_bias: bool = False
    group_size: int = -1
    with_scaling: bool = False
    with_zeros: bool = False
    # original: (w - z) * s ; rescale: w * s - z ; quantized: (w - dequant(qz)) * s
    zeros_mode: Literal["original", "rescale", "quantized"] = "original"
    storage_dtype: str = "int8"
    fast_decoding: Optional[bool] = None
    propagate_a: Optional[TransformKind] = None
    propagate_b: Optional[TransformKind] = None
    optimize_stratety: Union[int, OptimizeStrategy] = OptimizeStrategy.SingleBatchDecodeOnly  # (sic)

    def _set(self, name, value):
        object.__setattr__(self, name, value)

    @staticmethod
    def _legalize_propagate(propagate):
        if isinstance(propagate, bool):
            return TransformKind.LDMatrixTransform if propagate else TransformKind.NonTransform
        if isinstance(propagate, int):
            return TransformKind(propagate)
        return propagate

    def _initialize_fast_decoding(self, fast_decoding):
        # general_matmul/__init__.py:163-184
        unsupported = any([
            "int" not in self.W_dtype,
            self.W_dtype == self.A_dtype,
            self.W_dtype in ["int8", "uint8"],
            self.W_dtype in ["int4", "uint4"] and self.A_dtype in ["int8"],
            self.A_dtype == "bfloat16",
        ])
        if fast_decoding is not None:
            self._set("fast_decoding", fast_decoding)
        else:
            self._set("fast_decoding", not unsupported)

    def __post_init__(self):
        if self.M is None:
            if self.optimize_stratety == OptimizeStrategy.SingleBatchDecodeOnly:
                self._set("M", [1, 16, 32, 64, 128, 256, 512, 1024])
            else:
                self._set("M", [16, 32, 64, 128, 256, 512, 1024])
        if self.N is None:
            raise ValueError("N should be specified currently.")
        if self.K is None:
            raise ValueError("K should be specified currently.")
        self._set("M", tuple(self.M) if isinstance(self.M, list) else self.M)
        if isinstance(self.optimize_stratety, int) and not isinstance(self.optimize_stratety, OptimizeStrategy):
            self._set("optimize_stratety", OptimizeStrategy(self.optimize_stratety))
        # Weight propagation (general_matmul/__init__.py:113-157).  The reference re-tiles W offline into mma.sync /
        # ldmatrix fragment order; wgmma operands are laid out in registers by the kernels themselves, so that particular
        # permutation has no meaning here.  What an offline layout still buys on H100 is DRAM / TMA locality: a requested
        # propagate_b selects the slab tiling BB_TILE_SLAB (include/bitblas_b200.h: [N/32][row_bytes/512][32][512 B]; one
        # work unit of the decode GEMV = one contiguous 16 KB block).  Default (None / False): the reference's row-major
        # storage, byte-compatible with its checkpoints.  propagate_a never applies (activations are consumed as they are).
        requested_b = self._legalize_propagate(self.propagate_b)
        want_tile = requested_b not in (None, TransformKind.NonTransform)
        if want_tile:
            wbits = {"int4": 4, "uint4": 4, "int2": 2, "uint2": 2}.get(self.W_dtype)
            ok = (wbits is not None and self.W_dtype != self.A_dtype and self.N % 128 == 0
                  and (self.K * wbits // 8) % _lib.BB_TILE_ROW_BYTES == 0 and (self.K * wbits) % 8 == 0)
            if not ok:
                logger.warning("propagate_b: slab tiling needs a 4/2-bit integer weight, N %% 128 == 0 and K*bits/8 %% 512 == 0 "
                               "(N=%s K=%s W_dtype=%s); keeping the row-major storage", self.N, self.K, self.W_dtype)
                want_tile = False
        self._set("propagate_a", TransformKind.NonTransform)
        self._set("propagate_b", TransformKind.LDMatrixTransform if want_tile else TransformKind.NonTransform)
        if self.zeros_mode is None:
            self._set("zeros_mode", "original")
        self._initialize_fast_decoding(self.fast_decoding)
        if self.with_bias is None:
            self._set("with_bias", False)
        if self.group_size is None:
            self._set("group_size", -1)
        if self.with_scaling is None:
            self._set("with_scaling", False)
        if self.with_zeros is None:
            self._set("with_zeros", False)
        if self.A_dtype == self.W_dtype and self.W_dtype in ["float16", "bfloat16", "int8", "e4m3_float8", "e5m2_float8"]:
            self._set("storage_dtype", self.W_dtype)


class WeightTransform:
    """Stand-in for the reference's ``OPExecutorCPU`` chain [QuantCompress][LOP3Permutate]
    (general_matmul/__init__.py:557-565, operator.py:529-556).  Callable on an int8 [N, K] tensor of unsigned
    field values; returns the packed (and, with fast decoding, interleaved) int8 [N, K*bits/8] tensor.  CPU
    tensors go through the C++ host routines, CUDA tensors through the single-pass device kernel."""

    def __init__(self, bits: int, interleave_target: int):
        self.bits = bits
        self.interleave_target = interleave_target  # 0: none, 8 / 16: LOP3 interleave
        self.operators = ["QuantCompress"] + (["LOP3Permutate"] if interleave_target else [])

    @property
    def size(self):
        return len(self.operators)

    def forward(self, weight: torch.Tensor) -> torch.Tensor:
        lib = _lib.load()
        if weight.dtype != torch.int8:
            weight = weight.to(torch.int8)
        weight = weight.contiguous()
        rows = weight.numel() // weight.shape[-1]
        cols = weight.shape[-1]
        epw = 32 // self.bits
        if cols % epw:
            raise ValueError(f"K={cols} must be a multiple of {epw} for {self.bits}-bit storage")
        out = torch.empty(weight.shape[:-1] + (cols * self.bits // 8,), dtype=torch.int8, device=weight.device)
        if weight.is_cuda:
            _lib.ensure_init(weight.device.index or 0)
            stream = torch.cuda.current_stream(weight.device).cuda_stream
            with torch.cuda.device(weight.device):
                _lib.check(lib.bb_transform_weight_device(weight.data_ptr(), out.data_ptr(), rows, cols, self.bits,
                                                          self.interleave_target, stream), "bb_transform_weight_device")
            return out
        _lib.check(lib.bb_compress_host(weight.data_ptr(), out.data_ptr(), rows, cols, self.bits), "bb_compress_host")
        if self.interleave_target:
            out2 = torch.empty_like(out)
            _lib.check(lib.bb_interleave_host(out.data_ptr(), out2.data_ptr(), out.numel(), self.bits,
                                              self.interleave_target), "bb_interleave_host")
            out = out2
        return out

    __call__ = forward


class _LibShim:
    """``matmul.lib``: exposes ``init()`` and ``call(*ptrs, [m], stream)`` with the reference's positional order
    A, B, [LUT], [Scale], [Zeros|Qzeros], [Bias], C, [m], stream (builder/wrapper/base.py:5-19; callers:
    ops/operator.py:458-463, module/__init__.py:275-287)."""

    def __init__(self, op: "Matmul"):
        self._op = op
        self._c = _lib.load()

    def init(self):
        if torch.cuda.is_available():
            _lib.ensure_init(torch.cuda.current_device())

    @staticmethod
    def _ptr(v):
        if isinstance(v, ctypes.c_void_p):
            return v.value or 0
        if isinstance(v, torch.Tensor):
            return v.data_ptr()
        return int(v) if v is not None else 0

    def call(self, *args):
        op = self._op
        args = list(args)
        stream = self._ptr(args.pop())
        m = int(args.pop()) if op.dynamic_range is not None else int(op.M)
        ptrs = [self._ptr(a) for a in args]
        expect = 3 + int(op.lut is not None) + int(op.with_scaling) + int(op.with_zeros) + int(op.with_bias)
        if op.lut is not None and len(ptrs) == expect - 1:
            # bitblas.Linear-style callers pass A, qweight, [scales], [zeros], [bias], C and never the NF4 table
            # (module/__init__.py:275-287 has the same omission): supply the operator's own
            ptrs.insert(2, op.lut.data_ptr())
        if len(ptrs) != expect:
            raise TypeError(f"lib.call expected {expect} buffers (A, W, [lut], [scale], [zeros], [bias], C), got {len(ptrs)}")
        it = iter(ptrs)
        A = next(it); W = next(it)
        lut = next(it) if op.lut is not None else 0
        scale = next(it) if op.with_scaling else 0
        zeros = next(it) if op.with_zeros else 0
        bias = next(it) if op.with_bias else 0
        C = next(it)
        ws_ptr, ws_bytes = op._workspace_for(m, torch.device("cuda", torch.cuda.current_device())) if torch.cuda.is_available() else (0, 0)
        rc = self._c.bb_matmul(ctypes.byref(op._desc), A, W, lut, scale, zeros, bias, C, m, ws_ptr, ws_bytes, stream)
        if rc != 0:
            raise RuntimeError(f"bb_matmul failed (code {rc}): {_lib.last_error()}")


class Matmul(Operator):
    BITBLAS_TRICK_DTYPE_MAP = {  # general_matmul/__init__.py:324-345
        "float64": ("fp", 64), "float32": ("fp", 32), "float16": ("fp", 16), "bfloat16": ("bf", 16),
        "int32": ("int", 32), "uint32": ("uint", 32), "int16": ("int", 16), "uint16": ("uint", 16),
        "int8": ("int", 8), "uint8": ("uint", 8), "int4": ("int", 4), "uint4": ("uint", 4),
        "int2": ("int", 2), "uint2": ("uint", 2), "int1": ("int", 1), "uint1": ("uint", 1),
        "nf4": ("nf", 4), "fp4_e2m1": ("fp", 4), "e4m3_float8": ("fp_e4m3", 8), "e5m2_float8": ("fp_e5m2", 8),
    }
    NF4_LUT = [  # general_matmul/__init__.py:414-432
        -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
        -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
        0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0,
    ]

    def __init__(self, config: MatmulConfig, name: str = "matmul", target=None, enable_tuning: bool = True,
                 from_database: bool = False, backend: str = "b200"):
        if target is None:
            from ...utils import auto_detect_nvidia_target
            target = auto_detect_nvidia_target()
        assert config.A_dtype in self.BITBLAS_TRICK_DTYPE_MAP, f"Unsupported input dtype {config.A_dtype}"
        assert config.W_dtype in self.BITBLAS_TRICK_DTYPE_MAP, f"Unsupported weight dtype {config.W_dtype}"
        source_format, bit = self.BITBLAS_TRICK_DTYPE_MAP[config.W_dtype]
        self.source_format = source_format
        self.bit = bit
        super().__init__(name, config, target, backend)
        if config.layout != "nt":
            # the dequantize path of the reference supports only "nt" (tirscript/matmul_dequantize_impl.py:912-915)
            raise ValueError(f"Unsupported layout: {config.layout} (only 'nt' is supported)")
        if source_format == "int" and self.with_zeros:
            logger.warning("[BitBLAS][Warning] with_zeros is not supported for int source format as int has a "
                           "constant zeropoints already.")
        self.consistent = is_native_compute(config.A_dtype, config.W_dtype)
        self.dynamic_range = {"m": self.M} if isinstance(self.M, tuple) else None
        self.workspace = None
        self.torch_output_dtype = getattr(torch, self.out_dtype)
        self.lut = None
        if source_format == "nf":
            self.lut = torch.tensor(self.NF4_LUT, dtype=getattr(torch, self.A_dtype))
            if torch.cuda.is_available():
                self.lut = self.lut.cuda()
        self._desc = None
        self._ws = {}
        self._ws_need = {}
        self._checked_key = None
        self._torch_a_dtype = getattr(torch, config.A_dtype, None)
        self._desc_ref = None
        self.weight_executors = None
        self.input_executors = None
        if not self.consistent:
            self._desc = self._make_desc()
            self._desc_ref = ctypes.byref(self._desc)
            if bit in (1, 2, 4):
                tgt = 0
                if self.fast_decoding:
                    assert source_format in ("int", "uint"), "fast decoding needs an integer weight format"
                    tgt = 8 if self.A_dtype == "int8" else 16
                self.weight_executors = WeightTransform(bit, tgt)
        self.lib = _LibShim(self) if not self.consistent else None
        if self.lib is not None:
            self.lib.init()

    # ---- descriptor --------------------------------------------------------------------------
    def _make_desc(self) -> _lib.MatmulDesc:
        c = self.config
        if c.A_dtype not in ("float16", "bfloat16", "int8"):
            raise ValueError(f"A_dtype {c.A_dtype} is not supported by the dequantize path (float16 | bfloat16 | int8)")
        fmt = self.source_format
        if fmt not in _lib.WFMT_IDS:
            raise ValueError(f"W_dtype {c.W_dtype} is not a supported low-bit weight format")
        d = _lib.MatmulDesc()
        d.N, d.K = int(c.N), int(c.K)
        d.a_dtype = _lib.DTYPE_IDS[c.A_dtype]
        d.w_fmt = _lib.WFMT_IDS[fmt]
        d.w_bits = int(self.bit)
        if c.A_dtype == "int8":
            if c.accum_dtype != "int32":
                raise ValueError("int8 activations require accum_dtype='int32'")
            d.accum_dtype = _lib.BB_I32
        else:
            if c.accum_dtype not in ("float16", "float32", "bfloat16"):
                raise ValueError(f"accum_dtype {c.accum_dtype} is not valid for {c.A_dtype} activations")
            # tensor-core accumulation is always fp32 (DESIGN.md: fp16 accumulate of the reference is not reproduced)
            d.accum_dtype = _lib.BB_F32
        if c.out_dtype not in _lib.DTYPE_IDS:
            raise ValueError(f"out_dtype {c.out_dtype} not supported")
        d.out_dtype = _lib.DTYPE_IDS[c.out_dtype]
        d.group_size = int(c.group_size) if c.group_size and c.group_size > 0 else -1
        d.with_scaling = int(bool(c.with_scaling))
        d.with_zeros = int(bool(c.with_zeros))
        d.zeros_mode = _lib.ZEROS_IDS[c.zeros_mode]
        d.with_bias = int(bool(c.with_bias))
        if self.bit < 8 and c.fast_decoding:
            d.w_layout = _lib.BB_LAYOUT_INTERLEAVED_8 if c.A_dtype == "int8" else _lib.BB_LAYOUT_INTERLEAVED_16
        else:
            d.w_layout = _lib.BB_LAYOUT_COMPRESSED
        d.w_tile = _lib.BB_TILE_SLAB if self.weight_tiled else _lib.BB_TILE_ROW_MAJOR
        return d

    @property
    def weight_tiled(self) -> bool:
        """stored weight is in the slab tiling (MatmulConfig.propagate_b)"""
        return self.config.propagate_b != TransformKind.NonTransform

    def tile_weight(self, w: torch.Tensor, inverse: bool = False) -> torch.Tensor:
        """row-major packed storage [N, K*bits/8] <-> BB_TILE_SLAB (same shape and bytes, 512-byte row segments re-ordered as
        [N/32][row_bytes/512][32][512]).  CUDA tensors: bb_retile_weight_device; CPU tensors: a torch permute."""
        R, B = _lib.BB_TILE_ROWS, _lib.BB_TILE_ROW_BYTES
        w = w.contiguous()
        n, rb = w.shape[0], w.shape[1] * w.element_size()
        if n % R or rb % B:
            raise ValueError(f"slab tiling needs rows % {R} == 0 and row bytes % {B} == 0 (got {n} x {rb})")
        if w.is_cuda:
            out = torch.empty_like(w)
            _lib.ensure_init(w.device.index or 0)
            with torch.cuda.device(w.device):
                _lib.check(_lib.load().bb_retile_weight_device(w.data_ptr(), out.data_ptr(), n, rb, int(inverse),
                                                               torch.cuda.current_stream(w.device).cuda_stream), "bb_retile_weight_device")
            return out
        b = w.view(torch.int8).reshape(n, rb)
        if inverse:
            t = b.reshape(n // R, rb // B, R, B).permute(0, 2, 1, 3)
        else:
            t = b.reshape(n // R, R, rb // B, B).permute(0, 2, 1, 3)
        return t.contiguous().reshape(n, rb).view(w.dtype).reshape(w.shape)

    # ---- weight / input preparation -------------------------------------------------------------
    def retrieve_weight_shape(self):
        if self.consistent or self.bit >= 8:
            return [int(self.N), int(self.K)]
        return [int(self.N), int(self.K) // 8 * self.bit]

    def transform_weight(self, weight, scale=None, zeros=None, bias=None):
        """general_matmul/__init__.py:662-711 (including its quirk of returning only the weight)."""
        weight = weight.contiguous()
        if self.W_dtype == self.A_dtype:
            return weight
        source_format, bit = self.source_format, self.bit
        if source_format == "int" and bit < 8:
            assert not self.with_scaling, "scale should be False for int source format"
            assert not self.with_zeros, "zeros should be False for int source format"
            maxq = 2 ** (bit - 1)
            weight = torch.clamp(weight, -maxq, maxq).char() + maxq
        elif source_format in ["fp_e5m2", "fp_e4m3"]:
            weight = weight.view(torch.int8)
        else:
            weight = weight.char()
        if self.weight_transform is not None:
            weight = self.weight_transform(weight).contiguous()
        if self.weight_tiled:
            weight = self.tile_weight(weight)
        return weight

    def transform_input(self, input_tensor):
        return input_tensor  # no ladder propagation on H100

    # ---- forward ------------------------------------------------------------------------------------
    def _check_tensor(self, t: torch.Tensor, name: str, dtype: torch.dtype, numel: Optional[int] = None):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor: bitblas_b200 has no CPU path")
        if t.dtype != dtype:
            raise TypeError(f"{name} has dtype {t.dtype}, expected {dtype}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
        if numel is not None and t.numel() != numel:
            raise ValueError(f"{name} has {t.numel()} elements, expected {numel}")

    def _check_params(self, W, scale, zeros, bias):
        """full validation of the (static) parameter tensors; forward() runs it once per distinct set of tensors."""
        c = self.config
        adt = getattr(torch, c.A_dtype)
        wshape = self.retrieve_weight_shape()
        self._check_tensor(W, "W", torch.int8 if W.dtype != torch.uint8 else torch.uint8, wshape[0] * wshape[1])
        G = c.K // (c.group_size if c.group_size and c.group_size > 0 else c.K)
        if c.with_scaling:
            if scale is None:
                raise ValueError("with_scaling=True but scale is None")
            self._check_tensor(scale, "scale", adt, c.N * G)
        if c.with_zeros:
            if zeros is None:
                raise ValueError("with_zeros=True but zeros is None")
            if c.zeros_mode == "quantized":
                self._check_tensor(zeros, "zeros", torch.int8, G * (c.N * self.bit // 8))
            else:
                self._check_tensor(zeros, "zeros", adt, c.N * G)
        if c.with_bias:
            if bias is None:
                raise ValueError("with_bias=True but bias is None")
            self._check_tensor(bias, "bias", adt, c.N)

    def forward(self, A, W, scale=None, zeros=None, bias=None, output=None) -> Any:
        if self.consistent:
            return self._forward_consistent(A, W, bias, output)
        c = self.config
        # the parameter tensors of a layer do not change between calls: validate each distinct set once (keyed on the storage
        # pointers; a new tensor -- or a re-allocated one -- is validated again).  The activations are checked every call.
        key = (W.data_ptr(), scale.data_ptr() if scale is not None else 0, zeros.data_ptr() if zeros is not None else 0,
               bias.data_ptr() if bias is not None else 0)
        if key != self._checked_key:
            self._check_params(W, scale, zeros, bias)
            self._checked_key = key
        if not (A.is_cuda and A.dtype == self._torch_a_dtype and A.is_contiguous()):
            self._check_tensor(A, "A", self._torch_a_dtype)
        K = c.K
        if A.shape[-1] != K:
            raise ValueError(f"A has inner dimension {A.shape[-1]}, expected K={K}")
        m = A.numel() // K
        if self.dynamic_range is None and m != int(c.M):
            raise ValueError(f"operator was created for static M={c.M}, got {m} rows")
        dev = A.device
        if output is None:
            output = torch.empty(A.shape[:-1] + (c.N,), dtype=self.torch_output_dtype, device=dev)
        elif not (output.is_cuda and output.dtype == self.torch_output_dtype and output.is_contiguous() and output.numel() == m * c.N):
            self._check_tensor(output, "output", self.torch_output_dtype, m * c.N)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if idx not in _lib._inited:
            _lib.ensure_init(idx)
        stream = torch.cuda.current_stream(dev).cuda_stream
        lut = self.lut
        if lut is not None and lut.device != dev:
            lut = self.lut = lut.to(dev)
        ws_ptr, ws_bytes = self._workspace_for(m, dev, stream)
        if idx != torch.cuda.current_device():
            with torch.cuda.device(dev):   # the kernels launch on the calling thread's current device
                rc = self.lib._c.bb_matmul(self._desc_ref, A.data_ptr(), key[0], lut.data_ptr() if lut is not None else 0,
                                           key[1], key[2], key[3], output.data_ptr(), m, ws_ptr, ws_bytes, stream)
        else:
            rc = self.lib._c.bb_matmul(self._desc_ref, A.data_ptr(), key[0], lut.data_ptr() if lut is not None else 0,
                                       key[1], key[2], key[3], output.data_ptr(), m, ws_ptr, ws_bytes, stream)
        if rc != 0:
            raise RuntimeError(f"bb_matmul failed (code {rc}): {_lib.last_error()}")
        return output

    def _workspace_for(self, m: int, device, stream=None):
        """scratch the kernel picked for `m` needs (bb_workspace_bytes: split-K partials, stream-K exchange slots); one cached,
        ZERO-INITIALISED buffer per operator, device and stream, grown on demand.  The stream-K kernels leave their slots
        zero-tagged, so the buffer is reused by later calls on the same stream without clearing (include/bitblas_b200.h)."""
        key = (int(m), _lib.OVERRIDE_GEN)
        need = self._ws_need.get(key)
        if need is None:
            need = self._ws_need[key] = int(self.lib._c.bb_workspace_bytes(ctypes.byref(self._desc), int(m)))
        if need == 0:
            return 0, 0
        wkey = (device, stream if stream is not None else torch.cuda.current_stream(device).cuda_stream)
        ws = self._ws.get(wkey)
        if ws is None or ws.numel() < need:
            ws = torch.zeros(need, dtype=torch.uint8, device=device)
            self._ws[wkey] = ws
        return ws.data_ptr(), ws.numel()

    def forward_scatter(self, A, W, scale=None, zeros=None, bias=None, *, peer_ptrs, ldc: int, col_offset: int):
        """Column-parallel forward (bb_matmul_scatter): this operator's N is the local shard; the kernel epilogue stores the
        [m, N] result into columns [col_offset, col_offset+N) of every buffer in `peer_ptrs` (device pointers of the
        ranks' [m, ldc] outputs, e.g. torch symmetric memory).  Returns nothing: the caller barriers, then reads."""
        if self.consistent:
            raise NotImplementedError("forward_scatter needs a low-bit weight operator")
        c = self.config
        adt = getattr(torch, c.A_dtype)
        self._check_tensor(A, "A", adt)
        if A.shape[-1] != c.K:
            raise ValueError(f"A has inner dimension {A.shape[-1]}, expected K={c.K}")
        m = reduce(_operator.mul, A.shape[:-1], 1)
        n = len(peer_ptrs)
        if isinstance(peer_ptrs, ctypes.Array):   # prebuilt (c_void_p * n) array: callers on a hot path build it once per buffer
            arr = peer_ptrs
        else:
            arr = (ctypes.c_void_p * n)(*[ctypes.c_void_p(int(x)) for x in peer_ptrs])
        dev = A.device.index if A.device.index is not None else torch.cuda.current_device()
        _lib.ensure_init(dev)
        stream = torch.cuda.current_stream(device=A.device).cuda_stream
        lut = self.lut
        if lut is not None and lut.device != A.device:
            lut = self.lut = lut.to(A.device)
        rc = self.lib._c.bb_matmul_scatter(ctypes.byref(self._desc), A.data_ptr(), W.data_ptr(),
                                           lut.data_ptr() if lut is not None else 0,
                                           scale.data_ptr() if c.with_scaling else 0,
                                           zeros.data_ptr() if c.with_zeros else 0,
                                           bias.data_ptr() if c.with_bias else 0,
                                           arr, n, int(ldc), int(col_offset), int(m), *self._workspace_for(int(m), A.device), stream)
        if rc != 0:
            raise RuntimeError(f"bb_matmul_scatter failed (code {rc}): {_lib.last_error()}")

    def _forward_consistent(self, A, W, bias, output):
        """A_dtype == W_dtype (no sub-byte decode; general_matmul/__init__.py:33-51,568-580): a plain library GEMM, outside the
        hot path (SURVEY.md 8f-3).  float16 / bfloat16: cuBLAS through torch.matmul (fp32 accumulate).  int8: EXACT int32
        accumulation through cuBLASLt (torch._int_mm), like the reference's INT8xINT8 kernels -- never through fp32, whose
        partial sums stop being exact at 2^24.  float8: operands widened to float16 (exact), fp32 accumulate."""
        if not A.is_cuda or not W.is_cuda:
            raise RuntimeError("A and W must be CUDA tensors: bitblas_b200 has no CPU path")
        c = self.config
        if W.shape[-1] != c.K or W.shape[0] != c.N or A.shape[-1] != c.K:
            raise ValueError(f"expected A[..., {c.K}] and W[{c.N}, {c.K}], got {tuple(A.shape)} and {tuple(W.shape)}")
        a2 = A.reshape(-1, c.K)
        if c.A_dtype in ("int8", "uint8"):
            if a2.dtype != torch.int8 or W.dtype != torch.int8:
                raise TypeError("the int8 dense path takes int8 A and W")
            acc = self._int8_gemm_exact(a2.contiguous(), W.contiguous())
            if bias is not None:
                acc = acc + bias.to(torch.int32)
            out = acc.to(self.torch_output_dtype)
        else:
            if c.A_dtype in ("e4m3_float8", "e5m2_float8"):
                a2, W = a2.to(torch.float16), W.to(torch.float16)
            out = torch.matmul(a2, W.t()).to(self.torch_output_dtype)
            if bias is not None:
                out = out + bias.to(out.dtype)
        out = out.reshape(A.shape[:-1] + (c.N,))
        if output is not None:
            output.copy_(out)
            return output
        return out

    @staticmethod
    def _int8_gemm_exact(a2: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
        """int32 = int8 [m, K] x int8 [N, K]^T.  torch._int_mm needs m > 16 and K, N multiples of 8: rows are zero-padded,
        other shapes take the (exact, slower) float64 GEMM."""
        m, K = a2.shape
        N = W.shape[0]
        if K % 8 == 0 and N % 8 == 0:
            rows = max(32, (m + 7) // 8 * 8)
            if rows != m:
                pad = torch.zeros((rows, K), dtype=torch.int8, device=a2.device)
                pad[:m] = a2
                a2 = pad
            return torch._int_mm(a2, W.t())[:m]
        return torch.matmul(a2.double(), W.double().t()).to(torch.int32)

    def __call__(self, *args: Any, **kwds: Any) -> Any:
        return self.forward(*args, **kwds)

    # ---- introspection ------------------------------------------------------------------------------
    def kernel_for(self, m: int) -> str:
        """name of the kernel family the dispatcher picks for `m` rows (bb_select_kernel)."""
        return _lib.kernel_name(_lib.load().bb_select_kernel(ctypes.byref(self._desc), int(m)))

    def get_source(self, target=None, kenrel_only=False) -> str:
        ms = self.M if isinstance(self.M, tuple) else (self.M,)
        lines = [f"// bitblas_b200 prebuilt sm_90a kernels ({_lib.LIB_PATH}); sources: bitblas_b200/csrc/*.cu"]
        if self._desc is not None:
            lines += [f"// m={m}: {self.kernel_for(m)}" for m in ms]
        return "\n".join(lines)

    def profile_latency(self, dynamic_symbolic_constraints: Optional[dict] = None) -> float:
        """mean latency in ms over 10 launches, CUDA events (reference: tvm time_evaluator(number=10),
        ops/operator.py:223-224,442-450)."""
        m = self.M
        if isinstance(m, tuple):
            m = (dynamic_symbolic_constraints or {}).get("m", m[-1])
        dev = torch.device("cuda")
        adt = getattr(torch, self.A_dtype)
        A = (torch.randn(m, self.K, device=dev) if adt.is_floating_point else torch.randint(-8, 8, (m, self.K), device=dev)).to(adt)
        if self.consistent:
            W = (torch.randn(self.N, self.K, device=dev)).to(adt)
            args = (A, W)
        else:
            W = torch.randint(-128, 127, self.retrieve_weight_shape(), dtype=torch.int8, device=dev)
            G = self.K // (self.group_size if self.group_size > 0 else self.K)
            scale = torch.rand(self.N, G, device=dev).to(adt) if self.with_scaling else None
            zeros = None
            if self.with_zeros:
                zeros = (torch.randint(-128, 127, (G, self.N * self.bit // 8), dtype=torch.int8, device=dev)
                         if self.zeros_mode == "quantized" else torch.rand(self.N, G, device=dev).to(adt))
            bias = torch.rand(self.N, device=dev).to(adt) if self.with_bias else None
            args = (A, W, scale, zeros, bias)
        for _ in range(3):
            self.forward(*args)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(10):
            self.forward(*args)
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / 10

    def cleanup(self):
        self.workspace = None

    # ---- config-mirroring properties (general_matmul/__init__.py:761-841) ----
    M = property(lambda self: self.config.M)
    N = property(lambda self: self.config.N)
    K = property(lambda self: self.config.K)
    A_dtype = property(lambda self: self.config.A_dtype)
    W_dtype = property(lambda self: self.config.W_dtype)
    out_dtype = property(lambda self: self.config.out_dtype)
    accum_dtype = property(lambda self: self.config.accum_dtype)
    storage_dtype = property(lambda self: self.config.storage_dtype)
    with_scaling = property(lambda self: self.config.with_scaling)
    with_zeros = property(lambda self: self.config.with_zeros)
    group_size = property(lambda self: self.config.group_size)
    fast_decoding = property(lambda self: self.config.fast_decoding)
    with_bias = property(lambda self: self.config.with_bias)
    propagate_a = property(lambda self: self.config.propagate_a)
    propagate_b = property(lambda self: self.config.propagate_b)
    layout = property(lambda self: self.config.layout)
    zeros_mode = property(lambda self: self.config.zeros_mode)

    @property
    def input_transform(self):
        return None

    @property
    def weight_transform(self):
        return self.weight_executors if (self.weight_executors is not None and self.weight_executors.size) else None


__all__ = ["Matmul", "MatmulConfig", "WeightTransform", "is_native_compute"]
