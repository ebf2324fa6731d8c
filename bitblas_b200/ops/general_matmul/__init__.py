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

# Matmul.forward_grouped runs the single grouped launch while T <= GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E rows (E groups);
# above it each non-empty group runs through bb_matmul, whose dispatcher picks the wgmma GEMM above 8 rows.  tools/moe_bench.py
# (NVIDIA H100 80GB HBM3, 700 W power limit): with 8 large experts (Mixtral-8x7B down, 4096 x 14336) the single launch is 1.6-2.7x
# faster up to 8 rows per expert, even at 16 and slower above (0.60x at 32); the fused gate/up (28672 x 4096) is already 0.67x
# at 16 rows per expert.  With 128 small experts (Qwen3-30B-A3B gate/up) the single launch stays ahead up to ~128 rows per
# expert because the per-group side issues one call per expert; the constant follows the large-expert crossover.
GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = 8

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
        want_tile = slab_tiled(self.propagate_b, self.N, self.K, self.W_dtype, self.A_dtype)
        if not want_tile and self._legalize_propagate(self.propagate_b) not in (None, TransformKind.NonTransform):
            logger.warning("propagate_b: slab tiling needs a 4/2-bit integer weight, N %% 128 == 0 and K*bits/8 %% 512 == 0 "
                           "(N=%s K=%s W_dtype=%s); keeping the row-major storage", self.N, self.K, self.W_dtype)
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


def slab_tiled(propagate_b, N: int, K: int, W_dtype: str, A_dtype: str) -> bool:
    """True when a requested propagate_b stores an [N, K] weight of W_dtype in the slab tiling BB_TILE_SLAB, False when it
    legalises to (or asked for) row-major storage.  The tiling needs a 4/2-bit integer weight, N % 128 == 0 and
    K*bits/8 % BB_TILE_ROW_BYTES == 0.  MatmulConfig legalises propagate_b with it, and the tensor-parallel loaders
    (bitblas_b200.parallel) use it to tell whether a FULL layer's weight is tiled when only its shard has an operator."""
    if MatmulConfig._legalize_propagate(propagate_b) in (None, TransformKind.NonTransform):
        return False
    wbits = {"int4": 4, "uint4": 4, "int2": 2, "uint2": 2}.get(W_dtype)
    return (wbits is not None and W_dtype != A_dtype and N % 128 == 0 and (K * wbits // 8) % _lib.BB_TILE_ROW_BYTES == 0
            and (K * wbits) % 8 == 0)


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
            _, idx, stream = _lib.device_stream(weight)
            _lib.call("bb_transform_weight_device", idx, weight.data_ptr(), out.data_ptr(), rows, cols, self.bits,
                      self.interleave_target, stream)
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
        # bare pointers name no device: like the reference's generated `call`, this launches on the current one
        op._launch_raw(A, W, lut, scale, zeros, bias, next(it), m, torch.cuda.current_device(), stream)


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
        self._grouped_checked_key = None
        self._grouped_gemm_ok = False   # bb_matmul_grouped_gemm covers the checked parameter set (N % 128 == 0)
        self._grouped_gemm_err = ""     # the library's message where it does not
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
            _, idx, stream = _lib.device_stream(w)
            _lib.call("bb_retile_weight_device", idx, w.data_ptr(), out.data_ptr(), n, rb, int(inverse), stream)
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
    def _check_params(self, W, scale, zeros, bias, device, scaled=False, w4a8=False):
        """full validation of the (static) parameter tensors, all of them on `device` (A's: the kernel gets bare pointers);
        forward() runs it once per distinct set of tensors.  scaled (forward_scaled): `scale` is the fp32 [N] w_scale and the
        bias is in the output dtype; w4a8 (forward_w4a8): `scale` is fp32 [N, K/g] and the bias is in the output dtype."""
        c = self.config
        adt = getattr(torch, c.A_dtype)
        wshape = self.retrieve_weight_shape()
        _lib.check_tensor(W, "W", torch.int8 if W.dtype != torch.uint8 else torch.uint8, numel=wshape[0] * wshape[1])
        G = c.K // (c.group_size if c.group_size and c.group_size > 0 else c.K)
        if w4a8:
            if scale is None:
                raise ValueError("forward_w4a8 needs scale (float32 [N, K/g])")
            _lib.check_tensor(scale, "scale", torch.float32, numel=c.N * G)
            scaled, adt = True, None   # the bias check below is forward_scaled's
        elif c.with_scaling:
            if scale is None:
                raise ValueError("with_scaling=True but scale is None")
            _lib.check_tensor(scale, "scale", adt, numel=c.N * G)
        if c.with_zeros:
            if zeros is None:
                raise ValueError("with_zeros=True but zeros is None")
            if c.zeros_mode == "quantized":
                _lib.check_tensor(zeros, "zeros", torch.int8, numel=G * (c.N * self.bit // 8))
            else:
                _lib.check_tensor(zeros, "zeros", adt, numel=c.N * G)
        if c.with_bias:
            if bias is None:
                raise ValueError("with_bias=True but bias is None")
            _lib.check_tensor(bias, "bias", self.torch_output_dtype if scaled else adt, numel=c.N)
        if scaled and not w4a8:
            if scale is None:
                raise ValueError("forward_scaled needs w_scale (float32 [N])")
            _lib.check_tensor(scale, "w_scale", torch.float32, numel=c.N)
        for t in (W, scale if c.with_scaling or scaled else None, zeros if c.with_zeros else None, bias if c.with_bias else None):
            if t is not None and t.device != device:
                raise ValueError(f"the layer's buffers must be on A's device {device} (a buffer is on {t.device})")

    def _output_for(self, A, output, N):
        """the output of A [.., K]: a new [.., N] tensor on A's device, or the caller's, checked to hold the m * N values"""
        if output is None:
            return torch.empty(A.shape[:-1] + (N,), dtype=self.torch_output_dtype, device=A.device)
        numel = A.numel() // self.config.K * N
        if not (output.is_cuda and output.dtype == self.torch_output_dtype and output.is_contiguous() and output.numel() == numel):
            _lib.check_tensor(output, "output", self.torch_output_dtype, numel=numel)
        return output

    def forward(self, A, W, scale=None, zeros=None, bias=None, output=None) -> Any:
        if self.consistent:
            return self._forward_consistent(A, W, bias, output)
        output, ptrs = self._check_forward(A, W, scale, zeros, bias, output)
        return self._launch(A, ptrs, output)

    def _check_forward(self, A, W, scale, zeros, bias, output, swiglu=False, scaled=False, w4a8=False):
        """the checking half of forward() (swiglu: of forward_swiglu, whose output has N / 2 columns; scaled: of forward_scaled,
        with `scale` the w_scale): validates every argument and launches nothing.  Returns the output and, for _launch, the data
        pointers of W, scale, zeros and bias."""
        c = self.config
        if not (A.is_cuda and A.dtype == self._torch_a_dtype and A.is_contiguous()):
            _lib.check_tensor(A, "A", self._torch_a_dtype)
        # the parameter tensors of a layer do not change between calls: validate each distinct set once (keyed on the storage
        # pointers and A's device; a new tensor -- or a re-allocated one -- is validated again).  The activations are checked
        # every call.
        key = (W.data_ptr(), scale.data_ptr() if scale is not None else 0, zeros.data_ptr() if zeros is not None else 0,
               bias.data_ptr() if bias is not None else 0, A.device, scaled, w4a8)
        if key != self._checked_key:
            self._check_params(W, scale, zeros, bias, A.device, scaled, w4a8)
            self._checked_key = key
        K = c.K
        if A.shape[-1] != K:
            raise ValueError(f"A has inner dimension {A.shape[-1]}, expected K={K}")
        if self.dynamic_range is None and A.numel() // K != int(c.M):
            raise ValueError(f"operator was created for static M={c.M}, got {A.numel() // K} rows")
        return self._output_for(A, output, c.N // 2 if swiglu else c.N), key

    def _launch(self, A, ptrs, output, swiglu=False):
        """the launching half of forward() (swiglu: of forward_swiglu): A is the checked activations, or a column gather of them
        (Linear's and SwiGLUMLP's act-order)"""
        dev, idx, stream = _lib.device_stream(A)
        lut = self.lut
        if lut is not None and lut.device != dev:
            lut = self.lut = lut.to(dev)
        self._launch_raw(A.data_ptr(), ptrs[0], lut.data_ptr() if lut is not None else 0, ptrs[1], ptrs[2], ptrs[3],
                        output.data_ptr(), A.numel() // self.config.K, idx, stream, swiglu)
        return output

    def _launch_raw(self, A, W, lut, scale, zeros, bias, C, m, device, stream, swiglu=False, a_scale=None, w4a8=False):
        """the package's one bb_matmul (swiglu: bb_matmul_swiglu; a_scale, the pointer of the fp32 [m] activation scales:
        bb_matmul_scaled with `scale` the w_scale, or with w4a8 bb_matmul_w4a8 with `scale` the fp32 group scales) call: raw
        pointers (0 = absent), m rows, on the device of ordinal `device`"""
        ws_ptr, ws_bytes = self._workspace_for(m, device, stream, w4a8)
        if w4a8:
            _lib.call("bb_matmul_w4a8", device, self._desc_ref, A, W, a_scale, scale, zeros, bias, C, m, ws_ptr, ws_bytes, stream)
            return
        if a_scale is not None:
            _lib.call("bb_matmul_scaled", device, self._desc_ref, A, W, a_scale, scale, bias, C, m, ws_ptr, ws_bytes, stream)
            return
        _lib.call("bb_matmul_swiglu" if swiglu else "bb_matmul", device, self._desc_ref, A, W, lut, scale, zeros, bias, C, m,
                  ws_ptr, ws_bytes, stream)

    def check_swiglu(self) -> None:
        """raise unless forward_swiglu covers this operator: NotImplementedError for a consistent (A_dtype == W_dtype) operator,
        ValueError for int8 activations or N % 16 != 0 (the gate/up interleave moves blocks of 8 gate and 8 up rows)"""
        if self.consistent:
            raise NotImplementedError("forward_swiglu needs a low-bit weight operator")
        c = self.config
        if c.A_dtype == "int8":
            raise ValueError("forward_swiglu needs float16 or bfloat16 activations (int8 is not supported)")
        if c.N % 16:
            raise ValueError(f"forward_swiglu needs N = 2I with I % 8 == 0 (gate/up interleave; N={c.N})")

    def forward_swiglu(self, A, W, scale=None, zeros=None, bias=None, output=None):
        """The gate/up projection of a dense SwiGLU MLP in one launch (bb_matmul_swiglu): this operator's N = 2I rows hold gate and
        up in the gate/up interleave (bitblas_b200.moe.interleave_gate_up; scale, zeros and bias rows follow it), and the output
        [.., I] is silu(gate) * up, formed in the kernel epilogue from exactly the values forward() would store for the two rows.
        The kernel is the one forward() picks for the same m, with the same workspace.  Arguments as in forward()."""
        self.check_swiglu()
        output, ptrs = self._check_forward(A, W, scale, zeros, bias, output, swiglu=True)
        return self._launch(A, ptrs, output, swiglu=True)

    def check_scaled(self) -> None:
        """raise unless forward_scaled covers this operator: NotImplementedError for a consistent (A_dtype == W_dtype) operator,
        ValueError for 16-bit activations, an integer out_dtype, or group scales / zeros (the weight's scale is w_scale)"""
        if self.consistent:
            raise NotImplementedError("forward_scaled needs a low-bit weight operator")
        c = self.config
        if c.A_dtype != "int8":
            raise ValueError(f"forward_scaled needs int8 activations (A_dtype={c.A_dtype}; quantize_act_int8 makes them from "
                             "float16 / bfloat16)")
        if c.out_dtype not in ("float16", "bfloat16", "float32"):
            raise ValueError(f"forward_scaled needs out_dtype float16, bfloat16 or float32 (got {c.out_dtype})")
        if c.with_scaling or c.with_zeros:
            raise ValueError("forward_scaled takes the weight's scale as w_scale: the operator needs with_scaling=False and "
                             "with_zeros=False")

    def forward_scaled(self, A, W, a_scale, w_scale, bias=None, output=None):
        """The int8 matmul with a dequantizing epilogue in one launch (bb_matmul_scaled; two with split-K): A int8 [.., K] (e.g.
        from quantize_act_int8), a_scale float32 [m] one quantization scale per row of A, w_scale float32 [N] one per output
        row of W, and output [.., N] = round((float(acc) / a_scale[r]) / w_scale[n]) (+ bias, [N] in the output dtype, added
        after the rounding), acc the exact int32 sum forward() forms.  The kernel is the one forward() picks for the same m,
        with the same workspace."""
        self.check_scaled()
        output, ptrs = self._check_forward(A, W, w_scale, None, bias, output, scaled=True)
        m = A.numel() // self.config.K
        if not (isinstance(a_scale, torch.Tensor) and a_scale.is_cuda and a_scale.dtype == torch.float32
                and a_scale.is_contiguous() and a_scale.numel() == m):
            _lib.check_tensor(a_scale, "a_scale", torch.float32, numel=m)
        if a_scale.device != A.device:
            raise ValueError(f"a_scale must be on A's device {A.device} (got {a_scale.device})")
        _, idx, stream = _lib.device_stream(A)
        self._launch_raw(A.data_ptr(), ptrs[0], 0, ptrs[1], 0, ptrs[3], output.data_ptr(), m, idx, stream,
                         a_scale=a_scale.data_ptr())
        return output

    def _workspace_for(self, m: int, device: int, stream: int, w4a8: bool = False, fp8: bool = False):
        """scratch the kernel picked for `m` needs (bb_workspace_bytes: split-K partials, stream-K exchange slots; w4a8: of the
        descriptor without group scales and zeros, which bb_matmul_w4a8's kernels need at most; fp8: bb_workspace_bytes_fp8);
        one cached, ZERO-INITIALISED buffer per operator, device (ordinal) and stream, grown on demand.  The m = 1 slab kernel
        leaves its slots zero-tagged, so the buffer is reused by later calls on the same stream without clearing
        (include/bitblas_b200.h)."""
        key = (int(m), _lib.OVERRIDE_GEN, w4a8, fp8)
        need = self._ws_need.get(key)
        if need is None:
            if fp8:
                need = int(_lib.load().bb_workspace_bytes_fp8(ctypes.byref(self._fp8_desc()), int(m)))
            else:
                need = int(self.lib._c.bb_workspace_bytes(ctypes.byref(self._w4a8_cleared_desc() if w4a8 else self._desc), int(m)))
            self._ws_need[key] = need
        if need == 0:
            return 0, 0
        wkey = (device, stream)
        ws = self._ws.get(wkey)
        if ws is None or ws.numel() < need:
            ws = torch.zeros(need, dtype=torch.uint8, device=torch.device("cuda", device))
            self._ws[wkey] = ws
        return ws.data_ptr(), ws.numel()

    def check_w4a8(self) -> None:
        """raise unless forward_w4a8 covers this operator: NotImplementedError for a consistent (A_dtype == W_dtype) operator,
        ValueError for 16-bit activations, an integer out_dtype, no group scales, zeros other than "quantized", weights other than
        4-bit uint / int, or int weights with zeros"""
        if self.consistent:
            raise NotImplementedError("forward_w4a8 needs a low-bit weight operator")
        c = self.config
        if c.A_dtype != "int8":
            raise ValueError(f"forward_w4a8 needs int8 activations (A_dtype={c.A_dtype}; quantize_act_int8 makes them from "
                             "float16 / bfloat16)")
        if c.out_dtype not in ("float16", "bfloat16", "float32"):
            raise ValueError(f"forward_w4a8 needs out_dtype float16, bfloat16 or float32 (got {c.out_dtype})")
        if not c.with_scaling:
            raise ValueError("forward_w4a8 needs with_scaling=True (float32 group scales)")
        if c.with_zeros and c.zeros_mode != "quantized":
            raise ValueError(f"forward_w4a8 needs zeros_mode='quantized' (got {c.zeros_mode})")
        if c.W_dtype not in ("uint4", "int4"):
            raise ValueError(f"forward_w4a8 needs uint4 or int4 weights (got {c.W_dtype})")
        if c.with_zeros and c.W_dtype == "int4":
            raise ValueError("forward_w4a8: int4 weights take no zero points")

    def _w4a8_cleared_desc(self) -> _lib.MatmulDesc:
        """this operator's descriptor without group scales and zeros: its bb_workspace_bytes sizes bb_matmul_w4a8's workspace"""
        d = getattr(self, "_w4a8_desc", None)
        if d is None:
            d = self._w4a8_desc = _lib.MatmulDesc.from_buffer_copy(self._desc)
            d.with_scaling = d.with_zeros = 0
        return d

    def kernel_for_w4a8(self, m: int) -> str:
        """the kernel family forward_w4a8 runs for m rows (bb_select_kernel_w4a8)"""
        return _lib.kernel_name(self.lib._c.bb_select_kernel_w4a8(ctypes.byref(self._desc), int(m)))

    def forward_w4a8(self, A_q, W, a_scale, scale, zeros=None, bias=None, output=None):
        """GPTQ-style 4-bit weights against int8 activations in one launch (bb_matmul_w4a8; two with split-K): A_q int8 [.., K]
        (e.g. from quantize_act_int8), a_scale float32 [m] one quantization scale per row of A_q, scale float32 [N, K/g] the group
        scales, zeros the packed quantized zero points [K/g, N/2] (with_zeros), and output [.., N] = round(S / a_scale[r])
        (+ bias, [N] in the output dtype, added after the rounding) with S = sum_g float(acc_g) * scale[n, g] in fp32 and acc_g
        the exact int32 dot product of group g.  The kernel is kernel_for_w4a8(m)."""
        self.check_w4a8()
        c = self.config
        output, ptrs = self._check_forward(A_q, W, scale, zeros, bias, output, scaled=True, w4a8=True)
        m = A_q.numel() // c.K
        if not (isinstance(a_scale, torch.Tensor) and a_scale.is_cuda and a_scale.dtype == torch.float32
                and a_scale.is_contiguous() and a_scale.numel() == m):
            _lib.check_tensor(a_scale, "a_scale", torch.float32, numel=m)
        if a_scale.device != A_q.device:
            raise ValueError(f"a_scale must be on A's device {A_q.device} (got {a_scale.device})")
        _, idx, stream = _lib.device_stream(A_q)
        self._launch_raw(A_q.data_ptr(), ptrs[0], 0, ptrs[1], ptrs[2], ptrs[3], output.data_ptr(), m, idx, stream,
                         a_scale=a_scale.data_ptr(), w4a8=True)
        return output

    def check_fp8(self) -> None:
        """raise ValueError unless forward_fp8 covers this operator: A_dtype = W_dtype = "e4m3_float8", accum_dtype float32,
        out_dtype float16 / bfloat16 / float32, N % 16 == 0 and K % 128 == 0"""
        c = self.config
        if c.A_dtype != "e4m3_float8" or c.W_dtype != "e4m3_float8":
            raise ValueError(f"forward_fp8 needs A_dtype = W_dtype = 'e4m3_float8' (got {c.A_dtype}, {c.W_dtype})")
        if c.accum_dtype != "float32":
            raise ValueError(f"forward_fp8 needs accum_dtype='float32' (got {c.accum_dtype})")
        if c.out_dtype not in ("float16", "bfloat16", "float32"):
            raise ValueError(f"forward_fp8 needs out_dtype float16, bfloat16 or float32 (got {c.out_dtype})")
        if c.N % 16 or c.K % 128:
            raise ValueError(f"forward_fp8 needs N % 16 == 0 and K % 128 == 0 (N={c.N}, K={c.K})")

    def _fp8_desc(self) -> _lib.MatmulDesc:
        """the bb_matmul_fp8 descriptor of this operator: e4m3 x e4m3, fp32 scales in 128 x 128 blocks"""
        d = getattr(self, "_fp8_desc_c", None)
        if d is None:
            c = self.config
            d = self._fp8_desc_c = _lib.MatmulDesc()
            d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = int(c.N), int(c.K), _lib.BB_E4M3, _lib.BB_W_FP8_E4M3, 8
            d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.DTYPE_IDS[c.out_dtype], 128
            d.with_scaling, d.with_bias = 1, int(bool(c.with_bias))
        return d

    def kernel_for_fp8(self, m: int) -> str:
        """the kernel family forward_fp8 runs for m rows (bb_select_kernel_fp8)"""
        self.check_fp8()
        return _lib.kernel_name(_lib.load().bb_select_kernel_fp8(ctypes.byref(self._fp8_desc()), int(m)))

    def forward_fp8(self, A_q, W, a_scale, w_scale, bias=None, output=None):
        """Block-scaled FP8 matmul on the FP8 tensor cores in one launch (bb_matmul_fp8; two with split-K): A_q float8_e4m3fn
        [.., K] with a_scale float32 [m, K/128] (quantize_act_fp8's transposed view of a k-block-major buffer: a_scale[r, b] at
        b * ld + r), W float8_e4m3fn [N, K] with w_scale float32 [ceil(N/128), K/128], and output [.., N] = round(S) (+ bias, [N]
        in the output dtype, added after the rounding) with S = sum_b P_b * (a_scale[r, b] * w_scale[n / 128, b]) in fp32 and
        P_b the tensor core's sum over the 128 k of block b.  The kernel is kernel_for_fp8(m).  forward() on this operator
        stays the fp16 widening path."""
        self.check_fp8()
        c = self.config
        N, K, KB = int(c.N), int(c.K), int(c.K) // 128
        e4m3 = torch.float8_e4m3fn
        if not (isinstance(A_q, torch.Tensor) and A_q.is_cuda and A_q.dtype == e4m3 and A_q.is_contiguous()):
            _lib.check_tensor(A_q, "A_q", e4m3)
        if A_q.dim() < 1 or A_q.shape[-1] != K:
            raise ValueError(f"A_q has inner dimension {A_q.shape[-1] if A_q.dim() else None}, expected K={K}")
        m = A_q.numel() // K
        dev = A_q.device
        _lib.check_tensor(W, "W", e4m3, numel=N * K)
        _lib.check_tensor(w_scale, "w_scale", torch.float32, numel=((N + 127) // 128) * KB)
        ld = self._fp8_a_scale_ld(a_scale, m)
        if c.with_bias:
            if bias is None:
                raise ValueError("with_bias=True but bias is None")
            _lib.check_tensor(bias, "bias", self.torch_output_dtype, numel=N)
        elif bias is not None:
            raise ValueError("the operator was built with with_bias=False but a bias was given")
        for t in (W, w_scale, a_scale, bias):
            if t is not None and t.device != dev:
                raise ValueError(f"every operand must be on A_q's device {dev} (one is on {t.device})")
        output = self._output_for(A_q, output, N)
        _, idx, stream = _lib.device_stream(A_q)
        ws_ptr, ws_bytes = self._workspace_for(m, idx, stream, fp8=True)
        _lib.call("bb_matmul_fp8", idx, ctypes.byref(self._fp8_desc()), A_q.data_ptr(), a_scale.data_ptr(), ld, W.data_ptr(),
                  w_scale.data_ptr(), bias.data_ptr() if bias is not None else 0, output.data_ptr(), m, ws_ptr, ws_bytes, stream)
        return output

    def _fp8_a_scale_ld(self, a_scale, m: int) -> int:
        """the a_scale_ld of quantize_act_fp8's scales for m rows: a float32 CUDA [m, K/128] transposed view of a k-block-major
        [K/128, ld] buffer"""
        KB = int(self.config.K) // 128
        if not isinstance(a_scale, torch.Tensor) or a_scale.dtype != torch.float32 or tuple(a_scale.shape) != (m, KB):
            raise TypeError(f"a_scale must be a float32 [{m}, {KB}] torch.Tensor (quantize_act_fp8's scales)")
        if not a_scale.is_cuda:
            raise RuntimeError("a_scale must be a CUDA tensor: bitblas_b200 has no CPU path")
        if m > 1 and a_scale.stride(0) != 1:
            raise ValueError("a_scale must be k-block-major: the [m, K/128] transposed view of a [K/128, ld] buffer (stride(0) == 1)")
        return a_scale.stride(1) if KB > 1 else (m + 3) // 4 * 4

    # ---- grouped (mixture-of-experts) block-scaled FP8 --------------------------------------------------------------------------
    def check_grouped_fp8(self, num_groups: int, swiglu: bool = False) -> None:
        """raise ValueError unless bb_matmul_grouped_fp8 (swiglu: bb_matmul_grouped_fp8_swiglu) covers this operator with
        `num_groups` experts: check_fp8, then the library's own checks with total_rows = 0 (nothing touches the device)"""
        self.check_fp8()
        name = "bb_matmul_grouped_fp8_swiglu" if swiglu else "bb_matmul_grouped_fp8"
        rc = getattr(_lib.load(), name)(ctypes.byref(self._fp8_desc()), int(num_groups), 0, 0, 0, 0, 0, 0, 0, 0, 0)
        if rc != 0:
            raise ValueError(f"{name} does not cover this configuration: {_lib.last_error()}")

    def forward_grouped_fp8(self, A_q, W, offsets, a_scale, w_scale, output=None):
        """Grouped block-scaled FP8 matmul for mixture-of-experts layers in ONE graph-capturable launch (bb_matmul_grouped_fp8):
        A_q float8_e4m3fn [T, K] sorted so that expert e owns rows [offsets[e], offsets[e+1]) (offsets int32 CUDA [E + 1], read
        on the device), a_scale quantize_act_fp8's float32 [T, K/128] scales of A_q, W float8_e4m3fn [E, N, K] and w_scale
        float32 [E, N/128, K/128].  For every expert e, output[offsets[e]:offsets[e+1]] is forward_fp8 of those rows against W[e]
        run unsplit, bit for bit.  Offsets are clamped to [0, T]; rows no expert claims are not written."""
        N = int(self.config.N)
        return self._grouped_fp8("bb_matmul_grouped_fp8", A_q, W, offsets, a_scale, w_scale, output, N // 128, N)

    def forward_grouped_fp8_swiglu(self, A_q, W, offsets, a_scale, w_scale, output=None):
        """The gate/up projection of a block-scaled FP8 SwiGLU expert block in ONE launch (bb_matmul_grouped_fp8_swiglu): this
        operator's N = 2I rows of W [E, 2I, K] hold gate and up in the gate/up interleave (moe.interleave_gate_up kind "weight")
        and w_scale [E, 2 ceil(I/128), K/128] their scales interleaved by block (kind "block_scale").  output [T, I] =
        silu(g) * u, rounded once, with g and u exactly what forward_grouped_fp8 stores for the gate and up rows.  Operands and
        offsets otherwise as forward_grouped_fp8."""
        I = int(self.config.N) // 2
        return self._grouped_fp8("bb_matmul_grouped_fp8_swiglu", A_q, W, offsets, a_scale, w_scale, output, 2 * -(-I // 128), I,
                                 swiglu=True)

    def _grouped_fp8(self, name, A_q, W, offsets, a_scale, w_scale, output, s_rows, out_cols, swiglu=False):
        c = self.config
        N, K, KB = int(c.N), int(c.K), int(c.K) // 128
        e4m3 = torch.float8_e4m3fn
        if not isinstance(offsets, torch.Tensor) or offsets.dtype != torch.int32:
            raise TypeError("offsets must be an int32 torch.Tensor of num_groups + 1 row offsets")
        if offsets.dim() != 1 or not 2 <= offsets.numel() <= _lib.BB_GROUPED_MAX_GROUPS + 1:
            raise ValueError(f"offsets must be 1-D with num_groups + 1 entries, 1 <= num_groups <= {_lib.BB_GROUPED_MAX_GROUPS} "
                             f"(got shape {tuple(offsets.shape)})")
        E = offsets.numel() - 1
        key = (name, E)
        if key != getattr(self, "_grouped_fp8_checked", None):
            self.check_grouped_fp8(E, swiglu)
            self._grouped_fp8_checked = key
        _lib.check_tensor(A_q, "A_q", e4m3, 2)
        if A_q.shape[1] != K:
            raise ValueError(f"A_q must be [T, K={K}], got {tuple(A_q.shape)}")
        T = A_q.shape[0]
        _lib.check_tensor(W, "W", e4m3, 3)
        if tuple(W.shape) != (E, N, K):
            raise ValueError(f"W must be [E={E}, {N}, {K}] (got {tuple(W.shape)})")
        _lib.check_tensor(w_scale, "w_scale", torch.float32, 3)
        if tuple(w_scale.shape) != (E, s_rows, KB):
            raise ValueError(f"w_scale must be [E={E}, {s_rows}, {KB}] (got {tuple(w_scale.shape)})")
        _lib.check_tensor(offsets, "offsets", torch.int32)
        ld = self._fp8_a_scale_ld(a_scale, T)
        if output is None:
            output = torch.empty((T, out_cols), dtype=self.torch_output_dtype, device=A_q.device)
        else:
            _lib.check_tensor(output, "output", self.torch_output_dtype)
            if tuple(output.shape) != (T, out_cols):
                raise ValueError(f"output must be [T={T}, {out_cols}] (got {tuple(output.shape)})")
        for t in (W, w_scale, a_scale, offsets, output):
            if t.device != A_q.device:
                raise ValueError(f"every operand must be on A_q's device {A_q.device} (one is on {t.device})")
        _, idx, stream = _lib.device_stream(A_q)
        _lib.call(name, idx, ctypes.byref(self._fp8_desc()), E, offsets.data_ptr(), A_q.data_ptr(), a_scale.data_ptr(), ld,
                  W.data_ptr(), w_scale.data_ptr(), output.data_ptr(), T, stream)
        return output

    def forward_scatter(self, A, W, scale=None, zeros=None, bias=None, *, peer_ptrs, ldc: int, col_offset: int):
        """Column-parallel forward (bb_matmul_scatter): this operator's N is the local shard; the kernel epilogue stores the
        [m, N] result into columns [col_offset, col_offset+N) of every buffer in `peer_ptrs` (device pointers of the
        ranks' [m, ldc] outputs, e.g. torch symmetric memory).  Returns nothing: the caller barriers, then reads."""
        if self.consistent:
            raise NotImplementedError("forward_scatter needs a low-bit weight operator")
        c = self.config
        _lib.check_tensor(A, "A", self._torch_a_dtype)
        if A.shape[-1] != c.K:
            raise ValueError(f"A has inner dimension {A.shape[-1]}, expected K={c.K}")
        m = reduce(_operator.mul, A.shape[:-1], 1)
        n = len(peer_ptrs)
        if isinstance(peer_ptrs, ctypes.Array):   # prebuilt (c_void_p * n) array: callers on a hot path build it once per buffer
            arr = peer_ptrs
        else:
            arr = (ctypes.c_void_p * n)(*[ctypes.c_void_p(int(x)) for x in peer_ptrs])
        dev, idx, stream = _lib.device_stream(A)
        lut = self.lut
        if lut is not None and lut.device != dev:
            lut = self.lut = lut.to(dev)
        _lib.call("bb_matmul_scatter", idx, self._desc_ref, A.data_ptr(), W.data_ptr(),
                  lut.data_ptr() if lut is not None else 0,
                  scale.data_ptr() if c.with_scaling else 0,
                  zeros.data_ptr() if c.with_zeros else 0,
                  bias.data_ptr() if c.with_bias else 0,
                  arr, n, int(ldc), int(col_offset), int(m), *self._workspace_for(int(m), idx, stream), stream)

    # ---- grouped (mixture-of-experts) forward -----------------------------------------------------------------------------
    def check_grouped(self, num_groups: int, swiglu: bool = False) -> None:
        """raise ValueError unless bb_matmul_grouped (swiglu: bb_matmul_grouped_swiglu) covers this operator's config with
        `num_groups` groups (validated by the library with total_rows = 0: nothing touches the device)."""
        if self.consistent:
            raise ValueError("the grouped matmul needs a low-bit weight operator (A_dtype != W_dtype)")
        name = "bb_matmul_grouped_swiglu" if swiglu else "bb_matmul_grouped"
        rc = getattr(self.lib._c, name)(self._desc_ref, int(num_groups), 0, 0, 0, 0, 0, 0, 0, 0, 0)
        if rc != 0:
            raise ValueError(f"{name} does not cover this configuration: {_lib.last_error()}")

    def _check_grouped_params(self, E, W, scale, zeros, bias):
        """stacked parameter tensors: W [E, N, K*bits/8], scale [E, N, K/g], zeros [E, N, K/g] ([E, K/g, N*bits/8] quantized),
        bias [E, N].  Shapes and dtypes are checked before the device, so a CPU tensor of the wrong shape reports its shape."""
        c = self.config
        adt = self._torch_a_dtype
        G = c.K // (c.group_size if c.group_size and c.group_size > 0 else c.K)
        specs = [("W", W, torch.int8, (E, *self.retrieve_weight_shape()), True),
                 ("scale", scale, adt, (E, c.N, G), c.with_scaling),
                 ("zeros", zeros, torch.int8 if c.zeros_mode == "quantized" else adt,
                  (E, G, c.N * self.bit // 8) if c.zeros_mode == "quantized" else (E, c.N, G), c.with_zeros),
                 ("bias", bias, adt, (E, c.N), c.with_bias)]
        specs = [s for s in specs if s[4]]
        for name, t, dtype, shape, _ in specs:
            if t is None:
                raise ValueError(f"the operator's config needs {name}, got None")
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{name} must be a torch.Tensor")
            if tuple(t.shape) != shape:
                raise ValueError(f"{name} has shape {tuple(t.shape)}, expected the stacked shape {shape}")
        for name, t, dtype, shape, _ in specs:
            _lib.check_tensor(t, name, dtype)

    def forward_grouped(self, A, W, offsets, scale=None, zeros=None, bias=None, output=None, capturable=False):
        """Grouped matmul for mixture-of-experts layers (bb_matmul_grouped): E problems of this operator's config.  A [T, K] holds
        every group's rows, sorted so that group e owns rows [offsets[e], offsets[e+1]); `offsets` is an int32 CUDA tensor of
        E + 1 entries.  W, scale, zeros and bias are stacked over the groups (see _check_grouped_params).  For every group e:
        output[offsets[e]:offsets[e+1]] = A[offsets[e]:offsets[e+1]] x dequant(W[e])^T (+ bias[e]).  Rows no group claims are not
        written.

        Up to GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E rows this is ONE kernel launch that reads the offsets on the device: no host
        synchronisation, CUDA-graph capturable.  Above it (prefill) the offsets are copied to the host once and every non-empty
        group runs through bb_matmul on its row slice, where the dispatcher picks the wgmma GEMM; that path synchronises with the
        device and cannot be captured in a graph.

        capturable=True (the meaning the flag has on torch's optimizers): the host never reads the offsets, so the call is one
        launch and graph-capturable at every T.  Above the threshold it runs the grouped wgmma GEMM (bb_matmul_grouped_gemm, the
        numerics of bb_matmul on the wgmma GEMM) where it covers the config (N % 128 == 0), and bb_matmul_grouped otherwise."""
        if self.consistent:
            raise NotImplementedError("forward_grouped needs a low-bit weight operator")
        E, T, ptrs, output, dev, stream = self._grouped_prepare(A, W, offsets, scale, zeros, bias, output, self.config.N)
        if T <= GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E or capturable:
            name = "bb_matmul_grouped" if self._grouped_single_launch(T, E) == "gemv" else "bb_matmul_grouped_gemm"
            _lib.call(name, dev, self._desc_ref, E, offsets.data_ptr(), A.data_ptr(), *ptrs, output.data_ptr(), T, stream)
        else:
            self._forward_grouped_per_group(A, W, offsets, scale, zeros, bias, output, dev, stream)
        return output

    def forward_grouped_swiglu(self, A, W, offsets, scale=None, zeros=None, bias=None, output=None, row_index=None):
        """The gate/up projection of a SwiGLU mixture-of-experts block in ONE graph-capturable launch: this operator's N = 2I rows
        hold gate and up in the gate/up interleave (bitblas_b200.moe.interleave_gate_up), and the output [T, I] is
        silu(gate) * up, formed in the kernel epilogue from exactly the values forward_grouped(capturable=True) would store
        (bb_matmul_grouped_swiglu / bb_matmul_grouped_gemm_swiglu, picked by the same rule).  Operands and offsets as in
        forward_grouped.

        row_index (int32 CUDA tensor of T entries, e.g. the row_token of bitblas_b200.moe.moe_route_index): sorted row r reads
        A[clamp(row_index[r], 0, a_rows - 1)] of A [a_rows, K] in the GEMM's producer, so the rows need not be gathered first;
        the output is [T, I].  This always runs the grouped wgmma GEMM (bb_matmul_grouped_gemm_swiglu_gather) and raises
        ValueError where it does not cover the config (2I % 128 != 0)."""
        if self.consistent:
            raise NotImplementedError("forward_grouped_swiglu needs a low-bit weight operator")
        if row_index is not None:
            return self._forward_grouped_swiglu_gather(A, W, offsets, scale, zeros, bias, output, row_index)
        E, T, ptrs, output, dev, stream = self._grouped_prepare(A, W, offsets, scale, zeros, bias, output, self.config.N // 2,
                                                                swiglu=True)
        name = "bb_matmul_grouped_swiglu" if self._grouped_single_launch(T, E) == "gemv" else "bb_matmul_grouped_gemm_swiglu"
        _lib.call(name, dev, self._desc_ref, E, offsets.data_ptr(), A.data_ptr(), *ptrs, output.data_ptr(), T, stream)
        return output

    def _forward_grouped_swiglu_gather(self, A, W, offsets, scale, zeros, bias, output, row_index):
        name = "bb_matmul_grouped_gemm_swiglu_gather"
        if not isinstance(row_index, torch.Tensor) or row_index.dtype != torch.int32 or row_index.dim() != 1:
            raise TypeError("row_index must be a 1-D int32 torch.Tensor (one row of A per sorted row)")
        E, T, ptrs, output, dev, stream = self._grouped_prepare(A, W, offsets, scale, zeros, bias, output, self.config.N // 2,
                                                                swiglu=True, rows=row_index.numel())
        if not self._grouped_gemm_ok:
            raise ValueError(f"{name} does not cover this configuration: {self._grouped_gemm_err}")
        _lib.check_tensor(row_index, "row_index", torch.int32)
        if row_index.device != A.device:
            raise ValueError("row_index must be on A's device")
        if T > 0 and A.shape[0] < 1:
            raise ValueError("A must have at least one row to gather from")
        _lib.call(name, dev, self._desc_ref, E, offsets.data_ptr(), row_index.data_ptr(), A.data_ptr(), A.shape[0], *ptrs,
                  output.data_ptr(), T, stream)
        return output

    def _grouped_single_launch(self, T: int, E: int) -> str:
        """the kernel of the one capturable grouped launch for T rows over E groups: the grouped GEMV ("gemv") up to
        GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E rows and where the grouped GEMM does not cover the config (N % 128 != 0),
        the grouped wgmma GEMM ("gemm") above"""
        return "gemm" if T > GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E and self._grouped_gemm_ok else "gemv"

    def _grouped_prepare(self, A, W, offsets, scale, zeros, bias, output, out_cols, swiglu=False, rows=None):
        """argument checks of the grouped forwards (parameters once per distinct set); returns (E, T, parameter pointers, output
        [T, out_cols], device ordinal, stream).  T is A's row count, or `rows` (the gathering call, whose A has any number of rows)."""
        c = self.config
        if not isinstance(offsets, torch.Tensor) or offsets.dtype != torch.int32:
            raise TypeError("offsets must be an int32 torch.Tensor of num_groups + 1 row offsets")
        if offsets.dim() != 1 or not 2 <= offsets.numel() <= _lib.BB_GROUPED_MAX_GROUPS + 1:
            raise ValueError(f"offsets must be 1-D with num_groups + 1 entries, 1 <= num_groups <= {_lib.BB_GROUPED_MAX_GROUPS} "
                             f"(got shape {tuple(offsets.shape)})")
        E = offsets.numel() - 1
        key = (E, W.data_ptr(), scale.data_ptr() if scale is not None else 0, zeros.data_ptr() if zeros is not None else 0,
               bias.data_ptr() if bias is not None else 0, swiglu)
        if key != self._grouped_checked_key:
            self._check_grouped_params(E, W, scale, zeros, bias)
            self.check_grouped(E, swiglu)
            self._grouped_gemm_ok = self.lib._c.bb_matmul_grouped_gemm(self._desc_ref, E, 0, 0, 0, 0, 0, 0, 0, 0, 0) == 0
            self._grouped_gemm_err = "" if self._grouped_gemm_ok else _lib.last_error()
            self._grouped_checked_key = key
        if not isinstance(A, torch.Tensor) or A.dim() != 2 or A.shape[1] != c.K:
            raise ValueError(f"A must be [T, K={c.K}], got {tuple(A.shape) if isinstance(A, torch.Tensor) else type(A)}")
        T = A.shape[0] if rows is None else rows
        if output is not None and (not isinstance(output, torch.Tensor) or tuple(output.shape) != (T, out_cols)):
            raise ValueError(f"output must be [T={T}, {out_cols}]")
        _lib.check_tensor(A, "A", self._torch_a_dtype)
        _lib.check_tensor(offsets, "offsets", torch.int32)
        if offsets.device != A.device or W.device != A.device:
            raise ValueError("A, W and offsets must be on the same device")
        if output is None:
            output = torch.empty((T, out_cols), dtype=self.torch_output_dtype, device=A.device)
        else:
            _lib.check_tensor(output, "output", self.torch_output_dtype)
        _, idx, stream = _lib.device_stream(A)
        return E, T, key[1:5], output, idx, stream

    def _forward_grouped_per_group(self, A, W, offsets, scale, zeros, bias, output, dev, stream):
        """prefill side of forward_grouped: one bb_matmul per non-empty group on its row slice, with the offsets clamped exactly as
        the grouped kernel clamps them ([0, T]; a group whose end is below its start is empty)."""
        T = A.shape[0]
        bounds = offsets.cpu().clamp(0, T).tolist()
        for e in range(len(bounds) - 1):
            r0, r1 = bounds[e], bounds[e + 1]
            if r1 <= r0:
                continue
            self._launch_raw(A[r0:r1].data_ptr(), W[e].data_ptr(), 0,
                            scale[e].data_ptr() if self.with_scaling else 0,
                            zeros[e].data_ptr() if self.with_zeros else 0,
                            bias[e].data_ptr() if self.with_bias else 0,
                            output[r0:r1].data_ptr(), r1 - r0, dev, stream)

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


__all__ = ["Matmul", "MatmulConfig", "WeightTransform", "is_native_compute", "slab_tiled"]
