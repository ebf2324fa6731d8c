"""GPU known-answer tests for the in-register LOP3 decode (bb_debug_decode), the analogue of the reference's
gtest DecodeTest.* suite (testing/cpp/lop3_type_conversion/lowprecision_to_float16.cu:51-101, lowprecision_to_int8.cu):
values -> compress -> interleave -> device decode -> exact equality.  The same packed words are also decoded by the
REFERENCE's device functions (oracle/ref_shim.cu) and compared bit for bit: live when oracle/_ref is built from a reference
checkout, otherwise against the stored outputs of such a run (tests/golden/ref_decode_golden.npz, written by
tests/golden/make_ref_decode_golden.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import bitblas_oracle as O
from bitblas_b200 import _lib

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libbitblas_ref.so")
GOLDEN = os.path.join(HERE, "golden", "ref_decode_golden.npz")


def _pack(values, bits, tgt, layout_il=True):
    packed = O.general_compress(values, bits)
    if layout_il:
        packed = O.interleave_weight(packed, bits, tgt)
    return torch.from_numpy(np.ascontiguousarray(packed)).cuda()


@pytest.mark.parametrize("bits", [4, 2])
@pytest.mark.parametrize("signed", [0, 1])
@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("il", [True, False])
def test_decode_to_16bit_exact(bits, signed, kind, il):
    lib = _lib.load()
    _lib.ensure_init(0)
    rng = np.random.RandomState(0)   # srand(0) in the reference KATs
    vals = rng.randint(0, 2**bits, size=(1, 4096)).astype(np.int8)
    dev = _pack(vals, bits, "float16", il)
    out = torch.empty(4096, dtype=torch.float16 if kind == 0 else torch.bfloat16, device="cuda")
    layout = _lib.BB_LAYOUT_INTERLEAVED_16 if il else _lib.BB_LAYOUT_COMPRESSED
    _lib.check(lib.bb_debug_decode(kind, bits, signed, layout, dev.data_ptr(), out.data_ptr(), dev.numel() // 4, 0))
    torch.cuda.synchronize()
    expect = vals.reshape(-1).astype(np.int32) - (2 ** (bits - 1) if signed else 0)
    assert np.array_equal(out.float().cpu().numpy().astype(np.int32), expect)


@pytest.mark.parametrize("bits", [4, 2])
@pytest.mark.parametrize("signed", [0, 1])
def test_decode_to_int8_exact(bits, signed):
    lib = _lib.load()
    _lib.ensure_init(0)
    rng = np.random.RandomState(0)
    vals = rng.randint(0, 2**bits, size=(1, 4096)).astype(np.int8)
    dev = _pack(vals, bits, "int8")
    out = torch.empty(4096, dtype=torch.int8, device="cuda")
    _lib.check(lib.bb_debug_decode(2, bits, signed, _lib.BB_LAYOUT_INTERLEAVED_8, dev.data_ptr(), out.data_ptr(), dev.numel() // 4, 0))
    torch.cuda.synchronize()
    expect = vals.reshape(-1).astype(np.int32) - (2 ** (bits - 1) if signed else 0)
    assert np.array_equal(out.cpu().numpy().astype(np.int32), expect)




@pytest.mark.parametrize("bits", [4, 2, 1])
@pytest.mark.parametrize("tgt", [0, 16, 8])
def test_device_weight_transform_matches_host(bits, tgt):
    from bitblas_b200.ops.general_matmul import WeightTransform
    rng = np.random.RandomState(7)
    w = torch.from_numpy(rng.randint(0, 2**bits, size=(64, 512)).astype(np.int8))
    wt = WeightTransform(bits, tgt)
    assert torch.equal(wt(w.cuda()).cpu(), wt(w))


# ---- the reference's full decode KAT matrix (testing/cpp/lop3_type_conversion/lowprecision_to_float16.cu:51-101: 20 TESTs,
# lowprecision_to_int8.cu: 6), run side by side with the product's decode / dequantise arithmetic on this GPU --------------
# kind ids of oracle/ref_shim.cu
REF_F16 = dict(I4U=0, I4S=1, I2U=2, I2S=3, I1U=4, I1S=5, I4U_SCALE=6, I4U_ZEROS_ORIGINAL=7, I4U_ZEROS_RESCALE=8,
               I4U_ZEROS_QUANTIZED=9, I2U_SCALE=10, I2U_ZEROS_ORIGINAL=11, I2U_ZEROS_RESCALE=12)
REF_I8 = dict(I4U=0, I4S=1, I2U=2, I2S=3, I1U=4, I1S=5)
# what the reference's SIGNED decodes subtract, per implementation of the device functions: the C++ test header
# (fast_decoding.hpp:17, MEDIAN 0x6407 / 0x6401; decode_i{4,2}s_to_i8s) subtracts 2^(b-1) - 1 -- SURVEY.md 8c defect (iii) --
# while the Python product's LOP3 library (lop3.py: MEDIAN 0x6408 / 0x6402, i8s 7 / 2) subtracts 2^(b-1) except for 4-bit -> int8.
# This library subtracts 2^(b-1) everywhere (lop3.py:23, general_matmul/__init__.py:688-690).
SIGNED_OFFSET = {"cpp": {("f16", 4): 7, ("f16", 2): 1, ("i8", 4): 7, ("i8", 2): 1},
                 "lop3": {("f16", 4): 8, ("f16", 2): 2, ("i8", 4): 7, ("i8", 2): 2}}


class RefLib:
    """the reference's decode entry points (oracle/ref_shim.cu) behind ctypes; `host` = its C++ pack helpers are usable"""

    def __init__(self, lib, host=True):
        lib.ref_decode_f16.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 4
        lib.ref_decode_i8.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        lib.ref_general_compress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.ref_general_interleave_fp16.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t]
        self.lib, self.host = lib, host

    def f16(self, kind, dev, n, scale=None, zeros=None, qz=None):
        out = torch.empty(n, dtype=torch.float16, device="cuda")
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        assert self.lib.ref_decode_f16(kind, dev.data_ptr(), out.data_ptr(), n // 8, ptr(scale), ptr(zeros), ptr(qz), None) == 0
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def i8(self, kind, dev, n):
        out = torch.empty(n, dtype=torch.int8, device="cuda")
        assert self.lib.ref_decode_i8(kind, dev.data_ptr(), out.data_ptr(), n // 16, None) == 0
        torch.cuda.synchronize()
        return out.cpu().numpy()


def bind_ref(lib, host=True):
    return RefLib(lib, host)


# Each case draws its seeded inputs, runs the reference on them and returns inputs + reference output ("ref").
def _case_unsigned_f16(bits, kind):
    def run(ref):
        vals = np.random.RandomState(5).randint(0, 2**bits, size=(1, 8192)).astype(np.int8)
        return dict(vals=vals, ref=ref.f16(REF_F16[kind], _pack(vals, bits, "float16"), 8192))
    return run


def _case_unsigned_i8(ref):
    vals = np.random.RandomState(6).randint(0, 4, size=(1, 4096)).astype(np.int8)
    return dict(vals=vals, ref=ref.i8(REF_I8["I2U"], _pack(vals, 2, "int8"), 4096))


def _case_signed_f16(bits, kind):
    def run(ref):
        vals = np.random.RandomState(11).randint(0, 2**bits, size=(1, 8192)).astype(np.int8)
        return dict(vals=vals, ref=ref.f16(REF_F16[kind], _pack(vals, bits, "float16"), 8192))
    return run


def _case_dequant(kind, bits, mode):
    def run(ref):
        rng = np.random.RandomState(12)
        n = 16384
        vals = rng.randint(0, 2**bits, size=(1, n)).astype(np.int8)
        g = n // 8
        scale = (rng.rand(g) * 3 + 0.013).astype(np.float16)
        zeros = (rng.rand(g) * (2**bits - 1)).astype(np.float16)
        if mode == 3:
            zeros = (zeros.astype(np.float32) * scale.astype(np.float32)).astype(np.float16)
        qz = rng.randint(0, 2**bits, size=g).astype(np.int32)
        c = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
        out = ref.f16(REF_F16[kind], _pack(vals, bits, "float16"), n, c(scale), c(zeros) if mode in (2, 3) else None,
                      c(qz) if mode == 4 else None)
        return dict(vals=vals, scale=scale, zeros=zeros, qz=qz, ref=out)
    return run


def _case_i8(kind, bits):
    def run(ref):
        vals = np.random.RandomState(13).randint(0, 2**bits, size=(1, 8192)).astype(np.int8)
        return dict(vals=vals, ref=ref.i8(REF_I8[kind], _pack(vals, bits, "int8"), 8192))
    return run


def _case_one_bit(kind):
    def run(ref):
        vals = np.random.RandomState(14).randint(0, 2, size=4096).astype(np.int8)
        if ref.host:   # the reference's own C++ compress + interleave
            comp = np.zeros(4096 // 8, dtype=np.int8)
            inter = np.zeros_like(comp)
            ref.lib.ref_general_compress(vals.ctypes.data, comp.ctypes.data, 1, 4096, 0)
            ref.lib.ref_general_interleave_fp16(comp.ctypes.data, inter.ctypes.data, 1, comp.nbytes)
        else:          # the oracle's packing, pinned to those C++ functions by tests/test_oracle_golden.py
            inter = O.interleave_weight(O.general_compress(vals.reshape(1, -1), 1), 1, "float16").reshape(-1)
        return dict(vals=vals, packed=inter, ref=ref.f16(REF_F16[kind], torch.from_numpy(inter).cuda(), 4096))
    return run


DEQUANT = [("I4U_SCALE", 4, 1), ("I4U_ZEROS_ORIGINAL", 4, 2), ("I4U_ZEROS_RESCALE", 4, 3), ("I4U_ZEROS_QUANTIZED", 4, 4),
           ("I2U_SCALE", 2, 1), ("I2U_ZEROS_ORIGINAL", 2, 2), ("I2U_ZEROS_RESCALE", 2, 3)]
I8_MATRIX = [("I4U", 4, 0), ("I4S", 4, 1), ("I2U", 2, 0), ("I2S", 2, 1)]
REF_CASES = {"u16_I4U": _case_unsigned_f16(4, "I4U"), "u16_I2U": _case_unsigned_f16(2, "I2U"), "u8_I2U": _case_unsigned_i8,
             "s16_I4S": _case_signed_f16(4, "I4S"), "s16_I2S": _case_signed_f16(2, "I2S"),
             **{f"dq_{k}": _case_dequant(k, b, m) for k, b, m in DEQUANT},
             **{f"i8_{k}": _case_i8(k, b) for k, b, _ in I8_MATRIX},
             "b1_I1U": _case_one_bit("I1U"), "b1_I1S": _case_one_bit("I1S")}


def _reference(name):
    """(source, case dict) of REF_CASES[name]: run live when oracle/_ref is built, else the stored run"""
    if os.path.exists(REF_SO):
        return "cpp", REF_CASES[name](bind_ref(ctypes.CDLL(REF_SO)))
    G = np.load(GOLDEN)
    pre = name + "/"
    return str(G["source"]), {k[len(pre):]: G[k] for k in G.files if k.startswith(pre)}


def _mine_f16(bits, signed, vals):
    lib = _lib.load()
    _lib.ensure_init(0)
    dev = _pack(vals, bits, "float16")
    mine = torch.empty(vals.size, dtype=torch.float16, device="cuda")
    _lib.check(lib.bb_debug_decode(0, bits, signed, _lib.BB_LAYOUT_INTERLEAVED_16, dev.data_ptr(), mine.data_ptr(), dev.numel() // 4, 0))
    torch.cuda.synchronize()
    return mine.cpu().numpy()


def _mine_i8(bits, signed, vals):
    lib = _lib.load()
    _lib.ensure_init(0)
    dev = _pack(vals, bits, "int8")
    mine = torch.empty(vals.size, dtype=torch.int8, device="cuda")
    _lib.check(lib.bb_debug_decode(2, bits, signed, _lib.BB_LAYOUT_INTERLEAVED_8, dev.data_ptr(), mine.data_ptr(), dev.numel() // 4, 0))
    torch.cuda.synchronize()
    return mine.cpu().numpy()


@pytest.mark.parametrize("bits,kind_ref", [(4, 0), (2, 2)])
def test_decode_matches_reference_device_functions(bits, kind_ref):
    """unsigned decode vs decode_i4u_to_f16 / decode_i2u_to_f16 of the reference's device functions."""
    _, c = _reference("u16_I4U" if bits == 4 else "u16_I2U")
    mine = _mine_f16(bits, 0, c["vals"])
    assert np.array_equal(mine.view(np.uint16), c["ref"].view(np.uint16))
    assert np.array_equal(c["ref"].astype(np.int32), c["vals"].reshape(-1))


def test_int8_decode_matches_reference_device_functions():
    _, c = _reference("u8_I2U")
    assert np.array_equal(_mine_i8(2, 0, c["vals"]), c["ref"])


@pytest.mark.parametrize("bits,kind", [(4, "I4S"), (2, "I2S")])
def test_signed_decode_vs_reference_device_functions(bits, kind):
    """decode_i{4,2}s_to_f16: the reference's signed offset depends on which of its implementations ran (SIGNED_OFFSET); this
    library follows its Python product and subtracts 2^(b-1) (SURVEY.md 8c)."""
    src, c = _reference("s16_" + kind)
    v = c["vals"].reshape(-1).astype(np.int32)
    mine = _mine_f16(bits, 1, c["vals"]).astype(np.int32)
    assert np.array_equal(mine, v - 2 ** (bits - 1))
    assert np.array_equal(c["ref"].astype(np.int32), v - SIGNED_OFFSET[src][("f16", bits)])


@pytest.mark.parametrize("kind,bits,mode", DEQUANT)
def test_dequant_arithmetic_vs_reference_device_functions(kind, bits, mode):
    """DecodeTest.*WithScaling / *WithZerosOriginal / *Rescale / *Quantized: the tensor-core GEMM path's dequantise arithmetic
    (dq_finish: fp16 sub, then mul -- or one fma for rescale) must reproduce the reference's rounding order bit for bit, with
    non-trivial fp16 scales and non-integer fp16 zero points (one per group of 8 outputs, as in the reference KATs)."""
    lib = _lib.load()
    _lib.ensure_init(0)
    _, c = _reference("dq_" + kind)
    n = c["vals"].size
    dev = _pack(c["vals"], bits, "float16")
    scale, zeros, qz = (torch.from_numpy(c[k]).cuda() for k in ("scale", "zeros", "qz"))
    mine = torch.empty(n, dtype=torch.float16, device="cuda")
    _lib.check(lib.bb_debug_dequant(0, bits, 0, _lib.BB_LAYOUT_INTERLEAVED_16, mode, dev.data_ptr(), scale.data_ptr(),
                                    zeros.data_ptr(), qz.data_ptr(), mine.data_ptr(), dev.numel() // 4, 0))
    torch.cuda.synchronize()
    assert np.array_equal(mine.cpu().numpy().view(np.uint16), c["ref"].view(np.uint16)), (mine[:16], c["ref"][:16])
    # and the oracle's A_dtype dequantise (the model every parity test is checked against) states the same numbers
    u = torch.from_numpy(c["vals"].reshape(-1).astype(np.float32)).half()
    s8, z8, q8 = (scale.cpu().repeat_interleave(8), zeros.cpu().repeat_interleave(8), qz.cpu().repeat_interleave(8).half())
    rescale = (u * s8 - z8) if bits == 2 else torch.addcmul(-z8.float(), u.float(), s8.float()).half()   # 2-bit: two roundings (lop3.py:633-635)
    expect = {1: u * s8, 2: (u - z8) * s8, 3: rescale, 4: (u - q8) * s8}[mode]
    assert torch.equal(mine.cpu(), expect)


@pytest.mark.parametrize("kind,bits,signed", I8_MATRIX)
def test_int8_decode_matrix_vs_reference_device_functions(kind, bits, signed):
    """lowprecision_to_int8.cu DecodeTest.{U,}Int{4,2}ToINT8.  Signed: the reference's offset per implementation is
    SIGNED_OFFSET (lop3.py:1016, SURVEY.md 8c defect (iii)); the Python product and this library subtract 2^(b-1)."""
    src, c = _reference("i8_" + kind)
    v = c["vals"].reshape(-1).astype(np.int32)
    assert np.array_equal(_mine_i8(bits, signed, c["vals"]).astype(np.int32), v - (2 ** (bits - 1) if signed else 0))
    assert np.array_equal(c["ref"].astype(np.int32), v - (SIGNED_OFFSET[src][("i8", bits)] if signed else 0))


@pytest.mark.parametrize("kind,signed", [("I1U", 0), ("I1S", 1)])
def test_one_bit_reference_decode_pins_the_generic_path(kind, signed):
    """DecodeTest.{U,}Int1ToFloat16: 1-bit weights run through the generic kernel here (no in-register fast path), whose
    arithmetic is the oracle's; the reference's device decode on the C++-interleaved words must agree with it: uint1 -> {0, 1},
    int1 -> {-1, +1} (lop3.py:723-727; SURVEY.md 8c defect (ii): the TIR decode would give {0, -1})."""
    _, c = _reference("b1_" + kind)
    assert np.array_equal(c["packed"], O.interleave_weight(O.general_compress(c["vals"].reshape(1, -1), 1), 1, "float16").reshape(-1))
    got = c["ref"].astype(np.int32)
    expect = O.decode_fields(torch.from_numpy(c["vals"].astype(np.int32)), "int" if signed else "uint", 1, torch.float32).numpy().astype(np.int32)
    assert np.array_equal(got, expect)
