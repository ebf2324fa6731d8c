"""Pin oracle/bitblas_oracle.py against the reference (CPU only).

(a) golden vectors produced by running the reference's own numpy functions (tests/golden/make_golden.py),
(b) vectors from the reference's C++ host functions (fast_decoding.hpp) and, when oracle/_ref is built,
    a live call into them,
(c) the worked examples in fast_decoding.hpp:32-46,609-627 and SURVEY.md §8a (0x76543210 -> 0x75316420),
(d) a numpy model of the LOP3 decode idiom (lop3.py:14-33, 958-1005): decoding the interleaved word
    must give the elements back in logical order -- the property the CUDA kernels rely on.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import bitblas_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "quant_golden.npz"))


@pytest.mark.parametrize("bits", [4, 2, 1])
def test_compress_matches_reference_numpy_and_cpp(bits):
    w = G[f"w_b{bits}"]
    got = O.general_compress(w, bits)
    assert np.array_equal(got, G[f"compress_b{bits}"])
    assert np.array_equal(got, G[f"ref_cpp_compress_b{bits}"])
    assert np.array_equal(O.general_decompress(got, bits), w)


@pytest.mark.parametrize("bits,tgt", [(4, "float16"), (4, "int8"), (2, "int8")])
def test_interleave_matches_reference_numpy(bits, tgt):
    got = O.interleave_weight(G[f"compress_b{bits}"], bits, tgt)
    assert np.array_equal(got, G[f"interleave_b{bits}_{tgt}"])


@pytest.mark.parametrize("bits", [4, 2, 1])
@pytest.mark.parametrize("tgt", ["float16", "int8"])
def test_interleave_matches_reference_cpp(bits, tgt):
    got = O.interleave_weight(G[f"compress_b{bits}"], bits, tgt)
    assert np.array_equal(got, G[f"ref_cpp_interleave_b{bits}_{tgt}"])


def test_interleave_live_against_ref_so():
    """the reference's C++ interleave (fast_decoding.hpp:30-95,607-668): called live when oracle/_ref is built from a reference
    checkout, otherwise its stored outputs (quant_golden.npz ref_cpp_*, written by tests/golden/make_golden.py) are the reference"""
    so = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libbitblas_ref.so")
    if not os.path.exists(so):
        for bits in (4, 2, 1):
            for tgt in ("float16", "int8"):
                got = O.interleave_weight(G[f"compress_b{bits}"], bits, tgt).reshape(-1)
                assert np.array_equal(got, G[f"ref_cpp_interleave_b{bits}_{tgt}"].reshape(-1)), (bits, tgt)
        return
    lib = ctypes.CDLL(so)
    rng = np.random.RandomState(1)
    for bits in (4, 2, 1):
        w = rng.randint(0, 2**bits, size=(8, 256)).astype(np.int8)
        packed = O.general_compress(w, bits)
        flat = np.ascontiguousarray(packed).reshape(-1)
        for tgt, fn in (("float16", lib.ref_general_interleave_fp16), ("int8", lib.ref_general_interleave_int8)):
            dst = np.zeros_like(flat)
            fn(flat.ctypes.data_as(ctypes.c_void_p), dst.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(bits),
               ctypes.c_size_t(flat.nbytes))
            assert np.array_equal(O.interleave_weight(packed, bits, tgt).reshape(-1), dst), (bits, tgt)


def test_worked_examples():
    # 4-bit / f16: {e7..e0} -> {e7,e5,e3,e1,e6,e4,e2,e0}   (fast_decoding.hpp:32-36)
    word = np.array([0x76543210], dtype=np.uint32).view(np.int8)
    assert O.interleave_weight(word, 4, "float16").view(np.uint32)[0] == 0x75316420
    # 4-bit / int8: {e7,e3,e6,e2,e5,e1,e4,e0}              (fast_decoding.hpp:609-613)
    assert O.interleave_weight(word, 4, "int8").view(np.uint32)[0] == 0x73625140
    assert list(O.interleave_perm(4, "float16")) == [0, 2, 4, 6, 1, 3, 5, 7]
    assert list(O.interleave_perm(4, "int8")) == [0, 4, 1, 5, 2, 6, 3, 7]


@pytest.mark.parametrize("bits,tgt", [(4, "float16"), (2, "float16"), (1, "float16"), (4, "int8"), (2, "int8"), (1, "int8")])
def test_deinterleave_roundtrip(bits, tgt):
    rng = np.random.RandomState(2)
    w = rng.randint(0, 2**bits, size=(4, 128)).astype(np.int8)
    packed = O.general_compress(w, bits)
    inter = O.interleave_weight(packed, bits, tgt)
    assert np.array_equal(O.deinterleave_weight(inter, bits, tgt), packed)


def _lop3_decode_f16_words(words_u32: np.ndarray, bits: int) -> np.ndarray:
    """numpy model of decode_i{4,2}{u}_to_f16 (lop3.py:14-33, 432-470): 8 values per 32/16-bit input."""
    out = []
    if bits == 4:
        for w in words_u32:
            for i in range(4):
                x = (int(w) >> (4 * i)) & 0x000F000F
                out += [x & 0xFFFF, x >> 16]
    elif bits == 2:
        for w in words_u32:
            for half in range(2):
                h = (int(w) >> (16 * half)) & 0xFFFF
                x = (h & 0xFF) | ((h & 0xFF00) << 8)
                for i in range(4):
                    y = (x >> (2 * i)) & 0x00030003
                    out += [y & 0xFFFF, y >> 16]
    return np.array(out, dtype=np.int8)


@pytest.mark.parametrize("bits", [4, 2])
def test_lop3_decode_model_recovers_logical_order_f16(bits):
    rng = np.random.RandomState(3)
    w = rng.randint(0, 2**bits, size=(1, 256)).astype(np.int8)
    inter = O.interleave_weight(O.general_compress(w, bits), bits, "float16").view(np.uint32).reshape(-1)
    assert np.array_equal(_lop3_decode_f16_words(inter, bits), w.reshape(-1))


@pytest.mark.parametrize("bits", [4, 2])
def test_lop3_decode_model_recovers_logical_order_i8(bits):
    # decode_i2b_to_i8s / decode_i4b_to_i8s (lop3.py:958-1055)
    rng = np.random.RandomState(4)
    w = rng.randint(0, 2**bits, size=(1, 256)).astype(np.int8)
    inter = O.interleave_weight(O.general_compress(w, bits), bits, "int8").view(np.uint32).reshape(-1)
    out = []
    mask = 0x03030303 if bits == 2 else 0x0F0F0F0F
    for word in inter:
        for i in range(8 // bits):
            x = (int(word) >> (bits * i)) & mask
            out += [(x >> (8 * b)) & 0xFF for b in range(4)]
    assert np.array_equal(np.array(out, dtype=np.int8), w.reshape(-1))


def test_decode_formulas_known_answers():
    u = torch.arange(16)
    assert O.decode_fields(u, "uint", 4, torch.float16).tolist() == list(range(16))
    assert O.decode_fields(u, "int", 4, torch.float16).tolist() == [i - 8 for i in range(16)]
    assert O.decode_fields(torch.arange(4), "int", 2, torch.float16).tolist() == [-2, -1, 0, 1]
    assert O.decode_fields(torch.arange(2), "int", 1, torch.float16).tolist() == [-1, 1]
    # "fp4" = sign + 3-bit exponent 2^(e-7), zero when e == 0 (quantization.py:141-156)
    fp4 = O.decode_fields(u, "fp", 4, torch.float16).tolist()
    assert fp4[:8] == [0.0] + [2.0 ** (e - 7) for e in range(1, 8)]
    assert fp4[8:] == [0.0] + [-(2.0 ** (e - 7)) for e in range(1, 8)]
    # e4m3 bit trick is exact for normal numbers (quantization.py:169-176)
    codes = torch.arange(256)
    ref = codes.to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float16)
    got = O.decode_fields(codes, "fp_e4m3", 8, torch.float16)
    normal = ((codes & 0x78) != 0) & ((codes & 0x7F) != 0x7F)
    assert torch.equal(got[normal], ref[normal])
    # nf4 LUT passthrough
    lut = torch.tensor(O.NF4_LUT, dtype=torch.float16)
    assert torch.equal(O.decode_fields(u, "nf", 4, torch.float16, lut), lut)


def test_matmul_dequant_matches_reference_style_ref_program():
    """Independent re-derivation of test_general_matmul_ops_backend_tl.py:227-273 on its own inputs."""
    torch.manual_seed(0)
    M, N, K, g = 4, 64, 256, 32
    A = torch.rand(M, K, dtype=torch.float16) - 0.5
    iw = torch.randint(0, 8, (N, K), dtype=torch.int8)
    scale = torch.rand(N, K // g, dtype=torch.float16)
    zeros = torch.full((N, K // g), 8.0, dtype=torch.float16)
    gi = torch.arange(K) // g
    for mode in ("original", "rescale"):
        z = zeros if mode == "original" else zeros * scale
        if mode == "original":
            Bd = (iw - z[:, gi]) * scale[:, gi]
        else:
            Bd = iw * scale[:, gi] - z[:, gi]
        ref = (A.float() @ Bd.T.float()).to(torch.float16)
        got = O.matmul_dequant(A, iw.to(torch.int32), W_dtype="uint4", group_size=g, with_scaling=True,
                               with_zeros=True, zeros_mode=mode, scale=scale, zeros=z, fast_decoding=False)
        O.torch_assert_close(got, ref, rtol=1e-2, atol=1e-2, max_mismatched_ratio=0.0)
    qz = torch.from_numpy(O.general_compress(np.full((K // g, N), 8, dtype=np.int8), 4))
    Bd = (iw - 8).to(torch.float16) * scale[:, gi]
    ref = (A.float() @ Bd.T.float()).to(torch.float16)
    got = O.matmul_dequant(A, iw.to(torch.int32), W_dtype="uint4", group_size=g, with_scaling=True,
                           with_zeros=True, zeros_mode="quantized", scale=scale, zeros=qz)
    assert torch.equal(got, ref)


def test_int_accumulate_exact():
    torch.manual_seed(0)
    A = torch.randint(-128, 128, (3, 512), dtype=torch.int8)
    W = torch.randint(-2, 2, (32, 512), dtype=torch.int8)
    got = O.matmul_dequant(A, (W + 2).to(torch.int32), W_dtype="int2", A_dtype="int8", accum_dtype="int32",
                           out_dtype="int32")
    assert torch.equal(got, (A.int() @ W.int().T))


def test_gptq_unpack():
    torch.manual_seed(0)
    z = torch.randint(0, 16, (4, 64), dtype=torch.int32)
    packed = torch.zeros(4, 8, dtype=torch.int32)
    for c in range(64):
        packed[:, c // 8] |= z[:, c] << (4 * (c % 8))
    assert torch.equal(O.unpack_qzeros(packed, 4, v2=True).int(), z)
    assert torch.equal(O.unpack_qzeros(packed, 4).int(), (z + 1) & 15)
    qw = packed.view(torch.int8)
    assert torch.equal(O.unpack_qweight(qw, 4).int(), z)
