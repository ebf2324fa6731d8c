"""GPU: every compiled kernel instance against a float64 reference, element by element.

The kernels are template grids; dispatch picks the instance from the dtype, bit width, layout, zeros mode and m.  The tables
below mirror the host-side instance selection (launch_mma_nt, launch_gemv_i8, launch_grouped's rows per pass, launch_ts_bm,
launch_slab, launch_generic), and every test forces its kernel family with bb_set_kernel_override, asserts
Matmul.kernel_for(m), and compares each output element with a reference computed in float64 on the CPU.

Dequantisation contract (what the reference computes; u = the stored field, w = its decoded value, s = scale, z = zeros):

  family                         | how the dequantised weight is formed
  -------------------------------+-----------------------------------------------------------------------------------------
  gemv_mma, grouped, gemv_slab   | exact: w, w*s, (w - z)*s, w*s - z, (u - qz)*s.  The kernels fold the decode magic and the
                                 | zero point into fp32 sums ((magic + u)*s and (magic + z)*s chains), never round a weight
  gemm_ts (wgmma)                | A_dtype arithmetic, one rounding per operation (dq_finish): (w - z) then * s; rescale is
                                 | one fma(w, s, -z) for 4-bit weights (both dtypes, both layouts) and w*s, then - z, for
                                 | 2-bit; table / fp8 formats: decoded value * s
  generic_simt                   | A_dtype arithmetic in the reference's order: rescale is one fma only where the reference's
                                 | LOP3 decode has one (fp16, interleaved integer weights, 4- or 1-bit); otherwise w*s, then - z
  int8 activations (all)         | exact integers; int32 accumulation; the epilogue is emulated bit for bit (torch.equal)

Error model of the floating-point outputs (checked per element, no mismatch allowance, bf16 included):

  |got - ref| <= k * ulp_out(m) + C_ACC * 2^-24 * sum_k |a_k| * |term_k|

  * ulp_out(m): one unit in the last place of out_dtype at m = |ref| (k = 1).  With bias the kernels round the fp32 sum to
    out_dtype and then add the rounded bias, so m = max(|ref|, |ref - bias|, |bias|) and k = 2.
  * The accumulation term bounds the fp32 (tensor-core) accumulation: every partial sum is at most sum_k |a_k| |term_k|, and
    each rounding or truncation step costs at most 2^-24 of it.  `term` is what the kernel actually accumulates: the
    dequantised weight for gemm_ts and generic_simt; for the GEMV family the magic-number chains |s| (magic + u) and
    |s| (magic + z) (plus |s| |z| for zero points that are not folded and |z| for rescale zeros, which a third MMA applies
    against the activation sums).  C_ACC (per rule, below) allows for the depth of the summation: the partial sums of random
    activations stay well below sum_k |a_k| |term_k|, so far fewer than one full step per k is ever lost.

The bound is compared with assert_fp_close's allowance (1e-2 * max(1, mean|ref|) + 1e-2 * |ref|) on every checked element;
test_bound_tightness (last in this file) requires it to be at least 5x tighter on 99 % of the gemm_ts / generic_simt elements
with fp16 or fp32 output.
"""
from __future__ import annotations

import contextlib
import ctypes
import itertools
import zlib

import pytest
import torch

import bitblas_oracle as O
import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS32 = 2.0 ** -24
# accumulation constant per dequantisation rule; the largest values needed on an H100 (NVIDIA H100 80GB HBM3) over this file
# were 3.0 (GEMV family, activations of one sign), 9.2 (gemm_ts, 48 wgmma k-steps in one CTA, fp32 output) and 0.02 (generic)
C_ACC = {"exact": 8.0, "gemm_ts": 32.0, "generic": 16.0}
MAGIC = {"float16": 1024.0, "bfloat16": 128.0}
# (mantissa bits, smallest normal exponent) of the output types
ULP = {"float16": (10, -14), "bfloat16": (7, -126), "float32": (23, -126)}

(K_GENERIC, K_GEMV_MMA, K_GEMV_I8, K_GEMM_TS, K_GEMM_TS_I8, K_GEMV_SLAB) = 1, 2, 3, 4, 5, 7
KERNEL_NAME = {K_GENERIC: "generic_simt", K_GEMV_MMA: "gemv_mma", K_GEMV_I8: "gemv_i8", K_GEMM_TS: "gemm_ts_wgmma",
               K_GEMM_TS_I8: "gemm_ts_wgmma_i8", K_GEMV_SLAB: "gemv_slab"}

MODES = ["none", "scale", "original", "rescale", "quantized"]
OUTS = ["float16", "bfloat16", "float32"]
GROUPS = [128, 384, -1]

_TIGHTNESS = []   # (rule, out_dtype, assert_fp_close allowance / this file's bound per element) for test_bound_tightness


# ---- host-side instance selection, mirrored ---------------------------------------------------------------------------------
def mma_nt(m):
    """launch_mma_nt / launch_gemv_i8: batch tiles of 8 rows per instance"""
    nt = (m + 7) // 8
    return 1 if nt <= 1 else (2 if nt == 2 else 4)


def grouped_nt(counts):
    """launch_grouped: rows per pass from the mean rows per active group"""
    T = sum(counts)
    active = min(len(counts), T)
    mean = -(-T // active)
    return 1 if mean <= 8 else (2 if mean <= 16 else 4)


def ts_bm(m):
    """launch_ts_bm: the wgmma N extent"""
    return 32 if m <= 32 else (64 if m <= 64 else 128)


def ts_splits(m, N, K, kb, sms):
    """launch_ts_inst / choose_splits: split-K factor (m <= 128 only)"""
    if m > 128:
        return 1
    tiles = -(-m // ts_bm(m)) * (N // 128)
    num_kb = K // kb
    if tiles >= sms:
        return 1
    best = 1
    for sp in range(2, 9):
        if num_kb % sp or num_kb // sp < 8:
            continue
        if tiles * sp <= sms:
            best = sp
    return best


# ---- inputs -----------------------------------------------------------------------------------------------------------------
def _fp8_codes(fmt):
    """finite 8-bit float codes of magnitude <= 16 (keeps every reference finite in fp16)"""
    u = torch.arange(256, dtype=torch.int32)
    v = O.decode_fields(u, fmt, 8, torch.float32)
    return u[torch.isfinite(v) & (v.abs() <= 16)]


def make_case(M, N, K, *, A_dtype="float16", W_dtype="uint4", out_dtype="float16", group_size=-1, mode="none", bias=False,
              fast_decoding=None, seed=0, zeros_value=None, A=None, a_range=128):
    """seeded inputs in helpers.make_case's layout, with the value edges of this file: signed scales, "original" zero points
    that are integers, fractions, negative and above the GEMV fold limit (MAXZ) in one tensor, signed "rescale" zeros"""
    g = torch.Generator().manual_seed(seed)
    fmt, bit = O.W_DTYPE_MAP[W_dtype]
    adt = O.TORCH_DTYPE[A_dtype]
    gs = K if group_size in (-1, None) else group_size
    G = K // gs
    if A is None:
        if A_dtype == "int8":
            A = torch.randint(-a_range, a_range, (M, K), generator=g, dtype=torch.int8)
        else:
            A = (torch.rand((M, K), generator=g) - 0.5).to(adt)
    if fmt in ("fp_e4m3", "fp_e5m2"):
        codes = _fp8_codes(fmt)
        fields = codes[torch.randint(0, codes.numel(), (N, K), generator=g)]
    else:
        fields = torch.randint(0, 2 ** bit, (N, K), generator=g, dtype=torch.int32)
    with_scaling = mode != "none"
    with_zeros = mode in ("original", "rescale", "quantized")
    scale = zeros = qz = b = None
    if with_scaling:
        sign = torch.where(torch.rand((N, G), generator=g) < 0.3, -1.0, 1.0)
        scale = ((torch.rand((N, G), generator=g) * (2.0 / 2 ** bit) + 0.01) * sign).to(adt)
    if mode == "original":
        if zeros_value is not None:
            zeros = torch.full((N, G), float(zeros_value)).to(adt)
        else:
            big = (50.0, 200.0) if A_dtype == "float16" else (120.0, 200.0)
            choices = torch.stack([
                torch.randint(0, 2 ** bit, (N, G), generator=g).float(),       # integer, folded by the GEMV kernels
                torch.rand((N, G), generator=g) * (2 ** bit - 1),                # fraction
                -torch.randint(1, 5, (N, G), generator=g).float() - torch.rand((N, G), generator=g).round() * 0.5,
                torch.full((N, G), big[0]), torch.full((N, G), big[1])])
            pick = torch.randint(0, 5, (N, G), generator=g)
            zeros = choices.gather(0, pick[None]).squeeze(0).to(adt)
    elif mode == "rescale":
        sign = torch.where(torch.rand((N, G), generator=g) < 0.3, -1.0, 1.0)
        zeros = ((torch.rand((N, G), generator=g) * (2 ** bit - 1)).to(adt) * scale * sign.to(adt)).to(adt)
    elif mode == "quantized":
        qz = torch.randint(0, 2 ** bit, (G, N), generator=g, dtype=torch.int32)
        zeros = torch.from_numpy(O.general_compress(qz.numpy(), bit))
    if bias:
        if A_dtype == "int8":
            b = torch.randint(-8, 8, (N,), generator=g, dtype=torch.int8)
        else:
            b = ((torch.rand((N,), generator=g) - 0.5) * 4).to(adt)
    cfg = dict(A_dtype=A_dtype, W_dtype=W_dtype, accum_dtype="int32" if A_dtype == "int8" else "float32",
               out_dtype=out_dtype, group_size=group_size, with_scaling=with_scaling, with_zeros=with_zeros,
               zeros_mode=mode if with_zeros else "original", with_bias=bias, fast_decoding=fast_decoding)
    return dict(M=M, N=N, K=K, A=A, fields=fields, scale=scale, zeros=zeros, qz=qz, bias=b, bit=bit, fmt=fmt, mode=mode,
                cfg=cfg)


# ---- float64 reference --------------------------------------------------------------------------------------------------------
def _decoded(case):
    """decoded weight values (float64) before scale / zeros"""
    u, fmt, bit = case["fields"].to(torch.int64), case["fmt"], case["bit"]
    if case["mode"] == "quantized":
        gidx = torch.arange(case["K"]) // (case["K"] // case["qz"].shape[0])
        return (u - case["qz"].to(torch.int64)[gidx, :].T).double()
    if fmt == "uint":
        return u.double()
    if fmt == "int":
        if bit == 1:
            return (2 * u - 1).double()
        if bit == 8:
            return u.to(torch.uint8).view(torch.int8).double()
        return (u - 2 ** (bit - 1)).double()
    adt = O.TORCH_DTYPE[case["cfg"]["A_dtype"]]
    lut = None
    if fmt == "nf":   # the operator's table: the standard NF4 one unless the case carries its own 16 entries
        lut = case["lut"].to(adt) if case.get("lut") is not None else torch.tensor(O.NF4_LUT, dtype=adt)
    return O.decode_fields(u.to(torch.int32), fmt, bit, adt, lut).double()


def dequant(case, rule, layout_il=False):
    """W [N, K] in float64 by the family's contract (module docstring); rule: exact | gemm_ts | generic"""
    mode, bit = case["mode"], case["bit"]
    w = _decoded(case)
    if mode == "none":
        return w
    gidx = torch.arange(case["K"]) // (case["K"] // case["scale"].shape[1])
    adt = O.TORCH_DTYPE[case["cfg"]["A_dtype"]]
    s = case["scale"][:, gidx]
    z = case["zeros"][:, gidx] if mode in ("original", "rescale") else None
    if rule == "exact":
        if mode == "original":
            return (w - z.double()) * s.double()
        if mode == "rescale":
            return w * s.double() - z.double()
        return w * s.double()
    t = w.to(adt)   # small integers and table values: exact in A_dtype
    if mode == "original":
        return ((t - z) * s).double()
    if mode == "rescale":
        if rule == "gemm_ts":
            fma = bit != 2
        else:
            fma = layout_il and case["fmt"] in ("uint", "int") and adt == torch.float16 and bit != 2
        if fma:
            return (t.double() * s.double() - z.double()).to(adt).double()
        return ((t * s) - z).double()
    return (t * s).double()


def acc_terms(case, rule, W):
    """|term| [N, K]: what the kernel accumulates in fp32 (module docstring)"""
    if rule != "exact" or case["fmt"] not in ("uint", "int"):
        return W.abs()
    mode, A_dtype = case["mode"], case["cfg"]["A_dtype"]
    M0 = MAGIC[A_dtype]
    u = case["fields"].double()
    zp = 2.0 ** (case["bit"] - 1) if case["fmt"] == "int" else 0.0
    if mode == "none":
        return 2 * M0 + u + zp
    gidx = torch.arange(case["K"]) // (case["K"] // case["scale"].shape[1])
    s = case["scale"][:, gidx].double().abs()
    if mode == "original":
        z = case["zeros"][:, gidx].double().abs()
        return s * (2 * M0 + u + 2 * z)
    if mode == "rescale":
        return s * (2 * M0 + u) + case["zeros"][:, gidx].double().abs()
    if mode == "quantized":
        return s * (2 * M0 + u + case["qz"].double()[gidx, :].T)
    return s * (2 * M0 + u + zp)


def _ulp(x, dtype):
    mant, emin = ULP[dtype]
    e = torch.floor(torch.log2(x.clamp_min(2.0 ** (emin - mant))))
    return torch.pow(2.0, torch.clamp(e, min=emin) - mant)


def float_reference(case, rule, layout_il=False, rows=None):
    """(reference, per-element bound) of the float output by the family's rule: what check_float compares with, computed once
    where several kernels of one rule run the same case"""
    A = case["A"] if rows is None else case["A"][rows]
    W = dequant(case, rule, layout_il)
    A64 = A.double()
    ref = A64 @ W.T
    acc = A64.abs() @ acc_terms(case, rule, W).T
    out = case["cfg"]["out_dtype"]
    mag = ref.abs()
    k_out = 1.0
    if case["bias"] is not None:
        b = case["bias"].double()
        ref_nb = ref
        ref = ref + b
        mag = torch.maximum(torch.maximum(ref.abs(), ref_nb.abs()), b.abs().expand_as(ref))
        k_out = 2.0
    odt = O.TORCH_DTYPE[out]
    assert torch.isfinite(ref.to(odt).float()).all(), f"reference not finite in {out}"
    return ref, k_out * _ulp(mag, out) + C_ACC[rule] * EPS32 * acc


def check_float(got, case, rule, what, layout_il=False, rows=None, reference=None):
    """got against float_reference(case, rule, layout_il, rows), or the `reference` pair already computed for it"""
    ref, bound = reference if reference is not None else float_reference(case, rule, layout_il, rows)
    out = case["cfg"]["out_dtype"]
    g = got.double()
    err = (g - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        idx = bad.nonzero()[:4].tolist()
        worst = float((err / bound).nan_to_num(float("inf")).max())
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements outside the bound (worst err/bound {worst:.2f}); "
                             f"first at {idx}: got {[float(g[i, j]) for i, j in idx]} ref {[float(ref[i, j]) for i, j in idx]}")
    allow = 1e-2 * max(1.0, float(ref.abs().mean())) + 1e-2 * ref.abs()
    _TIGHTNESS.append((rule, out, (allow / bound).flatten().float()))


def int_reference(case, rows=None):
    """int8 activations: exact int32 accumulation and the kernels' epilogue per out_dtype"""
    A = case["A"] if rows is None else case["A"][rows]
    W = _decoded(case).to(torch.int64)
    acc = A.to(torch.int64) @ W.T
    acc = (acc + 2 ** 31) % 2 ** 32 - 2 ** 31
    b = case["bias"].to(torch.int64) if case["bias"] is not None else torch.zeros(case["N"], dtype=torch.int64)
    out = case["cfg"]["out_dtype"]
    if out == "int32":
        return (acc + b).to(torch.int32)
    if out == "int8":
        return (((acc + 128) % 256 - 128) + b).to(torch.int8)    # int8(int8(acc) + b)
    if out == "float32":
        return acc.to(torch.float32) + b.to(torch.float32)
    odt = O.TORCH_DTYPE[out]
    return acc.to(torch.float32).to(odt) + b.to(odt)              # __hadd(__int2half_rn(acc), __int2half_rn(b))


# ---- running one forced kernel ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def forced(kernel_id):
    from bitblas_b200 import _lib
    lib = _lib.load()
    lib.bb_set_kernel_override(kernel_id)
    try:
        yield lib
    finally:
        lib.bb_set_kernel_override(0)


def run_forced(case, kernel_id, m=None):
    op = H.product_operator(case)
    m = case["M"] if m is None else m
    with forced(kernel_id):
        assert op.kernel_for(m) == KERNEL_NAME[kernel_id], (op.kernel_for(m), case["cfg"])
        got = H.run_product(op, case)
    return op, got


def _layout_il(op):
    return bool(op.fast_decoding) and op.bit < 8


def _id(d):
    return "-".join(f"{k}={v}" for k, v in d.items())


def _seed(d):
    return zlib.crc32(_id(d).encode()) % 100003


# ---- gemv_mma: T x bits x layout x NT x zeros = 120 instances -----------------------------------------------------------------
NT_ROWS = {1: (1, 8), 2: (9, 16), 4: (25, 32, 17)}


def _gemv_cells():
    cells = []
    for i, (T, bits, il, nt, mode) in enumerate(itertools.product(["float16", "bfloat16"], [4, 2], [True, False], [1, 2, 4], MODES)):
        signed = mode in ("none", "scale") and i % 2 == 1
        rows = NT_ROWS[nt]
        cells.append(dict(T=T, W=("int" if signed else "uint") + str(bits), il=il, nt=nt, mode=mode, m=rows[i % len(rows)],
                          out=OUTS[i % 3], bias=i % 4 < 2, g=GROUPS[i % 3]))
    return cells


GEMV_CELLS = _gemv_cells()


@pytest.mark.parametrize("c", GEMV_CELLS, ids=[_id(c) for c in GEMV_CELLS])
def test_gemv_mma_instance(c):
    assert mma_nt(c["m"]) == c["nt"]
    case = make_case(c["m"], 256, 768, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"],
                     bias=c["bias"], fast_decoding=c["il"], seed=_seed(c))
    op, got = run_forced(case, K_GEMV_MMA)
    assert _layout_il(op) == c["il"]
    check_float(got, case, "exact", f"gemv_mma {c}")


# ---- grouped: the same 120 cells, routings that make the host pick each NT ------------------------------------------------------
# each has an empty expert, counts that are not multiples of the rows per pass R = 8 NT, and one expert with more than R rows
ROUTINGS = {1: [3, 0, 11, 5, 1], 2: [13, 0, 21, 9, 20], 4: [40, 0, 17, 33, 30]}


@pytest.mark.parametrize("c", GEMV_CELLS, ids=[_id(c) for c in GEMV_CELLS])
def test_grouped_instance(c, monkeypatch):
    from bitblas_b200 import _lib
    from bitblas_b200.ops import general_matmul as GM
    monkeypatch.setattr(GM, "GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP", 1 << 20)   # the single launch at every row count
    counts = ROUTINGS[c["nt"]]
    assert grouped_nt(counts) == c["nt"]
    N, K, T = 128, 768, sum(counts)
    seed = _seed(c)
    kw = dict(A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"], bias=c["bias"],
              fast_decoding=c["il"])
    A = make_case(T, 8, K, seed=seed, **dict(kw, mode="none", bias=False))["A"]
    cases = [make_case(T, N, K, seed=seed * 31 + e, A=A, **kw) for e in range(len(counts))]
    op = H.product_operator(cases[0], M=[1, 16])
    st = lambda k: torch.stack([x[k] for x in cases]).to(DEV) if cases[0][k] is not None else None   # noqa: E731
    W = torch.stack([H.product_weight(op, x, DEV) for x in cases])
    off = [0] + list(itertools.accumulate(counts))
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    got = op.forward_grouped(A.to(DEV), W, torch.tensor(off, dtype=torch.int32, device=DEV), scale=st("scale"),
                             zeros=st("zeros"), bias=st("bias")).cpu()
    assert lib.bb_launch_count() - n0 == 1
    for e, x in enumerate(cases):
        if counts[e]:
            rows = slice(off[e], off[e + 1])
            check_float(got[rows], x, "exact", f"grouped expert {e} {c}", rows=rows)


# ---- gemm_ts (float): T x bits x BM x layout x mode = 120 instances; split-K on and off at m <= 128 ------------------------------
TS_ROWS_FOR_BM = {32: (1, 2, 31, 32), 64: (33, 63, 64), 128: (65, 127, 128, 129, 255, 257)}


def _ts_cells():
    cells = []
    for i, (T, bits, bm, il, mode) in enumerate(itertools.product(["float16", "bfloat16"], [4, 2], [32, 64, 128], [True, False], MODES)):
        signed = mode in ("none", "scale") and i % 2 == 1
        rows = TS_ROWS_FOR_BM[bm]
        cells.append(dict(T=T, W=("int" if signed else "uint") + str(bits), bm=bm, il=il, mode=mode, m=rows[i % len(rows)],
                          out=OUTS[i % 3], bias=i % 4 < 2, g=GROUPS[(i // 2) % 3], split=i % 2 == 0))
    return cells


TS_CELLS = _ts_cells()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check_split(op, m, split, kb, sms=None):
    """the split-K factor of the launch on `sms` SMs (default: the device's), read from bb_workspace_bytes: 0 without split-K,
    else the slab's slot region at the device's full SM count followed by f [m, N] fp32 partials"""
    from bitblas_b200 import _lib
    from exact_inputs import slab_slot_bytes
    ws = _lib.load().bb_workspace_bytes(ctypes.byref(op._desc), m)
    f = ts_splits(m, op.N, op.K, kb, sms or _sms())
    assert ws == (slab_slot_bytes(_sms()) + f * m * op.N * 4 if f > 1 else 0), (m, ws, f)
    if m <= 128:
        assert (f > 1) == split


@pytest.mark.parametrize("c", TS_CELLS, ids=[_id(c) for c in TS_CELLS])
def test_gemm_ts_instance(c):
    assert ts_bm(c["m"]) == c["bm"]
    K = 1536 if c["split"] else 768   # 24 k-blocks split 3 ways; 12 k-blocks cannot split (8 per split at least)
    case = make_case(c["m"], 256, K, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"],
                     bias=c["bias"], fast_decoding=c["il"], seed=_seed(c))
    op, got = run_forced(case, K_GEMM_TS)
    assert _layout_il(op) == c["il"]
    with forced(K_GEMM_TS):
        _check_split(op, c["m"], c["split"], 64)
    check_float(got, case, "gemm_ts", f"gemm_ts {c}")


# ---- gemm_ts with int8 activations: bits x layout x BM x signedness; every output type +- bias, split-K on and off ----------------
I8_OUTS = ["int32", "int8", "float32", "float16", "bfloat16"]


def _ts_i8_cells():
    cells = []
    for i, (bits, il, bm, signed) in enumerate(itertools.product([4, 2], [True, False], [32, 64, 128], [True, False])):
        rows = TS_ROWS_FOR_BM[bm]
        cells.append(dict(W=("int" if signed else "uint") + str(bits), il=il, bm=bm, m=rows[i % len(rows)],
                          out=I8_OUTS[i % 5], bias=i % 4 < 2, split=i % 2 == 0))
    for out, bias, split in itertools.product(I8_OUTS, [False, True], [False, True]):
        cells.append(dict(W="uint4", il=False, bm=32, m=5, out=out, bias=bias, split=split))
    return cells


TS_I8_CELLS = _ts_i8_cells()


def check_int(got, case, what):
    ref = int_reference(case)
    if not torch.equal(got, ref):
        bad = (got.double() != ref.double())
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements differ; first at {idx}: "
                             f"got {[got[i, j].item() for i, j in idx]} ref {[ref[i, j].item() for i, j in idx]}")


@pytest.mark.parametrize("c", TS_I8_CELLS, ids=[_id(c) for c in TS_I8_CELLS])
def test_gemm_ts_i8_instance(c):
    assert ts_bm(c["m"]) == c["bm"]
    K = 2048 if c["split"] else 1024   # 16 / 8 k-blocks of 128
    a_range = 32 if c["out"] in ("float16", "bfloat16") else 128   # keeps the sum finite in fp16
    case = make_case(c["m"], 256, K, A_dtype="int8", W_dtype=c["W"], out_dtype=c["out"], bias=c["bias"],
                     fast_decoding=c["il"], seed=_seed(c), a_range=a_range)
    op, got = run_forced(case, K_GEMM_TS_I8)
    assert _layout_il(op) == c["il"]
    with forced(K_GEMM_TS_I8):
        _check_split(op, c["m"], c["split"], 128)
    check_int(got, case, f"gemm_ts_i8 {c}")


# ---- gemm_ts table (NF4, fp4) and 8-bit float formats: T x BM ---------------------------------------------------------------------
TABLE_CELLS = [dict(W=W, T=T, bm=bm, m=TS_ROWS_FOR_BM[bm][i % 3], scale=i % 2 == 0, out=OUTS[i % 3])
               for i, (W, T, bm) in enumerate(itertools.product(["nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8"],
                                                                ["float16", "bfloat16"], [32, 64, 128]))]


@pytest.mark.parametrize("c", TABLE_CELLS, ids=[_id(c) for c in TABLE_CELLS])
def test_gemm_ts_table_and_fp8_instance(c):
    case = make_case(c["m"], 256, 768, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=128,
                     mode="scale" if c["scale"] else "none", seed=_seed(c))
    op, got = run_forced(case, K_GEMM_TS)
    check_float(got, case, "gemm_ts", f"gemm_ts {c}")


# ---- gemv_i8: bits x NT = 6 instances -------------------------------------------------------------------------------------------
GEMV_I8_CELLS = [dict(W=("int" if i % 2 else "uint") + str(bits), nt=nt, m=NT_ROWS[nt][i % len(NT_ROWS[nt])],
                      out=I8_OUTS[i % 5], bias=i % 3 == 0)
                 for i, (bits, nt) in enumerate(itertools.product([4, 2], [1, 2, 4]))]


@pytest.mark.parametrize("c", GEMV_I8_CELLS, ids=[_id(c) for c in GEMV_I8_CELLS])
def test_gemv_i8_instance(c):
    assert mma_nt(c["m"]) == c["nt"]
    a_range = 32 if c["out"] in ("float16", "bfloat16") else 128
    case = make_case(c["m"], 256, 1024, A_dtype="int8", W_dtype=c["W"], out_dtype=c["out"], bias=c["bias"], fast_decoding=True,
                     seed=_seed(c), a_range=a_range)
    op, got = run_forced(case, K_GEMV_I8)
    check_int(got, case, f"gemv_i8 {c}")


# ---- gemv_slab: 6 instances (T x {interleaved int, compressed int, table}) x modes ---------------------------------------------
SLAB_CELLS = ([dict(T=T, W="uint4" if mode not in ("none", "scale") or i % 2 == 0 else "int4", il=il, mode=mode,
                    out=OUTS[i % 3], bias=i % 4 < 2, g=GROUPS[i % 3], N=(16, 272, 512)[i % 3])
               for i, (T, il, mode) in enumerate(itertools.product(["float16", "bfloat16"], [True, False], MODES))]
              + [dict(T=T, W=W, il=False, mode=mode, out=OUTS[i % 3], bias=i % 2 == 0, g=128, N=(272, 512)[i % 2])
                 for i, (T, W, mode) in enumerate(itertools.product(["float16", "bfloat16"], ["nf4", "fp4_e2m1"], ["none", "scale"]))])


@pytest.mark.parametrize("c", SLAB_CELLS, ids=[_id(c) for c in SLAB_CELLS])
def test_gemv_slab_instance(c):
    K = 256 if c["g"] == 128 else 768    # K = 256: one slab unit; 768 for the 384 / per-row groups
    case = make_case(1, c["N"], K, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"],
                     bias=c["bias"], fast_decoding=c["il"] if c["W"] in ("uint4", "int4") else None, seed=_seed(c))
    op, got = run_forced(case, K_GEMV_SLAB)
    assert _layout_il(op) == c["il"]
    check_float(got, case, "exact", f"gemv_slab {c}")


# ---- generic_simt: mode x dtype x bits (1, 2, 4, 8) x layout, table / fp8 formats, int8 activations ------------------------------
def _generic_cells():
    cells = []
    for i, (T, bits, mode) in enumerate(itertools.product(["float16", "bfloat16"], [1, 2, 4, 8], MODES)):
        for il in ([True, False] if bits < 8 else [False]):
            signed = mode in ("none", "scale") and (i + il) % 2 == 1
            cells.append(dict(T=T, W=("int" if signed else "uint") + str(bits), il=il, mode=mode, m=(1, 3, 7)[i % 3],
                              out=OUTS[i % 3], bias=i % 2 == 0, g=(64, 384, -1)[i % 3]))
    for i, (T, W) in enumerate(itertools.product(["float16", "bfloat16"], ["nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8"])):
        cells.append(dict(T=T, W=W, il=False, mode=("none", "scale")[i % 2], m=5, out=OUTS[i % 3], bias=i % 2 == 1, g=64))
    for i, W in enumerate(["uint1", "int2", "uint4", "int4"]):
        cells.append(dict(T="int8", W=W, il=i % 2 == 0, mode="none", m=6, out=I8_OUTS[i], bias=i % 2 == 1, g=-1))
    return cells


GENERIC_CELLS = _generic_cells()


@pytest.mark.parametrize("c", GENERIC_CELLS, ids=[_id(c) for c in GENERIC_CELLS])
def test_generic_instance(c):
    table = c["W"] in ("nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8")
    case = make_case(c["m"], 72, 768, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"],
                     bias=c["bias"], fast_decoding=None if table else c["il"], seed=_seed(c),
                     a_range=32 if c["out"] in ("float16", "bfloat16") else 128)
    op, got = run_forced(case, K_GENERIC)
    assert _layout_il(op) == c["il"]
    if c["T"] == "int8":
        check_int(got, case, f"generic {c}")
    else:
        check_float(got, case, "generic", f"generic {c}", layout_il=c["il"])


# ---- shape edges ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", ["float16", "bfloat16"])
@pytest.mark.parametrize("m", range(1, 33))
def test_gemv_mma_every_m(m, T):
    kw = (dict(W_dtype="uint4", mode="original", fast_decoding=True, group_size=128, bias=True) if T == "float16"
          else dict(W_dtype="uint2", mode="rescale", fast_decoding=False, group_size=384, out_dtype="float32"))
    case = make_case(m, 128, 768, A_dtype=T, seed=m, **kw)
    _, got = run_forced(case, K_GEMV_MMA)
    check_float(got, case, "exact", f"gemv_mma m={m} {T}")


@pytest.mark.parametrize("m", range(1, 33))
def test_gemv_i8_every_m(m):
    case = make_case(m, 128, 512, A_dtype="int8", W_dtype="int2", out_dtype="int32", bias=True, fast_decoding=True, seed=m)
    _, got = run_forced(case, K_GEMV_I8)
    check_int(got, case, f"gemv_i8 m={m}")


@pytest.mark.parametrize("T", ["float16", "bfloat16"])
@pytest.mark.parametrize("m", [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 257])
def test_gemm_ts_m_edges(m, T):
    case = make_case(m, 256, 1024, A_dtype=T, W_dtype="uint4", mode="quantized", group_size=128, out_dtype="float16",
                     fast_decoding=T == "float16", seed=m)
    _, got = run_forced(case, K_GEMM_TS)
    check_float(got, case, "gemm_ts", f"gemm_ts m={m} {T}")


@pytest.mark.parametrize("K,m,g", [(64, 16, -1), (64, 129, -1), (576, 16, 64), (576, 200, 192), (1728, 16, -1)])
def test_gemm_ts_k_blocks(K, m, g):
    """one k-block; an odd number of k-blocks (the loop's tail step), also inside each split of a 3-way split-K (27 k-blocks)"""
    case = make_case(m, 128, K, W_dtype="uint2", mode="original", group_size=g, bias=True, fast_decoding=True, seed=K + m)
    op, got = run_forced(case, K_GEMM_TS)
    with forced(K_GEMM_TS):
        _check_split(op, m, ts_splits(m, 128, K, 64, _sms()) > 1, 64)
    check_float(got, case, "gemm_ts", f"gemm_ts K={K} m={m}")


@pytest.mark.parametrize("T", ["float16", "bfloat16"])
@pytest.mark.parametrize("m", [1, 8, 20])
def test_gemv_mma_single_step(m, T):
    """K = 128: one 128-element step, one warp per row block"""
    case = make_case(m, 64, 128, A_dtype=T, W_dtype="uint4", mode="original", group_size=128, fast_decoding=True, seed=m)
    _, got = run_forced(case, K_GEMV_MMA)
    check_float(got, case, "exact", f"gemv_mma K=128 m={m} {T}")


@pytest.mark.parametrize("N,K,g", [(16, 256, 128), (48, 256, -1), (272, 1024, 128), (256, 1024, 128), (16, 2048, 256)])
def test_gemv_slab_shapes(N, K, g):
    """K = 256 (one unit), N = 16, N = 16 (mod 32); N % 32 == 0 with G = 8 one-step groups takes the vector parameter path"""
    case = make_case(1, N, K, W_dtype="uint4", mode="quantized", group_size=g, fast_decoding=True, seed=N + K)
    _, got = run_forced(case, K_GEMV_SLAB)
    check_float(got, case, "exact", f"gemv_slab N={N} K={K}")


# ---- value edges ------------------------------------------------------------------------------------------------------------------
# "original" zero points that no GEMV kernel can fold into its magic number (MAXZ: 47 on the fp16 4-bit path, 112 / 124 for bf16),
# uniform over the whole matrix, through every kernel that takes original zeros
ZEDGE = [("float16", 50.0), ("float16", 200.0), ("float16", -3.0), ("bfloat16", 120.0), ("bfloat16", 200.0), ("bfloat16", -2.5)]


@pytest.mark.parametrize("kernel", [K_GEMV_MMA, K_GEMV_SLAB, K_GEMM_TS, K_GENERIC], ids=lambda k: KERNEL_NAME[k])
@pytest.mark.parametrize("T,z", ZEDGE, ids=[f"{t}-z={z}" for t, z in ZEDGE])
def test_original_zeros_outside_fold_range(T, z, kernel):
    m = 1 if kernel == K_GEMV_SLAB else 4
    case = make_case(m, 256, 512, A_dtype=T, W_dtype="uint4", mode="original", group_size=128, fast_decoding=True,
                     zeros_value=z, seed=int(abs(z) * 10) + kernel)
    _, got = run_forced(case, kernel)
    rule = {K_GEMM_TS: "gemm_ts", K_GENERIC: "generic"}.get(kernel, "exact")
    check_float(got, case, rule, f"{KERNEL_NAME[kernel]} z={z} {T}", layout_il=True)


def test_grouped_original_zeros_outside_fold_range(monkeypatch):
    from bitblas_b200.ops import general_matmul as GM
    monkeypatch.setattr(GM, "GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP", 1 << 20)
    for T, z in ZEDGE:
        counts = [2, 0, 9]
        A = make_case(11, 8, 512, A_dtype=T, seed=1)["A"]
        cases = [make_case(11, 128, 512, A_dtype=T, W_dtype="uint4", mode="original", group_size=128, fast_decoding=True,
                           zeros_value=z, seed=e, A=A) for e in range(3)]
        op = H.product_operator(cases[0], M=[1, 16])
        W = torch.stack([H.product_weight(op, x, DEV) for x in cases])
        off = [0, 2, 2, 11]
        got = op.forward_grouped(A.to(DEV), W, torch.tensor(off, dtype=torch.int32, device=DEV),
                                 scale=torch.stack([x["scale"] for x in cases]).to(DEV),
                                 zeros=torch.stack([x["zeros"] for x in cases]).to(DEV)).cpu()
        for e in (0, 2):
            rows = slice(off[e], off[e + 1])
            check_float(got[rows], cases[e], "exact", f"grouped z={z} {T} expert {e}", rows=rows)


def _adversarial(K, g):
    return {
        "one_sign_large": (torch.rand((4, K), generator=g) * 8 + 2).half(),
        "tiny": ((torch.rand((4, K), generator=g) - 0.5) * 2e-4).half(),
        "wide_range": (torch.randn((4, K), generator=g) * torch.pow(10.0, torch.randint(-4, 2, (4, K), generator=g).float())).half(),
        "alternating": (torch.tensor([1.0, -1.0]).repeat(2 * K).reshape(4, K) * 300).half(),
    }


@pytest.mark.parametrize("name", ["one_sign_large", "tiny", "wide_range", "alternating"])
@pytest.mark.parametrize("mode", ["original", "rescale", "quantized"])
def test_adversarial_activations_gemv_mma_and_grouped(mode, name, monkeypatch):
    """activations whose sums cancel badly, are all of one sign, are tiny, or span 1e-4 .. 10: the magic number and the zero
    point are removed through fp32 activation sums, not per element"""
    from bitblas_b200.ops import general_matmul as GM
    monkeypatch.setattr(GM, "GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP", 1 << 20)
    K = 1024
    A = _adversarial(K, torch.Generator().manual_seed(7))[name]
    kw = dict(W_dtype="uint4", mode=mode, group_size=128, fast_decoding=True, out_dtype="float32")
    case = make_case(4, 256, K, A=A, seed=3, **kw)
    if mode == "original":   # integer / fractional zero points in range: the fold and the third-MMA paths
        case["zeros"] = (case["zeros"].float().clamp(-4, 15)).half()
    _, got = run_forced(case, K_GEMV_MMA)
    check_float(got, case, "exact", f"gemv_mma {name} {mode}")
    cases = [case, make_case(4, 256, K, A=A, seed=4, **kw)]
    if mode == "original":
        cases[1]["zeros"] = (cases[1]["zeros"].float().clamp(-4, 15)).half()
    op = H.product_operator(case, M=[1, 16])
    W = torch.stack([H.product_weight(op, x, DEV) for x in cases])
    st = lambda k: torch.stack([x[k] for x in cases]).to(DEV)   # noqa: E731
    got = op.forward_grouped(A.to(DEV), W, torch.tensor([0, 1, 4], dtype=torch.int32, device=DEV), scale=st("scale"),
                             zeros=st("zeros")).cpu()
    check_float(got[0:1], cases[0], "exact", f"grouped {name} {mode} expert 0", rows=slice(0, 1))
    check_float(got[1:4], cases[1], "exact", f"grouped {name} {mode} expert 1", rows=slice(1, 4))


# ---- the tolerance itself ----------------------------------------------------------------------------------------------------------
def test_bound_tightness():
    """over every fp16 / fp32 output element this file checked with an A_dtype-rounded reference (gemm_ts, generic_simt), the
    per-element bound is at least 5x tighter than assert_fp_close in 99 %.  Not held to that target: bfloat16 outputs, whose one
    ulp is 0.4-0.8 % of the value against assert_fp_close's 1 %, and the GEMV family, whose bound carries the magic-number
    chains (2 * 1024 |s| per weight in fp16)."""
    if len(_TIGHTNESS) < 100:
        pytest.skip("needs the grid tests of this file to have run first")
    r = torch.cat([t for rule, out, t in _TIGHTNESS if rule != "exact" and out != "bfloat16"])
    share = float((r >= 5).float().mean())
    assert share >= 0.99, f"only {share:.4f} of {r.numel()} elements have a bound 5x tighter than assert_fp_close " \
                          f"(median ratio {float(r.median()):.1f})"
