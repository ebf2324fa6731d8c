"""The library's dispatch table restated in Python: validate(), the five support predicates and the select() ladder of
bb_api.cu, and bb_workspace_bytes.  Each predicate is a list of named clauses, so a descriptor can be told which clause put it on
which side (`explain`).

Every clause is written with & | ~ and numpy-compatible arithmetic, so one function evaluates a single descriptor (fields are ints)
or a whole grid at once (fields are int64 arrays of one length; m an int or an array of that length).

Sources restated here (keep them in step):
  validate, select, bb_workspace_bytes   bitblas_b200/csrc/bb_api.cu
  generic_supported                      bitblas_b200/csrc/bb_generic.cu
  gemv_mma_supported, gemv_i8_supported  bitblas_b200/csrc/bb_gemv.cu
  gemm_ts_supported, choose_splits,      bitblas_b200/csrc/bb_gemm_ts.cu
  gemm_ts_workspace_bytes
  gemv_slab_supported, slot bytes        bitblas_b200/csrc/bb_gemv_slab.cu
  tile_shape_ok                          bitblas_b200/csrc/bb_common.cuh
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

F16, BF16, F32, I8, I32 = 0, 1, 2, 3, 4
W_UINT, W_INT, W_NF, W_FP4, W_E4M3, W_E5M2 = 0, 1, 2, 3, 4, 5
Z_ORIGINAL, Z_RESCALE, Z_QUANTIZED = 0, 1, 2
L_COMP, L_IL16, L_IL8 = 0, 1, 2
T_ROW, T_SLAB = 0, 1
AUTO, GENERIC, GEMV_MMA, GEMV_I8, GEMM_TS, GEMM_TS_I8, GEMV_SLAB = 0, 1, 2, 3, 4, 5, 7
FAMILIES = (GENERIC, GEMV_MMA, GEMV_I8, GEMM_TS, GEMM_TS_I8, GEMV_SLAB)
NAME = {GENERIC: "generic_simt", GEMV_MMA: "gemv_mma", GEMV_I8: "gemv_i8", GEMM_TS: "gemm_ts_wgmma", GEMM_TS_I8: "gemm_ts_wgmma_i8",
        GEMV_SLAB: "gemv_slab", -1: "unknown"}
FIELDS = ("N", "K", "a_dtype", "w_fmt", "w_bits", "accum_dtype", "out_dtype", "group_size", "with_scaling", "with_zeros",
          "zeros_mode", "with_bias", "w_layout", "w_tile", "r0", "r1")   # bb_matmul_desc, in order (r0, r1: reserved[2])
TILE_ROWS, TILE_ROW_BYTES = 32, 512        # BB_TILE_ROWS, BB_TILE_ROW_BYTES
GS_ROWS, GS_KU, GS_MINB, GS_NG = 32, 1024, 2, 2   # the slab kernel's rows and k per unit, CTAs per SM, consumer groups
TS_ROWS = 128                              # weight rows per wgmma CTA tile


def _in(x, values):
    out = x == values[0]
    for v in values[1:]:
        out = out | (x == v)
    return out


def _g(d):
    """the group size (group_size <= 0: one group of K), never 0"""
    g = np.where(d.group_size <= 0, d.K, d.group_size)
    return np.maximum(g, 1)


def _table(d):
    return _in(d.w_fmt, (W_NF, W_FP4))


def _fp8(d):
    return _in(d.w_fmt, (W_E4M3, W_E5M2))


def _integer(d):
    return _in(d.w_fmt, (W_UINT, W_INT))


def _zeros(d):
    return d.with_zeros != 0


def _scaling(d):
    return d.with_scaling != 0


def _a16(d):
    return _in(d.a_dtype, (F16, BF16))


def _float_out(d):
    return _in(d.out_dtype, (F16, BF16, F32))


def _qzeros(d):
    return _zeros(d) & (d.zeros_mode == Z_QUANTIZED)


def tile_shape_ok(d):
    return (d.N % TILE_ROWS == 0) & ((d.K * d.w_bits // 8) % TILE_ROW_BYTES == 0) & ((d.K * d.w_bits) % 8 == 0)


# ---- the clauses: (name, f(d, m)) -> True where the descriptor passes ----------------------------------------------------------
GENERIC_CLAUSES = [
    ("bits in {1, 2, 4, 8}", lambda d, m: _in(d.w_bits, (1, 2, 4, 8))),
    ("K * bits % 32 (below 8 bits)", lambda d, m: (d.w_bits == 8) | ((d.K * d.w_bits) % 32 == 0)),
    ("int8 A: integer format", lambda d, m: (d.a_dtype != I8) | _integer(d)),
    ("A in {f16, bf16, i8}", lambda d, m: _in(d.a_dtype, (F16, BF16, I8))),
]

VALIDATE_CLAUSES = [
    ("N > 0 and K > 0", lambda d, m: (d.N > 0) & (d.K > 0)),
    ("A in {f16, bf16, i8}", lambda d, m: _in(d.a_dtype, (F16, BF16, I8))),
    ("bits in {1, 2, 4, 8}", lambda d, m: _in(d.w_bits, (1, 2, 4, 8))),
    ("format id", lambda d, m: (d.w_fmt >= W_UINT) & (d.w_fmt <= W_E5M2)),
    ("nf4 / fp4: 4-bit", lambda d, m: ~_table(d) | (d.w_bits == 4)),
    ("fp8: 8-bit", lambda d, m: ~_fp8(d) | (d.w_bits == 8)),
    ("K % g", lambda d, m: d.K % _g(d) == 0),
    ("zeros_mode in 0..2", lambda d, m: ~_zeros(d) | ((d.zeros_mode >= 0) & (d.zeros_mode <= 2))),
    ("layout id", lambda d, m: (d.w_layout >= 0) & (d.w_layout <= 2)),
    ("8-bit: compressed", lambda d, m: (d.w_layout == L_COMP) | (d.w_bits != 8)),
    ("int8 A: int32 accum", lambda d, m: (d.a_dtype != I8) | (d.accum_dtype == I32)),
    ("int32 accum: int8 A", lambda d, m: (d.a_dtype == I8) | (d.accum_dtype != I32)),
    ("16-bit A: out f16/bf16/f32", lambda d, m: (d.a_dtype == I8) | _float_out(d)),
    ("reserved == 0", lambda d, m: (d.r0 == 0) & (d.r1 == 0)),
    ("tile id", lambda d, m: _in(d.w_tile, (T_ROW, T_SLAB))),
    ("slab tile: 4/2-bit integer", lambda d, m: (d.w_tile != T_SLAB) | (_integer(d) & _in(d.w_bits, (4, 2)))),
    ("slab tile: N % 32, K*bits/8 % 512", lambda d, m: (d.w_tile != T_SLAB) | tile_shape_ok(d)),
] + [("generic: " + n, f) for n, f in GENERIC_CLAUSES]

SLAB_CLAUSES = [
    ("m == 1", lambda d, m: m == 1),
    ("A f16/bf16", lambda d, m: _a16(d)),
    ("table format: compressed, no zeros", lambda d, m: ~_table(d) | ((d.w_layout == L_COMP) & ~_zeros(d))),
    ("format: uint/int/nf4/fp4", lambda d, m: _table(d) | _integer(d)),
    ("4-bit", lambda d, m: d.w_bits == 4),
    ("layout != interleaved-8", lambda d, m: d.w_layout != L_IL8),
    ("N % 16", lambda d, m: d.N % 16 == 0),
    ("K % 256", lambda d, m: d.K % 256 == 0),
    ("slab tile: N % 32, K % 1024", lambda d, m: (d.w_tile != T_SLAB) | ((d.N % GS_ROWS == 0) & (d.K % GS_KU == 0))),
    ("g % 128", lambda d, m: _g(d) % 128 == 0),
    ("K % g", lambda d, m: d.K % _g(d) == 0),
    ("zeros need scaling", lambda d, m: ~_zeros(d) | _scaling(d)),
    ("int format: no zeros", lambda d, m: (d.w_fmt != W_INT) | ~_zeros(d)),
    ("out f16/bf16/f32", lambda d, m: _float_out(d)),
    ("quantized zeros: N % 2", lambda d, m: ~_qzeros(d) | (d.N % 2 == 0)),
    ("work units < 2^30", lambda d, m: ((d.N + GS_ROWS - 1) // GS_ROWS + 4) * ((d.K + GS_KU - 1) // GS_KU) < (1 << 30)),
]

GEMV_MMA_CLAUSES = [
    ("1 <= m <= 32", lambda d, m: (m >= 1) & (m <= 32)),
    ("row-major", lambda d, m: d.w_tile == T_ROW),
    ("A f16/bf16", lambda d, m: _a16(d)),
    ("format: uint/int", lambda d, m: _integer(d)),
    ("4- or 2-bit", lambda d, m: _in(d.w_bits, (4, 2))),
    ("layout != interleaved-8", lambda d, m: d.w_layout != L_IL8),
    ("N % 16", lambda d, m: d.N % 16 == 0),
    ("K % 128", lambda d, m: d.K % 128 == 0),
    ("g % 128", lambda d, m: _g(d) % 128 == 0),
    ("K % g", lambda d, m: d.K % _g(d) == 0),
    ("zeros need scaling", lambda d, m: ~_zeros(d) | _scaling(d)),
    ("int format: no zeros", lambda d, m: (d.w_fmt != W_INT) | ~_zeros(d)),
    ("out f16/bf16/f32", lambda d, m: _float_out(d)),
    ("quantized zeros: N * bits % 8", lambda d, m: ~_qzeros(d) | ((d.N * d.w_bits) % 8 == 0)),
]

GEMV_I8_CLAUSES = [
    ("1 <= m <= 32", lambda d, m: (m >= 1) & (m <= 32)),
    ("row-major", lambda d, m: d.w_tile == T_ROW),
    ("A int8, int32 accum", lambda d, m: (d.a_dtype == I8) & (d.accum_dtype == I32)),
    ("format: uint/int", lambda d, m: _integer(d)),
    ("4- or 2-bit", lambda d, m: _in(d.w_bits, (4, 2))),
    ("layout == interleaved-8", lambda d, m: d.w_layout == L_IL8),
    ("no scale, no zeros", lambda d, m: ~_scaling(d) & ~_zeros(d)),
    ("N % 16", lambda d, m: d.N % 16 == 0),
    ("K % 128", lambda d, m: d.K % 128 == 0),
]

_I8, _A16 = (lambda d: d.a_dtype == I8), (lambda d: d.a_dtype != I8)
GEMM_TS_CLAUSES = [
    ("m >= 1", lambda d, m: m >= 1),
    ("table format: 4-bit compressed, no zeros, 16-bit A",
     lambda d, m: ~_table(d) | ((d.w_bits == 4) & (d.w_layout == L_COMP) & ~_zeros(d) & (d.a_dtype != I8))),
    ("fp8: 8-bit compressed, no zeros, 16-bit A",
     lambda d, m: ~_fp8(d) | ((d.w_bits == 8) & (d.w_layout == L_COMP) & ~_zeros(d) & (d.a_dtype != I8))),
    ("format: uint/int/table/fp8", lambda d, m: _table(d) | _fp8(d) | _integer(d)),
    ("bits: 4 or 2 (8 for fp8)", lambda d, m: _in(d.w_bits, (4, 2)) | ((d.w_bits == 8) & _fp8(d))),
    ("N % 128", lambda d, m: d.N % TS_ROWS == 0),
    ("int8 A: int32 accum, not interleaved-16", lambda d, m: ~_I8(d) | ((d.accum_dtype == I32) & (d.w_layout != L_IL16))),
    ("int8 A: no scale, no zeros", lambda d, m: ~_I8(d) | (~_scaling(d) & ~_zeros(d))),
    ("int8 A: K % 128", lambda d, m: ~_I8(d) | (d.K % 128 == 0)),
    ("A f16/bf16/i8", lambda d, m: _I8(d) | _a16(d)),
    ("16-bit A: layout != interleaved-8", lambda d, m: ~_A16(d) | (d.w_layout != L_IL8)),
    ("16-bit A: K % 64", lambda d, m: ~_A16(d) | (d.K % 64 == 0)),
    ("16-bit A: g % 64", lambda d, m: ~_A16(d) | (_g(d) % 64 == 0)),
    ("16-bit A: K % g", lambda d, m: ~_A16(d) | (d.K % _g(d) == 0)),
    ("16-bit A: zeros need scaling", lambda d, m: ~_A16(d) | ~_zeros(d) | _scaling(d)),
    ("16-bit A: int format: no zeros", lambda d, m: ~_A16(d) | (d.w_fmt != W_INT) | ~_zeros(d)),
    ("16-bit A: out f16/bf16/f32", lambda d, m: ~_A16(d) | _float_out(d)),
    ("16-bit A: quantized zeros: N * bits % 8", lambda d, m: ~_A16(d) | ~_qzeros(d) | ((d.N * d.w_bits) % 8 == 0)),
]

PREDICATES = {"validate": VALIDATE_CLAUSES, "generic_supported": GENERIC_CLAUSES, "gemv_slab_supported": SLAB_CLAUSES,
              "gemv_mma_supported": GEMV_MMA_CLAUSES, "gemv_i8_supported": GEMV_I8_CLAUSES, "gemm_ts_supported": GEMM_TS_CLAUSES}


def holds(clauses, d, m=1):
    """the conjunction of the clauses (every field and m are numpy integers or arrays: ~ is a logical not on them)"""
    m = np.asarray(m, dtype=np.int64)
    out = np.True_
    for _, f in clauses:
        out = out & f(d, m)
    return out


def explain(d, m=1):
    """{predicate: the first clause the single descriptor d fails at m, or None where it holds}"""
    m = np.int64(m)
    return {p: next((n for n, f in cl if not bool(f(d, m))), None) for p, cl in PREDICATES.items()}


# ---- select() and bb_workspace_bytes ----------------------------------------------------------------------------------------
def select(d, m, override=AUTO):
    """bb_select_kernel(d, m) under bb_set_kernel_override(override): a family id, or -1 (rejected by validate, or the forced
    family does not cover it)"""
    m = np.asarray(m, dtype=np.int64)
    valid = holds(VALIDATE_CLAUSES, d, m)
    slab, mma = holds(SLAB_CLAUSES, d, m), holds(GEMV_MMA_CLAUSES, d, m)
    i8, ts = holds(GEMV_I8_CLAUSES, d, m), holds(GEMM_TS_CLAUSES, d, m)
    a8 = d.a_dtype == I8
    if override != AUTO:
        ok = {GENERIC: True, GEMV_MMA: mma, GEMV_I8: i8, GEMM_TS: ~a8 & ts, GEMM_TS_I8: a8 & ts, GEMV_SLAB: slab}.get(override, False)
        return np.where(valid & ok, override, -1)
    ts_id = np.where(a8, GEMM_TS_I8, GEMM_TS)
    tiled = d.w_tile == T_SLAB
    small, mid = m <= 8, m <= 32
    ladder = [(tiled & slab, GEMV_SLAB), (tiled & ts, ts_id), (tiled, GENERIC),
              (small & slab, GEMV_SLAB), (small & mma, GEMV_MMA), (small & i8, GEMV_I8),
              (ts, ts_id),
              (mid & mma, GEMV_MMA), (mid & i8, GEMV_I8)]
    out = np.full(np.shape(valid), GENERIC)
    for cond, k in reversed(ladder):
        out = np.where(cond, k, out)
    return np.where(valid, out, -1)


def slab_slot_bytes(sms):
    return GS_MINB * GS_NG * sms * GS_ROWS * 8 + 256


def ts_bm(m):
    return np.where(m <= 32, 32, np.where(m <= 64, 64, 128))


def choose_splits(tiles, num_kb, sms):
    best = np.ones(np.shape(tiles), dtype=np.int64)
    for sp in range(2, 9):
        ok = (num_kb % sp == 0) & (num_kb // sp >= 8) & (tiles * sp <= sms)
        best = np.where(ok, sp, best)
    return np.where(tiles >= sms, 1, best)


def ts_splits(d, m, sms):
    """the wgmma GEMM's split-K factor (launch_ts_inst): 1 above m = 128"""
    kb = np.where(d.a_dtype == I8, 128, 64)
    tiles = ((m + ts_bm(m) - 1) // ts_bm(m)) * (d.N // TS_ROWS)
    return np.where(m > 128, 1, choose_splits(tiles, d.K // kb, sms))


def workspace_bytes(d, m, sms, sms_uncapped=None, override=AUTO):
    """bb_workspace_bytes(d, m): the slab's slots (at the capped count), the split-K partials past the slots of the full device,
    0 for every other family"""
    sms_uncapped = sms if sms_uncapped is None else sms_uncapped
    m = np.asarray(m, dtype=np.int64)
    k = select(d, m, override)
    sp = ts_splits(d, m, sms)
    ts = np.where(sp > 1, slab_slot_bytes(sms_uncapped) + sp * m * d.N * 4, 0)
    return np.where(_in(k, (GEMM_TS, GEMM_TS_I8)), ts, np.where(k == GEMV_SLAB, slab_slot_bytes(sms), 0)).astype(np.int64)


# ---- descriptors ---------------------------------------------------------------------------------------------------------------
def desc(**kw):
    """one descriptor as a namespace of ints (defaults: f16 x uint4, fp32 accumulation, f16 out, row-major, compressed)"""
    base = dict(N=128, K=1024, a_dtype=F16, w_fmt=W_UINT, w_bits=4, accum_dtype=F32, out_dtype=F16, group_size=-1, with_scaling=0,
                with_zeros=0, zeros_mode=0, with_bias=0, w_layout=L_COMP, w_tile=T_ROW, r0=0, r1=0)
    base.update(kw)
    return SimpleNamespace(**{k: np.int64(v) for k, v in base.items()})


def from_struct(c):
    """the namespace of a ctypes bb_matmul_desc (bitblas_b200._lib.MatmulDesc)"""
    vals = {f: np.int64(getattr(c, f)) for f in FIELDS[:-2]}
    return SimpleNamespace(**vals, r0=np.int64(c.reserved[0]), r1=np.int64(c.reserved[1]))


def grid_view(rec):
    """the namespace of a numpy record array with FIELDS (int32): int64 columns, for the vectorised clauses"""
    return SimpleNamespace(**{f: rec[f].astype(np.int64) for f in FIELDS})


def record_dtype():
    return np.dtype([(f, np.int32) for f in FIELDS])
