"""GPU: every configuration the dispatcher accepts, at the edges of each kernel family's support, against the float64 reference.

Production calls reach bb_matmul through select() (bb_api.cu) at whatever shape a model or a tensor-parallel shard has, and land
on the first family whose support predicate holds.  The grid tests (test_gpu_kernel_grid.py) force each family at one comfortable
shape.  This file walks the boundaries instead: each case is a configuration next to one of the predicates' clauses (the
boundary classes below, BOUNDARY_CLASSES), and for each case it

  * runs Matmul.forward under auto dispatch and asserts that kernel_for(m) is the choice of the Python mirror of the dispatch
    table (dispatch_table.py);
  * runs every other family the mirror says accepts the configuration, forced with bb_set_kernel_override;
  * checks every output against float64 by the family's rule (check_float: exact / gemm_ts / generic), or bit for bit
    (int_reference for int8 activations; exact_inputs at the production shard shapes, where every family must return the
    exact result and prove_exact holds).

Rejected configurations are in the list too: misaligned A or W on a TMA or streaming family, sub-word-aligned W on generic_simt,
K % g != 0 and forward_swiglu at N % 16 != 0 must raise and launch nothing.

The case list is fixed; tests/test_dispatch_table.py checks on the CPU that it reaches every boundary class (classes_of, at 132
SMs: an H100 SXM; the split-K classes depend on the SM count).
"""
from __future__ import annotations

import zlib

import pytest
import torch

import dispatch_table as D
import exact_inputs as X
from test_gpu_bitnet import case_ref, scaled_case
from test_gpu_kernel_grid import (KERNEL_NAME, check_float, float_reference, forced, int_reference, make_case)
from test_gpu_moe import swiglu_bound

pytestmark = pytest.mark.gpu

DEV = "cuda"
W_INFO = {"uint1": (D.W_UINT, 1), "int1": (D.W_INT, 1), "uint2": (D.W_UINT, 2), "int2": (D.W_INT, 2), "uint4": (D.W_UINT, 4),
          "int4": (D.W_INT, 4), "uint8": (D.W_UINT, 8), "int8": (D.W_INT, 8), "nf4": (D.W_NF, 4), "fp4_e2m1": (D.W_FP4, 4),
          "e4m3_float8": (D.W_E4M3, 8), "e5m2_float8": (D.W_E5M2, 8)}
DT = {"float16": D.F16, "bfloat16": D.BF16, "float32": D.F32, "int8": D.I8, "int32": D.I32}
ZMODE = {"original": D.Z_ORIGINAL, "rescale": D.Z_RESCALE, "quantized": D.Z_QUANTIZED}
RULE = {D.GEMV_MMA: "exact", D.GEMV_SLAB: "exact", D.GEMM_TS: "gemm_ts", D.GENERIC: "generic"}
# a 16-entry table that is not NF4's: unsorted, asymmetric, exact in bfloat16
CUSTOM_LUT = [0.75, -1.5, 0.125, 2.0, -0.25, 1.0, -3.0, 0.5, 0.0, -0.625, 1.25, -2.0, 0.375, -0.875, 3.5, -0.0625]


def _case(**kw):
    c = dict(A="float16", W="uint4", out="float16", g=-1, mode="none", bias=False, il=None, tile=False, N=256, K=1024, m=1,
             exact=False, api="forward", unaligned=None, lut=None, reject=None)
    c.update(kw)
    if c["il"] is None:   # interleaved (fast decoding) storage for sub-byte integer weights unless a case says otherwise
        c["il"] = W_INFO[c["W"]][0] in (D.W_UINT, D.W_INT) and W_INFO[c["W"]][1] < 8
    flags = [f for f in ("bias", "tile", "exact") if c[f]] + [f"{k}={c[k]}" for k in ("api", "unaligned", "lut", "reject")
                                                            if c[k] not in (None, "forward")]
    c["id"] = "-".join([c["A"], c["W"], "il" if c["il"] else "cmp", f"N{c['N']}", f"K{c['K']}", f"m{c['m']}", f"g{c['g']}",
                        c["mode"], c["out"]] + flags)
    return c


MODES = ["none", "scale", "original", "rescale", "quantized"]


def _cases():
    L = []
    add = lambda **kw: L.append(_case(**kw))   # noqa: E731
    # ---- gemv_slab (m = 1, 4-bit) ----
    for N, mode in ((272, "quantized"), (144, "original"), (400, "scale")):                  # N % 32 = 16: the half row block
        add(N=N, K=1024, g=128, mode=mode, bias=N == 144)
    add(N=256, K=1024, g=256, mode="rescale", A="bfloat16", out="float32")                    # slow parameters: g != 128
    add(N=256, K=768, g=128, mode="scale", out="bfloat16", A="bfloat16")                      # G = 6: G % 8 != 0
    for mode in ("original", "rescale", "quantized", "scale"):                                # parameter views off 16 bytes
        add(N=256, K=1024, g=128, mode=mode, unaligned="params", bias=mode == "scale")
    for K in (1280, 1536, 768, 256):                                                          # ragged last unit; one 256-k unit
        add(N=512, K=K, g=256 if K == 1536 else -1 if K == 1280 else 128, mode="original", out="float32")
    for i, (W, g) in enumerate((("nf4", 128), ("nf4", 256), ("fp4_e2m1", 384), ("fp4_e2m1", -1), ("nf4", -1), ("fp4_e2m1", 256))):
        add(W=W, N=272 if i % 2 else 256, K=768 if g == 384 else 1024, g=g, mode="scale" if i != 4 else "none", bias=i % 2 == 1,
            A="bfloat16" if i % 3 == 0 else "float16", out=("float16", "bfloat16", "float32")[i % 3])
    add(W="nf4", N=256, K=1024, g=128, mode="scale", A="bfloat16", out="bfloat16", lut="custom", bias=True)
    add(W="nf4", N=272, K=1024, g=-1, mode="none", lut="custom")
    for i, mode in enumerate(MODES):                                                          # slab-tiled storage
        add(W="int4" if mode == "none" else "uint4", N=256, K=2048, g=128 if i % 2 else 512, mode=mode, tile=True,
            il=i % 2 == 0, bias=i == 2)
    # ---- gemv_mma ----
    for i, N in enumerate((144, 400)):                                                        # N % 128 != 0 at m = 1
        add(W="uint2", N=N, K=1024, g=128, mode="original", m=1, bias=i == 0)
        add(W="uint4", N=N, K=640, g=128, mode="quantized", m=1, A="bfloat16")
    for i, (N, m) in enumerate(((144, 9), (400, 17), (144, 32), (400, 24))):                 # N % 128 != 0 at m = 9..32, auto
        for j, mode in enumerate(MODES):
            add(W="uint4" if (i + j) % 2 else "uint2", N=N, K=768 if j % 2 else 1024, g=(128, 384, -1, 256, 128)[j] if j % 2 == 0
                else (384 if i % 2 else -1), mode=mode, m=m, bias=(i + j) % 3 == 0, out=("float16", "bfloat16", "float32")[(i + j) % 3],
                A="bfloat16" if i % 2 else "float16", il=(i + j) % 2 == 0)
    for K, m in ((640, 4), (1152, 20), (640, 32)):                                            # K = 128 * odd
        add(W="uint4", N=256, K=K, g=128, mode="rescale", m=m, out="float32")
    add(W="uint2", N=256, K=1024, g=256, mode="original", m=5)
    add(W="int4", N=144, K=768, g=384, mode="scale", m=12, A="bfloat16")
    # ---- gemv_i8 ----
    for i, out in enumerate(("int32", "int8", "float32", "float16", "bfloat16")):
        add(A="int8", W=("uint4", "int2")[i % 2], N=(144, 400)[i % 2], K=1024, m=(1, 5, 9, 20, 32)[i], out=out, bias=i % 2 == 0)
    for i, out in enumerate(("float32", "float16", "bfloat16")):
        add(A="int8", W=("uint4", "int2")[i % 2], N=(144, 400)[i % 2], K=1024, m=(1, 12, 32)[i], out=out, bias=i != 1,
            api="scaled")
    # ---- gemm_ts, 16-bit activations ----
    for i, (K, g) in enumerate(((576, 64), (960, 192), (960, 320), (320, 320))):             # K % 128 = 64
        add(W="uint4" if i % 2 else "uint2", N=256, K=K, g=g, mode=MODES[1 + i % 4], m=(16, 40, 100, 300)[i], bias=i % 2 == 0,
            A="bfloat16" if i % 2 else "float16")
    add(W="uint4", N=384, K=1536, g=128, mode="original", m=16, out="float32")                 # N = 128 * odd, split-K
    add(W="uint2", N=640, K=1536, g=192, mode="rescale", m=100, A="bfloat16", il=False)
    add(W="uint4", N=384, K=1024, g=-1, mode="quantized", m=257)
    for i, W in enumerate(("nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8")):                  # table / fp8 formats
        for j, split in enumerate((True, False)):
            g = (64, 192, -1)[(2 * i + j) % 3]
            add(W=W, N=256, K=1536 if split else 768, g=g, mode="scale" if (i + j) % 3 else "none", m=16 if split else 65,
                bias=(i + j) % 2 == 0, A="bfloat16" if i % 2 else "float16", out=("float16", "bfloat16", "float32")[(i + j) % 3])
    for i, mode in enumerate(MODES):                                                          # slab-tiled x BM x split-K
        add(W="int4" if mode == "none" else "uint4", N=256, K=2048, g=(128, 512, 256, 128, -1)[i], mode=mode, tile=True,
            m=(16, 40, 100, 300, 64)[i], il=i % 2 == 1, bias=i % 2 == 0, A="bfloat16" if i == 3 else "float16")
    add(W="uint2", N=256, K=2048, g=128, mode="original", tile=True, m=33)
    for c in ((dict(W="uint4", N=256, K=1536, g=192, mode="original", m=40)), (dict(W="nf4", N=256, K=768, g=64, mode="scale", m=16)),
              (dict(W="uint4", N=144, K=1024, g=128, mode="quantized", m=20)), (dict(W="uint4", N=272, K=1024, g=128, mode="scale", m=1)),
              (dict(W="uint2", N=48, K=256, g=32, mode="original", m=5))):
        add(api="swiglu", bias=True, **c)
    # ---- gemm_ts, int8 activations ----
    for i, W in enumerate(("uint4", "int2", "int4", "uint2")):                                # compressed, K % 256 = 128
        add(A="int8", W=W, il=False, N=256, K=3456 if i < 2 else 1152, m=(16, 40, 100, 300)[i], out=("int32", "float16")[i % 2])
    add(A="int8", W="uint4", N=256, K=2048, m=64, tile=True, out="int32", bias=True)
    add(A="int8", W="int4", N=256, K=2048, m=16, tile=True, out="int8")
    add(A="int8", W="uint4", il=False, N=256, K=3456, m=16, out="float32", api="scaled")
    add(A="int8", W="int2", N=384, K=1024, m=40, out="bfloat16", api="scaled", bias=True)
    # ---- generic_simt ----
    for i, N in enumerate((8, 24, 200)):                                                      # N % 16 != 0
        add(W=("uint4", "uint2", "int4")[i], N=N, K=256, g=(128, 64, -1)[i], mode=("original", "rescale", "scale")[i], m=(1, 9, 40)[i],
            bias=i != 1, out=("float16", "float32", "bfloat16")[i], A="bfloat16" if i == 1 else "float16")
    for i, (W, K) in enumerate((("uint1", 32), ("int1", 96), ("uint4", 96), ("uint4", 1376), ("uint1", 96))):   # K % 64 != 0
        add(W=W, N=72, K=K, g=32 if i == 2 else -1, mode="scale" if i % 2 == 0 else "none", m=(1, 3, 16, 33, 8)[i],
            bias=i % 2 == 1)
    add(W="uint4", N=112, K=256, g=32, mode="original", m=6)                                   # g = 32
    add(W="uint2", N=112, K=512, g=32, mode="rescale", m=1, A="bfloat16", il=False)
    add(W="int1", N=128, K=512, g=-1, mode="none", m=4, out="float32")                        # 1- and 8-bit integers
    add(W="uint8", N=128, K=512, g=64, mode="original", m=12, A="bfloat16")
    add(W="int8", N=72, K=256, g=-1, mode="scale", m=2, bias=True)
    add(A="int8", W="uint1", N=72, K=512, m=7, out="int32", bias=True)
    add(A="int8", W="uint8", N=128, K=512, m=40, out="float32")
    add(W="nf4", N=128, K=512, g=128, mode="original", m=3)                                   # table formats with zero points
    add(W="fp4_e2m1", N=128, K=512, g=-1, mode="rescale", m=20, A="bfloat16", out="float32")
    add(W="nf4", N=256, K=512, g=128, mode="quantized", m=1, lut="custom", out="float32")
    add(W="uint4", N=400, K=1024, g=128, mode="scale", m=40)                                  # m > 32 at N % 128 != 0
    add(W="uint2", N=144, K=768, g=-1, mode="original", m=300, out="float32")
    add(W="uint4", N=72, K=512, g=-1, mode="scale", m=5, unaligned="A2")                      # generic reads A element-wise
    add(W="uint4", N=72, K=512, g=-1, mode="none", m=5, unaligned="W4")                       # and W in aligned 32-bit words
    # ---- production shard shapes, exact inputs ----
    for N, K, ms, g, mode in ((1376, 4096, (1, 16, 33), 128, "quantized"), (4096, 1376, (1, 16), 32, "original"),
                              (2368, 4096, (1, 24, 100), 128, "scale"), (4096, 2368, (1, 64), 64, "rescale"),
                              (2752, 8192, (1, 20), 128, "original"), (8192, 2752, (1, 40), 64, "quantized"),
                              (3696, 8192, (1, 9, 40), 128, "scale"), (8192, 3696, (1, 8), -1, "none")):
        for m in ms:
            add(N=N, K=K, m=m, g=g, mode=mode, exact=True, bias=m % 2 == 0, A="bfloat16" if N == 2368 else "float16")
    add(N=19328, K=2048, m=16, g=128, mode="original", exact=True)                            # 151 wgmma tiles: wider than a wave
    add(N=3696, K=8192, m=1, g=128, mode="quantized", exact=True, unaligned="params")
    add(A="int8", W="int2", N=1376, K=4096, m=16, exact=True, out="int32")
    add(A="int8", W="int2", N=4096, K=1376, m=4, exact=True, out="int32")
    # ---- rejected ----
    add(N=256, K=1024, g=128, mode="scale", m=1, unaligned="A2", reject="align")             # slab
    add(N=256, K=1024, g=128, mode="scale", m=4, unaligned="W1", reject="align")             # gemv_mma
    add(N=256, K=1024, g=128, mode="scale", m=40, unaligned="W2", reject="align")            # gemm_ts
    add(A="int8", W="int2", N=256, K=1024, m=8, out="int32", unaligned="A2", reject="align")  # gemv_i8
    add(W="uint4", N=72, K=512, m=5, unaligned="W1", reject="align")                         # generic: 32-bit weight words
    add(W="uint2", N=72, K=512, m=40, unaligned="W2", reject="align")
    add(N=256, K=768, g=512, mode="scale", m=4, reject="K%g")
    add(N=256, K=1000, g=128, mode="scale", m=1, W="uint8", reject="K%g")
    add(N=24, K=256, mode="none", m=4, api="swiglu", reject="swiglu")
    add(N=200, K=512, g=128, mode="scale", m=1, api="swiglu", reject="swiglu")
    return L


CASES = _cases()


# ---- descriptors and boundary classes (CPU) -------------------------------------------------------------------------------------
def desc_of(c):
    """the bb_matmul_desc Matmul builds for case c, as a dispatch_table namespace"""
    fmt, bits = W_INFO[c["W"]]
    a8 = c["A"] == "int8"
    layout = (D.L_IL8 if a8 else D.L_IL16) if (bits < 8 and c["il"]) else D.L_COMP
    ws, wz = int(c["mode"] != "none"), int(c["mode"] in ZMODE)
    tile = c["tile"] and fmt in (D.W_UINT, D.W_INT) and bits in (2, 4) and c["N"] % 128 == 0 and (c["K"] * bits // 8) % 512 == 0
    return D.desc(N=c["N"], K=c["K"], a_dtype=DT[c["A"]], w_fmt=fmt, w_bits=bits, accum_dtype=D.I32 if a8 else D.F32,
                  out_dtype=DT[c["out"]], group_size=c["g"] if c["g"] > 0 else -1, with_scaling=ws, with_zeros=wz,
                  zeros_mode=ZMODE.get(c["mode"], D.Z_ORIGINAL), with_bias=int(c["bias"]), w_layout=layout,
                  w_tile=D.T_SLAB if tile else D.T_ROW)


def operator_of(c):
    import bitblas_b200 as bitblas
    cfg = bitblas.MatmulConfig(M=[1, c["m"]], N=c["N"], K=c["K"], A_dtype=c["A"], W_dtype=c["W"],
                               accum_dtype="int32" if c["A"] == "int8" else "float32", out_dtype=c["out"], layout="nt",
                               with_bias=c["bias"], group_size=c["g"], with_scaling=c["mode"] != "none",
                               with_zeros=c["mode"] in ZMODE, zeros_mode=c["mode"] if c["mode"] in ZMODE else "original",
                               fast_decoding=c["il"], propagate_b=c["tile"])
    return bitblas.Matmul(cfg, enable_tuning=False)


def families_of(c):
    """(the auto choice, every family that accepts the case) by the mirror"""
    d, m = desc_of(c), c["m"]
    return int(D.select(d, m)), [f for f in D.FAMILIES if int(D.select(d, m, f)) == f]


BOUNDARY_CLASSES = (
    ["slab: N % 32 = 16", "slab slow params: N % 32 != 0", "slab slow params: g != 128", "slab slow params: G % 8 != 0",
     "slab slow params: unaligned scale/zeros", "slab: ragged last unit", "slab: K = 256", "slab: nf4", "slab: fp4",
     "slab: table + bias", "slab: table bf16", "slab: custom nf4 table"]
    + [f"slab: table g={g}" for g in (128, 256, 384, -1)] + [f"slab: tiled {m}" for m in MODES]
    + ["mma: N % 128 != 0 at m = 1 (2-bit)", "mma: N % 128 != 0 at m = 1 (K % 256 != 0)", "mma auto: N % 128 != 0 at m = 9..32",
       "mma: K = 128 * odd"] + [f"mma: N = {n}" for n in (144, 400, 1376, 3696)] + [f"mma: g = {g}" for g in (256, 384, -1)]
    + [f"mma: {m} at N % 128 != 0" for m in MODES]
    + ["i8: N % 128 != 0"] + [f"i8: out {o}" for o in ("int32", "int8", "float32", "float16", "bfloat16")] + ["i8: scaled"]
    + [f"ts: K % 128 = 64, g = {g}" for g in (64, 192, 320)]
    + ["ts: N = 128 * odd", "ts: N = 128 * odd, split-K", "ts: grid wider than one wave"]
    + [f"ts: {w} split-K {s}" for w in ("nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8") for s in ("on", "off")]
    + ["ts: table/fp8 + bias"] + [f"ts: table/fp8 g = {g}" for g in (64, 192, -1)]
    + [f"ts: tiled {m}" for m in MODES] + [f"ts: tiled BM {b}" for b in (32, 64, 128)] + ["ts: tiled split-K", "ts: swiglu"]
    + ["ts_i8: 4-bit compressed, K % 256 = 128, split-K", "ts_i8: 2-bit compressed, K % 256 = 128, split-K", "ts_i8: tiled int4",
       "ts_i8: scaled"]
    + [f"generic: N = {n}" for n in (8, 24, 200)]
    + ["generic: 1-bit K = 32", "generic: 1-bit K = 96", "generic: 4-bit K = 96", "generic: K = 1376", "generic: g = 32",
       "generic: 1-bit", "generic: 8-bit integer", "generic: table format with zeros", "generic: m > 32 at N % 128 != 0",
       "generic: A at a 2-byte offset"]
    + ["reject: unaligned A", "reject: unaligned W", "reject: generic W off a 32-bit word", "reject: K % g", "reject: swiglu N % 16"])


def classes_of(c, sms=132):
    """the boundary classes case c reaches, from the mirror's view of its descriptor"""
    d, m, N, K, W = desc_of(c), c["m"], c["N"], c["K"], c["W"]
    fmt, bits = W_INFO[W]
    g = c["g"] if c["g"] > 0 else K
    out = set()
    if c["reject"]:
        if c["reject"] == "align":
            auto = int(D.select(d, m))
            if auto == D.GENERIC:
                if c["unaligned"] in ("W1", "W2") and bits < 8:
                    out.add("reject: generic W off a 32-bit word")
            else:
                out.add("reject: unaligned A" if c["unaligned"].startswith("A") else "reject: unaligned W")
        elif c["reject"] == "K%g":
            if K % g:
                out.add("reject: K % g")
        elif c["reject"] == "swiglu" and N % 16:
            out.add("reject: swiglu N % 16")
        return out
    auto, fams = families_of(c)
    assert auto in fams, c["id"]
    table = fmt in (D.W_NF, D.W_FP4)
    if D.GEMV_SLAB in fams:
        G = K // g
        if N % 32 == 16:
            out.add("slab: N % 32 = 16")
        if c["mode"] != "none":
            if N % 32:
                out.add("slab slow params: N % 32 != 0")
            if g != 128:
                out.add("slab slow params: g != 128")
            if G % 8:
                out.add("slab slow params: G % 8 != 0")
            if c["unaligned"] == "params":
                out.add("slab slow params: unaligned scale/zeros")
        if K % 1024 and K > 256:
            out.add("slab: ragged last unit")
        if K == 256:
            out.add("slab: K = 256")
        if table:
            out.add("slab: nf4" if fmt == D.W_NF else "slab: fp4")
            out.add(f"slab: table g={c['g'] if c['g'] > 0 else -1}")
            if c["bias"]:
                out.add("slab: table + bias")
            if c["A"] == "bfloat16":
                out.add("slab: table bf16")
            if c["lut"] == "custom":
                out.add("slab: custom nf4 table")
        if d.w_tile == D.T_SLAB:
            out.add(f"slab: tiled {c['mode']}")
    if D.GEMV_MMA in fams:
        if N % 128 and m == 1:
            out.add("mma: N % 128 != 0 at m = 1 (2-bit)" if bits == 2 else "mma: N % 128 != 0 at m = 1 (K % 256 != 0)"
                    if K % 256 else "mma: N % 128 = 0")
        if N % 128 and 9 <= m <= 32 and auto == D.GEMV_MMA:
            out.add("mma auto: N % 128 != 0 at m = 9..32")
        if (K // 128) % 2:
            out.add("mma: K = 128 * odd")
        out.add(f"mma: N = {N}")
        out.add(f"mma: g = {c['g'] if c['g'] > 0 else -1}")
        if N % 128:
            out.add(f"mma: {c['mode']} at N % 128 != 0")
    if D.GEMV_I8 in fams:
        if N % 128:
            out.add("i8: N % 128 != 0")
        out.add(f"i8: out {c['out']}")
        if c["api"] == "scaled":
            out.add("i8: scaled")
    ts = [f for f in fams if f in (D.GEMM_TS, D.GEMM_TS_I8)]
    if ts:
        split = int(D.ts_splits(d, m, sms)) > 1
        if ts[0] == D.GEMM_TS:
            if K % 128 == 64:
                out.add(f"ts: K % 128 = 64, g = {c['g']}")
            if (N // 128) % 2:
                out.add("ts: N = 128 * odd")
                if split:
                    out.add("ts: N = 128 * odd, split-K")
            if -(-m // int(D.ts_bm(m))) * (N // 128) > sms:
                out.add("ts: grid wider than one wave")
            if table or fmt in (D.W_E4M3, D.W_E5M2):
                out.add(f"ts: {W} split-K {'on' if split else 'off'}")
                if c["bias"]:
                    out.add("ts: table/fp8 + bias")
                out.add(f"ts: table/fp8 g = {c['g'] if c['g'] > 0 else -1}")
            if d.w_tile == D.T_SLAB:
                out.add(f"ts: tiled {c['mode']}")
                out.add(f"ts: tiled BM {int(D.ts_bm(m))}")
                if split:
                    out.add("ts: tiled split-K")
            if c["api"] == "swiglu":
                out.add("ts: swiglu")
        else:
            if d.w_layout == D.L_COMP and K % 256 == 128 and split and bits in (2, 4):
                out.add(f"ts_i8: {bits}-bit compressed, K % 256 = 128, split-K")
            if d.w_tile == D.T_SLAB and bits == 4:
                out.add("ts_i8: tiled int4")
            if c["api"] == "scaled":
                out.add("ts_i8: scaled")
    if auto == D.GENERIC:
        if N % 16:
            out.add(f"generic: N = {N}")
        if bits == 1 and K in (32, 96):
            out.add(f"generic: 1-bit K = {K}")
        if bits == 4 and K == 96:
            out.add("generic: 4-bit K = 96")
        if K == 1376:
            out.add("generic: K = 1376")
        if c["g"] == 32:
            out.add("generic: g = 32")
        if bits == 1:
            out.add("generic: 1-bit")
        if bits == 8 and fmt in (D.W_UINT, D.W_INT):
            out.add("generic: 8-bit integer")
        if table and c["mode"] in ZMODE:
            out.add("generic: table format with zeros")
        if m > 32 and N % 128:
            out.add("generic: m > 32 at N % 128 != 0")
        if c["unaligned"] == "A2":
            out.add("generic: A at a 2-byte offset")
    return out


# ---- running (GPU) ---------------------------------------------------------------------------------------------------------------
def _seed(c):
    return zlib.crc32(c["id"].encode()) % 100003


def _inputs(c):
    seed = _seed(c)
    if c["api"] == "scaled":
        case = scaled_case(c["m"], c["N"], c["K"], c["W"], c["il"], c["out"], c["bias"], per_row=True, seed=seed)
    elif c["exact"]:
        A = None
        if c["K"] % 32 and c["A"] != "int8":   # (3696 = 32 * 115.5) the exact activations of the next multiple of 32, cut
            A = X.dyadic_activations(c["m"], -(-c["K"] // 32) * 32, torch.Generator().manual_seed(seed), 0.1)[:, :c["K"]]
            for r in (A.sum(1) == 0).nonzero().flatten().tolist():   # the cut can cancel a row: one more 1/2 where it had a 0
                A[r, int((A[r] == 0).nonzero()[0])] = 0.5
            A = A.to(O_DTYPE[c["A"]])
        case = X.make_exact_case(c["m"], c["N"], c["K"], A_dtype=c["A"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"],
                                 mode=c["mode"], bias=c["bias"], fast_decoding=c["il"], seed=seed, propagate_b=c["tile"], A=A)
    else:
        case = make_case(c["m"], c["N"], c["K"], A_dtype=c["A"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"],
                         mode=c["mode"], bias=c["bias"], fast_decoding=c["il"], seed=seed,
                         a_range=32 if c["out"] in ("float16", "bfloat16") else 128)
    case["propagate_b"] = c["tile"]
    if c["lut"] == "custom":
        case["lut"] = torch.tensor(CUSTOM_LUT)
    return case


def _offset_copy(t, nbytes):
    """t copied into a view that starts `nbytes` past a 16-byte boundary (contiguous, same shape and dtype)"""
    es = t.element_size()
    assert nbytes % es == 0
    flat = torch.zeros(t.numel() + 16, dtype=t.dtype, device=DEV)
    v = flat[nbytes // es:nbytes // es + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == nbytes
    return v


def _tensors(c, op, case):
    t = dict(A=case["A"].to(DEV), W=X.product_weight(op, case, DEV))
    for k in ("scale", "zeros", "bias"):
        t[k] = case[k].to(DEV) if case.get(k) is not None else None
    if c["api"] == "scaled":
        t.update(a_scale=case["a_scale"].to(DEV), w_scale=case["w_scale"].to(DEV),
                 bias=case["obias"].to(DEV) if case["obias"] is not None else None)
    u = c["unaligned"]
    if u == "params":
        for k in ("scale", "zeros"):
            if t[k] is not None:
                t[k] = _offset_copy(t[k], 2)
    elif u:
        name, nbytes = u[0], int(u[1:])
        t[name] = _offset_copy(t[name], nbytes)
    if c["lut"] == "custom":
        op.lut = case["lut"].to(O_DTYPE[c["A"]]).to(DEV)
    return t


O_DTYPE = {"float16": torch.float16, "bfloat16": torch.bfloat16}


def _call(c, op, t):
    if c["api"] == "scaled":
        return op.forward_scaled(t["A"], t["W"], t["a_scale"], t["w_scale"], t["bias"])
    kw = dict(scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    if c["api"] == "swiglu":
        return op.forward(t["A"], t["W"], **kw), op.forward_swiglu(t["A"], t["W"], **kw)
    return op.forward(t["A"], t["W"], **kw)


def _rows(c):
    """the rows checked against float64: all, or a sample of 64 at m > 64 with N > 512"""
    if c["m"] <= 64 or c["N"] <= 512:
        return None
    return torch.unique(torch.linspace(0, c["m"] - 1, 64).long())


@pytest.mark.parametrize("c", [c for c in CASES if not c["reject"]], ids=lambda c: c["id"])
def test_dispatch_edge(c):
    from bitblas_b200 import _lib
    lib = _lib.load()
    case = _inputs(c)
    op = operator_of(c)
    assert vars(D.from_struct(op._desc)) == vars(desc_of(c))
    auto, fams = families_of(c)
    assert op.kernel_for(c["m"]) == KERNEL_NAME[auto], (op.kernel_for(c["m"]), D.explain(desc_of(c), c["m"]))
    t = _tensors(c, op, case)
    if c["exact"]:
        # the bounds of the families that run the case: the fp32 sum of every family, the magic chains of the two GEMVs
        X.prove_exact(case, families=("sum",) + (("slab",) if D.GEMV_SLAB in fams else ()) + (("gemv",) if D.GEMV_MMA in fams else ()),
                      device=DEV)
        ref = X.exact_reference(case, DEV).cpu()
    refs = {}
    rows = _rows(c)
    for fam in [auto] + [f for f in fams if f != auto]:
        what = f"{c['id']} on {KERNEL_NAME[fam]}{' (auto)' if fam == auto else ''}"
        with forced(D.AUTO if fam == auto else fam):
            assert op.kernel_for(c["m"]) == KERNEL_NAME[fam]
            n0 = lib.bb_launch_count()
            res = _call(c, op, t)
            torch.cuda.synchronize()
            assert lib.bb_launch_count() > n0
        pre, got = res if c["api"] == "swiglu" else (res, None)
        pre = pre.cpu()
        if c["api"] == "scaled":
            X.compare_exact(pre, case_ref(case), what)
        elif c["exact"]:
            X.compare_exact(pre, ref, what)
        elif c["A"] == "int8":
            X.compare_exact(pre, int_reference(case), what)
        else:
            rule = RULE[fam]
            il = c["il"] and W_INFO[c["W"]][1] < 8
            key = (rule, il and rule == "generic")
            if key not in refs:
                refs[key] = float_reference(case, rule, layout_il=il, rows=rows)
            check_float(pre if rows is None else pre[rows], case, rule, what, layout_il=il, rows=rows, reference=refs[key])
        if got is not None:
            swiglu_bound(got.cpu(), pre, c["out"], c["bias"])


@pytest.mark.parametrize("c", [c for c in CASES if c["reject"]], ids=lambda c: c["id"])
def test_dispatch_edge_rejected(c):
    """the call raises and launches nothing"""
    from bitblas_b200 import _lib
    lib = _lib.load()
    case = _inputs(c) if c["reject"] != "K%g" else None
    op = operator_of(c)
    if c["reject"] == "K%g":
        assert op.kernel_for(c["m"]) == "unknown"
        g = torch.Generator().manual_seed(1)
        A = torch.rand((c["m"], c["K"]), generator=g).half().to(DEV)
        W = torch.zeros(op.retrieve_weight_shape(), dtype=torch.int8, device=DEV)
        G = max(1, c["K"] // c["g"])
        t = dict(A=A, W=W, scale=torch.ones((c["N"], G), dtype=torch.float16, device=DEV), zeros=None, bias=None)
    else:
        t = _tensors(c, op, case)
    n0 = lib.bb_launch_count()
    if c["reject"] == "align":
        with pytest.raises(RuntimeError, match=r"code 5\)"):
            _call(c, op, t)
    elif c["reject"] == "swiglu":
        with pytest.raises(ValueError, match="N % 16|I % 8"):
            op.forward_swiglu(t["A"], t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    else:
        with pytest.raises((RuntimeError, ValueError), match="divisible|group"):
            _call(c, op, t)
    torch.cuda.synchronize()
    assert lib.bb_launch_count() == n0
