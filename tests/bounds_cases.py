"""Guarded device buffers and the case list of the memory-bounds tests (test_gpu_bounds.py).  Importable without a GPU.

A value test compares the elements a kernel was asked to write.  A store one row past C, a 128-bit vector store over an N tail,
a split-K partial past the workspace or a quantizer writing one scale too many lands in whatever the allocator placed next, and
no value test looks there.  So every operand of a bounds test is one `Guarded` allocation, [front guard | payload | back guard]:

  * each guard is at least MIN_GUARD bytes and at least one 128-row tile of the operand's rows, so a kernel with a missing row
    predicate still stays inside the allocation;
  * input guards (and input payload padding) hold a value that changes any stored result it reaches: NaN for floating-point
    operands, 0x7F (NaN) for e4m3, 127 for int8 activations, 0xFF for packed weights and quantized zeros, INT32_MAX / -2 for
    int32 offsets, ids, perm and row indices;
  * output payloads and guards hold a signalling-NaN pattern (or a byte pattern for integer outputs) that no kernel stores, so a
    store to an element the contract leaves unwritten shows even when it writes a plausible value.

After each call: (a) every guard byte is unchanged, (b) every input buffer is byte-identical to its snapshot, (c) output elements
the contract leaves unwritten keep their fill, (d) the written elements equal the reference.

The case list below names, per entry point, the kernel family (forced with bb_set_kernel_override), the shape, the types and the
SM-count cap.  test_bounds_cases.py checks on the CPU that it reaches every instance the host-side mirrors can select and every
row-count edge, that every export writing device memory has cases or a reason in EXCLUDED, and that every case is needed.
"""
import struct

import torch

import dispatch_table as D
import exact_inputs as X
from test_gpu_kernel_grid import grouped_nt, mma_nt, ts_bm

MIN_GUARD = 64 * 1024
FULL_SMS = 132     # H100 SXM; the mirrors' instance sets are computed at this count


def fp8_bm(rows_per_tile):
    """launch_fp8_bm / launch_grouped_fp8_bm / launch_grouped_gemm_bm: activation rows per tile"""
    return 32 if rows_per_tile <= 32 else (64 if rows_per_tile <= 64 else 128)


def grouped_bm(counts):
    """launch_grouped_gemm_bm and launch_grouped_fp8_bm: BM from the mean rows per active group"""
    T = sum(counts)
    return fp8_bm(-(-T // min(len(counts), T)))


# ---- fills ------------------------------------------------------------------------------------------------------------------------
def _le(fmt, *v):
    return struct.pack("<" + fmt, *v)


FILL = {   # inputs: guards and padding
    "float16": _le("H", 0x7E00), "bfloat16": _le("H", 0x7FC0), "float32": _le("I", 0x7FC00000),
    "e4m3": b"\x7f", "int8": b"\x7f", "packed": b"\xff", "int32": _le("ii", 0x7FFFFFFF, -2),
}
OUT_FILL = {   # outputs: payload and guards; signalling NaNs (kernels store quiet NaNs), byte patterns for integer outputs
    "float16": _le("H", 0x7C01), "bfloat16": _le("H", 0x7F81), "float32": _le("I", 0x7F800001),
    "e4m3": b"\x7f", "int8": b"\x5a", "int32": _le("I", 0x5AA5A55A), "packed": b"\x5a", "bytes": b"\xa5",
}


def _round_up(x, a):
    return -(-x // a) * a


def guard_for(row_bytes=0):
    """guard bytes for an operand whose rows are `row_bytes` long: one 128-row tile, at least MIN_GUARD, a multiple of 256"""
    return _round_up(max(MIN_GUARD, 128 * int(row_bytes)), 256)


class Guarded:
    """one device allocation [front guard | payload | back guard]; the payload starts `offset` bytes past a 256-byte boundary"""

    def __init__(self, payload_bytes, offset=0, guard=MIN_GUARD, fill=b"\xff", device="cuda"):
        assert 0 <= offset < 256 and guard % 256 == 0 and guard >= MIN_GUARD
        self.start = guard + offset
        self.nbytes = int(payload_bytes)
        total = _round_up(self.start + self.nbytes + guard, 256)
        pat = torch.tensor(list(fill), dtype=torch.uint8)
        self.buf = pat.repeat(-(-total // pat.numel()))[:total].to(device)
        self.snap = None

    @classmethod
    def input(cls, t, kind, offset=0, guard=MIN_GUARD):
        """a copy of the tensor `t` (any dtype) as payload, `kind` a key of FILL for the guards"""
        t = t.contiguous()
        g = cls(t.numel() * t.element_size(), offset, guard, FILL[kind], t.device if t.is_cuda else "cuda")
        g.payload().copy_(t.reshape(-1).view(torch.uint8).to(g.buf.device))
        return g

    @classmethod
    def output(cls, shape, dtype, kind, offset=0, guard=MIN_GUARD, device="cuda"):
        n = 1
        for s in shape:
            n *= s
        g = cls(n * torch.empty((), dtype=dtype).element_size(), offset, guard, OUT_FILL[kind], device)
        g.shape, g.dtype = tuple(shape), dtype
        return g

    def payload(self):
        return self.buf[self.start:self.start + self.nbytes]

    def view(self, dtype=None, shape=None):
        dtype = dtype or self.dtype
        shape = shape or self.shape
        return self.payload().view(dtype).view(shape)

    @property
    def ptr(self):
        return self.buf.data_ptr() + self.start

    def seal(self):
        self.snap = self.buf.cpu().clone()
        return self

    def check_guards(self, what):
        now = self.buf.cpu()
        for name, sl in (("front", slice(0, self.start)), ("back", slice(self.start + self.nbytes, None))):
            bad = (now[sl] != self.snap[sl]).nonzero()
            if bad.numel():
                first = int(bad[0]) + (0 if name == "front" else self.start + self.nbytes)
                rel = first - self.start if name == "front" else first - self.start - self.nbytes
                raise AssertionError(f"{what}: {bad.numel()} bytes of the {name} guard changed; first at payload "
                                     f"{'start' if name == 'front' else 'end'} {rel:+d}: {int(now[first]):#04x}")

    def check_unchanged(self, what):
        self.check_guards(what)
        now = self.buf.cpu()
        if not torch.equal(now, self.snap):
            bad = (now != self.snap).nonzero()
            raise AssertionError(f"{what}: an input was written: {bad.numel()} payload bytes changed, first at byte "
                                 f"{int(bad[0]) - self.start}")

    def check_kept(self, keep, what):
        """the elements of the [shape] output where `keep` (bool, same shape) is set still hold the fill"""
        now = self.buf.cpu()[self.start:self.start + self.nbytes].view(self.dtype).view(self.shape)
        was = self.snap[self.start:self.start + self.nbytes].view(self.dtype).view(self.shape)
        width = torch.empty((), dtype=self.dtype).element_size()
        iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[width]
        bad = keep & (now.view(iv) != was.view(iv))
        if bad.any():
            idx = bad.nonzero()[:4].tolist()
            raise AssertionError(f"{what}: {int(bad.sum())} elements the contract leaves unwritten were written; first at {idx}")


# ---- exports that write device memory, and those that do not -------------------------------------------------------------------
EXCLUDED = {
    "bb_peer_barrier": "writes peer-mapped flag blocks of other GPUs: multi-GPU, kept by test_gpu_multi.py",
    "bb_debug_decode": "test hook, its every output element compared by test_gpu_decode_kat.py",
    "bb_debug_dequant": "test hook, its every output element compared by test_gpu_decode_kat.py",
    "bb_init": "host-only: per-device setup, no caller buffer",
    "bb_select_kernel": "host-only", "bb_select_kernel_w4a8": "host-only", "bb_select_kernel_fp8": "host-only",
    "bb_workspace_bytes": "host-only", "bb_workspace_bytes_fp8": "host-only", "bb_kernel_name": "host-only",
    "bb_set_kernel_override": "host-only", "bb_set_sm_count_cap": "host-only", "bb_launch_count": "host-only",
    "bb_last_error": "host-only", "bb_version": "host-only",
    "bb_compress_host": "host-only: host memory in and out", "bb_interleave_host": "host-only: host memory in and out",
}

M_EDGES = (1, 7, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 300)
OUTS = ("float16", "bfloat16", "float32")
MODES = ("none", "scale", "original", "rescale", "quantized")
SPLIT_CAP = 66    # split-K factors 2 .. 8 are forced at this SM count (test_gpu_sm_counts.py's way)


# ---- the plain matmuls ---------------------------------------------------------------------------------------------------------
# per family: (N, K) with a tail where the family takes one, the rows it accepts
FAMILY = {
    "generic_simt": dict(kid=D.GENERIC, N=136, K=384, ms=M_EDGES),          # any N: 136 is no multiple of 16
    "gemv_mma": dict(kid=D.GEMV_MMA, N=144, K=384, ms=[m for m in M_EDGES if m <= 32]),   # N % 128 = 16, three 128-k steps
    "gemv_i8": dict(kid=D.GEMV_I8, N=144, K=384, ms=[m for m in M_EDGES if m <= 32]),
    "gemm_ts_wgmma": dict(kid=D.GEMM_TS, N=256, K=576, ms=M_EDGES, g=192),  # nine 64-k blocks, no split at 132 SMs
    "gemm_ts_wgmma_i8": dict(kid=D.GEMM_TS_I8, N=256, K=640, ms=M_EDGES),   # five 128-k blocks
    "gemv_slab": dict(kid=D.GEMV_SLAB, N=1040, K=2048, ms=(1,)),            # N % 32 = 16: a half row block
}
I8_FAMILIES = ("gemv_i8", "gemm_ts_wgmma_i8")


def split_shape(f, m, int8):
    """(N, K) that the wgmma GEMM splits exactly f ways at m rows on SPLIT_CAP SMs: 8 k-blocks per split, one m-tile column"""
    kb = 128 if int8 else 64
    N, K = 128, 8 * f * kb
    d = D.desc(N=N, K=K, a_dtype=D.I8 if int8 else D.F16, accum_dtype=D.I32 if int8 else D.F32)
    assert int(D.ts_splits(d, m, SPLIT_CAP)) == f
    return N, K


def _slab_cap(N, K, prop):
    return next(c for c in range(2, FULL_SMS + 1) if prop in X.slab_coverage(N, K, c))


def _matmul_cases():
    cases = []
    i = 0
    for fam, f in FAMILY.items():
        for m in f["ms"]:
            i += 1
            int8 = fam in I8_FAMILIES or (fam == "generic_simt" and m % 3 == 0)
            if int8:
                out = ("int32", "int8", "float16", "float32")[i % 4]
                W, mode = ("int4", "uint2", "uint4")[i % 3], "none"
            else:
                out, mode = OUTS[i % 3], MODES[i % 5]
                W = ("int4" if mode in ("none", "scale") and i % 2 else "uint4") if fam == "gemv_slab" or i % 4 else "uint2"
            A = "int8" if int8 else ("float16", "bfloat16")[i % 2]
            cases.append(dict(entry="bb_matmul", family=fam, m=m, N=f["N"], K=f["K"], A=A,
                              W=W, out=out, mode=mode, g=(f.get("g", 128), -1)[i % 2] if mode != "none" else -1, bias=i % 2 == 0,
                              il=fam in I8_FAMILIES or i % 3 != 0, tiled=False, cap=None))
    for int8, fam in ((False, "gemm_ts_wgmma"), (True, "gemm_ts_wgmma_i8")):
        for f in range(2, 9):
            m = (1, 17, 40, 100, 128)[f % 5]
            N, K = split_shape(f, m, int8)
            cases.append(dict(entry="bb_matmul", family=fam, m=m, N=N, K=K, A="int8" if int8 else "bfloat16", W="uint4",
                              out=("int32" if int8 else "float16", "float32", "bfloat16" if not int8 else "int8")[f % 3],
                              mode="none" if int8 else MODES[f % 5], g=-1 if int8 or f % 5 == 0 else 512, bias=f % 2 == 1,
                              il=True, tiled=False, cap=SPLIT_CAP, split=f))
    # the slab decode GEMV at SM counts where a stream-K range ends inside a row block, and slab-tiled weights
    for N, K, prop in ((1040, 3072, "range_inside_block"), (1040, 5120, "owner_stops_mid_block")):
        cases.append(dict(entry="bb_matmul", family="gemv_slab", m=1, N=N, K=K, A="bfloat16", W="uint4", out="float32",
                          mode="quantized",
                          g=128, bias=True, il=True, tiled=False, cap=_slab_cap(N, K, prop), prop=prop))
    for fam, m in (("gemv_slab", 1), ("gemm_ts_wgmma", 129)):
        cases.append(dict(entry="bb_matmul", family=fam, m=m, N=1024, K=2048, A="float16", W="uint4", out="bfloat16", mode="original",
                          g=256, bias=True, il=True, tiled=True, cap=None))
    return cases


def matmul_labels(c):
    fam, m = c["family"], c["m"]
    out = {f"{fam} m={m}" + (" tiled" if c["tiled"] else "") + (f" split{c['split']}" if c.get("split") else "")
           + (f" {c['prop']}" if c.get("prop") else "")}
    if fam in ("gemv_mma", "gemv_i8"):
        out.add(f"{fam} nt{mma_nt(m)}")
    if fam.startswith("gemm_ts"):
        out.add(f"{fam} bm{ts_bm(m)}")
        out.add(f"{fam} split{c.get('split', 1)}")
    if c.get("prop"):
        out.add(f"gemv_slab {c['prop']}")
    out |= {f"out:{c['out']}", "bias" if c["bias"] else "no bias", "slab-tiled W" if c["tiled"] else "row-major W"}
    return out


def matmul_required():
    req = {f"{fam} m={m}" for fam, f in FAMILY.items() for m in f["ms"]}
    req |= {f"{fam} nt{nt}" for fam in ("gemv_mma", "gemv_i8") for nt in (1, 2, 4)}
    req |= {f"{fam} bm{bm}" for fam in ("gemm_ts_wgmma", "gemm_ts_wgmma_i8") for bm in (32, 64, 128)}
    req |= {f"{fam} split{s}" for fam in ("gemm_ts_wgmma", "gemm_ts_wgmma_i8") for s in range(1, 9)}
    split_ms = (1, 17, 40, 100, 128)   # the row count of split factor s is split_ms[s % 5]
    req |= {f"{fam} m={split_ms[s % 5]} split{s}" for fam in ("gemm_ts_wgmma", "gemm_ts_wgmma_i8") for s in range(2, 9)}
    req |= {"gemv_slab range_inside_block", "gemv_slab owner_stops_mid_block", "gemv_slab m=1 tiled", "gemm_ts_wgmma m=129 tiled"}
    req |= {f"out:{o}" for o in OUTS + ("int32", "int8")} | {"bias", "no bias", "slab-tiled W", "row-major W"}
    return req


MATMUL = _matmul_cases()

# ---- the other matmul entry points ----------------------------------------------------------------------------------------------
# (family, m): N = 16 for the SwiGLU forms where the family takes it (the smallest I = 8), N = 128 on the wgmma GEMM
SWIGLU = [dict(entry="bb_matmul_swiglu", family=fam, m=m, N=N, K=K, A=("float16", "bfloat16")[i % 2],
               W=("uint4", "uint2")[i % 2] if fam != "gemv_slab" else "uint4",
               out=OUTS[i % 3], mode=MODES[(i + 2) % 5], g=192 if K == 576 else 128, bias=i % 2 == 1, cap=cap, split=split)
          for i, (fam, m, N, K, cap, split) in enumerate([
              ("generic_simt", 1, 16, 256, None, 1), ("generic_simt", 129, 16, 256, None, 1),
              ("gemv_mma", 7, 16, 384, None, 1), ("gemv_mma", 9, 16, 384, None, 1), ("gemv_mma", 17, 16, 384, None, 1),
              ("gemm_ts_wgmma", 1, 128, 576, None, 1), ("gemm_ts_wgmma", 33, 128, 576, None, 1),
              ("gemm_ts_wgmma", 65, 128, 576, None, 1), ("gemm_ts_wgmma", 300, 128, 576, None, 1),
              ("gemm_ts_wgmma", 17, 128, 2048, SPLIT_CAP, 4), ("gemv_slab", 1, 48, 1024, None, 1)])]

SCALED = [dict(entry="bb_matmul_scaled", family=fam, m=m, N=N, K=K, W=W, out=OUTS[i % 3], bias=i % 2 == 0, cap=cap, split=split)
          for i, (fam, m, N, K, W, cap, split) in enumerate([
              ("generic_simt", 9, 136, 256, "int2", None, 1), ("gemv_i8", 1, 144, 384, "int2", None, 1),
              ("gemv_i8", 16, 144, 384, "uint4", None, 1), ("gemv_i8", 32, 144, 384, "int4", None, 1),
              ("gemm_ts_wgmma_i8", 32, 256, 640, "int2", None, 1), ("gemm_ts_wgmma_i8", 64, 256, 640, "uint2", None, 1),
              ("gemm_ts_wgmma_i8", 129, 256, 640, "int4", None, 1), ("gemm_ts_wgmma_i8", 17, 128, 3072, "int2", SPLIT_CAP, 3)])]

W4A8 = [dict(entry="bb_matmul_w4a8", family=fam, m=m, N=N, K=K, W=W, g=g, zeros=W == "uint4", out=OUTS[i % 3], bias=i % 2 == 1,
             cap=cap, split=split)
        for i, (fam, m, N, K, W, g, cap, split) in enumerate([
            ("generic_simt", 7, 144, 384, "uint4", 128, None, 1), ("gemv_i8", 8, 144, 384, "int4", 128, None, 1),
            ("gemv_i8", 9, 144, 384, "uint4", -1, None, 1), ("gemv_i8", 25, 144, 384, "uint4", 128, None, 1),
            ("gemm_ts_wgmma_i8", 33, 256, 640, "int4", 128, None, 1), ("gemm_ts_wgmma_i8", 64, 256, 640, "uint4", 128, None, 1),
            ("gemm_ts_wgmma_i8", 300, 256, 640, "uint4", -1, None, 1), ("gemm_ts_wgmma_i8", 1, 128, 2048, "uint4", 128, SPLIT_CAP, 2)])]

FP8 = [dict(entry="bb_matmul_fp8", m=m, N=N, K=K, out=OUTS[i % 3], bias=i % 2 == 0, pad=(i % 3) * 4, cap=cap, split=split)
       for i, (m, N, K, cap, split) in enumerate([
           (1, 144, 128, None, 1), (32, 1040, 384, None, 1), (33, 144, 1152, None, 1), (64, 272, 128, None, 1), (65, 16, 384, None, 1),
           (129, 144, 256, None, 1), (300, 1040, 128, None, 1), (1, 576, 2048, None, 2), (20, 144, 3072, SPLIT_CAP, 3)])]


def _gemm_labels(c):
    fam = c.get("family", "gemm_fp8")
    out = {f"{fam} m={c['m']}" + (f" split{c['split']}" if c["split"] > 1 else "")}
    if c["split"] > 1:
        out = {f"{fam} m={c['m']} split{c['split']}"}
    if fam in ("gemv_mma", "gemv_i8"):
        out.add(f"{fam} nt{mma_nt(c['m'])}")
    elif fam.startswith("gemm_ts"):
        out.add(f"{fam} bm{ts_bm(c['m'])}")
    elif fam == "gemm_fp8":
        out.add(f"bm{fp8_bm(c['m'])}")
    if c["split"] > 1:
        out.add(f"{fam} split")
    return out


# ---- quantizers ----------------------------------------------------------------------------------------------------------------
QUANT_INT8 = [dict(entry="bb_quantize_act_int8", rows=r, K=K, A=("float16", "bfloat16")[i % 2])
              for i, (r, K) in enumerate([(1, 8), (7, 136), (129, 1000), (300, 2560)])]
QUANT_FP8 = [dict(entry="bb_quantize_act_fp8", rows=r, K=K, A=("float16", "bfloat16")[i % 2], ld=ld)
             for i, (r, K, ld) in enumerate([(1, 128, 4), (7, 384, 12), (129, 1152, 136), (300, 256, 300)])]

# ---- grouped calls -------------------------------------------------------------------------------------------------------------
# counts: an empty expert, a first expert of a count that is not = 0 mod 4 (the next expert starts off a 4-row boundary), E = 1
# and E = 256; `bucket` the instance the host picks (grouped_nt for the GEMV, grouped_bm for the GEMMs)
E256 = [(7 * e) % 6 if e % 9 else 0 for e in range(255)] + [3]
GROUPED_ROUTINGS = {
    "bb_matmul_grouped": {"nt1": [3, 0, 11, 5, 1], "nt2": [13, 0, 21, 9, 20], "nt4": [41, 0, 17, 33, 30], "e1": [9], "e256": E256},
    "bb_matmul_grouped_gemm": {"bm32": [3, 0, 40, 20, 17], "bm64": [70, 0, 50, 33, 90], "bm128": [201, 0, 130, 77, 300],
                               "e1": [129], "e256": E256},
}
GROUPED_ROUTINGS["bb_matmul_grouped_swiglu"] = GROUPED_ROUTINGS["bb_matmul_grouped"]
GROUPED_ROUTINGS["bb_matmul_grouped_gemm_swiglu"] = GROUPED_ROUTINGS["bb_matmul_grouped_gemm"]
GROUPED_ROUTINGS["bb_matmul_grouped_gemm_swiglu_gather"] = GROUPED_ROUTINGS["bb_matmul_grouped_gemm"]
GROUPED_ROUTINGS["bb_matmul_grouped_fp8"] = GROUPED_ROUTINGS["bb_matmul_grouped_gemm"]
GROUPED_ROUTINGS["bb_matmul_grouped_fp8_swiglu"] = GROUPED_ROUTINGS["bb_matmul_grouped_gemm"]


def grouped_bucket(entry, counts):
    return f"nt{grouped_nt(counts)}" if entry in ("bb_matmul_grouped", "bb_matmul_grouped_swiglu") else f"bm{grouped_bm(counts)}"


GROUPED = [dict(entry=entry, name=name, counts=counts, unclaimed=3, i=i)
           for entry, routings in GROUPED_ROUTINGS.items() for i, (name, counts) in enumerate(routings.items())]


def _grouped_labels(c):
    out = {f"{c['entry']} routing {c['name']}", f"{c['entry']} {grouped_bucket(c['entry'], c['counts'])}"}
    counts = c["counts"]
    if 0 in counts:
        out.add(f"{c['entry']} empty expert")
    if counts[0] % 4:
        out.add(f"{c['entry']} expert off a 4-row boundary")
    return out


def _grouped_required(entry):
    buckets = ("nt1", "nt2", "nt4") if entry in ("bb_matmul_grouped", "bb_matmul_grouped_swiglu") else ("bm32", "bm64", "bm128")
    return ({f"{entry} {b}" for b in buckets} | {f"{entry} routing {n}" for n in buckets + ("e1", "e256")}
            | {f"{entry} empty expert", f"{entry} expert off a 4-row boundary"})


# ---- routing, combine, top-k, permute, scatter -------------------------------------------------------------------------------------
ROUTE = [dict(entry=e, T=T, k=k, E=E, K=64, drop=drop) for e in ("bb_moe_route", "bb_moe_route_index")
         for T, k, E, drop in ((1, 1, 1, False), (37, 2, 8, True), (300, 8, 256, True))]
COMBINE = [dict(entry="bb_moe_combine", T=T, k=k, N=N, out=out) for T, k, N, out in
           ((1, 1, 8, "float16"), (37, 2, 72, "bfloat16"), (129, 6, 1024, "float32"))]
TOPK = [dict(entry="bb_moe_topk", T=T, E=E, k=k, logits=lg, scoring=sc, groups=gr) for T, E, k, lg, sc, gr in
        ((0, 8, 2, "float32", 0, 1), (7, 64, 32, "float16", 0, 1), (33, 256, 8, "bfloat16", 1, 8), (129, 32, 1, "float32", 1, 1))]
PERMUTE = [dict(entry="bb_permute_cols", rows=r, K=K, A=a, counts=c) for r, K, a, c in
           ((1, 8, "float16", None), (129, 136, "bfloat16", None), (40, 264, "float16", [5, 0, 13, 9]),
            (300, 128, "bfloat16", [1] * 256))]
SCATTER = [dict(entry="bb_matmul_scatter", family=fam, m=m, N=N, K=K, peers=p) for fam, m, N, K, p in
           (("gemv_slab", 1, 256, 1024, 1), ("gemv_mma", 9, 144, 384, 2), ("gemm_ts_wgmma", 65, 256, 1024, 2),
            ("gemm_ts_wgmma", 300, 384, 1024, 1), ("gemv_i8", 17, 144, 384, 1))]

# ---- device prep kernels ---------------------------------------------------------------------------------------------------------
PREP = ([dict(entry="bb_transform_weight_device", rows=r, cols=c, bits=b, target=t) for r, c, b, t in
         ((1, 32, 4, 0), (37, 256, 2, 16), (129, 384, 4, 16), (16, 128, 4, 8), (33, 1024, 1, 16), (7, 64, 2, 8))]
        + [dict(entry="bb_repack_gptq_qweight_device", K=K, N=N, bits=b, target=t) for K, N, b, t in
           ((128, 40, 4, 16), (256, 72, 2, 0), (384, 8, 4, 8))]
        + [dict(entry="bb_repack_gptq_qzeros_device", groups=gr, N=N, bits=b, mode=mo, A=a, v2=v2) for gr, N, b, mo, a, v2 in
           ((3, 40, 4, 0, "float16", 0), (1, 80, 2, 1, "bfloat16", 1), (5, 64, 4, 2, "float16", 0), (2, 16, 2, 2, "bfloat16", 1))]
        + [dict(entry="bb_retile_weight_device", rows=r, row_bytes=rb, inverse=inv) for r, rb, inv in ((32, 512, 0), (96, 1536, 1))])

# ---- Python layers that take output= ----------------------------------------------------------------------------------------------
LAYERS = [dict(entry="python", layer=n) for n in ("Matmul.forward", "Matmul.forward_swiglu", "Matmul.forward_grouped",
                                                   "Matmul.forward_grouped_swiglu", "moe_combine")]


# ---- the whole list ------------------------------------------------------------------------------------------------------------
CASES = (MATMUL + SWIGLU + SCALED + W4A8 + FP8 + QUANT_INT8 + QUANT_FP8 + GROUPED + ROUTE + COMBINE + TOPK + PERMUTE + SCATTER + PREP
         + LAYERS)


def labels(c):
    """the instances and edges case `c` reaches, each prefixed with its entry point"""
    e = c["entry"]
    if e == "bb_matmul":
        raw = matmul_labels(c)
    elif e in ("bb_matmul_swiglu", "bb_matmul_scaled", "bb_matmul_w4a8", "bb_matmul_fp8"):
        raw = _gemm_labels(c)
    elif e in GROUPED_ROUTINGS:
        return _grouped_labels(c)
    elif e in ("bb_quantize_act_int8", "bb_quantize_act_fp8", "bb_permute_cols"):
        raw = {f"rows={c['rows']}"} | ({"scale_ld > rows"} if c.get("ld", 0) > c["rows"] else set()) | (
            {"grouped" if c.get("counts") else "dense"} if e == "bb_permute_cols" else set())
    elif e in ("bb_moe_route", "bb_moe_route_index"):
        raw = {f"T={c['T']} k={c['k']} E={c['E']}"} | ({"dropped ids"} if c["drop"] else set())
    elif e == "bb_moe_combine":
        raw = {f"T={c['T']}", f"out:{c['out']}"}
    elif e == "bb_moe_topk":
        raw = {f"T={c['T']}", f"k={c['k']}", f"logits:{c['logits']}"}
    elif e == "bb_matmul_scatter":
        raw = {f"{c['family']} m={c['m']}"}
    elif e == "python":
        raw = {c["layer"]}
    elif e in ("bb_transform_weight_device", "bb_repack_gptq_qweight_device"):
        raw = {f"bits={c['bits']} target={c['target']}"}
    elif e == "bb_repack_gptq_qzeros_device":
        raw = {f"mode={c['mode']} v2={c['v2']}"}
    else:
        raw = {f"inverse={c['inverse']}"}
    return {f"{e}: {r}" for r in raw}


REQUIRED_M = {   # the row counts each GEMM entry point runs at, per family ("" split factor 1)
    "bb_matmul_swiglu": {"generic_simt": (1, 129), "gemv_mma": (7, 9, 17), "gemm_ts_wgmma": (1, 33, 65, 300, "17 split4"),
                         "gemv_slab": (1,)},
    "bb_matmul_scaled": {"generic_simt": (9,), "gemv_i8": (1, 16, 32), "gemm_ts_wgmma_i8": (32, 64, 129, "17 split3")},
    "bb_matmul_w4a8": {"generic_simt": (7,), "gemv_i8": (8, 9, 25), "gemm_ts_wgmma_i8": (33, 64, 300, "1 split2")},
    "bb_matmul_fp8": {"gemm_fp8": (1, 32, 33, 64, 65, 129, 300, "1 split2", "20 split3")},
}


def required():
    """the labels the list must reach: every instance the mirrors can select at FULL_SMS SMs, and the edges named in the docstrings"""
    req = {f"bb_matmul: {r}" for r in matmul_required()}
    for e, fams in REQUIRED_M.items():
        for fam, ms in fams.items():
            req |= {f"{e}: {fam} m={m}" for m in ms}
            if fam in ("gemv_mma", "gemv_i8"):
                req |= {f"{e}: {fam} nt{nt}" for nt in (1, 2, 4)}
            if fam.startswith("gemm_ts"):
                req |= {f"{e}: {fam} bm{bm}" for bm in (32, 64, 128)} | {f"{e}: {fam} split"}
            if fam == "gemm_fp8":
                req |= {f"{e}: bm{bm}" for bm in (32, 64, 128)} | {f"{e}: gemm_fp8 split"}
    for e in GROUPED_ROUTINGS:
        req |= _grouped_required(e)
    req |= {f"bb_quantize_act_int8: rows={r}" for r in (1, 7, 129, 300)}
    req |= {f"bb_quantize_act_fp8: rows={r}" for r in (1, 7, 129, 300)} | {"bb_quantize_act_fp8: scale_ld > rows"}
    req |= {f"bb_permute_cols: rows={r}" for r in (1, 129, 40, 300)} | {"bb_permute_cols: dense", "bb_permute_cols: grouped"}
    for e in ("bb_moe_route", "bb_moe_route_index"):
        req |= {f"{e}: T={t} k={k} E={x}" for t, k, x in ((1, 1, 1), (37, 2, 8), (300, 8, 256))} | {f"{e}: dropped ids"}
    req |= {f"bb_moe_combine: T={t}" for t in (1, 37, 129)} | {f"bb_moe_combine: out:{o}" for o in OUTS}
    req |= {f"bb_moe_topk: T={t}" for t in (0, 7, 33, 129)} | {"bb_moe_topk: k=32"} | {f"bb_moe_topk: logits:{o}" for o in OUTS}
    req |= {f"bb_matmul_scatter: {f}" for f in ("gemv_slab m=1", "gemv_mma m=9", "gemm_ts_wgmma m=65", "gemm_ts_wgmma m=300",
                                                 "gemv_i8 m=17")}
    req |= {f"python: {n}" for n in ("Matmul.forward", "Matmul.forward_swiglu", "Matmul.forward_grouped",
                                       "Matmul.forward_grouped_swiglu", "moe_combine")}
    req |= {f"bb_transform_weight_device: bits={b} target={t}" for b, t in ((4, 0), (2, 16), (4, 16), (4, 8), (1, 16), (2, 8))}
    req |= {f"bb_repack_gptq_qweight_device: bits={b} target={t}" for b, t in ((4, 16), (2, 0), (4, 8))}
    req |= {f"bb_repack_gptq_qzeros_device: mode={m} v2={v}" for m, v in ((0, 0), (1, 1), (2, 0), (2, 1))}
    req |= {f"bb_retile_weight_device: inverse={i}" for i in (0, 1)}
    return req


def entries():
    """the entry points the list covers"""
    return {c["entry"] for c in CASES} - {"python"}
