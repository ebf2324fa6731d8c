"""GPU: every kernel entry point reads and writes only the memory its contract names.

Each case of bounds_cases.py runs through the C ABI with every operand in a `Guarded` allocation: guards of at least one 128-row
tile, poisoned padding (NaN, 0x7F, 0xFF, INT32_MAX / -2: a read of it reaches the stored values), output payloads pre-filled with
a pattern no kernel stores, payloads at 0 and at the least alignment the contract allows.  After each call (a) every guard is
unchanged, (b) every input is byte-identical to its snapshot, (c) output elements the contract leaves unwritten keep their fill,
(d) the written elements equal the reference: bit for bit where the contract is exact (exact_inputs, fp8_restate, the BitNet and
W4A8 restatements, route_reference), within the existing float64 bounds where it is not (SwiGLU, combine, top-k weights).
"""
import contextlib
import ctypes
import itertools

import numpy as np
import pytest
import torch

import bounds_cases as B
import exact_inputs as X
import fp8_restate as R
from bounds_cases import Guarded, guard_for
from test_gpu_kernel_grid import forced
from test_gpu_moe import route_reference, swiglu_bound

pytestmark = pytest.mark.gpu

DEV = "cuda"
TORCH = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32, "int8": torch.int8, "int32": torch.int32}
E4M3 = torch.float8_e4m3fn


def _lib():
    from bitblas_b200 import _lib as L
    return L


def _call(name, *args):
    L = _lib()
    L.ensure_init(torch.cuda.current_device())
    L.call(name, torch.cuda.current_device(), *args)


def _stream():
    return torch.cuda.current_stream().cuda_stream


@contextlib.contextmanager
def sm_cap(cap):
    if not cap:
        yield
        return
    lib = _lib().load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if cap > sms:
        pytest.skip(f"{cap} SMs is above this device's {sms}")
    prev = lib.bb_set_sm_count_cap(cap)
    assert prev >= 0, _lib().last_error()
    try:
        yield
    finally:
        lib.bb_set_sm_count_cap(prev)


class Buffers:
    """the guarded operands of one call: inputs (checked unchanged) and outputs (guards checked)"""

    def __init__(self, what):
        self.what, self.inputs, self.outputs = what, [], []

    def inp(self, t, kind, offset=0, row_bytes=0):
        if t is None:
            return None
        g = Guarded.input(t, kind, offset, guard_for(row_bytes))
        self.inputs.append(g)
        return g

    def out(self, shape, dtype, kind, offset=0, row_bytes=0):
        g = Guarded.output(shape, dtype, kind, offset, guard_for(row_bytes))
        self.outputs.append(g)
        return g

    def seal(self):
        for g in self.inputs + self.outputs:
            g.seal()

    def check(self):
        torch.cuda.synchronize()
        for g in self.inputs:
            g.check_unchanged(f"{self.what}: input")
        for g in self.outputs:
            g.check_guards(f"{self.what}: output")


def ptr(g):
    return 0 if g is None else g.ptr


def _zeros_kind(case):
    return "packed" if case["mode"] == "quantized" else case["cfg"]["A_dtype"]


def _operands(bufs, case, W, i):
    """A, W, scale, zeros, bias of an exact case as guarded inputs; payloads at 0 or 16 bytes past a 256-byte boundary"""
    off = 16 * (i % 2)
    K = case["K"]
    A = bufs.inp(case["A"], case["cfg"]["A_dtype"], off, K * case["A"].element_size())
    Wg = bufs.inp(W.view(torch.int8), "packed", off, W.shape[-1])
    s = bufs.inp(case["scale"], case["cfg"]["A_dtype"], off)
    z = bufs.inp(case["zeros"], _zeros_kind(case), off)
    b = bufs.inp(case["bias"], "int8" if case["bias"] is not None and case["bias"].dtype == torch.int8 else case["cfg"]["A_dtype"], off)
    return A, Wg, s, z, b


def _families(fam):
    return {"gemv_slab": ("sum", "slab", "gemv"), "gemv_mma": ("sum", "gemv")}.get(fam, ("sum",))


def _exact(c, i, **kw):
    return X.make_exact_case(c["m"], c["N"], c["K"], A_dtype=c["A"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"],
                             mode=c["mode"], bias=c["bias"], fast_decoding=c.get("il", True), seed=1000 + i,
                             propagate_b=c.get("tiled", False), **kw)


def _cid(c):
    return "-".join(f"{k}={v}" for k, v in c.items() if k not in ("entry", "i") and not isinstance(v, list))


# ---- bb_matmul on its six families, with its workspace ------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(B.MATMUL)), ids=[_cid(c) for c in B.MATMUL])
def test_matmul(i):
    c = B.MATMUL[i]
    kid, m = B.FAMILY[c["family"]]["kid"], c["m"]
    case = _exact(c, i)
    what = f"bb_matmul {_cid(c)}"
    with sm_cap(c["cap"]), forced(kid) as lib:
        op = X.product_operator(case)
        assert op.kernel_for(m) == c["family"], op.kernel_for(m)
        W = X.product_weight(op, case, DEV)
        ws_bytes = lib.bb_workspace_bytes(op._desc_ref, m)
        assert (ws_bytes > 0) == (c["family"] == "gemv_slab" or c.get("split", 1) > 1), ws_bytes
        bufs = Buffers(what)
        A, Wg, s, z, b = _operands(bufs, case, W, i)
        odt = TORCH[c["out"]]
        C = bufs.out((m, c["N"]), odt, c["out"], 16 * (i % 2), c["N"] * 4)
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        if ws is not None:
            ws.payload().zero_()
        bufs.seal()
        _call("bb_matmul", op._desc_ref, A.ptr, Wg.ptr, 0, ptr(s), ptr(z), ptr(b), C.ptr, m, ptr(ws), ws_bytes, _stream())
        bufs.check()
    if ws is not None and c["family"] == "gemv_slab":
        assert int(ws.payload().count_nonzero()) == 0, "the slab call left its slots dirty"
    X.prove_exact(case, _families(c["family"]), device=DEV)
    X.compare_exact(C.view().cpu(), X.exact_reference(case, DEV).cpu(), what)


# ---- the SwiGLU, scaled, W4A8 and FP8 matmuls -----------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(B.SWIGLU)), ids=[_cid(c) for c in B.SWIGLU])
def test_matmul_swiglu(i):
    c = B.SWIGLU[i]
    kid, m = B.FAMILY[c["family"]]["kid"], c["m"]
    case = _exact(c, i)
    what = f"bb_matmul_swiglu {_cid(c)}"
    with sm_cap(c["cap"]), forced(kid) as lib:
        op = X.product_operator(case)
        assert op.kernel_for(m) == c["family"]
        W = X.product_weight(op, case, DEV)
        ws_bytes = lib.bb_workspace_bytes(op._desc_ref, m)
        bufs = Buffers(what)
        A, Wg, s, z, b = _operands(bufs, case, W, i)
        C = bufs.out((m, c["N"] // 2), TORCH[c["out"]], c["out"], 16 * (i % 2))
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        if ws is not None:
            ws.payload().zero_()
        bufs.seal()
        _call("bb_matmul_swiglu", op._desc_ref, A.ptr, Wg.ptr, 0, ptr(s), ptr(z), ptr(b), C.ptr, m, ptr(ws), ws_bytes, _stream())
        bufs.check()
    X.prove_exact(case, _families(c["family"]), device=DEV)
    swiglu_bound(C.view().cpu(), X.exact_reference(case, DEV).cpu(), c["out"], c["bias"])


@pytest.mark.parametrize("i", range(len(B.SCALED)), ids=[_cid(c) for c in B.SCALED])
def test_matmul_scaled(i):
    from test_gpu_bitnet import case_ref, scaled_case
    import helpers as H
    c = B.SCALED[i]
    kid, m = B.FAMILY[c["family"]]["kid"], c["m"]
    case = scaled_case(m, c["N"], c["K"], c["W"], True, c["out"], c["bias"], i % 2 == 0, seed=2000 + i)
    what = f"bb_matmul_scaled {_cid(c)}"
    with sm_cap(c["cap"]), forced(kid) as lib:
        op = H.product_operator(case, M=[1, m])
        assert op.kernel_for(m) == c["family"]
        W = H.product_weight(op, case, DEV)
        ws_bytes = lib.bb_workspace_bytes(op._desc_ref, m)
        assert (ws_bytes > 0) == (c["split"] > 1)
        bufs = Buffers(what)
        off = 16 * (i % 2)
        A = bufs.inp(case["A"], "int8", off, c["K"])
        Wg = bufs.inp(W.view(torch.int8), "packed", off, W.shape[-1])
        sa = bufs.inp(case["a_scale"], "float32", 4 * (i % 2))
        sw = bufs.inp(case["w_scale"], "float32", 4 * (i % 2))
        b = bufs.inp(case["obias"], c["out"], off)
        C = bufs.out((m, c["N"]), TORCH[c["out"]], c["out"], off)
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        if ws is not None:
            ws.payload().zero_()
        bufs.seal()
        _call("bb_matmul_scaled", op._desc_ref, A.ptr, Wg.ptr, sa.ptr, sw.ptr, ptr(b), C.ptr, m, ptr(ws), ws_bytes, _stream())
        bufs.check()
    X.compare_exact(C.view().cpu(), case_ref(case), what)


@pytest.mark.parametrize("i", range(len(B.W4A8)), ids=[_cid(c) for c in B.W4A8])
def test_matmul_w4a8(i):
    from bitblas_b200.w4a8 import pack_zeros
    from test_gpu_w4a8 import Case
    c = B.W4A8[i]
    kid, m = B.FAMILY[c["family"]]["kid"], c["m"]
    case = Case(m, c["N"], c["K"], g=c["g"] if c["g"] > 0 else c["K"], W=c["W"], zeros=c["zeros"], out=c["out"], bias=c["bias"],
                exact=True, seed=3000 + i)
    what = f"bb_matmul_w4a8 {_cid(c)}"
    with sm_cap(c["cap"]), forced(kid) as lib:
        op = case.layer_op()
        assert op.kernel_for_w4a8(m) == c["family"]
        W = op.weight_transform(case.u.to(torch.int8)).to(DEV)
        ws_bytes = lib.bb_workspace_bytes(ctypes.byref(op._w4a8_cleared_desc()), m)
        assert (ws_bytes > 0) == (c["split"] > 1)
        bufs = Buffers(what)
        off = 16 * (i % 2)
        A = bufs.inp(case.q, "int8", off, c["K"])
        Wg = bufs.inp(W, "packed", off, W.shape[-1])
        sa = bufs.inp(case.a_scale, "float32", 4 * (i % 2))
        sc = bufs.inp(case.scales, "float32", 4 * (i % 2))
        z = bufs.inp(pack_zeros(case.z).view(torch.int8) if c["zeros"] else None, "packed", off)
        b = bufs.inp(case.bias, c["out"], off)
        C = bufs.out((m, c["N"]), TORCH[c["out"]], c["out"], off)
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        if ws is not None:
            ws.payload().zero_()
        bufs.seal()
        _call("bb_matmul_w4a8", op._desc_ref, A.ptr, Wg.ptr, sa.ptr, sc.ptr, ptr(z), ptr(b), C.ptr, m, ptr(ws), ws_bytes, _stream())
        bufs.check()
    X.compare_exact(C.view().cpu(), case.restate(), what)


def _a_scale_payload(sa, ld):
    """sa [rows, KB] in bb_quantize_act_fp8's k-block-major layout [KB, ld], the gap between blocks NaN"""
    rows, KB = sa.shape
    buf = torch.full((KB, ld), float("nan"))
    buf[:, :rows] = sa.t()
    return buf


@pytest.mark.parametrize("i", range(len(B.FP8)), ids=[_cid(c) for c in B.FP8])
def test_matmul_fp8(i):
    from test_gpu_fp8 import _op, exact_S, exact_case
    c = B.FP8[i]
    m, N, K = c["m"], c["N"], c["K"]
    qa, qw, sa, sw = exact_case(m, N, K, seed=4000 + i)
    bias = (torch.randn(N, generator=torch.Generator().manual_seed(i)) * 4).to(TORCH[c["out"]]) if c["bias"] else None
    what = f"bb_matmul_fp8 {_cid(c)}"
    ld = (m + 3) // 4 * 4 + c["pad"]
    with sm_cap(c["cap"]):
        op = _op(N, K, c["out"], c["bias"])
        desc = op._fp8_desc()
        lib = _lib().load()
        ws_bytes = lib.bb_workspace_bytes_fp8(ctypes.byref(desc), m)
        assert (ws_bytes > 0) == (c["split"] > 1)
        assert ws_bytes in (0, c["split"] * m * N * 4)
        bufs = Buffers(what)
        off = 16 * (i % 2)
        A = bufs.inp(qa.to(E4M3).view(torch.uint8), "e4m3", off, K)
        Wg = bufs.inp(qw.to(E4M3).view(torch.uint8), "e4m3", off, K)
        sa_g = bufs.inp(_a_scale_payload(sa, ld), "float32", off)
        sw_g = bufs.inp(sw, "float32", 4 * (i % 2))
        b = bufs.inp(bias, c["out"], off)
        C = bufs.out((m, N), TORCH[c["out"]], c["out"], off, N * 4)
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        bufs.seal()
        _call("bb_matmul_fp8", ctypes.byref(desc), A.ptr, sa_g.ptr, ld, Wg.ptr, sw_g.ptr, ptr(b), C.ptr, m, ptr(ws), ws_bytes,
              _stream())
        bufs.check()
    ref = R.round_out(exact_S(qa, qw, sa, sw).float(), c["out"], bias)
    X.compare_exact(C.view().cpu(), ref, what)


# ---- quantizers --------------------------------------------------------------------------------------------------------------------
def _activations(rows, K, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    mag = torch.exp2(torch.randint(-6, 7, (rows, 1), generator=g).float())
    return (torch.randn(rows, K, generator=g) * mag).to(TORCH[dtype])


@pytest.mark.parametrize("i", range(len(B.QUANT_INT8)), ids=[_cid(c) for c in B.QUANT_INT8])
def test_quantize_act_int8(i):
    from test_gpu_bitnet import quant_ref
    c = B.QUANT_INT8[i]
    rows, K = c["rows"], c["K"]
    x = _activations(rows, K, c["A"], 5000 + i)
    bufs = Buffers(f"bb_quantize_act_int8 {_cid(c)}")
    off = 16 * (i % 2)
    xg = bufs.inp(x, c["A"], off, 2 * K)
    q = bufs.out((rows, K), torch.int8, "int8", off, K)
    s = bufs.out((rows,), torch.float32, "float32", 4 * (i % 2))
    bufs.seal()
    _call("bb_quantize_act_int8", xg.ptr, _lib().dtype_id(TORCH[c["A"]]), rows, K, q.ptr, s.ptr, _stream())
    bufs.check()
    qr, sr = quant_ref(x)
    X.compare_exact(s.view().cpu(), sr, bufs.what + " scale")
    X.compare_exact(q.view().cpu(), qr, bufs.what + " q")


@pytest.mark.parametrize("i", range(len(B.QUANT_FP8)), ids=[_cid(c) for c in B.QUANT_FP8])
def test_quantize_act_fp8(i):
    from test_gpu_fp8 import quant_ref
    c = B.QUANT_FP8[i]
    rows, K, ld = c["rows"], c["K"], c["ld"]
    KB = K // 128
    x = _activations(rows, K, c["A"], 6000 + i)
    bufs = Buffers(f"bb_quantize_act_fp8 {_cid(c)}")
    off = 16 * (i % 2)
    xg = bufs.inp(x, c["A"], off, 2 * K)
    q = bufs.out((rows, K), torch.uint8, "e4m3", off, K)
    s = bufs.out((KB, ld), torch.float32, "float32", off)
    bufs.seal()
    _call("bb_quantize_act_fp8", xg.ptr, _lib().dtype_id(TORCH[c["A"]]), rows, K, q.ptr, s.ptr, ld, _stream())
    bufs.check()
    gap = torch.zeros(KB, ld, dtype=torch.bool)
    gap[:, rows:] = True
    s.check_kept(gap, bufs.what + ": the scale_ld gap")
    qr, sr = quant_ref(x.float().to(TORCH[c["A"]]))
    X.compare_exact(s.view().cpu()[:, :rows].t(), sr, bufs.what + " scale")
    X.compare_exact(q.view().cpu(), qr.view(torch.uint8), bufs.what + " q")


# ---- grouped matmuls -----------------------------------------------------------------------------------------------------------------
GROUPED_SHAPE = {   # (N, K) per entry point: N % 16 with a tail on the GEMV, N % 128 on the GEMMs; N = 2I for the SwiGLU forms
    "bb_matmul_grouped": (144, 384), "bb_matmul_grouped_swiglu": (144, 384), "bb_matmul_grouped_gemm": (256, 384),
    "bb_matmul_grouped_gemm_swiglu": (256, 384), "bb_matmul_grouped_gemm_swiglu_gather": (256, 384),
    "bb_matmul_grouped_fp8": (128, 256), "bb_matmul_grouped_fp8_swiglu": (256, 256),
}
LOWBIT_GROUPED = [c for c in B.GROUPED if "fp8" not in c["entry"]]
FP8_GROUPED = [c for c in B.GROUPED if "fp8" in c["entry"]]


def _offsets(counts):
    return torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32)


@pytest.mark.parametrize("c", LOWBIT_GROUPED, ids=lambda c: f"{c['entry']}-{c['name']}")
def test_grouped(c):
    entry, counts, i = c["entry"], c["counts"], c["i"]
    N, K = GROUPED_SHAPE[entry]
    swiglu, gather = "swiglu" in entry, "gather" in entry
    T = sum(counts)
    rows = T + c["unclaimed"]          # rows offsets[E] .. rows - 1 belong to no group
    E = len(counts)
    mode = B.MODES[(i + len(entry)) % 5]
    T_dt = ("float16", "bfloat16")[i % 2]
    W_dt = ("int4" if mode in ("none", "scale") else "uint4") if i % 2 else "uint2"
    g = (128, -1)[i % 2] if mode != "none" else -1
    gen = torch.Generator().manual_seed(7000 + i)
    a_rows = rows + 5 if gather else rows
    A = X.dyadic_activations(a_rows, K, gen, density=0.1, group=128).to(TORCH[T_dt])
    row_index = None
    if gather:   # claimed rows read random token rows; the unclaimed entries are poison (clamped by contract, never read)
        row_index = torch.full((rows,), -2, dtype=torch.int32)
        row_index[:T] = torch.randint(0, a_rows, (T,), generator=gen, dtype=torch.int32)
    A_rows = A[row_index[:T].long()] if gather else A[:T]
    E_used = min(E, 8)   # weights of experts past the eighth repeat the first eight (E = 256 stays small)
    cases = [X.make_exact_case(T, N, K, A_dtype=T_dt, W_dtype=W_dt, group_size=g, mode=mode, bias=i % 2 == 0,
                               out_dtype=B.OUTS[i % 3], fast_decoding=i % 3 != 0, seed=7100 + 13 * i + e, A=A_rows)
             for e in range(E_used)]
    op = X.product_operator(cases[0], M=[1, 16])
    Ws = [X.product_weight(op, x, DEV) for x in cases]
    st = lambda k: torch.stack([cases[e % E_used][k] for e in range(E)]) if cases[0][k] is not None else None   # noqa: E731
    W = torch.stack([Ws[e % E_used] for e in range(E)])
    off = _offsets(counts)
    what = f"{entry} {c['name']}"
    bufs = Buffers(what)
    o16 = 16 * (i % 2)
    Ag = bufs.inp(A, T_dt, o16, 2 * K)
    Wg = bufs.inp(W.view(torch.int8), "packed", o16, W.shape[-1])
    s = bufs.inp(st("scale"), T_dt, o16)
    z = bufs.inp(st("zeros"), _zeros_kind(cases[0]), o16)
    b = bufs.inp(st("bias"), T_dt, o16)
    offg = bufs.inp(off, "int32", 4 * (i % 2))
    rig = bufs.inp(row_index, "int32", 4 * (i % 2)) if gather else None
    cols = N // 2 if swiglu else N
    odt = TORCH[B.OUTS[i % 3]]
    C = bufs.out((rows, cols), odt, B.OUTS[i % 3], o16, cols * 4)
    bufs.seal()
    if gather:
        _call(entry, op._desc_ref, E, offg.ptr, rig.ptr, Ag.ptr, a_rows, Wg.ptr, ptr(s), ptr(z), ptr(b), C.ptr, rows, _stream())
    else:
        _call(entry, op._desc_ref, E, offg.ptr, Ag.ptr, Wg.ptr, ptr(s), ptr(z), ptr(b), C.ptr, rows, _stream())
    bufs.check()
    keep = torch.zeros(rows, cols, dtype=torch.bool)
    keep[T:] = True
    C.check_kept(keep, what + ": rows no group claims")
    got = C.view().cpu()
    fams = ("sum", "gemv") if entry in ("bb_matmul_grouped", "bb_matmul_grouped_swiglu") else ("sum",)
    for e in range(E):
        r0, r1 = int(off[e]), int(off[e + 1])
        if r1 == r0:
            continue
        x = cases[e % E_used]
        sub = dict(x, A=x["A"][r0:r1], M=r1 - r0)
        X.prove_exact(sub, fams, device=DEV)
        ref = X.exact_reference(sub, DEV).cpu()
        if swiglu:
            swiglu_bound(got[r0:r1], ref, B.OUTS[i % 3], x["bias"] is not None)
        else:
            X.compare_exact(got[r0:r1], ref, f"{what} expert {e}")


@pytest.mark.parametrize("c", FP8_GROUPED, ids=lambda c: f"{c['entry']}-{c['name']}")
def test_grouped_fp8(c):
    from test_gpu_grouped_fp8 import _op, exact_grouped, exact_reference
    entry, counts, i = c["entry"], c["counts"], c["i"]
    N, K = GROUPED_SHAPE[entry]
    swiglu = "swiglu" in entry
    T = sum(counts)
    rows = T + c["unclaimed"]
    offsets = _offsets(counts).tolist()
    out = B.OUTS[i % 3]
    (A, _, W, ws, _), qa, sa, host = exact_grouped(offsets, rows, N, K, seed=8000 + i, swiglu=swiglu)
    ld = (rows + 3) // 4 * 4 + 4 * (i % 2)
    op = _op(N, K, out)
    desc = op._fp8_desc()
    what = f"{entry} {c['name']}"
    bufs = Buffers(what)
    o16 = 16 * (i % 2)
    Ag = bufs.inp(A.view(torch.uint8), "e4m3", o16, K)
    sa_g = bufs.inp(_a_scale_payload(sa, ld), "float32", o16)
    Wg = bufs.inp(W.view(torch.uint8), "e4m3", o16, K)
    ws_g = bufs.inp(ws, "float32", 4 * (i % 2))
    offg = bufs.inp(torch.tensor(offsets, dtype=torch.int32), "int32", 4 * (i % 2))
    cols = N // 2 if swiglu else N
    C = bufs.out((rows, cols), TORCH[out], out, o16, cols * 4)
    bufs.seal()
    _call(entry, ctypes.byref(desc), len(counts), offg.ptr, Ag.ptr, sa_g.ptr, ld, Wg.ptr, ws_g.ptr, C.ptr, rows, _stream())
    bufs.check()
    keep = torch.zeros(rows, cols, dtype=torch.bool)
    keep[T:] = True
    C.check_kept(keep, what + ": rows no group claims")
    ref = exact_reference(qa, sa, host, offsets, rows, N, out, swiglu, sentinel=0.0).cpu()
    X.compare_exact(C.view().cpu()[:T], ref[:T], what)


# ---- routing, combine, top-k -------------------------------------------------------------------------------------------------------
def _ids(c, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, c["E"], (c["T"], c["k"]), generator=g, dtype=torch.int32)
    if c["drop"]:
        r = torch.rand((c["T"], c["k"]), generator=g)
        ids[r < 0.1] = -1
        ids[r > 0.9] = c["E"]
        ids.view(-1)[0] = -1
    return ids


@pytest.mark.parametrize("c", B.ROUTE, ids=lambda c: f"{c['entry']}-{_cid(c)}")
def test_route(c):
    T, k, E, K = c["T"], c["k"], c["E"], c["K"]
    ids = _ids(c, T * k + E)
    x = (torch.rand((T, K), generator=torch.Generator().manual_seed(T)) - 0.5).to(torch.float16)
    r_off, r_rows, r_xs, nvalid = route_reference(ids, x, E)
    what = f"{c['entry']} {_cid(c)}"
    bufs = Buffers(what)
    idg = bufs.inp(ids, "int32", 4)
    off = bufs.out((E + 1,), torch.int32, "int32", 4)
    rows = bufs.out((T * k,), torch.int32, "int32", 4)
    if c["entry"] == "bb_moe_route":
        xg = bufs.inp(x, "float16", 16, 2 * K)
        xs = bufs.out((T * k, K), torch.float16, "float16", 16, 2 * K)
        bufs.seal()
        _call("bb_moe_route", idg.ptr, T, k, E, xg.ptr, _lib().BB_F16, K, off.ptr, rows.ptr, xs.ptr, _stream())
        dest, ref_dest = xs, r_xs
    else:
        rt = bufs.out((T * k,), torch.int32, "int32", 4)
        bufs.seal()
        _call("bb_moe_route_index", idg.ptr, T, k, E, off.ptr, rows.ptr, rt.ptr, _stream())
        flat = ids.reshape(-1).long()
        valid = (flat >= 0) & (flat < E)
        order = torch.argsort(torch.where(valid, flat, E), stable=True)
        dest, ref_dest = rt, (order[:nvalid] // k).to(torch.int32)
    bufs.check()
    X.compare_exact(off.view().cpu(), r_off, what + " offsets")
    X.compare_exact(rows.view().cpu(), r_rows, what + " slot_rows")
    X.compare_exact(dest.view().cpu()[:nvalid], ref_dest, what + " sorted rows")
    keep = torch.zeros(dest.shape, dtype=torch.bool)
    keep[nvalid:] = True
    assert nvalid < T * k or not c["drop"]
    dest.check_kept(keep, what + ": sorted rows offsets[E] ..")


@pytest.mark.parametrize("c", B.COMBINE, ids=_cid)
def test_combine(c):
    from test_gpu_kernel_grid import EPS32, _ulp
    T, k, N, out = c["T"], c["k"], c["N"], c["out"]
    g = torch.Generator().manual_seed(T * k + N)
    Y = ((torch.rand((T * k, N), generator=g) - 0.5) * 8).to(TORCH[out])
    rows = torch.randperm(T * k, generator=g).to(torch.int32)
    rows[0] = -1
    if T * k > 1:
        rows[1] = T * k     # out of range: adds nothing
    w = torch.rand((T, k), generator=g)
    what = f"bb_moe_combine {_cid(c)}"
    bufs = Buffers(what)
    rg = bufs.inp(rows, "int32", 4)
    wg = bufs.inp(w, "float32", 4)
    Yg = bufs.inp(Y, out, 16, N * 4)
    o = bufs.out((T, N), TORCH[out], out, 16, N * 4)
    bufs.seal()
    _call("bb_moe_combine", rg.ptr, wg.ptr, Yg.ptr, _lib().dtype_id(TORCH[out]), o.ptr, T, k, N, _stream())
    bufs.check()
    got = o.view().cpu().double()
    valid = ((rows >= 0) & (rows < T * k)).reshape(T, k)
    Yv = Y.double()[rows.clamp(0, T * k - 1).long()].reshape(T, k, N) * valid[..., None]
    ref = (w.double()[..., None] * Yv).sum(1)
    bound = k * EPS32 * (w.double()[..., None].abs() * Yv.abs()).sum(1) + _ulp(ref.abs(), out)
    assert bool(((got - ref).abs() <= bound).all()), what


@pytest.mark.parametrize("c", B.TOPK, ids=_cid)
def test_topk(c):
    from test_gpu_moe_topk import _check_weights, _distinct_logits, reference
    T, E, k = c["T"], c["E"], c["k"]
    gen = torch.Generator().manual_seed(9000 + T + E)
    logits = _distinct_logits(T, E, gen).to(TORCH[c["logits"]])
    groups, tg = c["groups"], (4 if c["groups"] > 1 else 0)
    what = f"bb_moe_topk {_cid(c)}"
    bufs = Buffers(what)
    lg = bufs.inp(logits, c["logits"], 16, E * 4)
    ids = bufs.out((T, k), torch.int32, "int32", 4)
    wts = bufs.out((T, k), torch.float32, "float32", 4)
    bufs.seal()
    _call("bb_moe_topk", lg.ptr, _lib().dtype_id(TORCH[c["logits"]]), T, E, k, c["scoring"], 0, groups, tg, 0, 0, 1.0,
          ids.ptr, wts.ptr, _stream())
    bufs.check()
    if T == 0:
        return
    kw = dict(scoring="softmax" if c["scoring"] == 0 else "sigmoid")
    if groups > 1:
        kw.update(num_expert_group=groups, topk_group=tg)
    r_ids, r_w, ok = reference(logits, k, **kw)
    assert ok.all()
    X.compare_exact(ids.view().cpu(), r_ids, what + " ids")
    _check_weights(wts.view().cpu(), r_w)


# ---- permute ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", B.PERMUTE, ids=_cid)
def test_permute_cols(c):
    rows, K, counts = c["rows"], c["K"], c["counts"]
    gen = torch.Generator().manual_seed(rows + K)
    A = (torch.rand((rows, K), generator=gen) - 0.5).to(TORCH[c["A"]])
    E = len(counts) if counts else 1
    perm = torch.stack([torch.randperm(K, generator=gen) for _ in range(E)]).to(torch.int32)
    what = f"bb_permute_cols {_cid(c)}"
    bufs = Buffers(what)
    Ag = bufs.inp(A, c["A"], 16, 2 * K)
    pg = bufs.inp(perm, "int32", 4)
    offg = bufs.inp(_offsets(counts), "int32", 4) if counts else None
    o = bufs.out((rows, K), TORCH[c["A"]], c["A"], 16, 2 * K)
    bufs.seal()
    _call("bb_permute_cols", Ag.ptr, o.ptr, pg.ptr, rows, K, _lib().dtype_id(TORCH[c["A"]]), E, ptr(offg), _stream())
    bufs.check()
    got = o.view().cpu()
    off = _offsets(counts).tolist() if counts else [0, rows]
    for e in range(E):
        r0, r1 = off[e], off[e + 1]
        X.compare_exact(got[r0:r1], A[r0:r1][:, perm[e].long()], f"{what} group {e}")
    keep = torch.zeros(rows, K, dtype=torch.bool)
    keep[off[-1]:] = True
    o.check_kept(keep, what + ": rows no group claims")


# ---- scatter ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", B.SCATTER, ids=_cid)
def test_scatter(c):
    fam, m, N, K, peers = c["family"], c["m"], c["N"], c["K"], c["peers"]
    if fam == "gemv_i8":
        case = X.make_exact_case(m, N, K, A_dtype="int8", W_dtype="int4", out_dtype="int32", bias=True, fast_decoding=True, seed=N)
    else:
        case = X.make_exact_case(m, N, K, group_size=128, mode="quantized", bias=True, fast_decoding=True, seed=N + m)
    out = case["cfg"]["out_dtype"]
    ldc, col = N + 64, 32
    what = f"bb_matmul_scatter {_cid(c)}"
    with forced(B.FAMILY[fam]["kid"]) as lib:
        op = X.product_operator(case)
        assert op.kernel_for(m) == fam
        W = X.product_weight(op, case, DEV)
        ws_bytes = lib.bb_workspace_bytes(op._desc_ref, m)
        bufs = Buffers(what)
        A, Wg, s, z, b = _operands(bufs, case, W, 0)
        dests = [bufs.out((m, ldc), TORCH[out], out, 0, ldc * 4) for _ in range(peers)]
        ws = bufs.out((max(ws_bytes, 1),), torch.uint8, "bytes") if ws_bytes else None
        if ws is not None:
            ws.payload().zero_()
        bufs.seal()
        arr = (ctypes.c_void_p * peers)(*[d.ptr for d in dests])
        _call("bb_matmul_scatter", op._desc_ref, A.ptr, Wg.ptr, 0, ptr(s), ptr(z), ptr(b), arr, peers, ldc, col, m, ptr(ws),
              ws_bytes, _stream())
        bufs.check()
    ref = X.exact_reference(case, DEV).cpu()
    X.prove_exact(case, _families(fam), device=DEV)
    for d in dests:
        X.compare_exact(d.view().cpu()[:, col:col + N], ref, what)
        keep = torch.ones(m, ldc, dtype=torch.bool)
        keep[:, col:col + N] = False
        d.check_kept(keep, what + ": columns outside the window")


# ---- device prep kernels ---------------------------------------------------------------------------------------------------------
def _host_transform(vals, bits, target):
    """bb_compress_host (+ bb_interleave_host) of int8 values [rows, cols]: the host reference of the device transform"""
    lib = _lib().load()
    v = np.ascontiguousarray(vals.numpy().astype(np.int8))
    rows, cols = v.shape
    out = np.zeros((rows, cols * bits // 8), dtype=np.int8)
    assert lib.bb_compress_host(v.ctypes.data, out.ctypes.data, rows, cols, bits) == 0
    if target:
        il = np.zeros_like(out)
        assert lib.bb_interleave_host(out.ctypes.data, il.ctypes.data, out.size, bits, target) == 0
        out = il
    return torch.from_numpy(out)


PREP_TRANSFORM = [c for c in B.PREP if c["entry"] == "bb_transform_weight_device"]
PREP_QWEIGHT = [c for c in B.PREP if c["entry"] == "bb_repack_gptq_qweight_device"]
PREP_QZEROS = [c for c in B.PREP if c["entry"] == "bb_repack_gptq_qzeros_device"]
PREP_RETILE = [c for c in B.PREP if c["entry"] == "bb_retile_weight_device"]


@pytest.mark.parametrize("c", PREP_TRANSFORM, ids=_cid)
def test_transform_weight_device(c):
    rows, cols, bits, target = c["rows"], c["cols"], c["bits"], c["target"]
    vals = torch.randint(0, 2 ** bits, (rows, cols), generator=torch.Generator().manual_seed(rows * cols), dtype=torch.int8)
    what = f"bb_transform_weight_device {_cid(c)}"
    bufs = Buffers(what)
    wi = bufs.inp(vals, "packed", 16, cols)
    o = bufs.out((rows, cols * bits // 8), torch.int8, "packed", 16, cols)
    bufs.seal()
    _call("bb_transform_weight_device", wi.ptr, o.ptr, rows, cols, bits, target, _stream())
    bufs.check()
    X.compare_exact(o.view().cpu(), _host_transform(vals, bits, target), what)


@pytest.mark.parametrize("c", PREP_QWEIGHT, ids=_cid)
def test_repack_gptq_qweight_device(c):
    K, N, bits, target = c["K"], c["N"], c["bits"], c["target"]
    vals = torch.randint(0, 2 ** bits, (K, N), generator=torch.Generator().manual_seed(K + N))
    q = X._pack_int32(vals, bits, 0)
    what = f"bb_repack_gptq_qweight_device {_cid(c)}"
    bufs = Buffers(what)
    qi = bufs.inp(q, "int32", 16, N * 4)
    o = bufs.out((N, K * bits // 8), torch.int8, "packed", 16, K)
    bufs.seal()
    _call("bb_repack_gptq_qweight_device", qi.ptr, o.ptr, K, N, bits, target, _stream())
    bufs.check()
    X.compare_exact(o.view().cpu(), _host_transform(vals.T.contiguous().to(torch.int8), bits, target), what)


@pytest.mark.parametrize("c", PREP_QZEROS, ids=_cid)
def test_repack_gptq_qzeros_device(c):
    import bitblas_oracle as O
    G, N, bits, mode, adt, v2 = c["groups"], c["N"], c["bits"], c["mode"], TORCH[c["A"]], c["v2"]
    gen = torch.Generator().manual_seed(G * N + mode)
    stored = torch.randint(0, 2 ** bits, (G, N), generator=gen)
    qz = X._pack_int32(stored, bits, 1)
    scales = (2.0 ** -torch.randint(0, 3, (N, G), generator=gen).float()).to(adt)
    z = (stored + (0 if v2 else 1)) % 2 ** bits                     # [G, N]
    if mode == 2:
        shape, dt, kind = (G, N * bits // 8), torch.int8, "packed"
        ref = torch.from_numpy(O.general_compress(z.to(torch.int32).numpy(), bits)).view(torch.int8)
    else:
        shape, dt, kind = (N, G), adt, c["A"]
        ref = z.T.double() if mode == 0 else z.T.double() * scales.double()
        ref = ref.to(adt)
    what = f"bb_repack_gptq_qzeros_device {_cid(c)}"
    bufs = Buffers(what)
    qi = bufs.inp(qz, "int32", 16)
    si = bufs.inp(scales, c["A"], 16)
    o = bufs.out(shape, dt, kind, 16)
    bufs.seal()
    _call("bb_repack_gptq_qzeros_device", qi.ptr, si.ptr, o.ptr, G, N, bits, mode, _lib().dtype_id(adt), v2, _stream())
    bufs.check()
    X.compare_exact(o.view().cpu(), ref.reshape(shape), what)


@pytest.mark.parametrize("c", PREP_RETILE, ids=_cid)
def test_retile_weight_device(c):
    rows, rb, inv = c["rows"], c["row_bytes"], c["inverse"]
    w = torch.randint(-128, 128, (rows, rb), generator=torch.Generator().manual_seed(rows), dtype=torch.int8)
    tiled = w.view(rows // 32, 32, rb // 512, 512).permute(0, 2, 1, 3).reshape(rows, rb)
    src, ref = (tiled, w) if inv else (w, tiled)
    what = f"bb_retile_weight_device {_cid(c)}"
    bufs = Buffers(what)
    i_ = bufs.inp(src, "packed", 16, rb)
    o = bufs.out((rows, rb), torch.int8, "packed", 16, rb)
    bufs.seal()
    _call("bb_retile_weight_device", i_.ptr, o.ptr, rows, rb, inv, _stream())
    bufs.check()
    X.compare_exact(o.view().cpu(), ref, what)


# ---- Python layers writing into a preallocated slice -------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", [c["layer"] for c in B.LAYERS])
def test_python_layer_output_view(layer):
    """a serving stack hands in a view of a larger buffer: the layer writes that view and nothing around it"""
    what = f"{layer}(output=view)"
    m, N, K = 33, 256, 512
    case = X.make_exact_case(m, N, K, group_size=128, mode="quantized", bias=True, fast_decoding=True, seed=77)
    op = X.product_operator(case, M=[1, m])
    W = X.product_weight(op, case, DEV)
    t = {k: case[k].to(DEV) for k in ("scale", "zeros", "bias")}
    A = case["A"].to(DEV)
    counts = [5, 0, 20, 8]
    off = _offsets(counts).to(DEV)
    if layer == "Matmul.forward":
        run, shape = (lambda out: op.forward(A, W, **t, output=out)), (m, N)
    elif layer == "Matmul.forward_swiglu":
        run, shape = (lambda out: op.forward_swiglu(A, W, **t, output=out)), (m, N // 2)
    elif layer.startswith("Matmul.forward_grouped"):
        E = len(counts)
        Ws = W[None].expand(E, *W.shape).contiguous()
        ts = {k: v[None].expand(E, *v.shape).contiguous() for k, v in t.items()}
        fn = op.forward_grouped_swiglu if layer.endswith("swiglu") else op.forward_grouped
        run, shape = (lambda out: fn(A, Ws, off, **ts, output=out)), (m, N // 2 if layer.endswith("swiglu") else N)
    else:
        from bitblas_b200.moe import moe_combine
        Y = case["A"][:, :N].to(DEV)
        rows = torch.randperm(m, generator=torch.Generator().manual_seed(3)).to(torch.int32).to(DEV)
        w = torch.rand((m, 1), generator=torch.Generator().manual_seed(4)).to(DEV)
        run, shape = (lambda out: moe_combine(Y, rows, w, out)), (m, N)
    expect = run(None)
    torch.cuda.synchronize()
    g = Guarded.output(shape, torch.float16, "float16", 16, guard_for(shape[1] * 4)).seal()
    got = run(g.view())
    torch.cuda.synchronize()
    assert got.data_ptr() == g.ptr
    g.check_guards(what)
    X.compare_exact(g.view().cpu(), expect.cpu(), what)
    if layer == "Matmul.forward":
        X.compare_exact(g.view().cpu(), X.exact_reference(case, DEV).cpu(), what + " against the exact reference")
