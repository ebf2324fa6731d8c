"""GPU: the dense SwiGLU MLP.  bb_matmul_swiglu on every kernel family (gemv_slab, gemv_mma, gemm_ts with and without split-K,
generic_simt) against silu(g) * u formed from bb_matmul's output on the same buffers under the same kernel override, at production
shapes against the exact pre-activations, at capped SM counts, with a shared workspace, its rejections, and SwiGLUMLP end to end
(launch counts, graph replay, PDL, GPTQ loading, state_dict, slab tiling)."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import exact_inputs as X
from test_gpu_kernel_grid import (K_GEMM_TS, K_GEMV_MMA, K_GEMV_SLAB, K_GENERIC, KERNEL_NAME, MODES, OUTS, _seed, forced,
                                  make_case, ts_splits)
from test_gpu_act_order import GPTQ
from test_gpu_moe import _launches, swiglu_bound
from test_gpu_sm_counts import sm_cap

pytestmark = pytest.mark.gpu

DEV = "cuda"
K_AUTO = 0


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tensors(op, case):
    t = dict(W=X.product_weight(op, case, DEV))
    for k in ("scale", "zeros", "bias"):
        t[k] = case[k].to(DEV) if case[k] is not None else None
    return t


def _pair(op, case, t=None, A=None):
    """(plain [m, 2I] output of forward, forward_swiglu's [m, I]) on the same buffers"""
    t = t or _tensors(op, case)
    A = case["A"].to(DEV) if A is None else A
    kw = dict(scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    pre = op.forward(A, t["W"], **kw)
    got = op.forward_swiglu(A, t["W"], **kw)
    torch.cuda.synchronize()
    return pre.cpu(), got.cpu()


def _check_cell(case, kernel_id, m, what):
    op = X.product_operator(case, M=[1, m])
    t = _tensors(op, case)
    with forced(kernel_id):
        if kernel_id != K_AUTO:
            assert op.kernel_for(m) == KERNEL_NAME[kernel_id], (op.kernel_for(m), what)
        pre, got = _pair(op, case, t)
    assert got.shape == (m, case["N"] // 2)
    swiglu_bound(got, pre, case["cfg"]["out_dtype"], case["bias"] is not None)
    return op, t


# ---- every kernel instance -------------------------------------------------------------------------------------------------------
def _cells():
    cells = []
    i = 0
    # gemv_slab (m = 1, 4-bit): integer formats in both layouts and every zeros mode, the table formats, slab tiling
    for T in ("float16", "bfloat16"):
        for W, il in (("uint4", True), ("uint4", False), ("int4", True)):
            for mode in (MODES if W == "uint4" else ["none", "scale"]):
                cells.append(dict(k=K_GEMV_SLAB, m=1, T=T, W=W, il=il, mode=mode, out=OUTS[i % 3], bias=i % 2 == 0, K=2048))
                i += 1
        for W in ("nf4", "fp4_e2m1"):
            cells.append(dict(k=K_GEMV_SLAB, m=1, T=T, W=W, il=False, mode="scale", out=OUTS[i % 3], bias=i % 2 == 0, K=2048))
            i += 1
        cells.append(dict(k=K_GEMV_SLAB, m=1, T=T, W="uint4", il=True, mode="quantized", out="float16", bias=True, K=2048,
                          tile=True))
    # gemv_mma: m = 1 .. 32 over the NT = 1, 2, 4 instances, 4- and 2-bit, both layouts, every zeros mode
    rows = [1, 2, 5, 8, 9, 16, 17, 32]
    for T in ("float16", "bfloat16"):
        for W in ("uint4", "uint2", "int4"):
            for il in (True, False):
                for mode in (MODES if W.startswith("u") else ["none", "scale"]):
                    cells.append(dict(k=K_GEMV_MMA, m=rows[i % len(rows)], T=T, W=W, il=il, mode=mode, out=OUTS[i % 3],
                                      bias=i % 2 == 1, K=1024))
                    i += 1
    # gemm_ts: BM 32 / 64 / 128 and several m-tiles, with and without split-K (K = 1536: 3 splits at m <= 128 on >= 6 SMs)
    ts_rows = [9, 31, 33, 64, 65, 100, 128, 300]
    for T in ("float16", "bfloat16"):
        for W, il in (("uint4", True), ("uint4", False), ("uint2", True), ("uint2", False), ("int4", True)):
            for mode in (MODES if W.startswith("u") else ["none", "scale"]):
                m = ts_rows[i % len(ts_rows)]
                cells.append(dict(k=K_GEMM_TS, m=m, T=T, W=W, il=il, mode=mode, out=OUTS[i % 3], bias=i % 2 == 0,
                                  K=1536 if i % 2 else 768))
                i += 1
        for W in ("nf4", "fp4_e2m1", "e4m3_float8", "e5m2_float8"):
            for m in (40, 128):
                cells.append(dict(k=K_GEMM_TS, m=m, T=T, W=W, il=False, mode="scale", out=OUTS[i % 3], bias=i % 2 == 0, K=1536))
                i += 1
        cells.append(dict(k=K_GEMM_TS, m=65, T=T, W="uint4", il=True, mode="original", out="float16", bias=True, K=2048,
                          tile=True))
    # generic_simt: 1-bit weights, g = 32, a table format with zeros, several m
    for T in ("float16", "bfloat16"):
        for W, mode, g in (("uint1", "scale", -1), ("int1", "none", -1), ("uint4", "original", 32), ("uint2", "rescale", 32),
                           ("nf4", "scale", 128), ("nf4", "original", 128), ("uint4", "quantized", 128)):
            for m in (1, 5, 300):
                cells.append(dict(k=K_GENERIC, m=m, T=T, W=W, il=False, mode=mode, out=OUTS[i % 3], bias=i % 2 == 0, K=512,
                                  g=g))
                i += 1
    # AUTO: the dispatcher's own choice at each regime
    for m in (1, 4, 16, 100, 300):
        cells.append(dict(k=K_AUTO, m=m, T="float16", W="uint4", il=True, mode="quantized", out="float16", bias=True, K=2048))
    return cells


CELLS = _cells()


def _cid(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


@pytest.mark.parametrize("c", CELLS, ids=[_cid(c) for c in CELLS])
def test_swiglu_instance(c):
    N = 256 if not c.get("tile") else 512   # 2I; the tiled cells need N % 128 (gemm_ts) and whole 32-row units
    g = c.get("g", 128 if c["mode"] != "none" else -1)
    if c["W"].startswith("e") or c["W"] in ("nf4", "fp4_e2m1"):
        g = c.get("g", -1)
    integer = c["W"].startswith(("uint", "int"))
    case = make_case(c["m"], N, c["K"], A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=g, mode=c["mode"],
                     bias=c["bias"], fast_decoding=c["il"] if integer else None, seed=_seed(c))
    case["propagate_b"] = bool(c.get("tile"))
    op, _ = _check_cell(case, c["k"], c["m"], _cid(c))
    assert op.weight_tiled == bool(c.get("tile"))


# split-K factor f: K = 512 f gives 8 f k-blocks, which split f ways (8 k-blocks per split at least) while the 2 tiles leave SMs idle
SPLITS = [(2, 16), (3, 40), (4, 100), (5, 128), (6, 20), (7, 60), (8, 127)]


@pytest.mark.parametrize("f,m", SPLITS, ids=[f"split{f}-m{m}" for f, m in SPLITS])
def test_gemm_ts_split_factors_and_no_workspace(f, m):
    """every split-K factor (read from bb_workspace_bytes), and the same call through the C ABI without a workspace (no split-K)
    against bb_matmul without one"""
    from bitblas_b200 import _lib
    lib = _lib.load()
    K = 512 * f
    case = make_case(m, 256, K, W_dtype="uint4", group_size=128, mode="original", bias=True, fast_decoding=True, seed=m)
    op = X.product_operator(case, M=[1, m])
    t = _tensors(op, case)
    with forced(K_GEMM_TS):
        assert ts_splits(m, 256, K, 64, _sms()) == f
        ws = lib.bb_workspace_bytes(ctypes.byref(op._desc), m)
        assert ws == X.slab_slot_bytes(_sms()) + f * m * 256 * 4
        pre, got = _pair(op, case, t)
        swiglu_bound(got, pre, "float16", True)
        A = case["A"].to(DEV)
        pre0 = torch.empty((m, 256), dtype=torch.float16, device=DEV)
        got0 = torch.empty((m, 128), dtype=torch.float16, device=DEV)
        args = (A.data_ptr(), t["W"].data_ptr(), 0, t["scale"].data_ptr(), t["zeros"].data_ptr(), t["bias"].data_ptr())
        _lib.check(lib.bb_matmul(ctypes.byref(op._desc), *args, pre0.data_ptr(), m, None, 0, None), "bb_matmul")
        _lib.check(lib.bb_matmul_swiglu(ctypes.byref(op._desc), *args, got0.data_ptr(), m, None, 0, None), "bb_matmul_swiglu")
        torch.cuda.synchronize()
    swiglu_bound(got0.cpu(), pre0.cpu(), "float16", True)


def test_swiglu_launch_count_matches_bb_matmul():
    """one step of bb_launch_count per kernel, as bb_matmul: 1 for the GEMVs, 2 with split-K"""
    case = make_case(16, 256, 8192, W_dtype="uint4", group_size=128, mode="scale", fast_decoding=True, seed=1)
    op = X.product_operator(case, M=[1, 4, 16])
    t = _tensors(op, case)
    kw = dict(scale=t["scale"])
    for m, expect in ((1, 1), (4, 1), (16, 2)):
        A = case["A"][:m].to(DEV)
        _, n_plain = _launches(lambda: op.forward(A, t["W"], **kw))
        _, n_sw = _launches(lambda: op.forward_swiglu(A, t["W"], **kw))
        assert n_plain == n_sw == expect, (m, n_plain, n_sw)


# ---- production shapes, exact pre-activations ------------------------------------------------------------------------------------
# (2I, K): Llama-2-70B gate/up, Llama-3-8B gate/up, and a shape with N % 32 == 16 (a half row block in the slab kernel)
PROD = [(57344, 8192), (28672, 4096), (4112, 4096)]


@pytest.mark.parametrize("N,K", PROD, ids=[f"{n}x{k}" for n, k in PROD])
def test_production_shapes_exact(N, K):
    case = X.make_exact_case(4096, N, K, group_size=128, mode="quantized", fast_decoding=True, seed=N % 97)
    X.prove_exact(case, device=DEV)
    ref = X.exact_reference(case, DEV)   # the exact [4096, N] pre-activations, rounded as bb_matmul stores them
    op = X.product_operator(case, M=[1, 16, 128, 4096])
    t = _tensors(op, case)
    A = case["A"].to(DEV)
    for m in (1, 16, 128, 4096):
        got = op.forward_swiglu(A[:m], t["W"], scale=t["scale"], zeros=t["zeros"])
        torch.cuda.synchronize()
        swiglu_bound(got.cpu(), ref[:m].cpu(), "float16", False)
    del ref, got, t


# ---- capped SM counts ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 7, 33, 114])
def test_slab_at_caps_and_reproducible(cap):
    """m = 1 at SM counts where row blocks are split across CTAs (the stream-K fix-up runs): exact pre-activations, and three
    calls bit-identical"""
    N, K = 4112, 8192
    case = X.make_exact_case(1, N, K, group_size=128, mode="original", bias=True, fast_decoding=True, seed=cap)
    X.prove_exact(case, device=DEV)
    ref = X.exact_reference(case, DEV).cpu()
    op = X.product_operator(case, M=[1])
    t = _tensors(op, case)
    with sm_cap(min(cap, _sms())):
        assert op.kernel_for(1) == KERNEL_NAME[K_GEMV_SLAB]
        outs = [_pair(op, case, t)[1] for _ in range(3)]
    swiglu_bound(outs[0], ref, "float16", True)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize("cap", [8, 16, 33, 66, 114])
def test_split_k_at_caps(cap):
    cap = min(cap, _sms())
    N, K, m = 1024, 8192, 40
    case = X.make_exact_case(m, N, K, group_size=128, mode="rescale", bias=True, fast_decoding=True, seed=cap)
    X.prove_exact(case, ("sum",), device=DEV)
    ref = X.exact_reference(case, DEV).cpu()
    op = X.product_operator(case, M=[1, m])
    t = _tensors(op, case)
    with sm_cap(cap):
        assert op.kernel_for(m) == KERNEL_NAME[K_GEMM_TS]
        f = ts_splits(m, N, K, 64, cap)
        outs = [_pair(op, case, t)[1] for _ in range(2)]
    swiglu_bound(outs[0], ref, "float16", True)
    assert torch.equal(outs[0], outs[1]), f


# ---- one workspace for every m ---------------------------------------------------------------------------------------------------
def test_shared_workspace_split_k_then_m1():
    """a split-K forward_swiglu, then an m = 1 forward_swiglu on the operator's one buffer: the slab slots are zero after both
    calls and both outputs are right"""
    N, K = 4096, 4096
    case = X.make_exact_case(16, N, K, group_size=128, mode="original", bias=True, fast_decoding=True, seed=16)
    X.prove_exact(case, ("sum",), device=DEV)
    ref = X.exact_reference(case, DEV).cpu()
    op = X.product_operator(case, M=[1, 16])
    assert op.kernel_for(16) == KERNEL_NAME[K_GEMM_TS] and op.kernel_for(1) == KERNEL_NAME[K_GEMV_SLAB]
    assert ts_splits(16, N, K, 64, _sms()) > 1
    t = _tensors(op, case)
    A = case["A"].to(DEV)
    kw = dict(scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    got16 = op.forward_swiglu(A, t["W"], **kw)
    got1 = op.forward_swiglu(A[:1], t["W"], **kw)
    torch.cuda.synchronize()
    ws = op._ws[(0, torch.cuda.current_stream().cuda_stream)]
    slots = X.slab_slot_bytes(_sms())
    assert int(ws[:slots].count_nonzero()) == 0
    swiglu_bound(got16.cpu(), ref, "float16", True)
    swiglu_bound(got1.cpu(), ref[:1], "float16", True)


# ---- rejections ------------------------------------------------------------------------------------------------------------------
def test_rejections_through_the_abi_and_forward_swiglu():
    from bitblas_b200 import _lib
    lib = _lib.load()
    case = make_case(4, 256, 1024, W_dtype="uint4", group_size=128, mode="scale", fast_decoding=True, seed=5)
    op = X.product_operator(case, M=[1, 4])
    t = _tensors(op, case)
    A = case["A"].to(DEV)
    C = torch.empty((4, 128), dtype=torch.float16, device=DEV)
    d = ctypes.byref(op._desc)
    args = (A.data_ptr(), t["W"].data_ptr(), 0, t["scale"].data_ptr(), 0, 0)
    assert lib.bb_matmul_swiglu(d, *args, None, 4, None, 0, None) == 1 and "non-null" in _lib.last_error()
    assert lib.bb_matmul_swiglu(d, *args, C.data_ptr(), -1, None, 0, None) == 1 and "m must be" in _lib.last_error()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    assert lib.bb_matmul_swiglu(d, *args, C.data_ptr(), 0, None, 0, None) == 0
    assert lib.bb_launch_count() == n0
    i8 = X.product_operator(make_case(4, 256, 1024, A_dtype="int8", W_dtype="int4", out_dtype="int32", seed=6), M=[4])
    with pytest.raises(ValueError, match="int8"):
        i8.forward_swiglu(torch.zeros((4, 1024), dtype=torch.int8, device=DEV), t["W"])
    assert lib.bb_matmul_swiglu(ctypes.byref(i8._desc), *args, C.data_ptr(), 4, None, 0, None) == 1
    assert "int8 activations" in _lib.last_error()
    odd = X.product_operator(make_case(4, 272 - 8, 1024, W_dtype="uint4", seed=7), M=[4])
    with pytest.raises(ValueError, match="I % 8 == 0"):
        odd.forward_swiglu(A, t["W"])
    with pytest.raises(ValueError, match="output"):
        op.forward_swiglu(A, t["W"], scale=t["scale"], output=torch.empty((4, 256), dtype=torch.float16, device=DEV))


# ---- SwiGLUMLP ---------------------------------------------------------------------------------------------------------------------
H, I = 1024, 512


def _mlp_parts(seed, bits=4, g=128, T="float16", bias=False):
    """exact gate / up / down cases (unsigned fields, quantized zeros): gate and up share their activations"""
    cg = X.make_exact_case(16, I, H, A_dtype=T, out_dtype=T, group_size=g, mode="quantized", bias=bias, seed=seed,
                           W_dtype=f"uint{bits}")
    cu = X.make_exact_case(16, I, H, A_dtype=T, out_dtype=T, group_size=g, mode="quantized", bias=bias, seed=seed + 1,
                           W_dtype=f"uint{bits}", A=cg["A"])
    cd = X.make_exact_case(16, H, I, A_dtype=T, out_dtype=T, group_size=g, mode="quantized", bias=bias, seed=seed + 2,
                           W_dtype=f"uint{bits}")
    return cg, cu, cd


def _loaded_mlp(cg, cu, cd, **kw):
    import bitblas_b200 as bitblas
    T = cg["cfg"]["A_dtype"]
    mlp = bitblas.SwiGLUMLP(H, I, bias=cg["bias"] is not None, A_dtype=T, W_dtype=cg["cfg"]["W_dtype"], out_dtype=T,
                            accum_dtype="float32", group_size=cg["cfg"]["group_size"], with_scaling=True, with_zeros=True,
                            zeros_mode="quantized", opt_M=[1, 4, 16, 64], **kw)
    parts = [(c["fields"].to(torch.int8), c["scale"], c["zeros"], c["bias"]) for c in (cg, cu, cd)]
    mlp.load_and_transform_weight(*parts)
    return mlp.to(DEV)


def _separate(cg, cu, cd):
    """gate, up and down as three Linears (the same fields and parameters)"""
    import bitblas_b200 as bitblas
    T = cg["cfg"]["A_dtype"]
    outs = []
    for c, (n, k) in zip((cg, cu, cd), ((I, H), (I, H), (H, I))):
        lin = bitblas.Linear(k, n, bias=c["bias"] is not None, A_dtype=T, W_dtype=c["cfg"]["W_dtype"], out_dtype=T,
                             accum_dtype="float32", group_size=c["cfg"]["group_size"], with_scaling=True, with_zeros=True,
                             zeros_mode="quantized", opt_M=[1, 4, 16, 64])
        lin.load_and_transform_weight(c["fields"].to(torch.int8), c["scale"], c["zeros"], c["bias"])
        outs.append(lin.to(DEV))
    return outs


@pytest.mark.parametrize("T,bias", [("float16", False), ("bfloat16", True)])
def test_mlp_matches_separate_linears(T, bias):
    from bitblas_b200.moe import interleave_gate_up
    cg, cu, cd = _mlp_parts(11, T=T, bias=bias)
    mlp = _loaded_mlp(cg, cu, cd)
    lg, lu, ld = _separate(cg, cu, cd)
    for m in (1, 4, 16, 64):
        x = (torch.rand((m, H), generator=torch.Generator().manual_seed(m)) - 0.5).to(getattr(torch, T)).to(DEV)
        h = mlp.gate_up.bitblas_matmul.forward_swiglu(x, mlp.gate_up.qweight, mlp.gate_up.scales, mlp.gate_up.zeros,
                                                      mlp.gate_up.bias)
        pre = interleave_gate_up(lg(x), lu(x), "bias")
        swiglu_bound(h.cpu(), pre.cpu(), T, bias)
        y, n = _launches(lambda: mlp(x))
        _, n_parts = _launches(lambda: (mlp.gate_up.bitblas_matmul.forward_swiglu(x, mlp.gate_up.qweight, mlp.gate_up.scales,
                                                                                  mlp.gate_up.zeros, mlp.gate_up.bias),
                                        mlp.down(h)))
        assert n == n_parts and (m > 8 or n == 2), (m, n, n_parts)   # (split-K adds its reduce launch above m = 8)
        assert torch.equal(y, ld(h)), m


def test_mlp_graph_replay_and_leading_dims():
    import bitblas_b200 as bitblas
    cg, cu, cd = _mlp_parts(21)
    mlp = _loaded_mlp(cg, cu, cd)
    for m in (1, 4, 64):
        x = (torch.rand((2, m, H), generator=torch.Generator().manual_seed(m)) - 0.5).half().to(DEV)
        eager = mlp(x)
        assert eager.shape == (2, m, H)
        out = torch.empty_like(eager)
        step = bitblas.CapturedStep(lambda: mlp(x, output=out))
        out.zero_()
        step()
        assert torch.equal(out, eager), m


MLP_CHAIN = r"""
import sys, torch
sys.path[:0] = [{tests!r}, {oracle!r}]
import bitblas_b200 as bitblas
from test_gpu_swiglu import _mlp_parts, _loaded_mlp
cg, cu, cd = _mlp_parts(31)
mlp = _loaded_mlp(cg, cu, cd)
outs = []
for m in (1, 4):
    xs = [(torch.rand((m, 1024), generator=torch.Generator().manual_seed(8 * m + i)) - 0.5).half().cuda() for i in range(4)]
    ys = [mlp(x) for x in xs]   # enqueued back to back: each down reads the h its gate/up launch wrote
    torch.cuda.synchronize()
    outs += [y.cpu() for y in ys]
torch.save(outs, {out!r})
"""


def test_mlp_pdl_chain_matches_plain_stream_order(tmp_path):
    """MLP calls enqueued back to back (gate/up -> down -> gate/up ...) with PDL on (default) and off (BB_PDL=0) in fresh
    processes: the same bits"""
    tests = os.path.dirname(os.path.abspath(__file__))
    res = []
    for pdl in ("1", "0"):
        out = str(tmp_path / f"pdl{pdl}.pt")
        env = dict(os.environ, BB_PDL=pdl)
        code = MLP_CHAIN.format(tests=tests, oracle=os.path.join(os.path.dirname(tests), "oracle"), out=out)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        res.append(torch.load(out))
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))   # bit for bit (the exact-case weights saturate some outputs)


def _gptq_mods(seed, act_gate_up, act_down, v2=False):
    """GPTQ modules of gate, up (H -> I; one g_idx: they read the same input) and down (I -> H)"""
    gm = GPTQ(H, I, 128, 4, seed=seed, act_order=act_gate_up, v2=v2)
    um = GPTQ(H, I, 128, 4, seed=seed + 1, act_order=act_gate_up, v2=v2)
    um.g_idx = gm.g_idx
    return gm, um, GPTQ(I, H, 128, 4, seed=seed + 2, act_order=act_down, v2=v2)


def _mlp_for_gptq(T, **kw):
    import bitblas_b200 as bitblas
    return bitblas.SwiGLUMLP(H, I, A_dtype=T, W_dtype="uint4", out_dtype=T, accum_dtype="float32", group_size=128,
                             with_scaling=True, with_zeros=True, zeros_mode="quantized", opt_M=[1, 4, 16, 64], **kw).to(DEV)


def _x(m, T="float16", seed=0):
    return (torch.rand((m, H), generator=torch.Generator().manual_seed(seed)) - 0.5).to(getattr(torch, T)).to(DEV)


@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("T", ["float16", "bfloat16"])
@pytest.mark.parametrize("act", ["none", "gate_up", "down", "both"])
def test_mlp_gptq_loading(v2, T, act):
    """repack_from_gptq[_v2] of three GPTQ modules against gate, up and down loaded as three Linears from the same modules (each
    Linear gathers its own act-order columns): h within the SwiGLU bound of the Linears' gate and up, and y equal bit for bit to
    the down Linear applied to h (down's column order is absorbed into the stored gate/up rows)"""
    import bitblas_b200 as bitblas
    from bitblas_b200.moe import interleave_gate_up
    mods = _gptq_mods(51 + v2, act in ("gate_up", "both"), act in ("down", "both"), v2)
    mlp = _mlp_for_gptq(T)
    (mlp.repack_from_gptq_v2 if v2 else mlp.repack_from_gptq)(*mods)
    assert (mlp.gate_up.perm is not None) == (act in ("gate_up", "both")) and mlp.down.perm is None
    lins = []
    for mod, (k, n) in zip(mods, ((H, I), (H, I), (I, H))):
        lin = bitblas.Linear(k, n, A_dtype=T, W_dtype="uint4", out_dtype=T, accum_dtype="float32", group_size=128,
                             with_scaling=True, with_zeros=True, zeros_mode="quantized", opt_M=[1, 4, 16, 64]).to(DEV)
        (lin.repack_from_gptq_v2 if v2 else lin.repack_from_gptq)(mod)
        lins.append(lin)
    lg, lu, ld = lins
    for m in (1, 4):
        x = _x(m, T, seed=m)
        y, n = _launches(lambda: mlp(x))
        assert n == (3 if act in ("gate_up", "both") else 2)
        gu = mlp.gate_up
        xs = x if gu.perm is None else x[:, gu.perm.long()].contiguous()
        h = gu.bitblas_matmul.forward_swiglu(xs, gu.qweight, gu.scales, gu.zeros)   # in down's sorted K order
        pd = torch.sort(mods[2].g_idx.long(), stable=True).indices.to(DEV)
        h_orig = h[:, torch.argsort(pd)].contiguous()
        swiglu_bound(h_orig.cpu(), interleave_gate_up(lg(x), lu(x), "bias").cpu(), T, False)
        assert torch.equal(y, ld(h_orig)), m


def test_mlp_mismatched_gate_up_g_idx():
    g, u, d = _gptq_mods(61, True, False)
    u.g_idx = torch.arange(H, dtype=torch.int32) // 128
    with pytest.raises(ValueError, match="gate and up have different g_idx"):
        _mlp_for_gptq("float16").repack_from_gptq(g, u, d)


def test_mlp_state_dict_round_trip():
    mlp = _mlp_for_gptq("float16")
    mlp.repack_from_gptq(*_gptq_mods(41, True, True))
    assert mlp.gate_up.perm is not None and mlp.down.perm is None
    x = _x(4, seed=4)
    y = mlp(x)
    fresh = _mlp_for_gptq("float16")
    fresh.load_state_dict(mlp.state_dict())
    assert fresh.gate_up.perm is not None and fresh.down.perm is None
    assert torch.equal(fresh(x), y)


def test_mlp_slab_tiled_equals_row_major():
    """propagate_b: interleave, then tile.  At m = 1 both layouts run gemv_slab and agree bit for bit; elsewhere within the bound"""
    cg, cu, cd = _mlp_parts(71)
    a = _loaded_mlp(cg, cu, cd)
    b = _loaded_mlp(cg, cu, cd, propagate_b=True)
    assert b.gate_up.bitblas_matmul.weight_tiled and not a.gate_up.bitblas_matmul.weight_tiled
    assert a.gate_up.bitblas_matmul.kernel_for(1) == b.gate_up.bitblas_matmul.kernel_for(1) == KERNEL_NAME[K_GEMV_SLAB]
    for m in (1, 16, 64):
        x = (torch.rand((m, H), generator=torch.Generator().manual_seed(m)) - 0.5).half().to(DEV)
        ga, gb = (mm.gate_up.bitblas_matmul.forward_swiglu(x, mm.gate_up.qweight, mm.gate_up.scales, mm.gate_up.zeros)
                  for mm in (a, b))
        if m == 1:
            assert torch.equal(ga, gb)
            assert torch.equal(a(x), b(x))
        else:
            pre = a.gate_up(x)
            swiglu_bound(gb.cpu(), pre.cpu(), "float16", False)
