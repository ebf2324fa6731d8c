"""GPU: every work decomposition at the SM counts of smaller Hopper parts, bit for bit.

Every launcher sizes its work from device_sm_count(): the m = 1 slab GEMV's stream-K ranges (R = 2 x SMs) and its workspace
slots, the wgmma GEMM's split-K factor, the streaming GEMV's K split (pick_ks), and the persistent grids of the grouped GEMV,
the grouped GEMM and the routing kernel.  On one device the rest of the suite runs one partition per shape.  Here
bb_set_sm_count_cap makes the library size everything as if the device had fewer SMs (an H100 PCIe has 114; a MIG slice
reports its own), and each kernel runs on the exact inputs of exact_inputs.py, compared with torch.equal against the exact
reference (SwiGLU within swiglu_bound).  Operators are built inside the capped region, so no workspace sized at another count
is reused.  A cap only ever shrinks grids: the library refuses one above the real count.

Also: the split-K partials of the wgmma GEMM and the slab's tagged slots share one workspace without overlapping, and PDL chains
give the bits of plain stream order while the capped grids leave SMs idle for the next launch's prologue.
"""
import contextlib
import ctypes
import itertools

import pytest
import torch

import exact_inputs as X
import helpers as H
import test_gpu_exact_shapes as exact_shapes   # modules, not their test functions: pytest would collect those here again
import test_gpu_grouped
import test_gpu_grouped_gemm
import test_gpu_parity
from test_exact_inputs import SLAB_CAPS, SLAB_PROPERTIES, SLAB_SHAPES, slab_cap_coverage
from test_gpu_exact_shapes import (MOE, MODES, OUTS, SLAB_CELLS, _activations, _check_experts, _experts, _routing, _slab_context,
                                   _sms, _split_shape, _tensors, check, run)
from test_gpu_kernel_grid import K_GEMM_TS, K_GEMM_TS_I8, K_GEMV_SLAB, KERNEL_NAME, _check_split, forced, ts_splits
from test_gpu_moe import CHAIN as BLOCK_CHAIN
from test_gpu_moe import _check_route, pdl_chain_matches_plain_stream_order
from test_gpu_moe_gather import CHAIN as GATHER_CHAIN
from test_gpu_moe_gather import _check_route_index

pytestmark = pytest.mark.gpu

DEV = "cuda"
SHARD = (1024, 3584)   # a tensor-parallel shard of SLAB_SHAPES, run at every SM count


def _slab_witness_desc():
    """an m = 1 configuration the slab kernel takes: its bb_workspace_bytes is the slot region at the current count"""
    from bitblas_b200 import _lib
    d = _lib.MatmulDesc()
    d.N, d.K, d.a_dtype, d.w_fmt, d.w_bits = 1024, 1024, _lib.BB_F16, _lib.BB_W_UINT, 4
    d.accum_dtype, d.out_dtype, d.group_size = _lib.BB_F32, _lib.BB_F16, -1
    return d


@contextlib.contextmanager
def sm_cap(cap):
    """the library sizes every decomposition for `cap` SMs inside the block (checked through the slab's workspace size:
    [2 CTAs per SM][2 groups][32 rows] 8-byte slots + 256); the previous cap is restored on the way out"""
    from bitblas_b200 import _lib
    lib = _lib.load()
    prev = lib.bb_set_sm_count_cap(cap)
    assert prev >= 0, _lib.last_error()
    try:
        assert lib.bb_workspace_bytes(ctypes.byref(_slab_witness_desc()), 1) == X.slab_slot_bytes(cap), cap
        yield cap
    finally:
        lib.bb_set_sm_count_cap(prev)


def test_cap_is_refused_above_the_device_count():
    from bitblas_b200 import _lib
    lib = _lib.load()
    with sm_cap(7):
        assert lib.bb_set_sm_count_cap(_sms() + 1) < 0 and b"bb_set_sm_count_cap" in lib.bb_last_error()
        assert lib.bb_set_sm_count_cap(-1) < 0
        assert lib.bb_workspace_bytes(ctypes.byref(_slab_witness_desc()), 1) == X.slab_slot_bytes(7)
    assert lib.bb_workspace_bytes(ctypes.byref(_slab_witness_desc()), 1) == X.slab_slot_bytes(_sms())


# ---- slab decode GEMV: stream-K ranges and fix-up ----------------------------------------------------------------------------------
def test_slab_caps_cover_stream_k_properties():
    hit = slab_cap_coverage(_sms())
    print(f"\nslab stream-K coverage of SLAB_SHAPES at capped SM counts on {torch.cuda.get_device_name()} ({_sms()} SMs):")
    for p in sorted(SLAB_PROPERTIES):
        print(f"  {p:28s} {hit.get(p, [])}")
    for p in SLAB_PROPERTIES:
        assert len(hit.get(p, [])) >= 3 and min(hit[p]) < 8, (p, hit.get(p))


@pytest.mark.parametrize("first", range(1, 133, 33))
def test_slab_shard_every_sm_count(first):
    """the shard shape at every SM count 1 .. device count (R = 2 .. 2 x SMs ranges), 33 counts per test: the device side of
    test_slab_fixup_protocol_every_sm_count; mode, activation type, output type, group size and storage rotate with the count"""
    N, K = SHARD
    if first > _sms():
        pytest.skip(f"this device has {_sms()} SMs")
    for cap in range(first, min(first + 33, _sms() + 1)):
        mode, T = MODES[cap % 5], ("float16", "bfloat16")[(cap // 5) % 2]
        case = X.make_exact_case(1, N, K, A_dtype=T, W_dtype="int4" if mode in ("none", "scale") and cap % 2 else "uint4",
                                 out_dtype=OUTS[cap % 3], group_size=(128, 512, 896, -1)[cap % 4] if mode != "none" else -1,
                                 mode=mode, bias=cap % 2 == 0, fast_decoding=cap % 4 < 2, seed=cap)
        with sm_cap(cap):
            _, got = run(case, K_GEMV_SLAB)
        check(case, got, f"gemv_slab {N}x{K} {mode} {T} on {cap} SMs", _slab_context(N, K, cap))


@pytest.mark.parametrize("N,K", [s for s in SLAB_SHAPES if s != SHARD], ids=str)
def test_slab_shapes_at_caps(N, K):
    """the production and padding shapes at SLAB_CAPS and the device count, rotating over the shape's cells of test_slab_exact"""
    cells = [c for c in SLAB_CELLS if (c["N"], c["K"]) == (N, K)]
    for j, cap in enumerate(sorted(set(SLAB_CAPS) | {_sms()})):
        c = cells[j % len(cells)]
        case = X.make_exact_case(1, N, K, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"], mode=c["mode"],
                                 bias=c["bias"], fast_decoding=c["il"], seed=N + K + cap)
        with sm_cap(cap):
            _, got = run(case, K_GEMV_SLAB)
        check(case, got, f"gemv_slab on {cap} SMs {c}", _slab_context(N, K, cap))


@pytest.mark.parametrize("cap", [2, 66])
def test_slab_fp4_and_tiled_storage_at_caps(cap):
    with sm_cap(cap):
        for N, K in [(8192, 8192), SHARD]:
            case = X.make_exact_case(1, N, K, A_dtype="bfloat16" if N == K else "float16", W_dtype="fp4_e2m1", group_size=128,
                                     mode="scale", bias=True, out_dtype="float32", seed=N + cap)
            _, got = run(case, K_GEMV_SLAB)
            check(case, got, f"gemv_slab fp4 {N}x{K} on {cap} SMs", _slab_context(N, K, cap), families=("sum",))
        for N, K in [(8192, 8192), (1024, 8192)]:
            case = X.make_exact_case(1, N, K, group_size=128, mode="quantized", bias=True, fast_decoding=True, seed=N + cap,
                                     propagate_b=True)
            op, got = run(case, K_GEMV_SLAB)
            assert op.weight_tiled
            check(case, got, f"gemv_slab tiled {N}x{K} on {cap} SMs", _slab_context(N, K, cap))


@pytest.mark.parametrize("cap", [1, 33, None], ids=["1", "33", "device"])
def test_slab_reproducible_at_a_cap(cap):
    """random (inexact) inputs: two runs on the same SM count are bit-identical (the fix-up adds the parked partials in a fixed
    order).  Runs on different counts may differ: the summation order follows the ranges"""
    cap = cap or _sms()
    case = H.make_case(1, 12288, 12288, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                       zeros_mode="quantized", seed=cap)
    with sm_cap(cap):
        op = H.product_operator(case)
        assert op.kernel_for(1) == "gemv_slab"
        first = H.run_product(op, case)
        second = H.run_product(op, case)
    assert torch.equal(first, second)


# ---- streaming GEMV: the K split of pick_ks ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 8, 33, 114])
def test_gemv_k_split_at_caps(cap):
    """with fewer SMs pick_ks keeps fewer warps per CTA, or takes the full split over several waves, at grids where the device
    count keeps the full split in one wave"""
    if cap > _sms():
        pytest.skip(f"{cap} SMs is above this device's {_sms()}")
    with sm_cap(cap):
        for m in (1, 2, 5, 8, 9, 17, 32):
            exact_shapes.test_gemv_mma_k_split_mid_group(m)
        for m, N in ((4, 12288), (24, 28672)):
            exact_shapes.test_gemv_mma_k_split_grid_sizes(m, N)
        for i, (N, K) in enumerate([(8192, 8192), (28672, 8192), (8192, 28672), (12288, 12288)]):
            exact_shapes.test_gemv_mma_bench_shapes(N, K, (2, 8, 16)[(i + cap) % 3])
        for m in (1, 12):
            exact_shapes.test_gemv_i8_k_split(m)


# ---- wgmma GEMM: split-K --------------------------------------------------------------------------------------------------------
SPLIT_CAPS = [8, 16, 33, 66, 114]
SPLIT_ROWS = [(1, "float16", "original"), (40, "bfloat16", "rescale"), (100, "float16", "quantized")]


@pytest.mark.parametrize("cap", SPLIT_CAPS)
def test_gemm_ts_every_split_factor_at_cap(cap):
    """every factor f = 2..8 on `cap` SMs, for 16-bit and int8 activations; the factor asserted through bb_workspace_bytes"""
    if cap > _sms():
        pytest.skip(f"{cap} SMs is above this device's {_sms()}")
    with sm_cap(cap):
        for f in range(2, 9):
            m, T, mode = SPLIT_ROWS[(f + cap) % 3]
            N, K, g = _split_shape(f, m, 64, cap)
            case = X.make_exact_case(m, N, K, A_dtype=T, group_size=g, mode=mode, bias=f % 2 == 0, out_dtype=OUTS[(f + cap) % 3],
                                     fast_decoding=m % 2 == 0, seed=f * 7 + m + cap)
            op, got = run(case, K_GEMM_TS)
            with forced(K_GEMM_TS):
                _check_split(op, m, True, 64, sms=cap)
            check(case, got, f"gemm_ts split {f} ({N}x{K} g={g} m={m}) on {cap} SMs", families=("sum",))

            N, K, _ = _split_shape(f, 16, 128, cap)
            out = ("int32", "int8", "float32", "float16", "bfloat16")[(f + cap) % 5]
            case = X.make_exact_case(16, N, K, A_dtype="int8", W_dtype="int2", out_dtype=out, bias=f % 2 == 1, fast_decoding=True,
                                     seed=f + cap)
            if out in ("float16", "bfloat16"):
                case["A"] = (case["A"] // 8).to(torch.int8)   # keeps the int32 sum inside fp16's exact integers
            op, got = run(case, K_GEMM_TS_I8)
            with forced(K_GEMM_TS_I8):
                _check_split(op, 16, True, 128, sms=cap)
            X.compare_exact(got, X.exact_reference(case), f"gemm_ts_i8 split {f} ({N}x{K}) out={out} on {cap} SMs")


def test_gemm_ts_does_not_split_on_one_sm():
    """shapes that split 2..8 ways on the device run unsplit on one SM (bb_workspace_bytes 0), and stay exact"""
    with sm_cap(1):
        for f in (2, 4, 8):
            m, T, mode = SPLIT_ROWS[f % 3]
            N, K, g = _split_shape(f, m, 64, _sms())
            assert ts_splits(m, N, K, 64, 1) == 1
            case = X.make_exact_case(m, N, K, A_dtype=T, group_size=g, mode=mode, bias=True, out_dtype=OUTS[f % 3], seed=f)
            op, got = run(case, K_GEMM_TS)
            with forced(K_GEMM_TS):
                _check_split(op, m, False, 64, sms=1)
            check(case, got, f"gemm_ts unsplit ({N}x{K} m={m}) on 1 SM", families=("sum",))


# ---- grouped kernels and routing -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [1, 7, 66])
@pytest.mark.parametrize("model", list(MOE))
def test_grouped_moe_at_caps(model, cap):
    """gate/up of each model on `cap` SMs: the grouped GEMV at the single-launch limit, the grouped wgmma GEMM above it (on one
    SM one or two CTAs walk every tile through one mbarrier ring), both SwiGLU forms, and the GEMM gathering token rows"""
    from bitblas_b200.ops import general_matmul as GM
    E, topk = MOE[model]["E"], MOE[model]["topk"]
    limit = GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP
    with sm_cap(cap):
        op, cases, W, s, z, b = _experts(model, "gate_up", seed=len(model) + cap)
        for tokens, path, seed in [(limit * E // topk, "gemv", 11), ((limit + 4) * E * 2 // topk, "gemm", 12)]:
            counts, row_token = _routing(E, topk, tokens, seed + cap)
            T = sum(counts)
            off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
            A = _activations(model, "gate_up", T, seed)
            what = f"{model} {path} T={T} on {cap} SMs"
            got = op.forward_grouped(A.to(DEV), W, off, scale=s, zeros=z, bias=b, capturable=path == "gemm").cpu()
            _check_experts(cases, A, counts, got, what, path)
            got = op.forward_grouped_swiglu(A.to(DEV), W, off, scale=s, zeros=z, bias=b).cpu()
            _check_experts(cases, A, counts, got, f"swiglu {what}", path, swiglu=True)
            if path == "gemm":
                A_tok = _activations(model, "gate_up", tokens, seed)
                got = op.forward_grouped_swiglu(A_tok.to(DEV), W, off, scale=s, zeros=z, bias=b, row_index=row_token.to(DEV)).cpu()
                _check_experts(cases, A_tok[row_token.long()], counts, got, f"gathering swiglu {what}", path, swiglu=True)


@pytest.mark.parametrize("cap", [1, 2, 66])
def test_route_at_caps(cap):
    """moe_route against route_reference and moe_route_index against moe_route, k = 8, up to 4100 tokens (32800 slots)"""
    with sm_cap(cap):
        for E, T in [(8, 1), (128, 300), (64, 4100), (256, 4100)]:
            g = torch.Generator().manual_seed(E * 1000 + T + cap)
            ids = torch.randint(0, E, (T, 8), generator=g, dtype=torch.int32)
            drop = torch.rand((T, 8), generator=g)
            ids[drop < 0.05] = -1
            ids[drop > 0.95] = E
            x = (torch.rand((T, 64), generator=g) - 0.5).to(torch.bfloat16 if T % 2 else torch.float16)
            _check_route(ids, x, E)
            _check_route_index(ids, E)


# ---- PDL chains with idle SMs ------------------------------------------------------------------------------------------------------
# on a capped count the next kernel's pre-wait prologue (weight and parameter prefetch) overlaps the whole of its predecessor, not
# only its tail.  Each chain runs once.
@pytest.mark.parametrize("cap", [33, 66])
def test_pdl_chains_with_idle_sms(cap):
    """the decode GEMV, grouped GEMV and grouped GEMM chains against the same calls with a synchronisation after each"""
    with sm_cap(cap):
        test_gpu_parity.test_gemv_pdl_dependent_chain()
        test_gpu_grouped.test_grouped_pdl_dependent_chain()
        test_gpu_grouped_gemm.test_grouped_gemm_pdl_dependent_chain()


@pytest.mark.parametrize("chain", ["block", "gathering_block"])
@pytest.mark.parametrize("cap", [33, 66])
def test_moe_block_pdl_chains_with_idle_sms(cap, chain, tmp_path):
    """the mixture-of-experts block chains in child processes against BB_PDL=0 (read once per process); the child sets the cap"""
    prologue = f"from bitblas_b200 import _lib\nassert _lib.load().bb_set_sm_count_cap({cap}) == 0, _lib.last_error()"
    pdl_chain_matches_plain_stream_order(BLOCK_CHAIN if chain == "block" else GATHER_CHAIN, tmp_path, prologue)


# ---- one workspace for every m ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap,N", [(None, 4096), (33, 1024)], ids=["device", "33"])   # split-K 4 ways on 132 and on 33 SMs
def test_splitk_partials_leave_the_slab_slots_zero(cap, N):
    """include/bitblas_b200.h: a zero-initialised buffer serves later calls on the same stream.  A split-K call at m = 16 and then
    an m = 1 slab call share one buffer: the slots (the first slab_slot_bytes) are still zero when the m = 1 call starts, and
    both outputs are exact.  Through the C ABI with a caller-owned buffer, then through Matmul.forward's own workspace."""
    from bitblas_b200 import _lib
    K = 4096
    with sm_cap(cap) if cap else contextlib.nullcontext():
        cap = cap or _sms()
        c16 = X.make_exact_case(16, N, K, group_size=128, mode="original", bias=True, fast_decoding=True, seed=16)
        c1 = dict(c16, A=c16["A"][:1], M=1)
        slots = X.slab_slot_bytes(cap)
        ref16, ref1 = X.exact_reference(c16, DEV).cpu(), X.exact_reference(c1, DEV).cpu()
        X.prove_exact(c16, ("sum",), device=DEV)
        X.prove_exact(c1, device=DEV)

        op = X.product_operator(c16, M=[1, 16])
        assert op.kernel_for(16) == KERNEL_NAME[K_GEMM_TS] and op.kernel_for(1) == KERNEL_NAME[K_GEMV_SLAB]
        assert ts_splits(16, N, K, 64, cap) > 1   # (the exact size of the split-K workspace is checked at the end)
        t = _tensors(op, c16)
        lib = _lib.load()
        need = [lib.bb_workspace_bytes(ctypes.byref(op._desc), m) for m in (16, 1)]
        assert need[1] == slots and need[0] > 0
        ws = torch.zeros(max(need), dtype=torch.uint8, device=DEV)
        A = c16["A"].to(DEV)
        outs = [torch.empty((m, N), dtype=torch.float16, device=DEV) for m in (16, 1)]
        stream = torch.cuda.current_stream().cuda_stream
        for m, C in zip((16, 1), outs):
            if m == 1:
                torch.cuda.synchronize()
                assert int(ws[:slots].count_nonzero()) == 0, "the split-K call left data in the slab's slots"
            _lib.call("bb_matmul", torch.cuda.current_device(), op._desc_ref, A.data_ptr(), t["W"].data_ptr(), 0,
                      t["scale"].data_ptr(), t["zeros"].data_ptr(), t["bias"].data_ptr(), C.data_ptr(), m, ws.data_ptr(),
                      ws.numel(), stream)
        torch.cuda.synchronize()
        X.compare_exact(outs[0].cpu(), ref16, f"C ABI m = 16 on {cap} SMs")
        X.compare_exact(outs[1].cpu(), ref1, f"C ABI m = 1 after split-K on {cap} SMs")

        op = X.product_operator(c16, M=[1, 16])
        t = _tensors(op, c16)
        got16 = op.forward(A, t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
        torch.cuda.synchronize()
        (buf,) = op._ws.values()
        assert buf.numel() >= slots and int(buf[:slots].count_nonzero()) == 0, "the split-K call left data in the slab's slots"
        got1 = op.forward(A[:1], t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
        torch.cuda.synchronize()
        X.compare_exact(got16.cpu(), ref16, f"Matmul.forward m = 16 on {cap} SMs")
        X.compare_exact(got1.cpu(), ref1, f"Matmul.forward m = 1 after split-K on {cap} SMs")
        with forced(K_GEMM_TS):
            _check_split(op, 16, True, 64, sms=cap)
