"""GPU: every work decomposition at production shapes, bit for bit, on inputs for which every kernel must be exact.

The inputs (exact_inputs.py) are dyadic and small enough that every fp32 partial sum any kernel forms is exact whatever its
summation order, split-K factor, stream-K ranges or K split; `prove_exact` checks that precondition per case.  Each kernel's
output must then equal round(V) of the exact result (with bias round(round(V) + b)) in every bit: `torch.equal`, no tolerance.
The float64 reference is computed on the device (exact under the precondition; test_reference_device_equals_cpu shows it).

Decompositions covered: the slab decode GEMV's stream-K ranges and fix-up at the bench.py and tensor-parallel shard shapes (the
partition is mirrored and its coverage asserted on this device's SM count), the streaming GEMV's K split with warps starting
inside a group, every wgmma split-K factor 2..8 with splits starting inside a group, M = 4096 with all rows, the grouped GEMV,
grouped GEMM and per-expert path at mixture-of-experts shapes, their SwiGLU epilogues (grouped GEMV, grouped GEMM, and the GEMM
that gathers token rows; compared with silu(g) * u from the exact pre-activations within one ulp), and the scatter epilogue with
1, 2 and 8 destinations.
"""
import itertools

import pytest
import torch

import exact_inputs as X
from test_exact_inputs import SLAB_PROPERTIES, SLAB_SHAPES, SMALL_SM_PROPERTIES
from test_gpu_moe import swiglu_bound
from test_gpu_kernel_grid import (K_GEMM_TS, K_GEMM_TS_I8, K_GEMV_I8, K_GEMV_MMA, K_GEMV_SLAB, K_GENERIC, KERNEL_NAME, _check_split,
                                  forced, ts_bm, ts_splits)

pytestmark = pytest.mark.gpu

DEV = "cuda"
OUTS = ["float16", "bfloat16", "float32"]
MODES = ["none", "scale", "original", "rescale", "quantized"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tensors(op, case):
    t = dict(W=X.product_weight(op, case, DEV))
    for k in ("scale", "zeros", "bias"):
        t[k] = case[k].to(DEV) if case[k] is not None else None
    return t


def run(case, kernel_id=None, m=None, t=None, op=None):
    """the case through Matmul.forward (kernel_id: forced, and asserted through kernel_for); returns (op, output on the host)"""
    op = op or X.product_operator(case)
    m = case["M"] if m is None else m
    t = t or _tensors(op, case)
    A = case["A"].to(DEV)
    if kernel_id is None:
        out = op.forward(A, t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    else:
        with forced(kernel_id):
            assert op.kernel_for(m) == KERNEL_NAME[kernel_id], (op.kernel_for(m), case["cfg"])
            out = op.forward(A, t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"])
    torch.cuda.synchronize()
    return op, out.cpu()


def check(case, got, what, context=None, families=("sum", "slab", "gemv")):
    X.prove_exact(case, families, device=DEV)
    X.compare_exact(got, X.exact_reference(case, DEV), what, context)


# ---- the reference itself ------------------------------------------------------------------------------------------------------------
def test_reference_device_equals_cpu():
    case = X.make_exact_case(64, 512, 3840, mode="original", group_size=384, bias=True, out_dtype="bfloat16", seed=3)
    X.compare_exact(X.exact_reference(case, DEV), X.exact_reference(case, "cpu"), "device vs CPU reference")
    assert torch.equal(X.exact_value(case, DEV).cpu(), X.exact_value(case, "cpu"))


def test_generic_simt_reproduces_the_exact_reference():
    """IEEE fmaf on CUDA cores: if this is not exact the inputs are wrong, not the fast kernels"""
    for i, (mode, T) in enumerate(itertools.product(MODES, ["float16", "bfloat16"])):
        case = X.make_exact_case(3, 256, 8192, A_dtype=T, W_dtype="int4" if mode == "none" else "uint4", group_size=512,
                                 mode=mode, bias=i % 2 == 0, out_dtype=OUTS[i % 3], fast_decoding=i % 2 == 1, seed=i)
        _, got = run(case, K_GENERIC)
        check(case, got, f"generic_simt {mode} {T}")


# ---- slab decode GEMV: stream-K at production shapes ------------------------------------------------------------------------------
def _slab_context(N, K, sms=None):
    sms = sms or _sms()
    UPR, NRB, T, R = X.slab_geometry(N, K, sms)
    spans = X.slab_ranges_of_block(N, K, sms)
    return lambda r, n: f"(row block {n // 32}, CTAs {[R - 1 - ri for ri in spans.get(n // 32, [])]} of {R})"


def test_slab_shapes_cover_stream_k_properties_here():
    hit = {}
    for N, K in SLAB_SHAPES:
        for p in X.slab_coverage(N, K, _sms()):
            hit.setdefault(p, []).append((N, K))
    print(f"\nslab stream-K coverage on {torch.cuda.get_device_name()} ({_sms()} SMs):")
    for p in sorted(SLAB_PROPERTIES):
        print(f"  {p:28s} {hit.get(p, [])}")
    want = SLAB_PROPERTIES - SMALL_SM_PROPERTIES   # the rest: test_gpu_sm_counts.py at capped SM counts
    assert want <= set(hit), want - set(hit)


def _slab_cells():
    cells = []
    for i, (N, K) in enumerate(SLAB_SHAPES):
        for j, (mode, T) in enumerate(itertools.product(MODES, ["float16", "bfloat16"])):
            k = i + j
            if k % 2:   # half of the mode x dtype cells per shape, alternating between shapes
                continue
            cells.append(dict(N=N, K=K, mode=mode, T=T, W="int4" if mode in ("none", "scale") and k % 4 else "uint4",
                              il=k % 4 == 0, out=OUTS[k % 3], bias=k % 4 < 2, g=(128, -1, 256)[k % 3] if mode != "none" else -1))
    return cells


SLAB_CELLS = _slab_cells()


@pytest.mark.parametrize("c", SLAB_CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_slab_exact(c):
    case = X.make_exact_case(1, c["N"], c["K"], A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"], group_size=c["g"],
                             mode=c["mode"], bias=c["bias"], fast_decoding=c["il"], seed=c["N"] + c["K"] + len(c["mode"]))
    _, got = run(case, K_GEMV_SLAB)
    check(case, got, f"gemv_slab {c}", _slab_context(c["N"], c["K"]))


@pytest.mark.parametrize("N,K", [(8192, 8192), (1024, 3584), (4112, 6144)], ids=str)
@pytest.mark.parametrize("T", ["float16", "bfloat16"])
def test_slab_fp4_exact(N, K, T):
    case = X.make_exact_case(1, N, K, A_dtype=T, W_dtype="fp4_e2m1", group_size=128, mode="scale", bias=True,
                             out_dtype="float32" if T == "float16" else "bfloat16", seed=N + K)
    _, got = run(case, K_GEMV_SLAB)
    check(case, got, f"gemv_slab fp4 {N}x{K} {T}", _slab_context(N, K), families=("sum",))


@pytest.mark.parametrize("mode", ["original", "rescale", "quantized", "scale"])
def test_slab_fast_and_slow_parameter_paths(mode):
    """g = 128, N % 32 == 0: the 16-byte parameter copies; the same case with the scale (and zeros) tensor starting 8 bytes into
    its buffer takes the synchronous loads; both exact"""
    N, K = 8192, 8192
    case = X.make_exact_case(1, N, K, group_size=128, mode=mode, bias=True, fast_decoding=True, seed=11)
    op = X.product_operator(case)
    t = _tensors(op, case)
    _, fast = run(case, K_GEMV_SLAB, op=op, t=t)
    check(case, fast, f"slab fast params {mode}", _slab_context(N, K))
    for k in ("scale", "zeros") if mode in ("original", "rescale") else ("scale",):
        buf = torch.empty(t[k].numel() * t[k].element_size() + 8, dtype=torch.uint8, device=DEV)
        view = buf[8:].view(t[k].dtype).view(t[k].shape)
        view.copy_(t[k])
        assert view.data_ptr() % 16 == 8
        t[k] = view
    _, slow = run(case, K_GEMV_SLAB, op=X.product_operator(case), t=t)
    X.compare_exact(slow, fast, f"slab slow params {mode}")


@pytest.mark.parametrize("N,K", [(8192, 8192), (1024, 8192), (12288, 12288)], ids=str)
def test_slab_tiled_storage_exact(N, K):
    case = X.make_exact_case(1, N, K, group_size=128, mode="quantized", bias=True, fast_decoding=True, seed=N, propagate_b=True)
    op, got = run(case, K_GEMV_SLAB)
    assert op.weight_tiled
    check(case, got, f"slab tiled {N}x{K}", _slab_context(N, K))


# ---- gemv_mma / gemv_i8: the K split ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", list(range(1, 33)))
def test_gemv_mma_k_split_mid_group(m):
    """K = 3840 (30 steps) at g = 256, 384, 640: whichever ks the host picks, some warp starts inside a group for one of them;
    m = 2..8 through the dispatcher, 1 and 9..32 forced"""
    kid = None if 2 <= m <= 8 else K_GEMV_MMA
    for i, g in enumerate((256, 384, 640)):
        mode = MODES[(m + i) % 5]
        T = ("float16", "bfloat16")[(m + i) % 2]
        case = X.make_exact_case(m, 1024, 3840, A_dtype=T, W_dtype="uint4" if mode != "none" else "int4",
                                 group_size=g if mode != "none" else -1, mode=mode, bias=(m + i) % 3 == 0,
                                 out_dtype=OUTS[(m + i) % 3], fast_decoding=(m + i) % 2 == 0, seed=100 * m + i)
        op, got = run(case, kid)
        if kid is None:
            assert op.kernel_for(m) == "gemv_mma"
        check(case, got, f"gemv_mma m={m} g={g} {mode} {T}", families=("sum", "gemv"))


@pytest.mark.parametrize("N", [12288, 16384, 28672])
@pytest.mark.parametrize("m", [4, 24])
def test_gemv_mma_k_split_grid_sizes(m, N):
    """the same K = 3840 groups at row counts whose grids (768 .. 1792 CTAs) no longer fit the full K split in one wave, so the
    host picks a smaller ks, or the full split again over several waves (pick_ks); the ks itself is not visible from outside,
    and test_gemv_k_split_starts_mid_group shows that every ks = 2..8 has a mid-group start for one of these g"""
    for i, g in enumerate((256, 384, 640)):
        mode = ("original", "rescale", "quantized")[i]
        T = ("float16", "bfloat16")[(m + i) % 2]
        case = X.make_exact_case(m, N, 3840, A_dtype=T, group_size=g, mode=mode, bias=i == 1, out_dtype=OUTS[(m + i) % 3],
                                 fast_decoding=i != 2, seed=N + m + i)
        _, got = run(case, K_GEMV_MMA)
        check(case, got, f"gemv_mma m={m} N={N} g={g} {mode} {T}", families=("sum", "gemv"))


@pytest.mark.parametrize("K", [29 * 128, 31 * 128])
@pytest.mark.parametrize("m", [1, 4, 16, 32])
def test_gemv_mma_prime_steps(K, m):
    for g in (128, -1):
        for mode, T in (("original", "float16"), ("rescale", "bfloat16"), ("quantized", "float16")):
            case = X.make_exact_case(m, 2048, K, A_dtype=T, group_size=g, mode=mode, bias=True, fast_decoding=g == 128, seed=K + m)
            _, got = run(case, K_GEMV_MMA)
            check(case, got, f"gemv_mma K={K} m={m} g={g} {mode}", families=("sum", "gemv"))


@pytest.mark.parametrize("N,K", [(8192, 8192), (28672, 8192), (8192, 28672), (12288, 12288)], ids=str)
@pytest.mark.parametrize("m", [2, 8, 16])
def test_gemv_mma_bench_shapes(N, K, m):
    """multi-wave grids at the bench.py shapes"""
    case = X.make_exact_case(m, N, K, group_size=128, mode="quantized", bias=m == 8, fast_decoding=True, seed=N + K + m,
                             out_dtype="bfloat16" if m == 16 else "float16")
    _, got = run(case, K_GEMV_MMA)
    check(case, got, f"gemv_mma m={m} {N}x{K}", families=("sum", "gemv"))


@pytest.mark.parametrize("m", [1, 5, 12, 32])
def test_gemv_i8_k_split(m):
    for K in (3840, 31 * 128, 8192):
        case = X.make_exact_case(m, 2048, K, A_dtype="int8", W_dtype="int2", out_dtype="int32", bias=True, fast_decoding=True,
                                 seed=K + m)
        _, got = run(case, K_GEMV_I8)
        X.compare_exact(got, X.exact_reference(case), f"gemv_i8 m={m} K={K}")


# ---- wgmma GEMM: every split-K factor ----------------------------------------------------------------------------------------------
def _split_shape(f, m, kb, sms):
    """(N, K, g) whose split-K factor is f at m rows, preferring K of production shards and a group size that makes a split start
    inside a group"""
    for K in (3584, 2560, 3072, 4096, 5120, 6144, 7168, 8192, 1536, 1024, 2048, 12288, 14336):
        for N in (128 * t for t in range(1, 64)):
            if ts_splits(m, N, K, kb, sms) == f:
                per = K // f
                g = next((g for g in range(128, K, 128) if K % g == 0 and per % g), 128)
                return N, K, g
    raise AssertionError(f"no shape splits {f} ways on {sms} SMs")


# the output type follows f (every triple meets all three over f = 2..8), bias follows f + the triple: each triple gets every
# (output type, bias) pair
SPLIT_CELLS = [dict(f=f, m=m, T=T, mode=mode, out=OUTS[(i // 3) % 3], bias=i % 2 == 0)
               for i, (f, (m, T, mode)) in enumerate(itertools.product(range(2, 9), [(1, "float16", "original"), (40, "bfloat16", "rescale"),
                                                                                     (100, "float16", "quantized")]))]


@pytest.mark.parametrize("c", SPLIT_CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_gemm_ts_split_factor(c):
    N, K, g = _split_shape(c["f"], c["m"], 64, _sms())
    case = X.make_exact_case(c["m"], N, K, A_dtype=c["T"], group_size=g, mode=c["mode"], bias=c["bias"], out_dtype=c["out"],
                             fast_decoding=c["m"] % 2 == 0, seed=c["f"] * 7 + c["m"])
    op, got = run(case, K_GEMM_TS)
    with forced(K_GEMM_TS):
        _check_split(op, c["m"], True, 64)
    check(case, got, f"gemm_ts split {c['f']} ({N}x{K} g={g}) {c}", families=("sum",))


@pytest.mark.parametrize("f", range(2, 9))
@pytest.mark.parametrize("out", ["int32", "int8", "float32", "float16", "bfloat16"])
def test_gemm_ts_i8_split_factor(f, out):
    N, K, _ = _split_shape(f, 16, 128, _sms())
    case = X.make_exact_case(16, N, K, A_dtype="int8", W_dtype="int2", out_dtype=out, bias=f % 2 == 0, fast_decoding=True,
                             seed=f)
    if out in ("float16", "bfloat16"):
        case["A"] = (case["A"] // 8).to(torch.int8)   # keeps the int32 sum inside fp16's exact integers
    op, got = run(case, K_GEMM_TS_I8)
    with forced(K_GEMM_TS_I8):
        _check_split(op, 16, True, 128)
    X.compare_exact(got, X.exact_reference(case), f"gemm_ts_i8 split {f} out={out}")


@pytest.mark.parametrize("W", ["fp4_e2m1", "e4m3_float8", "e5m2_float8"])
@pytest.mark.parametrize("m", [20, 64, 200])
def test_gemm_ts_fp4_fp8_exact(W, m):
    N, K, g = (1024, 3584, 512) if m <= 128 else (2048, 4096, 128)
    case = X.make_exact_case(m, N, K, A_dtype="bfloat16" if m == 64 else "float16", W_dtype=W, group_size=g, mode="scale",
                             bias=True, out_dtype=OUTS[m % 3], seed=m)
    _, got = run(case, K_GEMM_TS)
    check(case, got, f"gemm_ts {W} m={m}", families=("sum",))


@pytest.mark.parametrize("m", [32, 64, 128])
def test_gemm_ts_tiled_storage(m):
    case = X.make_exact_case(m, 4096, 4096, group_size=128, mode="original", bias=True, fast_decoding=True, seed=m,
                             propagate_b=True)
    assert ts_bm(m) == m
    op, got = run(case, K_GEMM_TS)
    assert op.weight_tiled
    check(case, got, f"gemm_ts tiled m={m}", families=("sum",))


@pytest.mark.parametrize("N,K", [(12288, 12288), (8192, 8192), (28672, 8192), (8192, 28672)], ids=str)
def test_gemm_ts_m4096_all_rows(N, K):
    case = X.make_exact_case(4096, N, K, group_size=128, mode="quantized", fast_decoding=True, seed=N + K,
                             out_dtype="float16" if N == K else "bfloat16")
    _, got = run(case, K_GEMM_TS)
    check(case, got, f"gemm_ts M=4096 {N}x{K}", families=("sum",))


# ---- grouped kernels at mixture-of-experts shapes ---------------------------------------------------------------------------------
MOE = {"mixtral-8x7b": dict(E=8, topk=2, gate_up=(28672, 4096), down=(4096, 14336)),
       "qwen3-30b-a3b": dict(E=128, topk=8, gate_up=(1536, 2048), down=(2048, 768)),
       "deepseek-v2-lite": dict(E=64, topk=6, gate_up=(2816, 2048), down=(2048, 1408))}
# one expert configuration per model: activation type, zero-point mode, bias and output type all vary across the shapes
MOE_CFG = {"mixtral-8x7b": dict(A_dtype="float16", mode="quantized", bias=False, out_dtype="float16"),
           "qwen3-30b-a3b": dict(A_dtype="bfloat16", mode="original", bias=True, out_dtype="bfloat16"),
           "deepseek-v2-lite": dict(A_dtype="float16", mode="rescale", bias=True, out_dtype="float32")}


def _experts(model, proj, seed):
    """E experts of the model's projection (one row of activations each; the tests pass their own)"""
    N, K = MOE[model][proj]
    cases = [X.make_exact_case(1, N, K, group_size=128, fast_decoding=True, seed=seed * 131 + e, **MOE_CFG[model])
             for e in range(MOE[model]["E"])]
    op = X.product_operator(cases[0], M=[1, 16])
    W = torch.stack([X.product_weight(op, x, DEV) for x in cases])
    st = lambda k: torch.stack([x[k] for x in cases]).to(DEV) if cases[0][k] is not None else None   # noqa: E731
    return op, cases, W, st("scale"), st("zeros"), st("bias")


def _activations(model, proj, rows, seed):
    N, K = MOE[model][proj]
    return X.make_exact_case(rows, 32, K, group_size=128, seed=seed, **MOE_CFG[model])["A"]


def _routing(E, topk, tokens, seed):
    """top-k distinct experts per token, sorted by expert: (counts, row_token of each sorted row)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.rand((tokens, E), generator=g).argsort(1)[:, :topk].flatten()
    order = torch.argsort(ids, stable=True)
    return torch.bincount(ids, minlength=E).tolist(), (order // topk).to(torch.int32)


def _expected_path(op, T, E, single):
    """the host rule of forward_grouped, mirrored: one grouped launch up to GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E rows (the
    grouped GEMV); above it the grouped wgmma GEMM when the call must be one launch (capturable, SwiGLU) and N % 128 == 0,
    else one bb_matmul per expert"""
    from bitblas_b200.ops import general_matmul as GM
    if T <= GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E:
        return "gemv"
    return "gemm" if single and op.N % 128 == 0 else "per_group"


def _launches(fn):
    from bitblas_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out.cpu(), lib.bb_launch_count() - n0


def _check_experts(cases, A, counts, got, what, path, swiglu=False):
    off = [0] + list(itertools.accumulate(counts))
    for e, x in enumerate(cases):
        if not counts[e]:
            continue
        xe = dict(x, A=A[off[e]:off[e + 1]], M=counts[e])
        X.prove_exact(xe, ("sum", "gemv") if path == "gemv" else ("sum",), device=DEV)
        ref = X.exact_reference(xe, DEV).cpu()
        rows = slice(off[e], off[e + 1])
        if swiglu:   # silu(g) * u in float64 from the exact pre-activations, within swiglu_bound's one ulp (fp32: four)
            swiglu_bound(got[rows], ref, x["cfg"]["out_dtype"], x["bias"] is not None)
        else:
            X.compare_exact(got[rows], ref, f"{what} expert {e} of {len(counts)}")


@pytest.mark.parametrize("proj", ["gate_up", "down"])
@pytest.mark.parametrize("model", list(MOE))
def test_grouped_moe_shapes(model, proj):
    """a decode routing at the single-launch limit (GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP rows per expert on average: the
    grouped GEMV) and a prefill routing above it through the grouped wgmma GEMM (capturable) and the per-expert path"""
    from bitblas_b200.ops import general_matmul as GM
    E, topk = MOE[model]["E"], MOE[model]["topk"]
    limit = GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP
    op, cases, W, s, z, b = _experts(model, proj, seed=len(model) + len(proj))
    runs = [(limit * E // topk, False, 2), ((limit + 4) * E * 2 // topk, True, 3)]
    if model != "qwen3-30b-a3b":   # 128 experts: the per-expert host path is the slow path, covered at the other two shapes
        runs.append(((limit + 4) * E * 2 // topk, False, 4))
    for tokens, capturable, seed in runs:
        counts, _ = _routing(E, topk, tokens, seed)
        T = sum(counts)
        A = _activations(model, proj, T, seed)
        off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
        path = _expected_path(op, T, E, capturable)
        got, n = _launches(lambda: op.forward_grouped(A.to(DEV), W, off, scale=s, zeros=z, bias=b, capturable=capturable))
        if path == "per_group":
            assert n >= sum(1 for c in counts if c), (path, n)
        else:
            assert n == 1, (path, n)
        _check_experts(cases, A, counts, got, f"{model} {proj} {path} T={T}", path)


@pytest.mark.parametrize("model", list(MOE))
def test_grouped_swiglu_moe_shapes(model):
    """the gate/up projection with SwiGLU fused: at the single-launch limit (grouped GEMV), above it (grouped wgmma GEMM), and
    gathering the token rows through row_index (the gathering grouped GEMM).  The rows of W are taken as stored (gate/up
    interleave); the reference is silu(g) * u in float64 from the exact pre-activations round(round(V) + b)"""
    from bitblas_b200.ops import general_matmul as GM
    E, topk = MOE[model]["E"], MOE[model]["topk"]
    limit = GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP
    op, cases, W, s, z, b = _experts(model, "gate_up", seed=len(model))
    for tokens, seed, gather in [(limit * E // topk, 5, False), ((limit + 4) * E * 2 // topk, 6, False),
                                 ((limit + 4) * E * 2 // topk, 7, True)]:
        counts, row_token = _routing(E, topk, tokens, seed)
        T = sum(counts)
        off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
        if gather:
            A_tok = _activations(model, "gate_up", tokens, seed)
            A = A_tok[row_token.long()]
            got, n = _launches(lambda: op.forward_grouped_swiglu(A_tok.to(DEV), W, off, scale=s, zeros=z, bias=b,
                                                                 row_index=row_token.to(DEV)))
            path = "gemm"
        else:
            A = _activations(model, "gate_up", T, seed)
            path = _expected_path(op, T, E, True)
            got, n = _launches(lambda: op.forward_grouped_swiglu(A.to(DEV), W, off, scale=s, zeros=z, bias=b))
        assert n == 1 and got.shape == (T, op.N // 2), (n, got.shape)
        _check_experts(cases, A, counts, got, f"{model} swiglu {path} gather={gather} T={T}", path, swiglu=True)


# ---- scatter epilogue on one device ----------------------------------------------------------------------------------------------
SCATTER_CASES = [
    # kernel, M, N, K: the wgmma split-K reduce, the slab, gemv_mma
    (K_GEMM_TS, 16, 1024, 3584),
    (K_GEMV_SLAB, 1, 1024, 8192),
    (K_GEMV_MMA, 4, 1024, 8192),
]


@pytest.mark.parametrize("peers", [1, 2, 8])
@pytest.mark.parametrize("kernel,M,N,K", SCATTER_CASES, ids=["gemm_ts_split_k", "gemv_slab", "gemv_mma"])
def test_scatter_exact(kernel, M, N, K, peers):
    for out in OUTS:
        case = X.make_exact_case(M, N, K, group_size=128, mode="original", bias=out != "float32", out_dtype=out,
                                 fast_decoding=True, seed=peers + M)
        op = X.product_operator(case)
        t = _tensors(op, case)
        ref = X.exact_reference(case, DEV).cpu()
        X.prove_exact(case, device=DEV)
        ldc, off = 2 * N + 64, N + 32
        odt = getattr(torch, out)
        bufs = [torch.full((M, ldc), 7.0, dtype=odt, device=DEV) for _ in range(peers)]
        with forced(kernel):
            assert op.kernel_for(M) == KERNEL_NAME[kernel]
            if kernel == K_GEMM_TS:
                _check_split(op, M, True, 64)
            op.forward_scatter(case["A"].to(DEV), t["W"], scale=t["scale"], zeros=t["zeros"], bias=t["bias"],
                               peer_ptrs=[b.data_ptr() for b in bufs], ldc=ldc, col_offset=off)
        torch.cuda.synchronize()
        for i, b in enumerate(bufs):
            b = b.cpu()
            X.compare_exact(b[:, off:off + N], ref, f"scatter {KERNEL_NAME[kernel]} out={out} destination {i}/{peers}")
            assert bool((b[:, :off] == 7.0).all()) and bool((b[:, off + N:] == 7.0).all()), "stores outside the column window"
