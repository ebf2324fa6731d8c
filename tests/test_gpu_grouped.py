"""GPU: the grouped (mixture-of-experts) matmul -- Matmul.forward_grouped / bb_matmul_grouped / GroupedLinear -- against the CPU
oracle, group by group, on seeded inputs."""
import contextlib

import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _experts(E, N, K, seed=0, **kw):
    """E seeded single-expert cases of one config (fields, scale, zeros, bias per expert)"""
    return [H.make_case(1, N, K, seed=seed * 1000 + e, **kw) for e in range(E)]


def _stack(op, cases):
    W = torch.stack([H.product_weight(op, c, DEV) for c in cases])
    st = lambda k: torch.stack([c[k] for c in cases]).to(DEV) if cases[0][k] is not None else None   # noqa: E731
    return W, st("scale"), st("zeros"), st("bias")


def _counts_to_offsets(counts):
    off = [0]
    for c in counts:
        off.append(off[-1] + c)
    return off


def _check_groups(op, cases, A, offsets, got, what):
    """the oracle on each group's rows; the normwise error per group, the elementwise criterion over all claimed rows (with the
    bfloat16 mismatch allowance of the single-matrix tests, which is a share of the whole output)"""
    import bitblas_oracle as O
    bf16 = cases[0]["cfg"]["out_dtype"] == "bfloat16" or cases[0]["cfg"]["A_dtype"] == "bfloat16"
    gots, refs = [], []
    for e, c in enumerate(cases):
        r0, r1 = offsets[e], offsets[e + 1]
        if r1 <= r0:
            continue
        ref = H.oracle_output(dict(c, A=A[r0:r1]), fast_decoding=bool(op.fast_decoding))
        err = O.rel_fro_error(got[r0:r1], ref)
        assert err <= 1e-2, f"{what} group {e} rows [{r0}, {r1}): normwise rel err {err:.3e}"
        gots.append(got[r0:r1])
        refs.append(ref)
    H.assert_fp_close(torch.cat(gots), torch.cat(refs), what, max_mismatched_ratio=2e-3 if bf16 else 0.0)


@contextlib.contextmanager
def single_launch():
    """run forward_grouped's single grouped launch at any row count (the kernel itself is correct for any m_e)"""
    from bitblas_b200.ops import general_matmul as GM
    old = GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP
    GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = 1 << 20
    try:
        yield
    finally:
        GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = old


def _run(kw, counts, N=128, K=512, seed=0, single=True):
    from bitblas_b200 import _lib
    E = len(counts)
    cases = _experts(E, N, K, seed=seed, **kw)
    op = H.product_operator(cases[0], M=[1, 16])
    W, s, z, b = _stack(op, cases)
    offsets = _counts_to_offsets(counts)
    T = offsets[-1]
    g = torch.Generator().manual_seed(seed + 7)
    A = (torch.rand((T, K), generator=g) - 0.5).to(cases[0]["A"].dtype)
    off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    with single_launch() if single else contextlib.nullcontext():
        got = op.forward_grouped(A.to(DEV), W, off, scale=s, zeros=z, bias=b)
    torch.cuda.synchronize()
    if single:
        assert lib.bb_launch_count() - n0 == 1
    _check_groups(op, cases, A, offsets, got.cpu(), f"{kw} counts={counts}")
    return op, got


CONFIGS = [
    dict(W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", with_bias=True,
         fast_decoding=False),
    dict(W_dtype="uint4", group_size=-1, with_scaling=True, with_zeros=True, zeros_mode="rescale"),
    dict(W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", int_zeros=False),
    dict(W_dtype="int4", group_size=128, with_scaling=True),
    dict(W_dtype="uint4"),
    dict(W_dtype="uint2", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized"),
    dict(W_dtype="uint2", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original", fast_decoding=False),
    dict(W_dtype="int2", group_size=-1, with_scaling=True, with_bias=True),
    dict(W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", group_size=128, with_scaling=True, with_zeros=True,
         zeros_mode="original"),
    dict(W_dtype="uint4", A_dtype="bfloat16", out_dtype="bfloat16", fast_decoding=True, group_size=128, with_scaling=True,
         with_zeros=True, zeros_mode="quantized", with_bias=True),
    dict(W_dtype="int2", A_dtype="bfloat16", out_dtype="float32", accum_dtype="float32", group_size=128, with_scaling=True),
    dict(W_dtype="uint4", out_dtype="float32", accum_dtype="float32", group_size=128, with_scaling=True, with_zeros=True,
         zeros_mode="rescale", with_bias=True),
    dict(W_dtype="uint2", A_dtype="bfloat16", out_dtype="bfloat16", group_size=-1, with_scaling=True, with_zeros=True,
         zeros_mode="rescale"),
]


@pytest.mark.parametrize("kw", CONFIGS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_grouped_config_coverage(kw):
    # 8 experts: one empty, one with more than 32 rows, the others with a few (8 * NT row passes of every size)
    _run(kw, [3, 0, 1, 37, 2, 9, 5, 1], seed=1)


@pytest.mark.parametrize("counts", [
    [1], [2], [8], [33], [256],                        # one group: T in {1, 2, 8, 33, 256}
    [0, 0, 0, 80, 0, 0, 0, 0],                         # all rows in one group (three passes of 32 rows)
    [0, 4, 3, 2, 6], [4, 3, 2, 6, 0], [4, 3, 0, 0, 2, 6],   # empty first / last / middle groups
    [1, 1, 0, 0, 0, 0, 0, 0],                          # T = 2 over 8 groups
    [12, 13, 11, 14, 12, 13, 12, 13],                  # ~12 rows per group: 16-row passes
], ids=lambda c: f"E{len(c)}-T{sum(c)}")
def test_grouped_distributions(counts):
    _run(CONFIGS[0], counts, seed=2)


@pytest.mark.parametrize("E,T", [(8, 8), (64, 48), (128, 64), (128, 256), (64, 33)])
def test_grouped_uniform_routing(E, T):
    g = torch.Generator().manual_seed(E * 1000 + T)
    ids = torch.randint(0, E, (T,), generator=g)
    counts = torch.bincount(ids, minlength=E).tolist()
    _run(CONFIGS[0], counts, N=64, K=256, seed=3)


def test_grouped_single_launch_threshold():
    """up to GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E rows: exactly one launch; above it the groups run one bb_matmul each
    (the wgmma GEMM) with the same results"""
    from bitblas_b200 import _lib
    from bitblas_b200.ops.general_matmul import GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP as R
    lib = _lib.load()
    for counts, one in (([R, 0, 2 * R, R], True), ([R, 0, 2 * R + 1, R], False), ([3 * R, 0, 5 * R + 40, 7], False)):
        n0 = lib.bb_launch_count()
        _run(CONFIGS[0], counts, N=128, K=256, seed=4, single=False)
        n = lib.bb_launch_count() - n0
        assert n == 1 if one else n >= 3, (counts, n)   # per group: one launch, or a GEMM + split-K reduce


def test_grouped_malformed_offsets_stay_in_bounds():
    """offsets are clamped to [0, T] and a group whose end is below its start is empty: A / C carry 16 guard rows beyond T
    that keep their sentinel, and rows no group claims are not written"""
    from bitblas_b200 import _lib
    E, N, K, T = 4, 128, 256, 20
    cases = _experts(E, N, K, seed=5, **CONFIGS[0])
    op = H.product_operator(cases[0], M=[1, 16])
    W, s, z, _ = _stack(op, cases)
    g = torch.Generator().manual_seed(11)
    A_full = (torch.rand((T + 16, K), generator=g) - 0.5).half().to(DEV)
    sentinel = -1234.0

    @single_launch()
    def run(offsets):
        C_full = torch.full((T + 16, N), sentinel, dtype=torch.float16, device=DEV)
        off = torch.tensor(offsets, dtype=torch.int32, device=DEV)
        n0 = _lib.load().bb_launch_count()
        op.forward_grouped(A_full[:T], W, off, scale=s, zeros=z, output=C_full[:T])
        torch.cuda.synchronize()
        assert _lib.load().bb_launch_count() - n0 == 1
        C = C_full.cpu()
        assert torch.all(C[T:] == sentinel), "a guard row beyond T was written"
        return C

    A = A_full.cpu()
    # negative start, past-the-end stop: groups [0, 3), [3, 9), empty, [9, T)
    C = run([-5, 3, 9, 9, T + 16])
    _check_groups(op, cases, A, [0, 3, 9, 9, T], C[:T], "clamped")
    # rows 0..3 and 15..T-1 belong to no group
    C = run([4, 9, 9, 15, 15])
    assert torch.all(C[:4] == sentinel) and torch.all(C[15:] == sentinel)
    _check_groups(op, cases, A, [4, 9, 9, 15, 15], C, "unclaimed rows")
    # a decreasing entry: group 1 = [7, 2) is empty; group 2 = [2, 12) overlaps group 0 on rows 2..6
    C = run([0, 7, 2, 12, 12])
    _check_groups(op, cases[:1], A, [0, 2], C, "before the overlap")
    _check_groups(op, [cases[2]], A[7:12], [0, 5], C[7:12], "after the overlap")
    assert torch.all(C[12:T] == sentinel)


def test_grouped_graph_replay_with_changing_routing():
    """one CUDA graph; every replay refreshes the device offsets and the activations through pinned h2d copies"""
    import bitblas_b200 as bitblas
    E, N, K, T = 8, 128, 512, 16
    cases = _experts(E, N, K, seed=6, **CONFIGS[0])
    op = H.product_operator(cases[0], M=[1, 16])
    W, s, z, _ = _stack(op, cases)
    host_off = torch.zeros(E + 1, dtype=torch.int32).pin_memory()
    host_A = torch.zeros((T, K), dtype=torch.float16).pin_memory()
    host_C = torch.zeros((T, N), dtype=torch.float16).pin_memory()
    dev_off = torch.zeros(E + 1, dtype=torch.int32, device=DEV)
    dev_off[-1] = T
    dev_A = torch.zeros((T, K), dtype=torch.float16, device=DEV)
    dev_C = torch.zeros((T, N), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: op.forward_grouped(dev_A, W, dev_off, scale=s, zeros=z, output=dev_C),
                                h2d=[(dev_off, host_off), (dev_A, host_A)], d2h=[(host_C, dev_C)])
    for trial in range(4):
        g = torch.Generator().manual_seed(100 + trial)
        counts = torch.bincount(torch.randint(0, E, (T,), generator=g), minlength=E).tolist()
        offsets = _counts_to_offsets(counts)
        host_off.copy_(torch.tensor(offsets, dtype=torch.int32))
        A = (torch.rand((T, K), generator=g) - 0.5).half()
        host_A.copy_(A)
        step()
        _check_groups(op, cases, A, offsets, host_C.clone(), f"replay {trial}")


def test_grouped_pdl_dependent_chain():
    """offsets computed on the device (bincount + cumsum) right before each call, and a gate/up -> down chain of two grouped
    calls 16 times back to back without synchronisation: bit-identical to the same calls with a synchronisation after each
    launch"""
    E, T, K, N1, N2 = 8, 16, 512, 1024, 512
    c1 = _experts(E, N1, K, seed=7, **CONFIGS[0])
    c2 = _experts(E, N2, N1, seed=8, **CONFIGS[0])
    op1, op2 = H.product_operator(c1[0], M=[1, 16]), H.product_operator(c2[0], M=[1, 16])
    W1, s1, z1, _ = _stack(op1, c1)
    W2, s2, z2, _ = _stack(op2, c2)
    gen = torch.Generator(device=DEV).manual_seed(9)
    ids = [torch.randint(0, E, (T,), device=DEV, generator=gen) for _ in range(16)]
    xs = [((torch.rand((T, K), device=DEV, generator=gen) - 0.5) * 0.5).half() for _ in range(16)]
    mid = torch.empty((T, N1), dtype=torch.float16, device=DEV)
    outs = [torch.empty((T, N2), dtype=torch.float16, device=DEV) for _ in range(16)]
    offs = [torch.empty(E + 1, dtype=torch.int32, device=DEV) for _ in range(16)]

    def route(i, off):   # bincount + cumsum; scatter_add_ counts without torch.bincount's host read of max(ids)
        counts = torch.zeros(E, dtype=torch.int64, device=DEV).scatter_add_(0, ids[i], torch.ones_like(ids[i]))
        off[0] = 0
        off[1:] = torch.cumsum(counts, 0).to(torch.int32)

    torch.cuda.synchronize()
    for i in range(16):                 # no synchronisation anywhere in this loop
        route(i, offs[i])
        op1.forward_grouped(xs[i], W1, offs[i], scale=s1, zeros=z1, output=mid)
        op2.forward_grouped(mid, W2, offs[i], scale=s2, zeros=z2, output=outs[i])
    torch.cuda.synchronize()
    got = [o.cpu() for o in outs]
    off_ref = torch.empty(E + 1, dtype=torch.int32, device=DEV)
    for i in range(16):
        route(i, off_ref)
        torch.cuda.synchronize()
        op1.forward_grouped(xs[i], W1, off_ref, scale=s1, zeros=z1, output=mid)
        torch.cuda.synchronize()
        ref = op2.forward_grouped(mid, W2, off_ref, scale=s2, zeros=z2)
        torch.cuda.synchronize()
        assert torch.equal(got[i], ref.cpu()), f"chain step {i}"
        assert torch.equal(offs[i].cpu(), off_ref.cpu())
    offsets = offs[-1].cpu().tolist()
    _check_groups(op1, c1, xs[-1].cpu(), offsets, op1.forward_grouped(xs[-1], W1, offs[-1], scale=s1, zeros=z1).cpu(), "gate/up")


def _gptq_module(K, N, g, bits, seed, with_bias):
    gen = torch.Generator().manual_seed(seed)
    per = 32 // bits
    intw = torch.randint(0, 2**bits, (K, N), generator=gen, dtype=torch.int32)
    qweight = torch.zeros((K // per, N), dtype=torch.int32)
    for i in range(per):
        qweight |= intw[i::per] << (bits * i)
    zint = torch.randint(0, 2**bits - 1, (K // g, N), generator=gen, dtype=torch.int32)
    qzeros = torch.zeros((K // g, N // per), dtype=torch.int32)
    for i in range(per):
        qzeros |= zint[:, i::per] << (bits * i)

    class G:   # minimal stand-in for a GPTQ QuantLinear
        pass
    m = G()
    m.qweight, m.qzeros = qweight, qzeros
    m.scales = (torch.rand((K // g, N), generator=gen) * 0.1 + 0.01).half()
    m.bias = torch.nn.Parameter(torch.rand(N, generator=gen).half(), requires_grad=False) if with_bias else None
    return m


@pytest.mark.parametrize("mode", ["original", "rescale", "quantized"])
@pytest.mark.parametrize("bits", [4, 2])
def test_grouped_linear_matches_per_expert_linear(mode, bits):
    import bitblas_b200 as bitblas
    E, K, N, g = 4, 512, 256, 128
    kw = dict(A_dtype="float16", W_dtype=f"uint{bits}", group_size=g, with_scaling=True, with_zeros=True, zeros_mode=mode)
    mods = [_gptq_module(K, N, g, bits, seed=20 + e, with_bias=True) for e in range(E)]
    for v2 in (False, True):
        gl = bitblas.GroupedLinear(E, K, N, bias=True, **kw).cuda()
        (gl.repack_from_gptq_v2 if v2 else gl.repack_from_gptq)(mods)
        lins = []
        for e, m in enumerate(mods):
            lin = bitblas.Linear(K, N, bias=True, **kw).cuda()
            (lin.repack_from_gptq_v2 if v2 else lin.repack_from_gptq)(m)
            for name in ("qweight", "scales", "zeros", "bias"):
                assert torch.equal(getattr(gl, name)[e], getattr(lin, name)), (name, e, v2)
            lins.append(lin)
    counts = [3, 0, 5, 1]
    offsets = _counts_to_offsets(counts)
    A = ((torch.rand((sum(counts), K), generator=torch.Generator().manual_seed(1)) - 0.5)).half().to(DEV)
    got = gl(A, torch.tensor(offsets, dtype=torch.int32, device=DEV)).cpu()
    for e, lin in enumerate(lins):
        r0, r1 = offsets[e], offsets[e + 1]
        if r1 > r0:
            H.assert_fp_close(got[r0:r1], lin(A[r0:r1]).cpu(), f"GroupedLinear expert {e}")


def test_grouped_linear_load_and_transform_weight():
    import bitblas_b200 as bitblas
    E, K, N = 3, 512, 128
    for kw in (dict(W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="original"),
               dict(W_dtype="int4"),
               dict(W_dtype="uint2", A_dtype="bfloat16", group_size=-1, with_scaling=True)):
        gl = bitblas.GroupedLinear(E, K, N, **kw).cuda()
        lo = -8 if kw["W_dtype"] == "int4" else 0
        hi = 8 if kw["W_dtype"] == "int4" else 2 ** int(kw["W_dtype"][-1])
        w = torch.randint(lo, hi, (E, N, K), generator=torch.Generator().manual_seed(3), dtype=torch.int8).to(DEV)
        gl.load_and_transform_weight(w)
        for e in range(E):
            assert torch.equal(gl.qweight[e], gl.bitblas_matmul.transform_weight(w[e])), (kw, e)
