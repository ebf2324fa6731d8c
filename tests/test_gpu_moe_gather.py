"""GPU: the copy-free mixture-of-experts path.  bb_moe_route_index against bb_moe_route on the same ids; every instance of the
gathering grouped GEMM (bb_matmul_grouped_gemm_swiglu_gather) bit-identical to bb_matmul_grouped_gemm_swiglu on the gathered rows,
including malformed indices with guard rows; and the copy-free block (moe_route_index -> gathering gate/up -> down -> combine)
bit-identical to MoEExperts wherever its gate/up call runs the grouped GEMM, with its launch count, graph replay, a PDL chain and
its peak memory."""
import itertools

import pytest
import torch

from test_gpu_grouped_gemm import ROUTINGS as GEMM_ROUTINGS
from test_gpu_grouped_gemm import _build, grouped_bm
from test_gpu_kernel_grid import MODES, OUTS
from test_gpu_moe import _launches, _make_block, _routing, pdl_chain_matches_plain_stream_order

pytestmark = pytest.mark.gpu

DEV = "cuda"
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


# ---- routing -----------------------------------------------------------------------------------------------------------------
def _check_route_index(ids, E):
    from bitblas_b200.moe import moe_route, moe_route_index
    T, k = ids.shape
    ids = ids.to(DEV)
    x = torch.zeros((T, 8), dtype=torch.float16, device=DEV)
    off, rows, _ = moe_route(ids, x, E)
    off_i, rows_i, tok = moe_route_index(ids, E)
    assert torch.equal(off, off_i)
    assert torch.equal(rows, rows_i)
    rows, tok = rows.cpu().long(), tok.cpu()
    kept = (rows >= 0).nonzero().reshape(-1)
    assert torch.equal(tok[rows[kept]], (kept // k).to(torch.int32))
    assert int(off[-1]) == kept.numel()


@pytest.mark.parametrize("T", [1, 300, 4100])       # up to 32800 slots at k = 8
@pytest.mark.parametrize("k", [1, 6, 8])
@pytest.mark.parametrize("E", [1, 8, 128, 256])
def test_route_index_matches_route(E, k, T):
    g = torch.Generator().manual_seed(E * 1000 + k * 10 + T)
    ids = torch.randint(0, E, (T, k), generator=g, dtype=torch.int32)
    drop = torch.rand((T, k), generator=g)
    ids[drop < 0.05] = -1
    ids[drop > 0.95] = E
    _check_route_index(ids, E)


@pytest.mark.parametrize("case", ["one_expert", "all_dropped", "int_extremes"])
def test_route_index_edges(case):
    T, k, E = 1000, 4, 16
    if case == "one_expert":
        ids = torch.full((T, k), 5, dtype=torch.int32)
    elif case == "all_dropped":
        ids = torch.full((T, k), -1, dtype=torch.int32)
        ids[::2] = E
    else:
        ids = torch.randint(0, E, (T, k), dtype=torch.int32, generator=torch.Generator().manual_seed(4))
        ids[::3, 0] = INT_MAX
        ids[::5, 1] = INT_MIN
    _check_route_index(ids, E)


# ---- the gathering GEMM ------------------------------------------------------------------------------------------------------
def _plain_gemm(op, A, W, off, s, z, b, out_rows):
    """bb_matmul_grouped_gemm_swiglu itself (whatever forward_grouped_swiglu's rule would pick) on the rows of A"""
    C = torch.empty((out_rows, op.config.N // 2), dtype=op.torch_output_dtype, device=DEV)
    rc = op.lib._c.bb_matmul_grouped_gemm_swiglu(op._desc_ref, off.numel() - 1, off.data_ptr(), A.data_ptr(), W.data_ptr(),
                                                 s.data_ptr() if s is not None else 0, z.data_ptr() if z is not None else 0,
                                                 b.data_ptr() if b is not None else 0, C.data_ptr(), out_rows,
                                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return C


def _gather_vs_plain(op, A, W, counts, s, z, b, row_index, output=None):
    off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
    T = sum(counts)
    assert row_index.numel() == T
    ri = row_index.to(DEV)
    got, n = _launches(lambda: op.forward_grouped_swiglu(A, W, off, scale=s, zeros=z, bias=b, output=output, row_index=ri))
    assert n == 1 and got.shape == (T, op.config.N // 2)
    clamped = row_index.long().clamp(0, A.shape[0] - 1).to(DEV)
    ref = _plain_gemm(op, A[clamped].contiguous(), W, off, s, z, b, T)
    assert torch.equal(got, ref)
    return got


CELLS = [dict(T=T, bits=bits, il=il, bm=bm, mode=mode)
         for T, bits, il, bm, mode in itertools.product(["float16", "bfloat16"], [4, 2], [True, False], [32, 64, 128], MODES)]


@pytest.mark.parametrize("c", CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_gather_gemm_instance(c):
    """every instance (A dtype x bits x layout x BM) x scale/zero mode x output type x bias, against the plain call on the
    gathered rows: a_rows is not T, rows repeat, and tokens appear in any order"""
    counts = GEMM_ROUTINGS[c["bm"]]
    assert grouped_bm(counts) == c["bm"]
    T = sum(counts)
    for i, (out, bias) in enumerate(itertools.product(OUTS, [False, True])):
        W = ("int" if c["mode"] in ("none", "scale") and bias else "uint") + str(c["bits"])
        a_rows = [T // 3 + 1, T + 17, 40][i % 3]
        seed = 1000 * i + c["bm"] + len(c["mode"])
        op, _, A, Wq, s, z, b = _build(counts, 256, 768, seed=seed, A_dtype=c["T"], W=W, out=out, g=[128, 384, -1][i % 3],
                                       mode=c["mode"], bias=bias, il=c["il"], T=a_rows)
        ri = torch.randint(0, a_rows, (T,), generator=torch.Generator().manual_seed(seed), dtype=torch.int32)
        _gather_vs_plain(op, A.to(DEV), Wq, counts, s, z, b, ri)


def _sparse(E, T, active, seed):
    g = torch.Generator().manual_seed(seed)
    experts = torch.randperm(E, generator=g)[:active]
    counts = [0] * E
    for e in experts[torch.randint(0, active, (T,), generator=g)].tolist():
        counts[e] += 1
    return counts


ROUTES = {
    "empty_experts": [0, 0, 150, 0, 7, 0, 0, 90],
    "larger_than_a_tile": [300, 5, 129, 1],
    "one_expert": [0, 0, 0, 1000, 0],
    "E256": _sparse(256, 3000, 60, seed=1),
    "E256_all_on_one": [0] * 255 + [2100],
    "a_rows_1": [40, 0, 33],
}


@pytest.mark.parametrize("name", list(ROUTES))
@pytest.mark.parametrize("A_dtype", ["float16", "bfloat16"])
def test_gather_gemm_routings(name, A_dtype):
    counts = ROUTES[name]
    T = sum(counts)
    a_rows = 1 if name == "a_rows_1" else (16 if name.startswith("E256") else 257)   # E256: 256 reference cases of a_rows rows
    op, _, A, Wq, s, z, b = _build(counts, 384, 512, seed=len(name), A_dtype=A_dtype, W="uint4", out=A_dtype, bias=True, T=a_rows)
    ri = torch.randint(0, a_rows, (T,), generator=torch.Generator().manual_seed(T), dtype=torch.int32)
    _gather_vs_plain(op, A.to(DEV), Wq, counts, s, z, b, ri)


@pytest.mark.parametrize("bm", [32, 128])
def test_gather_gemm_malformed_indices_stay_inside_a_and_c(bm):
    """indices -1, a_rows, INT_MAX and INT_MIN are clamped: the result equals the call on the clamped index, nothing outside A is
    read (the guard rows around A hold values that would change the result) and nothing outside C is written"""
    counts = GEMM_ROUTINGS[bm]
    T, a_rows, guard = sum(counts), 97, 8
    op, _, A, Wq, s, z, b = _build(counts, 256, 768, seed=bm, T=a_rows, bias=True)
    A_big = torch.full((a_rows + 2 * guard, 768), 1000.0, dtype=torch.float16, device=DEV)
    A_big[guard:guard + a_rows] = A.to(DEV)
    ri = torch.randint(0, a_rows, (T,), generator=torch.Generator().manual_seed(bm), dtype=torch.int32)
    ri[::7], ri[1::7], ri[2::7], ri[3::7] = -1, a_rows, INT_MAX, INT_MIN
    ri[-1] = INT_MAX                                  # the last row of the last tile
    C_big = torch.full((T + 2 * guard, 128), -7.0, dtype=torch.float16, device=DEV)
    _gather_vs_plain(op, A_big[guard:guard + a_rows], Wq, counts, s, z, b, ri, output=C_big[guard:guard + T])
    assert torch.all(C_big[:guard] == -7.0) and torch.all(C_big[guard + T:] == -7.0)


def test_gather_raises_where_the_gemm_does_not_cover():
    import bitblas_b200 as bitblas
    gl = bitblas.GroupedLinear(8, 512, 144, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True,
                               with_zeros=True, zeros_mode="quantized").cuda()
    x = torch.zeros((100, 512), dtype=torch.float16, device=DEV)
    off = torch.tensor([0] + [100] * 8, dtype=torch.int32, device=DEV)
    ri = torch.zeros(100, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="bb_matmul_grouped_gemm_swiglu_gather does not cover this configuration.*N % 128"):
        gl.bitblas_matmul.forward_grouped_swiglu(x, gl.qweight, off, gl.scales, gl.zeros, row_index=ri)
    with pytest.raises(ValueError, match="num_groups \\+ 1 entries"):     # offsets are checked before the coverage
        gl.bitblas_matmul.forward_grouped_swiglu(x, gl.qweight, off[:0], gl.scales, gl.zeros, row_index=ri)


# ---- the block without the copy ------------------------------------------------------------------------------------------------
def _gathering(m, x, ids, w, output=None):
    """MoEExperts.forward with moe_route_index and the gathering gate/up call instead of moe_route's copy of x"""
    from bitblas_b200.moe import moe_combine, moe_route_index
    gu = m.gate_up
    off, slot_rows, row_token = moe_route_index(ids, m.num_experts)
    h = gu.bitblas_matmul.forward_grouped_swiglu(x, gu.qweight, off, gu.scales, gu.zeros, gu.bias, row_index=row_token)
    return moe_combine(m.down(h, off, capturable=True), slot_rows, w, output)


SHAPES = [dict(E=8, I=256, k=2), dict(E=32, I=128, k=4), dict(E=64, I=384, k=6)]


@pytest.mark.parametrize("T", [64, 300, 2048])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "E{E}-I{I}-k{k}".format(**s))
def test_gathering_block_matches_moe_experts(shape, T):
    """above 8 rows per expert (where MoEExperts' gate/up call runs the grouped GEMM) the copy-free composition gives MoEExperts'
    bits in 4 launches"""
    from bitblas_b200.ops.general_matmul import GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP as R
    E, I, k = shape["E"], shape["I"], shape["k"]
    if T * k <= R * E:
        pytest.skip("the gate/up call runs the grouped GEMV here")
    m, _ = _make_block(E=E, I=I, seed=T + E)
    x, ids, w = _routing(T, k, E, seed=T + 3)
    if T == 300:
        ids[::11, 0] = -1                                  # dropped slots
    x, ids, w = x.to(DEV), ids.to(DEV), w.to(DEV)
    got, n = _launches(lambda: _gathering(m, x, ids, w))
    assert n == 4
    assert torch.equal(got, m(x, ids, w))


def test_gathering_block_graph_replay_matches_eager():
    import bitblas_b200 as bitblas
    m, _ = _make_block(E=8, seed=5)
    T, k = 700, 2
    x_d = torch.zeros((T, 512), dtype=torch.float16, device=DEV)
    ids_d = torch.zeros((T, k), dtype=torch.int32, device=DEV)
    w_d = torch.zeros((T, k), dtype=torch.float32, device=DEV)
    out_d = torch.zeros((T, 512), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: _gathering(m, x_d, ids_d, w_d, output=out_d))
    for trial in range(4):
        x, ids, w = _routing(T, k, 8, seed=70 + trial)
        if trial == 0:
            ids[:] = 6                                  # every slot on one expert
        if trial == 1:
            ids[:, 1] = -1                              # half the slots dropped
        x_d.copy_(x)
        ids_d.copy_(ids)
        w_d.copy_(w)
        step()
        eager = _gathering(m, x.to(DEV), ids.to(DEV), w.to(DEV))
        ref = m(x.to(DEV), ids.to(DEV), w.to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(out_d, eager) and torch.equal(eager, ref), trial


CHAIN = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}, {oracle!r}]
{prologue}
from test_gpu_moe import _make_block, _routing
from test_gpu_moe_gather import _gathering
m, _ = _make_block(E=8, seed=23)
xs = [_routing(1024, 2, 8, seed=200 + i) for i in range(8)]
dev = [(x.cuda(), i.cuda(), w.cuda()) for x, i, w in xs]
torch.cuda.synchronize()
outs, h = [], None
for i in range(8):
    x, ids, w = dev[i]
    h = _gathering(m, x + h * 0.5 if i else x, ids, w)           # each step reads the previous step's output
    outs.append(h)
torch.cuda.synchronize()
torch.save([o.cpu() for o in outs], {path!r})
"""


def test_gathering_block_pdl_chain_matches_plain_stream_order(tmp_path):
    """8 copy-free blocks (2048 rows over 8 experts) back to back without synchronisation: PDL gives the bits of BB_PDL=0"""
    pdl_chain_matches_plain_stream_order(CHAIN, tmp_path)


def test_gathering_block_peak_memory_drops_by_the_copy():
    """T = 2048, k = 8, H = 2048: the copy-free block allocates at least the [T*k, H] copy less than MoEExperts; the allowance is
    row_token (T*k int32), which only the copy-free block allocates, plus 2 MiB of caching-allocator rounding"""
    import bitblas_b200 as bitblas
    T, k, E, H, I = 2048, 8, 64, 2048, 256
    m = bitblas.MoEExperts(E, H, I, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                           zeros_mode="quantized").cuda()
    g = torch.Generator(device=DEV).manual_seed(0)
    for gl in (m.gate_up, m.down):
        gl.qweight = torch.randint(-128, 128, tuple(gl.qweight.shape), dtype=torch.int8, device=DEV, generator=g)
        gl.scales = (torch.rand(tuple(gl.scales.shape), device=DEV, generator=g) * 0.01).half()
        gl.zeros = torch.randint(-128, 128, tuple(gl.zeros.shape), dtype=torch.int8, device=DEV, generator=g)
    x = (torch.rand((T, H), device=DEV, generator=g) - 0.5).half()
    ids = torch.rand((T, E), device=DEV, generator=g).argsort(dim=1)[:, :k].to(torch.int32).contiguous()
    w = torch.softmax(torch.randn((T, k), device=DEV, generator=g), dim=1)
    out = torch.empty((T, H), dtype=torch.float16, device=DEV)

    def peak(fn):
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    gathering, copying = peak(lambda: _gathering(m, x, ids, w, output=out)), peak(lambda: m(x, ids, w, output=out))
    assert copying - gathering >= T * k * H * 2 - T * k * 4 - (2 << 20), (gathering, copying)
    assert torch.equal(_gathering(m, x, ids, w), m(x, ids, w))
