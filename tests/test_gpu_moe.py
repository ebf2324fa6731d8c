"""GPU: the mixture-of-experts expert block.  Device routing (bb_moe_route) against a stable-argsort reference, the SwiGLU epilogue of
every grouped GEMV and GEMM instance against silu(g) * u formed from forward_grouped(capturable=True) on the same buffers, the
weighted top-k combine against float64, and MoEExperts end to end (launch count, graph replay, PDL, GPTQ loading)."""
import itertools
import os
import subprocess
import sys

import pytest
import torch

import bitblas_oracle as O
from test_gpu_grouped import _gptq_module
from test_gpu_grouped_gemm import ROUTINGS as GEMM_ROUTINGS
from test_gpu_grouped_gemm import _build, grouped_bm
from test_gpu_kernel_grid import EPS32, MODES, OUTS, ROUTINGS as GEMV_ROUTINGS, _ulp, grouped_nt

pytestmark = pytest.mark.gpu

DEV = "cuda"
TORCH = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}
CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")


def _launches(fn):
    from bitblas_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bb_launch_count() - n0


# ---- routing -----------------------------------------------------------------------------------------------------------------
def route_reference(ids, x, E):
    """stable argsort over the expert of each slot; dropped ids (outside [0, E)) sort last and get row -1"""
    flat = ids.reshape(-1).long()
    k = ids.shape[1]
    valid = (flat >= 0) & (flat < E)
    order = torch.argsort(torch.where(valid, flat, E), stable=True)
    nvalid = int(valid.sum())
    counts = torch.bincount(flat[valid], minlength=E)
    offsets = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(counts, 0)]).to(torch.int32)
    rows = torch.full((flat.numel(),), -1, dtype=torch.int32)
    rows[order[:nvalid]] = torch.arange(nvalid, dtype=torch.int32)
    return offsets, rows, x[order[:nvalid] // k], nvalid


def _check_route(ids, x, E):
    from bitblas_b200.moe import moe_route
    off, rows, xs = moe_route(ids.to(DEV), x.to(DEV), E)
    r_off, r_rows, r_xs, nvalid = route_reference(ids, x, E)
    assert torch.equal(off.cpu(), r_off)
    assert torch.equal(rows.cpu(), r_rows)
    assert torch.equal(xs[:nvalid].cpu(), r_xs)
    off2, rows2, xs2 = moe_route(ids.to(DEV), x.to(DEV), E)
    assert torch.equal(off, off2) and torch.equal(rows, rows2) and torch.equal(xs[:nvalid], xs2[:nvalid])


@pytest.mark.parametrize("T", [1, 7, 300, 4100])       # up to 32800 slots at k = 8
@pytest.mark.parametrize("k", [1, 2, 6, 8])
@pytest.mark.parametrize("E", [1, 8, 64, 128, 256])
def test_route_matches_stable_argsort(E, k, T):
    g = torch.Generator().manual_seed(E * 1000 + k * 10 + T)
    ids = torch.randint(0, E, (T, k), generator=g, dtype=torch.int32)   # with replacement: a token may pick one expert twice
    drop = torch.rand((T, k), generator=g)
    ids[drop < 0.05] = -1
    ids[drop > 0.95] = E
    K = 64 if T > 1000 else 136
    x = (torch.rand((T, K), generator=g) - 0.5).to(torch.bfloat16 if k % 2 else torch.float16)
    _check_route(ids, x, E)


@pytest.mark.parametrize("case", ["one_expert", "all_dropped", "twice_same", "empty_experts"])
def test_route_edges(case):
    T, k, E = 1000, 4, 16
    if case == "one_expert":
        ids = torch.full((T, k), 5, dtype=torch.int32)
    elif case == "all_dropped":
        ids = torch.full((T, k), -1, dtype=torch.int32)
        ids[::2] = E
    elif case == "twice_same":
        ids = torch.randint(0, E, (T, 1), dtype=torch.int32, generator=torch.Generator().manual_seed(1)).repeat(1, k)
    else:
        ids = torch.randint(0, 3, (T, k), dtype=torch.int32, generator=torch.Generator().manual_seed(2)) * 7
    x = (torch.rand((T, 256), generator=torch.Generator().manual_seed(3)) - 0.5).half()
    _check_route(ids, x, E)


# ---- SwiGLU epilogue ---------------------------------------------------------------------------------------------------------
def swiglu_bound(got, pre, out, bias):
    """got [T, I] against silu(g) * u in float64 from the de-interleaved plain output pre [T, 2I]: one ulp of the output type for
    fp16 / bf16 (fp32 errors of a few fp32 ulp cannot move a correctly rounded result by more); fp32 output: 4 ulp (expf is within
    2 ulp, then 1 + e, the division and the product each round once)"""
    from bitblas_b200.moe import deinterleave_gate_up
    g, u = deinterleave_gate_up(pre, "bias")
    g, u = g.double(), u.double()
    ref = g / (1 + torch.exp(-g)) * u
    # at or beyond the rounding boundary above the largest finite value, the kernel stores an infinity of that sign; values between
    # the largest finite value and that boundary round down to it and are covered by the one-ulp bound
    fmax = torch.finfo(TORCH[out]).max
    over = ref.abs() >= fmax + float(_ulp(torch.tensor([fmax], dtype=torch.float64), out)[0]) / 2
    assert torch.equal(got.double()[over], torch.sign(ref[over]) * float("inf"))
    k = 4.0 if out == "float32" else 1.0
    # 2^-100: below it silu(g) underflows in fp32 (exp(-g) overflows for g < -88) and the kernel stores (-)0
    bound = k * _ulp(ref.abs(), out) + 2.0 ** -100
    err = (got.double() - ref).abs()
    bad = ~(err <= bound) & ~over
    assert not bad.any(), f"{int(bad.sum())}/{bad.numel()} outside; worst err/bound {float((err / bound).max()):.2f}"


def _swiglu_cell(counts, N, K, seed, out, bias, **kw):
    op, _, A, W, s, z, b = _build(counts, N, K, seed=seed, out=out, bias=bias, **kw)
    off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
    Ad = A.to(DEV)
    pre = op.forward_grouped(Ad, W, off, scale=s, zeros=z, bias=b, capturable=True)
    got, n = _launches(lambda: op.forward_grouped_swiglu(Ad, W, off, scale=s, zeros=z, bias=b))
    assert n == 1 and got.shape == (sum(counts), N // 2) and got.dtype == TORCH[out]
    swiglu_bound(got.cpu(), pre.cpu(), out, bias)
    return op


GEMV_CELLS = [dict(T=T, bits=bits, il=il, nt=nt, mode=mode)
              for T, bits, il, nt, mode in itertools.product(["float16", "bfloat16"], [4, 2], [True, False], [1, 2, 4], MODES)]


@pytest.mark.parametrize("c", GEMV_CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_swiglu_grouped_gemv_instance(c, monkeypatch):
    from bitblas_b200.ops import general_matmul as GM
    monkeypatch.setattr(GM, "GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP", 1 << 20)   # the grouped GEMV at every row count
    counts = GEMV_ROUTINGS[c["nt"]]
    assert grouped_nt(counts) == c["nt"]
    for i, (out, bias) in enumerate(itertools.product(OUTS, [False, True])):
        W = ("int" if c["mode"] in ("none", "scale") and bias else "uint") + str(c["bits"])
        op = _swiglu_cell(counts, 128, 768, 7 * i + c["nt"] + len(c["mode"]), out, bias, A_dtype=c["T"], W=W,
                          g=[128, 384, -1][i % 3], mode=c["mode"], il=c["il"])
        assert op._grouped_single_launch(sum(counts), len(counts)) == "gemv"


GEMM_CELLS = [dict(T=T, bits=bits, il=il, bm=bm, mode=mode)
              for T, bits, il, bm, mode in itertools.product(["float16", "bfloat16"], [4, 2], [True, False], [32, 64, 128], MODES)]


@pytest.mark.parametrize("c", GEMM_CELLS, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_swiglu_grouped_gemm_instance(c):
    counts = GEMM_ROUTINGS[c["bm"]]
    assert grouped_bm(counts) == c["bm"]
    for i, (out, bias) in enumerate(itertools.product(OUTS, [False, True])):
        W = ("int" if c["mode"] in ("none", "scale") and bias else "uint") + str(c["bits"])
        op = _swiglu_cell(counts, 256, 768, 1000 * i + c["bm"] + len(c["mode"]), out, bias, A_dtype=c["T"], W=W,
                          g=[128, 384, -1][i % 3], mode=c["mode"], il=c["il"])
        assert op._grouped_single_launch(sum(counts), len(counts)) == "gemm"


@pytest.mark.parametrize("E", [4, 16])
def test_swiglu_both_sides_of_the_threshold(E):
    from bitblas_b200.ops.general_matmul import GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP as R
    for T in (R * E, R * E + 1):
        counts = torch.bincount(torch.randint(0, E, (T,), generator=torch.Generator().manual_seed(T)), minlength=E).tolist()
        op = _swiglu_cell(counts, 256, 512, T, "float16", True, mode="quantized")
        assert op._grouped_single_launch(T, E) == ("gemv" if T <= R * E else "gemm")


# ---- combine -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("T,k,N", [(1, 8, 2048), (37, 2, 64), (600, 6, 1024)])
def test_combine_matches_float64(T, k, N, out):
    from bitblas_b200.moe import moe_combine
    g = torch.Generator().manual_seed(T * k + N)
    Y = ((torch.rand((T * k, N), generator=g) - 0.5) * 8).to(TORCH[out])
    rows = torch.randperm(T * k, generator=g).to(torch.int32)
    r = torch.rand(T * k, generator=g)
    rows[r < 0.05] = -1
    rows[(r > 0.95)] = T * k          # out of range: dropped too
    rows[:k] = -1                      # token 0 has no valid slot
    w = torch.rand((T, k), generator=g)
    got = moe_combine(Y.to(DEV), rows.to(DEV), w.to(DEV))
    got2 = moe_combine(Y.to(DEV), rows.to(DEV), w.to(DEV))
    assert torch.equal(got, got2)
    got = got.cpu().double()
    valid = ((rows >= 0) & (rows < T * k)).reshape(T, k)
    Yv = Y.double()[rows.clamp(0, T * k - 1).long()].reshape(T, k, N) * valid[..., None]
    wv = w.double()[..., None]
    ref = (wv * Yv).sum(1)
    acc = (wv.abs() * Yv.abs()).sum(1)
    bound = k * EPS32 * acc + _ulp(ref.abs(), out)
    err = (got - ref).abs()
    assert (err <= bound).all(), f"worst err/bound {float((err / bound).max()):.2f}"
    assert torch.all(got[0] == 0)


# ---- the block -----------------------------------------------------------------------------------------------------------------
def _fields(E, N, K, bits, g, gen):
    """per-projection fields of the quantized-zeros config: weight values, scales [E, N, G], packed zeros [E, G, N*bits/8]"""
    G = K // g
    w = torch.randint(0, 2 ** bits, (E, N, K), generator=gen, dtype=torch.int8)
    s = (torch.rand((E, N, G), generator=gen) * 0.02 + 0.002).half()
    qz = torch.randint(0, 2 ** bits, (E, G, N), generator=gen, dtype=torch.int32)
    z = torch.stack([torch.from_numpy(O.general_compress(qz[e].numpy(), bits)) for e in range(E)])
    return w, s, z, qz


def _dequant(w, s, qz, g):
    gidx = torch.arange(w.shape[-1]) // g
    return (w.double() - qz.double()[:, gidx, :].transpose(1, 2)) * s.double()[:, :, gidx]


def _make_block(E=8, H=512, I=256, seed=0):
    import bitblas_b200 as bitblas
    gen = torch.Generator().manual_seed(seed)
    m = bitblas.MoEExperts(E, H, I, **CFG).cuda()
    fg, fu, fd = _fields(E, I, H, 4, 128, gen), _fields(E, I, H, 4, 128, gen), _fields(E, H, I, 4, 128, gen)
    m.load_and_transform_weight([t.to(DEV) for t in fg[:3]], [t.to(DEV) for t in fu[:3]], [t.to(DEV) for t in fd[:3]])
    dq = [_dequant(f[0], f[1], f[3], 128) for f in (fg, fu, fd)]
    return m, dq


def _routing(T, k, E, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.rand((T, E), generator=g).argsort(dim=1)[:, :k].to(torch.int32)
    w = torch.softmax(torch.randn((T, k), generator=g), dim=1)
    x = (torch.rand((T, 512), generator=g) - 0.5).half()
    return x, ids, w


def _oracle(dq, x, ids, w):
    Wg, Wu, Wd = dq
    x = x.double()
    out = torch.zeros((x.shape[0], Wd.shape[1]), dtype=torch.float64)
    for t in range(x.shape[0]):
        for j in range(ids.shape[1]):
            e = int(ids[t, j])
            gt, up = Wg[e] @ x[t], Wu[e] @ x[t]
            out[t] += float(w[t, j]) * (Wd[e] @ (gt / (1 + torch.exp(-gt)) * up))
    return out


def _composed(m, x, ids, w):
    """the same block from torch routing, forward_grouped(capturable=True), an fp32 silu * mul and a float64 combine"""
    from bitblas_b200.moe import deinterleave_gate_up
    T, k = ids.shape
    E = m.num_experts
    flat = ids.reshape(-1).long()
    order = torch.argsort(flat, stable=True)
    off = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.bincount(flat, minlength=E), 0)]).to(torch.int32)
    rows = torch.empty_like(order)
    rows[order] = torch.arange(order.numel())
    off_d = off.to(DEV)
    pre = m.gate_up(x[order // k].to(DEV), off_d, capturable=True)
    g, u = deinterleave_gate_up(pre, "bias")
    h = (torch.nn.functional.silu(g.float()) * u.float()).half()
    y = m.down(h, off_d, capturable=True).cpu().double()
    return (w.double()[..., None] * y[rows].reshape(T, k, -1)).sum(1)


def _normwise(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


@pytest.mark.parametrize("T", [1, 4, 64, 300])       # both grouped families: 8 experts take the grouped GEMM above 64 rows
def test_block_matches_composition_and_oracle(T):
    m, dq = _make_block(seed=T)
    x, ids, w = _routing(T, 2, 8, seed=T + 1)
    got, n = _launches(lambda: m(x.to(DEV), ids.to(DEV), w.to(DEV)))
    assert n == 4
    got = got.cpu()
    assert _normwise(got, _composed(m, x, ids, w)) <= 2e-3
    assert _normwise(got, _oracle(dq, x, ids, w)) <= 1e-2


def test_block_graph_replay_matches_eager():
    import bitblas_b200 as bitblas
    m, _ = _make_block(seed=11)
    T, k = 96, 2
    x_d = torch.zeros((T, 512), dtype=torch.float16, device=DEV)
    ids_d = torch.zeros((T, k), dtype=torch.int32, device=DEV)
    w_d = torch.zeros((T, k), dtype=torch.float32, device=DEV)
    out_d = torch.zeros((T, 512), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: m(x_d, ids_d, w_d, output=out_d))
    for trial in range(4):
        x, ids, w = _routing(T, k, 8, seed=50 + trial)
        if trial == 0:
            ids[:] = 3                                  # every slot on one expert
        x_d.copy_(x)
        ids_d.copy_(ids)
        w_d.copy_(w)
        step()
        eager = m(x.to(DEV), ids.to(DEV), w.to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(out_d, eager), trial


CHAIN = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}, {oracle!r}]
{prologue}
from test_gpu_moe import _make_block, _routing
m, _ = _make_block(seed=21)
outs = []
xs = [_routing(48, 2, 8, seed=100 + i) for i in range(16)]
dev = [(x.cuda(), i.cuda(), w.cuda()) for x, i, w in xs]
torch.cuda.synchronize()
h = dev[0][0]
for i in range(16):
    x, ids, w = dev[i]
    h = m(x + h * 0.5 if i else x, ids, w)           # each step reads the previous step's output
    outs.append(h)
torch.cuda.synchronize()
torch.save([o.cpu() for o in outs], {path!r})
"""


def pdl_chain_matches_plain_stream_order(chain, tmp_path, prologue=""):
    """runs the script `chain` (a template with the keys root, tests, oracle, path and prologue: code run before the chain) once
    with BB_PDL=1 and once with BB_PDL=0, which the library reads once per process, and asserts bit-identical step outputs"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = {}
    for pdl in ("1", "0"):
        path = str(tmp_path / f"chain{pdl}.pt")
        code = chain.format(root=root, tests=os.path.join(root, "tests"), oracle=os.path.join(root, "oracle"), path=path,
                            prologue=prologue)
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, BB_PDL=pdl), capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        res[pdl] = torch.load(path)
    for i, (a, b) in enumerate(zip(res["1"], res["0"])):
        assert torch.equal(a, b), f"step {i}"


def test_block_pdl_chain_matches_plain_stream_order(tmp_path):
    """16 blocks back to back, each fed by the previous one's output, without synchronisation: the launches chained with PDL give
    the same bits as BB_PDL=0 (plain stream order)"""
    pdl_chain_matches_plain_stream_order(CHAIN, tmp_path)


@pytest.mark.parametrize("v2", [False, True])
def test_block_gptq_loading_matches_fields(v2):
    """GPTQ modules per expert and projection give the same buffers and outputs as the same values loaded as fields"""
    import bitblas_b200 as bitblas
    from bitblas_b200.moe import interleave_gate_up
    E, H, I, g, bits = 4, 512, 256, 128, 4
    kw = dict(A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True, zeros_mode="quantized")
    mods = [[_gptq_module(K, N, g, bits, seed=100 * p + e, with_bias=False) for e in range(E)]
            for p, (K, N) in enumerate([(H, I), (H, I), (I, H)])]
    m = bitblas.MoEExperts(E, H, I, **kw).cuda()
    (m.repack_from_gptq_v2 if v2 else m.repack_from_gptq)(*mods)
    halves = []
    for p, (K, N) in enumerate([(H, I), (H, I), (I, H)]):
        gl = bitblas.GroupedLinear(E, K, N, **kw).cuda()
        (gl.repack_from_gptq_v2 if v2 else gl.repack_from_gptq)(mods[p])
        halves.append(gl)
    ref = bitblas.MoEExperts(E, H, I, **kw).cuda()
    ref.gate_up.qweight = interleave_gate_up(halves[0].qweight, halves[1].qweight, "weight")
    ref.gate_up.scales = interleave_gate_up(halves[0].scales, halves[1].scales, "scale")
    ref.gate_up.zeros = interleave_gate_up(halves[0].zeros, halves[1].zeros, "qzeros", bits)
    ref.down = halves[2]
    for name in ("qweight", "scales", "zeros"):
        assert torch.equal(getattr(m.gate_up, name), getattr(ref.gate_up, name)), name
        assert torch.equal(getattr(m.down, name), getattr(ref.down, name)), name
    x, ids, w = _routing(20, 2, E, seed=7)
    x, ids, w = x.to(DEV), ids.to(DEV), w.to(DEV)
    assert torch.equal(m(x, ids, w), ref(x, ids, w))
