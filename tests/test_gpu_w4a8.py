"""H100: bb_matmul_w4a8 and W4A8Linear.  Every new kernel instance (forced with the kernel override) against a CPU restatement of
the contract in include/bitblas_b200.h: bit for bit on exactly representable inputs (power-of-two scales and activation scales,
small integers: every fp32 step is exact in any order), and against float64 with a per-element error bound on random inputs.
The group order of generic_simt and the unsplit wgmma GEMM is restated too, so those two are also checked bit for bit on random
inputs.  Split-K factors, calls without a workspace, capped SM counts, repeat and graph-replay determinism, production shapes
under the dispatcher's own choice, GPTQ v1 / v2 / act-order loading, a PDL chain and rejections."""
import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.w4a8 import W4A8Linear, pack_zeros

pytestmark = pytest.mark.gpu

GENERIC, GEMV_I8, GEMM_TS_I8 = _lib.BB_KERNEL_GENERIC, _lib.BB_KERNEL_GEMV_I8, _lib.BB_KERNEL_GEMM_TS_I8
OUT = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}


def quant_ref(x):
    """BitNet's activation_quant on the CPU (bb_quantize_act_int8's contract): (q int8, scale float32 [rows])"""
    xf = x.cpu().float().reshape(-1, x.shape[-1])
    s = 127.0 / xf.abs().amax(-1, keepdim=True).clamp(min=1e-5)
    q = (xf * s).round().clamp(-128, 127).to(torch.int8)
    return q, s.reshape(-1)


class Case:
    """one W4A8 problem: q int8 [m, K], u [N, K] stored fields, z [N, G] zero points (None: 8 for int4, 0 for uint4), fp32
    scales [N, G], a_scale [m], bias [N] in out_dtype (or None)"""

    def __init__(self, m, N, K, g=128, W="uint4", zeros=True, out="float16", bias=False, exact=False, seed=0, layout="il"):
        gen = torch.Generator().manual_seed(seed)
        self.m, self.N, self.K, self.g, self.G = m, N, K, g, K // g
        self.W, self.zeros_on, self.out, self.layout = W, zeros, out, layout
        self.u = torch.randint(0, 16, (N, K), generator=gen)
        self.z = torch.randint(0, 16, (N, self.G), generator=gen) if zeros else None
        if exact:
            self.q = torch.randint(-8, 9, (m, K), generator=gen).to(torch.int8)
            self.scales = 2.0 ** -torch.randint(0, 3, (N, self.G), generator=gen).float()
            self.a_scale = 2.0 ** torch.randint(3, 7, (m,), generator=gen).float()
        else:
            self.q = torch.randint(-128, 128, (m, K), generator=gen).to(torch.int8)
            self.scales = (torch.rand(N, self.G, generator=gen) * 0.02 + 1e-3).float()
            self.a_scale = (torch.rand(m, generator=gen) * 100 + 20).float()
        self.bias = (torch.randn(N, generator=gen) * (0.25 if exact else 1)).to(OUT[out]) if bias else None

    def w(self):
        z = self.z.repeat_interleave(self.g, 1) if self.zeros_on else (8 if self.W == "int4" else 0)
        return self.u - z

    def group_acc(self):
        """acc[r, n, g] exact (int64)"""
        q = self.q.to(torch.int64).reshape(self.m, self.G, self.g)
        w = self.w().to(torch.int64).reshape(self.N, self.G, self.g)
        return torch.einsum("mgk,ngk->mng", q.double(), w.double()).to(torch.int64)   # |values| < 2^53: exact

    def restate(self):
        """the contract with the group order of generic_simt / unsplit gemm_ts: S = ((0 + p_0) + p_1) + ..., fp32 steps"""
        acc = self.group_acc().float()
        S = torch.zeros(self.m, self.N, dtype=torch.float32)
        for gi in range(self.G):
            S = S + acc[:, :, gi] * self.scales[:, gi][None, :]
        y = S / self.a_scale[:, None]
        return self._round(y)

    def _round(self, y):
        if self.out == "float32":
            return y + (self.bias.float() if self.bias is not None else 0)
        o = y.to(OUT[self.out])
        return o + self.bias if self.bias is not None else o

    def float64(self):
        """(y exact in float64 before the output rounding, the bound of the fp32 evaluation's error on y)"""
        p = self.group_acc().double() * self.scales.double()[None]
        y = p.sum(-1) / self.a_scale.double()[:, None]
        err = (self.G + 2) * 2.0 ** -24 * p.abs().sum(-1) / self.a_scale.double()[:, None] + 2.0 ** -24 * y.abs()
        return y, err

    def check_bound(self, got):
        y, err = self.float64()
        ulp_bits = {"float16": 10, "bfloat16": 7, "float32": 23}[self.out]
        tiny = {"float16": 2.0 ** -24, "bfloat16": 2.0 ** -133, "float32": 2.0 ** -149}[self.out]
        if self.bias is not None:
            yb = y + self.bias.double()
            mag = torch.maximum(y.abs(), yb.abs()) + err
            y = yb
        else:
            mag = y.abs() + err
        ulp = torch.clamp(2.0 ** (torch.floor(torch.log2(mag.clamp(min=1e-300))) - ulp_bits), min=tiny)
        bound = err + (2 if self.bias is not None else 1) * ulp
        diff = (got.cpu().double() - y).abs()
        bad = diff > bound
        assert not bool(bad.any()), f"{int(bad.sum())} elements outside the bound, worst {float((diff - bound).max())}"

    # ---- device operands ----
    def layer_op(self):
        layout = _lib.BB_LAYOUT_INTERLEAVED_8 if self.layout == "il" else _lib.BB_LAYOUT_COMPRESSED
        op = bitblas.Matmul(bitblas.MatmulConfig(N=self.N, K=self.K, A_dtype="int8", W_dtype=self.W, accum_dtype="int32",
                                                 out_dtype=self.out, group_size=self.g, with_scaling=True, with_zeros=self.zeros_on,
                                                 zeros_mode="quantized" if self.zeros_on else None, with_bias=self.bias is not None,
                                                 fast_decoding=self.layout == "il"), enable_tuning=False)
        assert op._desc.w_layout == layout
        return op

    def device(self, op):
        W = op.weight_transform(self.u.to(torch.int8)).cuda()
        return dict(A_q=self.q.cuda(), W=W, a_scale=self.a_scale.cuda(), scale=self.scales.cuda(),
                    zeros=pack_zeros(self.z).cuda() if self.zeros_on else None,
                    bias=self.bias.cuda() if self.bias is not None else None)


def _forced(kernel, fn):
    lib = _lib.load()
    prev = lib.bb_set_kernel_override(kernel)
    try:
        return fn()
    finally:
        lib.bb_set_kernel_override(prev)


def _run(case, kernel=None, op=None):
    op = op or case.layer_op()
    t = case.device(op)
    if kernel is not None:
        assert _forced(kernel, lambda: op.kernel_for_w4a8(case.m)) == _lib.kernel_name(kernel)
        out = _forced(kernel, lambda: op.forward_w4a8(**t))
    else:
        out = op.forward_w4a8(**t)
    torch.cuda.synchronize()
    return out.cpu(), op, t


# every new instance: gemv_i8 at NT = 1, 2, 4; gemm_ts_i8 at BM = 32 and 64 (one and several m-tiles), both layouts; generic
INSTANCES = [
    (GEMV_I8, 1, "il"), (GEMV_I8, 8, "il"), (GEMV_I8, 13, "il"), (GEMV_I8, 32, "il"),
    (GEMM_TS_I8, 5, "il"), (GEMM_TS_I8, 40, "il"), (GEMM_TS_I8, 100, "il"), (GEMM_TS_I8, 300, "il"),
    (GEMM_TS_I8, 5, "cmp"), (GEMM_TS_I8, 40, "cmp"), (GEMM_TS_I8, 100, "cmp"), (GEMM_TS_I8, 300, "cmp"),
    (GENERIC, 3, "il"), (GENERIC, 70, "cmp"),
]
FORMATS = [("uint4", True, 128, "float16", True), ("int4", False, 256, "bfloat16", False), ("uint4", False, -1, "float32", True),
           ("uint4", True, 512, "bfloat16", False)]


def _iid(p):
    return f"{_lib.kernel_name(p[0])}-m{p[1]}-{p[2]}"


@pytest.mark.parametrize("fmt", FORMATS, ids=lambda f: f"{f[0]}-z{int(f[1])}-g{f[2]}-{f[3]}-b{int(f[4])}")
@pytest.mark.parametrize("inst", INSTANCES, ids=_iid)
def test_instance(inst, fmt):
    kernel, m, layout = inst
    W, zeros, g, out, bias = fmt
    K = 1536
    g = K if g == -1 else g
    # exact inputs: bit for bit whatever the order; random inputs: the float64 bound, and bit for bit where the order is restated
    ex = Case(m, 256, K, g, W, zeros, out, bias, exact=True, seed=m * 7 + g, layout=layout)
    got, op, _ = _run(ex, kernel)
    assert torch.equal(got, ex.restate())
    rnd = Case(m, 256, K, g, W, zeros, out, bias, seed=m * 11 + g, layout=layout)
    got, _, _ = _run(rnd, kernel, op)
    rnd.check_bound(got)
    if kernel == GENERIC or (kernel == GEMM_TS_I8 and m > 128):   # no split-K: the restated group order
        assert torch.equal(got, rnd.restate())


def test_generic_fallback():
    """g not a multiple of 128 runs generic_simt under the dispatcher at every m; g = 384 (three k-blocks per group) stays on
    gemv_i8 and the wgmma GEMM"""
    for K, g, m, kernel in ((1024, 64, 1, "generic_simt"), (1024, 64, 20, "generic_simt"), (1024, 64, 200, "generic_simt"),
                            (1536, 384, 100, "gemm_ts_wgmma_i8"), (1536, 384, 300, "gemm_ts_wgmma_i8"), (1536, 384, 4, "gemv_i8")):
        c = Case(m, 256, K, g, exact=False, seed=m + g)
        got, op, _ = _run(c)
        assert op.kernel_for_w4a8(m) == kernel
        if kernel == "generic_simt" or m > 128:   # no split-K: the restated group order
            assert torch.equal(got, c.restate())
        else:
            c.check_bound(got)


def _expected_split(N, K, m, G):
    """the W4A8 split factor (launch_ts_inst): dispatch_table's choose_splits over the W4A8 tile grid (BM = 32 up to m = 32, else
    64), cut to the largest divisor of G"""
    import dispatch_table as DT
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bm = 32 if m <= 32 else 64
    sp = int(DT.choose_splits(((m + bm - 1) // bm) * (N // 128), K // 128, sms))
    while G % sp:
        sp -= 1
    return sp, DT.slab_slot_bytes(sms)


def _launches_with_workspace(op, t, m, N, ws_bytes):
    lib = _lib.load()
    ws = torch.zeros(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
    out = torch.empty(m, N, dtype=torch.float16, device="cuda")
    n0 = lib.bb_launch_count()
    rc = _forced(GEMM_TS_I8, lambda: lib.bb_matmul_w4a8(op._desc_ref, t["A_q"].data_ptr(), t["W"].data_ptr(), t["a_scale"].data_ptr(),
                                                         t["scale"].data_ptr(), t["zeros"].data_ptr(), 0, out.data_ptr(), m,
                                                         ws.data_ptr() if ws_bytes else 0, ws_bytes,
                                                         torch.cuda.current_stream().cuda_stream))
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return lib.bb_launch_count() - n0, out.cpu()


# (K, g) -> W4A8 split factors 2, 3, 4, 8 at m <= 128 on 132 SMs; (6144, 2048) and (6144, 384) cut the plain factor 6 to 3 and 4
@pytest.mark.parametrize("K,g", [(2048, 128), (3072, 1024), (4096, 512), (8192, 512), (6144, 2048), (6144, 384)])
@pytest.mark.parametrize("m", [1, 16, 64, 128])
def test_every_split_and_no_workspace(K, g, m):
    """gemm_ts at the split factor read from the workspace size: it splits (two launches) with exactly the partials of that
    factor and not with one byte less; the same call without a workspace is one launch.  All equal to each other and to the
    restatement on exact inputs; within the bound on random ones, and the unsplit call bit for bit in the restated order"""
    N = 256
    for exact in (True, False):
        c = Case(m, N, K, g, exact=exact, seed=K + g + m)
        got, op, t = _run(c, GEMM_TS_I8)
        sp, slots = _expected_split(N, K, m, K // g)
        assert sp > 1
        need = slots + sp * m * N * 4
        n, split_out = _launches_with_workspace(op, t, m, N, need)
        assert n == 2 and torch.equal(split_out, got)
        n, _ = _launches_with_workspace(op, t, m, N, need - 1)
        assert n == 1   # the factor is exactly sp: one byte less does not hold its partials
        n, plain = _launches_with_workspace(op, t, m, N, 0)
        assert n == 1
        if exact:
            assert torch.equal(got, c.restate()) and torch.equal(plain, got)
        else:
            c.check_bound(got)
            assert torch.equal(plain, c.restate())


def test_slab_tiled_weights():
    """BB_TILE_SLAB storage (propagate_b) on the wgmma GEMM (4-D tensor map) and the generic kernel (tiled_byte_offset)"""
    for kernel, m in ((GEMM_TS_I8, 16), (GEMM_TS_I8, 200), (GENERIC, 5)):
        c = Case(m, 256, 2048, 128, exact=True, seed=m)
        op = bitblas.Matmul(bitblas.MatmulConfig(N=256, K=2048, A_dtype="int8", W_dtype="uint4", accum_dtype="int32",
                                                 out_dtype="float16", group_size=128, with_scaling=True, with_zeros=True,
                                                 zeros_mode="quantized", fast_decoding=True, propagate_b=True), enable_tuning=False)
        assert op._desc.w_tile == _lib.BB_TILE_SLAB
        t = c.device(op)
        t["W"] = op.tile_weight(t["W"])
        assert _forced(kernel, lambda: op.kernel_for_w4a8(m)) == _lib.kernel_name(kernel)
        out = _forced(kernel, lambda: op.forward_w4a8(**t))
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), c.restate())


@pytest.mark.parametrize("cap", [16, 66, 114])
def test_capped_sm_counts(cap):
    lib = _lib.load()
    prev = lib.bb_set_sm_count_cap(cap)
    try:
        for kernel, m in ((GEMV_I8, 1), (GEMV_I8, 24), (GEMM_TS_I8, 16), (GEMM_TS_I8, 128)):
            c = Case(m, 1024, 4096, 128, exact=True, seed=cap + m)
            got, _, _ = _run(c, kernel)
            assert torch.equal(got, c.restate())
    finally:
        lib.bb_set_sm_count_cap(prev)


def test_repeat_and_graph_replay_bit_identical():
    for m in (1, 16, 100, 512):
        c = Case(m, 1024, 4096, 128, seed=m)
        op = c.layer_op()
        t = c.device(op)
        a = op.forward_w4a8(**t).clone()
        b = op.forward_w4a8(**t).clone()
        out = torch.empty_like(a)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            op.forward_w4a8(**t, output=out)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            op.forward_w4a8(**t, output=out)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, out)
        c.check_bound(a.cpu())


# Llama-2-70B's four linear shapes and Llama-3-8B's, (N, K)
PRODUCTION = [(10240, 8192), (8192, 8192), (57344, 8192), (8192, 28672), (6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]


@pytest.mark.parametrize("N,K", PRODUCTION, ids=lambda v: str(v))
def test_production_shapes(N, K):
    for m in (1, 16, 200):
        c = Case(m, N, K, 128, exact=True, seed=N + m)
        got, op, _ = _run(c)
        assert op.kernel_for_w4a8(m) == ("gemv_i8" if m <= 8 else "gemm_ts_wgmma_i8")
        assert torch.equal(got, c.restate())


# ---- W4A8Linear ---------------------------------------------------------------------------------------------------------------
def _gptq_module(K, N, g, v2, act_order, seed):
    gen = torch.Generator().manual_seed(seed)
    u = torch.randint(0, 16, (N, K), generator=gen)
    G = K // g
    z = torch.randint(0, 16, (N, G), generator=gen)
    scales = (torch.rand(G, N, generator=gen) * 0.02 + 0.001).half()
    g_idx = torch.randperm(K, generator=gen) // g if act_order else torch.arange(K) // g
    # qweight [K/8, N] int32: row k of K packs nibbles of u[:, k]
    uk = u.T.to(torch.int64).reshape(K // 8, 8, N)
    qweight = sum(uk[:, i, :] << (4 * i) for i in range(8)).to(torch.int64)
    qweight = torch.where(qweight >= 2 ** 31, qweight - 2 ** 32, qweight).to(torch.int32)
    zs = z.T.to(torch.int64) - (0 if v2 else 1)                       # [G, N]; v1 stores z - 1
    zs = zs & 15
    zk = zs.reshape(G, N // 8, 8)
    qzeros = sum(zk[:, :, i] << (4 * i) for i in range(8))
    qzeros = torch.where(qzeros >= 2 ** 31, qzeros - 2 ** 32, qzeros).to(torch.int32)

    class M:
        pass
    mod = M()
    mod.qweight, mod.qzeros, mod.scales, mod.g_idx, mod.bias = qweight, qzeros, scales, g_idx.to(torch.int32), None
    return mod, u, z, scales, g_idx


def _layer_ref(x, u, z, scales, g_idx, G):
    """the layer's formula in float64 from the unsorted checkpoint: groups by g_idx"""
    q, s = quant_ref(x)
    w = (u - z[:, g_idx.long()]).double()
    y = torch.zeros(q.shape[0], u.shape[0], dtype=torch.float64)
    absum = torch.zeros_like(y)
    for gi in range(G):
        cols = (g_idx == gi).nonzero().flatten()
        acc = q[:, cols].double() @ w[:, cols].T
        p = acc * scales[gi].float().double()[None, :]
        y += p
        absum += p.abs()
    return y / s.double()[:, None], (G + 2) * 2.0 ** -24 * absum / s.double()[:, None]


@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("act_order", [False, True])
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_gptq_loading(v2, act_order, dtype):
    K, N, g = 2048, 512, 128
    mod, u, z, scales, g_idx = _gptq_module(K, N, g, v2, act_order, seed=int(v2) + 2 * int(act_order))
    lin = W4A8Linear(K, N, A_dtype=dtype).cuda()
    (lin.repack_from_gptq_v2 if v2 else lin.repack_from_gptq)(mod)
    assert (lin.perm is not None) == act_order
    assert torch.equal(lin.scales.cpu(), scales.T.float())
    for m in (1, 20, 200):
        x = torch.randn(m, K, generator=torch.Generator().manual_seed(m)).to(getattr(torch, dtype)).cuda()
        got = lin(x).cpu().double()
        y, err = _layer_ref(x, u, z, scales, g_idx, K // g)
        ulp = 2.0 ** (torch.floor(torch.log2(y.abs() + err + 1e-30)) - (10 if dtype == "float16" else 7))
        assert bool(((got - y).abs() <= err + ulp).all())


def test_layer_graph_and_pdl_chain():
    """three W4A8Linear layers in a chain (quantize -> matmul, each layer's quantization writing its own q / scale), eager and
    replayed from a CUDA graph, equal to the layers run one by one with synchronisation in between"""
    torch.manual_seed(0)
    K = 1024
    layers = []
    for i in range(3):
        lin = W4A8Linear(K, K, bias=True).cuda()
        lin.load_quantized(torch.randint(0, 16, (K, K)), torch.rand(K, K // 128) * 0.01 + 1e-3, torch.randint(0, 16, (K, K // 128)),
                           torch.randn(K))
        layers.append(lin)
    for m in (1, 16, 256):
        x = torch.randn(m, K, device="cuda", dtype=torch.float16)
        ref = x
        for lin in layers:
            ref = lin(ref)
            torch.cuda.synchronize()
        y = x
        for lin in layers:
            y = lin(y)
        assert torch.equal(y, ref)
        xs = x.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                y = xs
                for lin in layers:
                    y = lin(y)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = xs
            for lin in layers:
                yg = lin(yg)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, ref)


def test_shared_scale_buffer_chain():
    """quantize -> matmul three times through one q / scale buffer pair (PDL: each quantization overwrites the scales the previous
    matmul reads, so it must wait for it), eager and replayed from a CUDA graph, against separate buffers per call"""
    K, N, m = 4096, 4096, 4
    c = Case(m, N, K, 128, seed=5)
    op = c.layer_op()
    t = c.device(op)
    q = torch.empty(m, K, dtype=torch.int8, device="cuda")
    s = torch.empty(m, dtype=torch.float32, device="cuda")
    xs = [torch.randn(m, K, device="cuda", dtype=torch.float16) * (i + 1) for i in range(3)]
    outs = [torch.empty(m, N, dtype=torch.float16, device="cuda") for _ in xs]

    def chain():
        for x, o in zip(xs, outs):
            bitblas.quantize_act_int8(x, q, s)
            op.forward_w4a8(q, t["W"], s, t["scale"], t["zeros"], output=o)

    refs = []
    for x in xs:
        qq, ss = bitblas.quantize_act_int8(x)
        refs.append(op.forward_w4a8(qq, t["W"], ss, t["scale"], t["zeros"]))
        torch.cuda.synchronize()
    chain()
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert torch.equal(o, r)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        chain()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        chain()
    for o in outs:
        o.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert torch.equal(o, r)


def test_rejections_launch_nothing():
    c = Case(4, 256, 1024, 128, seed=1)
    op = c.layer_op()
    t = c.device(op)
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    with pytest.raises(TypeError):
        op.forward_w4a8(t["A_q"].float(), t["W"], t["a_scale"], t["scale"], t["zeros"])
    with pytest.raises(ValueError):
        op.forward_w4a8(t["A_q"], t["W"], t["a_scale"][:2], t["scale"], t["zeros"])
    with pytest.raises(ValueError):
        op.forward_w4a8(t["A_q"], t["W"], t["a_scale"], t["scale"][:, :4].contiguous(), t["zeros"])
    out = torch.empty(4, 256, dtype=torch.float16, device="cuda")
    rc = lib.bb_matmul_w4a8(op._desc_ref, t["A_q"].data_ptr(), t["W"].data_ptr(), t["a_scale"].data_ptr() + 2,
                            t["scale"].data_ptr(), t["zeros"].data_ptr(), 0, out.data_ptr(), 4, 0, 0, 0)
    assert rc == 5
    assert lib.bb_launch_count() == n0
