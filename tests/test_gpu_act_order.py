"""GPU: GPTQ act-order checkpoints.  bb_permute_cols against torch indexing; Linear, GroupedLinear and MoEExperts loaded from act-order
GPTQ modules against the same checkpoint stored in sorted order (bit for bit), against float64 dequantisation through g_idx, and
their launch counts and graph replays."""
import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

DEV = "cuda"


# ---- fixtures: GPTQ stand-ins ---------------------------------------------------------------------------------------------------
def act_order_g_idx(K, g, gen):
    """as GPTQ builds it with desc_act: the columns quantized in order `perm` go to groups in that order, g_idx[perm[i]] = i // g"""
    perm = torch.randperm(K, generator=gen)
    g_idx = torch.empty(K, dtype=torch.int32)
    g_idx[perm] = torch.arange(K, dtype=torch.int32) // g
    return g_idx


class GPTQ:
    """minimal stand-in for a GPTQ QuantLinear: qweight int32 [K*bits/32, N], qzeros int32 [K/g, N*bits/32], scales [K/g, N],
    bias, g_idx; keeps the unpacked values (intw [K, N], zint [K/g, N]) for the references"""

    def __init__(self, K, N, g, bits, seed, act_order=True, with_bias=False, v2=False):
        gen = torch.Generator().manual_seed(seed)
        self.bits, self.g = bits, g
        self.intw = torch.randint(0, 2**bits, (K, N), generator=gen, dtype=torch.int32)
        self.zint = torch.randint(0, 2**bits - (0 if v2 else 1), (K // g, N), generator=gen, dtype=torch.int32)
        self.scales = (torch.rand((K // g, N), generator=gen) * 0.1 + 0.01).half()
        self.bias = torch.nn.Parameter(torch.rand(N, generator=gen).half(), requires_grad=False) if with_bias else None
        self.g_idx = act_order_g_idx(K, g, gen) if act_order else torch.arange(K, dtype=torch.int32) // g
        self._pack()

    def _pack(self):
        per = 32 // self.bits
        K, N = self.intw.shape
        self.qweight = torch.zeros((K // per, N), dtype=torch.int32)
        for i in range(per):
            self.qweight |= self.intw[i::per] << (self.bits * i)
        self.qzeros = torch.zeros((K // self.g, N // per), dtype=torch.int32)
        for i in range(per):
            self.qzeros |= self.zint[:, i::per] << (self.bits * i)

    def sorted(self):
        """the same checkpoint with its K axis stored in g_idx order and a trivial g_idx"""
        s = GPTQ.__new__(GPTQ)
        perm = torch.sort(self.g_idx.long(), stable=True).indices
        s.bits, s.g, s.zint, s.scales, s.bias = self.bits, self.g, self.zint, self.scales, self.bias
        s.intw = self.intw[perm].contiguous()
        s.g_idx = torch.arange(self.intw.shape[0], dtype=torch.int32) // self.g
        s._pack()
        return s, perm

    def dense(self, v2):
        """float64 [N, K]: W[k, n] = (q - z[g_idx[k], n]) * s[g_idx[k], n] (v1 stores the zero point minus one)"""
        gi = self.g_idx.long()
        z = self.zint.double() + (0 if v2 else 1)
        return ((self.intw.double() - z[gi]) * self.scales.double()[gi]).T


def _launches(fn):
    from bitblas_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.bb_launch_count() - n0


def _linear(K, N, bits, mode, **kw):
    import bitblas_b200 as bitblas
    return bitblas.Linear(K, N, A_dtype="float16", W_dtype=f"uint{bits}", group_size=128, with_scaling=True, with_zeros=True,
                          zeros_mode=mode, enable_tuning=False, **kw).cuda()


def _repack(layer, mod, v2):
    (layer.repack_from_gptq_v2 if v2 else layer.repack_from_gptq)(mod)
    return layer


# ---- bb_permute_cols ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows", [1, 7, 4096])
@pytest.mark.parametrize("K", [128, 1032, 8192, 28672])
def test_permute_cols_dense(dtype, rows, K):
    from bitblas_b200 import permute_cols
    gen = torch.Generator().manual_seed(rows * 7 + K)
    A = torch.randn((rows, K), generator=gen).to(dtype).to(DEV)
    perm = torch.randperm(K, generator=gen).to(torch.int32).to(DEV)
    assert torch.equal(permute_cols(A, perm), A[:, perm.long()])


def test_permute_cols_clamps_perm_values():
    from bitblas_b200 import permute_cols
    K = 256
    A = torch.randn((5, K)).half().to(DEV)
    perm = torch.randint(-3 * K, 4 * K, (K,), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
    perm[:4] = torch.tensor([-1, K, -2**31, 2**31 - 1], dtype=torch.int32)
    assert torch.equal(permute_cols(A, perm.to(DEV)), A[:, perm.long().clamp(0, K - 1).to(DEV)])


@pytest.mark.parametrize("case", ["sorted", "empty", "out_of_range", "unclaimed", "decreasing"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_permute_cols_grouped(case, dtype):
    from bitblas_b200 import permute_cols
    E, K, T = 6, 512, 300
    gen = torch.Generator().manual_seed(len(case))
    offsets = {"sorted": [0, 40, 41, 100, 180, 299, 300],
               "empty": [0, 0, 120, 120, 120, 300, 300],
               "out_of_range": [-50, 10, 20, 30, 40, 290, 1000],
               "unclaimed": [20, 60, 80, 80, 150, 200, 230],
               "decreasing": [100, 150, 20, 60, 100, 20, 0]}[case]   # groups 1, 4 and 5 end below their start
    A = torch.randn((T, K), generator=gen).to(dtype).to(DEV)
    perm = torch.stack([torch.randperm(K, generator=gen) for _ in range(E)]).to(torch.int32)
    out = torch.full((T, K), 7.0, dtype=dtype, device=DEV)
    permute_cols(A, perm.to(DEV), torch.tensor(offsets, dtype=torch.int32, device=DEV), output=out)
    ref = torch.full((T, K), 7.0, dtype=dtype)
    Ac = A.cpu()
    for e in range(E):
        b = min(max(offsets[e], 0), T)
        end = max(min(max(offsets[e + 1], 0), T), b)   # a group whose end is below its start is empty
        ref[b:end] = Ac[b:end][:, perm[e].long()]
    assert torch.equal(out.cpu(), ref)


# ---- Linear -------------------------------------------------------------------------------------------------------------------
LINEAR_CASES = [(m, bits, mode, v2) for m in (1, 4, 16, 256) for bits in (4, 2) for mode in ("original", "rescale", "quantized")
                for v2 in (False, True)]


@pytest.mark.parametrize("m,bits,mode,v2", LINEAR_CASES)
def test_linear_equals_sorted_checkpoint(m, bits, mode, v2):
    """the act-order layer and the same checkpoint stored in sorted order: equal buffers, and lin_act(A) == lin_plain(A[:, perm])"""
    K, N = 1024, 512
    mod = GPTQ(K, N, 128, bits, seed=m * 10 + bits, v2=v2, with_bias=m == 4)
    plain_mod, perm = mod.sorted()
    lin_act = _repack(_linear(K, N, bits, mode, bias=m == 4), mod, v2)
    lin_plain = _repack(_linear(K, N, bits, mode, bias=m == 4), plain_mod, v2)
    assert lin_plain.perm is None and torch.equal(lin_act.perm.cpu().long(), perm)
    for name in ("qweight", "scales", "zeros"):
        assert torch.equal(getattr(lin_act, name), getattr(lin_plain, name)), name
    A = (torch.rand((m, K), generator=torch.Generator().manual_seed(m)) - 0.5).half().to(DEV)
    assert torch.equal(lin_act(A), lin_plain(A[:, perm.to(DEV)]))


def test_linear_propagate_b_equals_sorted_checkpoint():
    K, N = 1024, 512
    mod = GPTQ(K, N, 128, 4, seed=3)
    plain_mod, perm = mod.sorted()
    lin_act = _repack(_linear(K, N, 4, "quantized", propagate_b=True), mod, False)
    lin_plain = _repack(_linear(K, N, 4, "quantized", propagate_b=True), plain_mod, False)
    assert torch.equal(lin_act.qweight, lin_plain.qweight)
    for m in (1, 16):
        A = (torch.rand((m, K)) - 0.5).half().to(DEV)
        assert torch.equal(lin_act(A), lin_plain(A[:, perm.to(DEV)]))


@pytest.mark.parametrize("bits", [4, 2])
@pytest.mark.parametrize("m", [1, 16, 256])
@pytest.mark.parametrize("v2", [False, True])
def test_linear_matches_float64_through_g_idx(bits, m, v2):
    K, N = 1024, 512
    mod = GPTQ(K, N, 128, bits, seed=40 + m, v2=v2, with_bias=True)
    lin = _repack(_linear(K, N, bits, "original", bias=True), mod, v2)
    A = (torch.rand((m, K), generator=torch.Generator().manual_seed(m)) - 0.5).half()
    ref = (A.double() @ mod.dense(v2).T + mod.bias.data.double()).half()
    H.assert_fp_close(lin(A.to(DEV)).cpu(), ref, f"act-order bits={bits} m={m} v2={v2}")


def test_linear_launch_counts_and_graph_replay():
    import bitblas_b200 as bitblas
    K, N = 1024, 512
    mod = GPTQ(K, N, 128, 4, seed=9)
    lin = _repack(_linear(K, N, 4, "quantized"), mod, False)
    A = (torch.rand((1, K)) - 0.5).half().to(DEV)
    _, n = _launches(lambda: lin(A))
    assert n == 2
    trivial = _repack(_linear(K, N, 4, "quantized"), GPTQ(K, N, 128, 4, seed=9, act_order=False), False)
    assert trivial.perm is None
    _, n = _launches(lambda: trivial(A))
    assert n == 1
    for m in (1, 64):
        a_d = torch.zeros((m, K), dtype=torch.float16, device=DEV)
        out_d = torch.zeros((m, N), dtype=torch.float16, device=DEV)
        step = bitblas.CapturedStep(lambda: lin(a_d, output=out_d))
        for trial in range(3):
            a_d.copy_((torch.rand((m, K), generator=torch.Generator().manual_seed(trial)) - 0.5).half())
            step()
            assert torch.equal(out_d, lin(a_d)), (m, trial)


# ---- GroupedLinear ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("counts", [[3, 0, 5, 1], [40, 0, 9, 64]])    # the grouped GEMV and the grouped GEMM
def test_grouped_linear_matches_per_expert_linear(counts):
    import bitblas_b200 as bitblas
    E, K, N, g = 4, 512, 256, 128
    kw = dict(A_dtype="float16", W_dtype="uint4", group_size=g, with_scaling=True, with_zeros=True, zeros_mode="quantized")
    mods = [GPTQ(K, N, g, 4, seed=60 + e, act_order=e != 1 and e != 3, with_bias=True) for e in range(E)]
    gl = bitblas.GroupedLinear(E, K, N, bias=True, **kw).cuda()
    gl.repack_from_gptq(mods)
    assert gl.perm.shape == (E, K)
    assert torch.equal(gl.perm[1].cpu(), torch.arange(K, dtype=torch.int32))
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + c)
    A = (torch.rand((offsets[-1], K), generator=torch.Generator().manual_seed(1)) - 0.5).half().to(DEV)
    got, n = _launches(lambda: gl(A, torch.tensor(offsets, dtype=torch.int32, device=DEV), capturable=True))
    assert n == 2
    for e, mod in enumerate(mods):
        lin = bitblas.Linear(K, N, bias=True, **kw).cuda()
        lin.repack_from_gptq(mod)
        assert (lin.perm is not None) == (e not in (1, 3))
        r0, r1 = offsets[e], offsets[e + 1]
        if r1 > r0:
            H.assert_fp_close(got[r0:r1].cpu(), lin(A[r0:r1]).cpu(), f"expert {e}")
            H.assert_fp_close(got[r0:r1].cpu(), (A[r0:r1].cpu().double() @ mod.dense(False).T + mod.bias.data.double()).half(),
                              f"expert {e} float64")


def test_grouped_linear_without_act_order_keeps_one_launch():
    import bitblas_b200 as bitblas
    E, K, N = 4, 512, 256
    gl = bitblas.GroupedLinear(E, K, N, A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
                               zeros_mode="quantized").cuda()
    gl.repack_from_gptq([GPTQ(K, N, 128, 4, seed=e, act_order=False) for e in range(E)])
    assert gl.perm is None
    A = (torch.rand((12, K)) - 0.5).half().to(DEV)
    _, n = _launches(lambda: gl(A, torch.tensor([0, 3, 6, 9, 12], dtype=torch.int32, device=DEV)))
    assert n == 1


# ---- MoEExperts ----------------------------------------------------------------------------------------------------------------
E_, H_, I_, G_ = 4, 512, 256, 128
MOE_KW = dict(A_dtype="float16", W_dtype="uint4", group_size=G_, with_scaling=True, with_zeros=True, zeros_mode="quantized")


def _moe_mods(seed, act_order=True):
    """gate and up of an expert share one g_idx (they read the same input); expert 1 is not act-order"""
    gate, up, down = [], [], []
    for e in range(E_):
        ao = act_order and e != 1
        gm, um = GPTQ(H_, I_, G_, 4, seed=seed + 3 * e, act_order=ao), GPTQ(H_, I_, G_, 4, seed=seed + 3 * e + 1, act_order=ao)
        um.g_idx = gm.g_idx
        gate.append(gm)
        up.append(um)
        down.append(GPTQ(I_, H_, G_, 4, seed=seed + 3 * e + 2, act_order=ao))
    return gate, up, down


def _moe(mods, v2=False):
    import bitblas_b200 as bitblas
    m = bitblas.MoEExperts(E_, H_, I_, **MOE_KW).cuda()
    (m.repack_from_gptq_v2 if v2 else m.repack_from_gptq)(*mods)
    return m


def _routing(T, k, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.rand((T, E_), generator=g).argsort(dim=1)[:, :k].to(torch.int32)
    w = torch.softmax(torch.randn((T, k), generator=g), dim=1)
    x = (torch.rand((T, H_), generator=g) - 0.5).half()
    return x, ids, w


def _composed(mods, x, ids, w):
    """per-expert act-order Linears: silu(gate(x)) * up(x) in fp32, rounded to fp16, down, float64 combine"""
    import bitblas_b200 as bitblas
    out = torch.zeros((x.shape[0], H_), dtype=torch.float64)
    xd = x.to(DEV)
    for e in range(E_):
        lins = []
        for mod, (K, N) in zip((mods[0][e], mods[1][e], mods[2][e]), ((H_, I_), (H_, I_), (I_, H_))):
            lin = bitblas.Linear(K, N, **MOE_KW).cuda()
            lin.repack_from_gptq(mod)
            lins.append(lin)
        h = (torch.nn.functional.silu(lins[0](xd).float()) * lins[1](xd).float()).half()
        y = lins[2](h).cpu().double()
        sel = (ids == e).double() * w.double()
        out += sel.sum(1, keepdim=True) * y
    return out


def _oracle(mods, x, ids, w):
    Wg, Wu, Wd = ([m.dense(False) for m in p] for p in mods)
    out = torch.zeros((x.shape[0], H_), dtype=torch.float64)
    xd = x.double()
    for t in range(x.shape[0]):
        for j in range(ids.shape[1]):
            e = int(ids[t, j])
            gt, up = Wg[e] @ xd[t], Wu[e] @ xd[t]
            out[t] += float(w[t, j]) * (Wd[e] @ (gt / (1 + torch.exp(-gt)) * up))
    return out


def _normwise(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


@pytest.mark.parametrize("T", [1, 512])
def test_moe_matches_composition_and_oracle(T):
    mods = _moe_mods(seed=T)
    m = _moe(mods)
    assert m.gate_up.perm.shape == (E_, H_) and m.down.perm is None
    x, ids, w = _routing(T, 2, seed=T + 1)
    got, n = _launches(lambda: m(x.to(DEV), ids.to(DEV), w.to(DEV)))
    assert n == 5
    got = got.cpu()
    assert _normwise(got, _composed(mods, x, ids, w)) <= 2e-3
    assert _normwise(got, _oracle(mods, x, ids, w)) <= 1e-2
    plain = _moe(_moe_mods(seed=T, act_order=False))
    assert plain.gate_up.perm is None
    _, n = _launches(lambda: plain(x.to(DEV), ids.to(DEV), w.to(DEV)))
    assert n == 4


def test_moe_down_perm_is_absorbed_into_gate_up_rows():
    """deinterleaving the stored gate/up rows and undoing the down projection's order gives each expert's own gate and up rows"""
    from bitblas_b200.moe import deinterleave_gate_up
    mods = _moe_mods(seed=5)
    m = _moe(mods)
    g, u = deinterleave_gate_up(m.gate_up.qweight, "weight")
    gs, us = deinterleave_gate_up(m.gate_up.scales, "scale")
    for e in range(E_):
        ref = {}
        for name, mod in (("gate", mods[0][e]), ("up", mods[1][e])):
            lin = _linear(H_, I_, 4, "quantized")
            lin.repack_from_gptq(mod)
            ref[name] = lin
        pd = torch.sort(mods[2][e].g_idx.long(), stable=True).indices.to(DEV)
        inv = torch.argsort(pd)
        assert torch.equal(g[e][inv], ref["gate"].qweight) and torch.equal(u[e][inv], ref["up"].qweight), e
        assert torch.equal(gs[e][inv], ref["gate"].scales) and torch.equal(us[e][inv], ref["up"].scales), e


def test_moe_graph_replay_matches_eager():
    import bitblas_b200 as bitblas
    m = _moe(_moe_mods(seed=11), v2=True)
    T, k = 96, 2
    x_d = torch.zeros((T, H_), dtype=torch.float16, device=DEV)
    ids_d = torch.zeros((T, k), dtype=torch.int32, device=DEV)
    w_d = torch.zeros((T, k), dtype=torch.float32, device=DEV)
    out_d = torch.zeros((T, H_), dtype=torch.float16, device=DEV)
    step = bitblas.CapturedStep(lambda: m(x_d, ids_d, w_d, output=out_d))
    for trial in range(3):
        x, ids, w = _routing(T, k, seed=50 + trial)
        x_d.copy_(x)
        ids_d.copy_(ids)
        w_d.copy_(w)
        step()
        eager = m(x.to(DEV), ids.to(DEV), w.to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(out_d, eager), trial


def test_moe_rejects_gate_and_up_with_different_g_idx():
    import bitblas_b200 as bitblas
    gate, up, down = _moe_mods(seed=13)
    up[2] = GPTQ(H_, I_, G_, 4, seed=99)
    with pytest.raises(ValueError, match="expert 2: gate and up have different g_idx"):
        bitblas.MoEExperts(E_, H_, I_, **MOE_KW).cuda().repack_from_gptq(gate, up, down)
