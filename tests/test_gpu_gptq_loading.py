"""GPU: GPTQ checkpoints loaded into Linear, GroupedLinear and MoEExperts, bit for bit, in float16 and bfloat16 from float16 and
bfloat16 checkpoint scales.

The checkpoints are built from exact cases (exact_inputs.gptq_checkpoint): integer zero points including 0 (stored by v1 as
2^bits - 1), scales +-2^e and quarter-integer biases, all exact in either 16-bit type, so every layer must return round(V) of the
float64 reference (with bias round(round(V) + b)) whatever the checkpoint's type and the layer's.  The reference is computed on the
device, as in test_gpu_exact_shapes.py.  Also: Linear.forward refuses buffers the kernel cannot read (wrong type, wrong size, on
the host) and outputs it cannot write before anything is launched.
"""
import itertools

import pytest
import torch

import bitblas_oracle as O
import exact_inputs as X
from test_gpu_exact_shapes import _check_experts, _expected_path, _launches
from test_gpu_kernel_grid import _check_split

pytestmark = pytest.mark.gpu

DEV = "cuda"
K, N, G = 2048, 512, 128
MS = (1, 4, 16, 256)   # slab (4-bit) / gemv_mma (2-bit), gemv_mma, gemm_ts with split-K, gemm_ts without
DTYPES = ("float16", "bfloat16")
MODES = ("original", "rescale", "quantized")
TORCH = {"float16": torch.float16, "bfloat16": torch.bfloat16}


# ---- cases --------------------------------------------------------------------------------------------------------------------------
def _linear_cells():
    """the full product A_dtype x checkpoint scale dtype x bits x zeros_mode x v1/v2; act-order, bias and propagate_b each run on
    and off within every (A_dtype, checkpoint dtype) pair, and the rescale cells without act-order use one group (g = -1)"""
    cells = []
    for p, (A_dtype, ckpt) in enumerate(itertools.product(DTYPES, DTYPES)):
        for (b, bits), (mi, mode), v2 in itertools.product(enumerate((4, 2)), enumerate(MODES), (False, True)):
            act = (mi + v2 + p) % 2 == 1
            cells.append(dict(A=A_dtype, ckpt=ckpt, bits=bits, mode=mode, v2=v2, act=act, bias=(b + mi + p // 2) % 2 == 1,
                              tiled=(b + v2 + mi + p) % 2 == 1, g=-1 if mode == "rescale" and not act else G))
    return cells


LINEAR_CELLS = _linear_cells()


def _cell_id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


def _seed(c):
    return LINEAR_CELLS.index(c) * 17 + 1


def linear_case(c, M=max(MS)):
    """(the sorted quantized-zeros case, its GPTQ checkpoint) of a Linear cell"""
    case = X.make_exact_case(M, N, K, A_dtype=c["A"], W_dtype=f"uint{c['bits']}", out_dtype=c["A"], group_size=c["g"],
                             mode="quantized", bias=c["bias"], seed=_seed(c))
    return case, X.gptq_checkpoint(case, v2=c["v2"], act_order=c["act"], scale_dtype=TORCH[c["ckpt"]], seed=_seed(c))


def expected_kernel(bits, tiled, m):
    """the dispatcher's pick (bb_select_kernel) at N = 512, K = 2048: the slab GEMV takes m = 1 for 4-bit weights in either
    storage; below 9 rows the streaming gemv_mma takes the rest, except slab-tiled storage, which only the TMA kernels read"""
    if m == 1 and bits == 4:
        return "gemv_slab"
    if m <= 8 and not tiled:
        return "gemv_mma"
    return "gemm_ts_wgmma"


def _linear(A_dtype, bits, mode, g=G, bias=False, tiled=False):
    import bitblas_b200 as bitblas
    return bitblas.Linear(K, N, bias=bias, A_dtype=A_dtype, W_dtype=f"uint{bits}", out_dtype=A_dtype, group_size=g,
                          with_scaling=True, with_zeros=True, zeros_mode=mode, propagate_b=tiled, enable_tuning=False)


def _repack(layer, ckpt, v2):
    (layer.repack_from_gptq_v2 if v2 else layer.repack_from_gptq)(ckpt)
    return layer


# ---- Linear -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", LINEAR_CELLS, ids=_cell_id)
def test_linear_gptq_exact(c):
    case, ckpt = linear_case(c)
    layer = _repack(_linear(c["A"], c["bits"], c["mode"], c["g"], c["bias"], c["tiled"]).cuda(), ckpt, c["v2"])
    op = layer.bitblas_matmul
    assert op.weight_tiled == c["tiled"]
    if c["act"]:
        assert torch.equal(layer.perm.cpu().long(), ckpt.perm)
    else:
        assert layer.perm is None
    ref_case = X.zeros_mode_case(case, c["mode"])
    A = ckpt.A.to(DEV)
    for m in MS:
        sub = dict(ref_case, A=ref_case["A"][:m], M=m)
        X.prove_exact(sub, device=DEV)
        kernel = expected_kernel(c["bits"], c["tiled"], m)
        assert op.kernel_for(m) == kernel, (m, op.kernel_for(m), kernel)
        split = kernel == "gemm_ts_wgmma" and m <= 128
        if kernel == "gemm_ts_wgmma":
            _check_split(op, m, split, 64)
        got = layer(A[:m])
        X.compare_exact(got, X.exact_reference(sub, DEV), f"Linear m={m} {kernel} {_cell_id(c)}")
        # steady state: the matmul (and split-K reduction) launches, plus the column gather of an act-order layer
        again, n = _launches(lambda: layer(A[:m]))
        assert n == 1 + split + c["act"], (m, kernel, n)
        assert torch.equal(again, got.cpu())


@pytest.mark.parametrize("v2", [False, True])
def test_linear_bf16_act_order_state_dict_round_trip(v2):
    """a bfloat16 act-order layer with bias, loaded from float16 scales, into a fresh layer through its state_dict"""
    case = X.make_exact_case(16, N, K, A_dtype="bfloat16", W_dtype="uint4", out_dtype="bfloat16", group_size=G, mode="quantized",
                             bias=True, seed=5 + v2)
    ckpt = X.gptq_checkpoint(case, v2=v2, act_order=True, scale_dtype=torch.float16, seed=5)
    layer = _repack(_linear("bfloat16", 4, "quantized", bias=True).cuda(), ckpt, v2)
    fresh = _linear("bfloat16", 4, "quantized", bias=True).cuda()
    fresh.load_state_dict(layer.state_dict(), strict=True)
    assert list(fresh.state_dict()) == ["qweight", "scales", "zeros", "bias", "perm"]
    for name, t in layer.state_dict().items():
        assert torch.equal(getattr(fresh, name), t), name
    A = ckpt.A.to(DEV)
    for m in (1, 16):
        got = fresh(A[:m])
        assert torch.equal(got, layer(A[:m]))
        X.compare_exact(got, X.exact_reference(dict(case, A=case["A"][:m]), DEV), f"state_dict round trip m={m} v2={v2}")


# ---- GroupedLinear ------------------------------------------------------------------------------------------------------------------
E_GROUPED = 4
ACT_EXPERTS = (0, 1)   # experts 0 and 1 are act-order, 2 and 3 are not; expert 1 gets no rows
ROUTINGS = ([3, 0, 5, 9], [40, 0, 9, 64])   # T = 17 and 113 around the single-launch limit 8 * E = 32
GROUPED_CELLS = [("float16", "quantized", False), ("float16", "original", True), ("bfloat16", "rescale", False),
                 ("bfloat16", "quantized", True)]


def grouped_cases(A_dtype, v2):
    """(the sorted quantized-zeros case, its GPTQ checkpoint with float16 scales) of every expert"""
    M = max(max(r) for r in ROUTINGS)
    cases = [X.make_exact_case(M, N, K, A_dtype=A_dtype, W_dtype="uint4", out_dtype=A_dtype, group_size=G, mode="quantized",
                               bias=True, seed=300 + e) for e in range(E_GROUPED)]
    return [(x, X.gptq_checkpoint(x, v2=v2, act_order=e in ACT_EXPERTS, scale_dtype=torch.float16, seed=300 + e))
            for e, x in enumerate(cases)]


@pytest.mark.parametrize("A_dtype,mode,v2", GROUPED_CELLS)
def test_grouped_linear_gptq_exact(A_dtype, mode, v2):
    """E = 4 experts from float16 checkpoint scales: the grouped GEMV below 8 E rows, the grouped wgmma GEMM (capturable) and the
    per-expert path above it; every expert's rows against its own exact reference"""
    import bitblas_b200 as bitblas
    E = E_GROUPED
    cases, ckpts = zip(*grouped_cases(A_dtype, v2))
    gl = bitblas.GroupedLinear(E, K, N, bias=True, A_dtype=A_dtype, W_dtype="uint4", out_dtype=A_dtype, group_size=G,
                               with_scaling=True, with_zeros=True, zeros_mode=mode).cuda()
    (gl.repack_from_gptq_v2 if v2 else gl.repack_from_gptq)(ckpts)
    for e, ck in enumerate(ckpts):
        want = ck.perm if ck.perm is not None else torch.arange(K)
        assert torch.equal(gl.perm[e].cpu().long(), want), e
    ref_cases = [X.zeros_mode_case(x, mode) for x in cases]
    op = gl.bitblas_matmul
    for counts in ROUTINGS:
        T = sum(counts)
        A_sorted = torch.cat([x["A"][:n] for x, n in zip(cases, counts)])
        A = torch.cat([ck.A[:n] for ck, n in zip(ckpts, counts)]).to(DEV)
        off = torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=DEV)
        for capturable in ((False,) if T <= 8 * E else (True, False)):
            path = _expected_path(op, T, E, capturable)
            gl(A, off, capturable=capturable)
            got, n = _launches(lambda: gl(A, off, capturable=capturable))
            if path == "per_group":
                assert n >= 1 + sum(1 for c in counts if c), (path, n)
            else:
                assert n == 2, (path, n)   # the grouped column gather and the one grouped launch
            _check_experts(ref_cases, A_sorted, counts, got, f"GroupedLinear {A_dtype} {mode} v2={v2} {path} T={T}", path)


# ---- MoEExperts ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("v2", [False, True])
def test_moe_bf16_gptq_matches_fields(v2, mode):
    """bfloat16 experts from float16 checkpoint scales, with bias, act-order gate/up and an act-order down projection: the GPTQ
    repack gives the buffers, and the outputs, of the same values loaded as fields (gate/up rows in the down projection's sorted
    order, the gate/up column order set as `perm`)"""
    import bitblas_b200 as bitblas
    E, H, I, bits = 4, 512, 256, 4
    kw = dict(A_dtype="bfloat16", W_dtype="uint4", out_dtype="bfloat16", group_size=G, with_scaling=True, with_zeros=True,
              zeros_mode=mode)

    def case(n, k, seed):
        return X.make_exact_case(1, n, k, A_dtype="bfloat16", W_dtype="uint4", out_dtype="bfloat16", group_size=G, mode="quantized",
                                 bias=True, seed=seed)

    gate, up, down = [case(I, H, 10 * e) for e in range(E)], [case(I, H, 10 * e + 1) for e in range(E)], \
        [case(H, I, 10 * e + 2) for e in range(E)]
    # gate and up read the same input, so they share one column order (one seed); the down projection has its own
    ck = [[X.gptq_checkpoint(x, v2=v2, act_order=True, scale_dtype=torch.float16, seed=e + (50 if p == 2 else 0))
           for e, x in enumerate(cs)] for p, cs in enumerate((gate, up, down))]
    assert all(torch.equal(ck[0][e].g_idx, ck[1][e].g_idx) for e in range(E))
    m = bitblas.MoEExperts(E, H, I, bias=True, **kw).cuda()
    (m.repack_from_gptq_v2 if v2 else m.repack_from_gptq)(*ck)

    def fields(cases, rows=None):
        """(weight, scales, zeros, bias) stacked over the experts on the device, each expert's rows in `rows[e]` order"""
        out = [[], [], [], []]
        for e, x in enumerate(cases):
            r = slice(None) if rows is None else rows[e]
            mx = X.zeros_mode_case(x, mode)
            out[0].append(x["fields"][r])
            out[1].append(x["scale"][r])
            out[2].append(torch.from_numpy(O.general_compress(x["qz"][:, r].numpy(), bits)) if mode == "quantized" else mx["zeros"][r])
            out[3].append(x["bias"][r])
        return tuple(torch.stack(t).to(DEV) for t in out)

    pd = [ck[2][e].perm for e in range(E)]   # the down projection's order, absorbed into the gate/up output rows
    ref = bitblas.MoEExperts(E, H, I, bias=True, **kw).cuda()
    ref.load_and_transform_weight(fields(gate, pd), fields(up, pd), fields(down))
    ref.gate_up.perm = torch.stack([ck[0][e].perm for e in range(E)]).to(torch.int32).to(DEV)
    for proj in ("gate_up", "down"):
        for name in ("qweight", "scales", "zeros", "bias", "perm"):
            a, b = getattr(getattr(m, proj), name), getattr(getattr(ref, proj), name)
            assert (a is None and b is None) or torch.equal(a, b), (proj, name)
    assert m.down.perm is None
    g = torch.Generator().manual_seed(3)
    for T in (8, 100):   # 16 rows: the grouped GEMVs; 200 rows: the grouped wgmma GEMMs
        ids = torch.rand((T, E), generator=g).argsort(1)[:, :2].to(torch.int32).to(DEV)
        w = torch.softmax(torch.randn((T, 2), generator=g), 1).to(DEV)
        x = (torch.rand((T, H), generator=g) - 0.5).to(torch.bfloat16).to(DEV)
        assert torch.equal(m(x, ids, w), ref(x, ids, w)), T


# ---- Linear.forward validation ------------------------------------------------------------------------------------------------------
def _valid_layer():
    """a bfloat16 act-order layer with bias from float16 scales (the column gather launches first: a check after it would be late)"""
    case = X.make_exact_case(4, N, K, A_dtype="bfloat16", W_dtype="uint4", out_dtype="bfloat16", group_size=G, mode="quantized",
                             bias=True, seed=77)
    ckpt = X.gptq_checkpoint(case, v2=False, act_order=True, scale_dtype=torch.float16, seed=77)
    layer = _repack(_linear("bfloat16", 4, "quantized", bias=True).cuda(), ckpt, False)
    return case, layer, ckpt.A.to(DEV)


def _refused(exc, match, layer, A, **kw):
    from bitblas_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    with pytest.raises(exc, match=match):
        layer(A, **kw)
    torch.cuda.synchronize()
    assert lib.bb_launch_count() == n0


def test_linear_forward_refuses_wrong_buffers_before_launch():
    import bitblas_b200 as bitblas
    case, layer, A = _valid_layer()
    ref = X.exact_reference(case, DEV)
    X.compare_exact(layer(A), ref, "valid layer")
    # float16 scales handed to a bfloat16 layer by load_and_transform_weight
    fields = bitblas.Linear(K, N, bias=True, A_dtype="bfloat16", W_dtype="uint4", out_dtype="bfloat16", group_size=G,
                            with_scaling=True, with_zeros=True, zeros_mode="quantized").cuda()
    fields.load_and_transform_weight(case["fields"].to(DEV), scales=case["scale"].half().to(DEV), zeros=case["zeros"].to(DEV),
                                     bias=case["bias"].to(DEV))
    _refused(TypeError, "scale has dtype torch.float16", fields, A)
    # a module never moved to the GPU
    _refused(RuntimeError, "W must be a CUDA tensor", _linear("bfloat16", 4, "quantized", bias=True), A)
    # a buffer that is not on A's device
    cpu_bias = _repack(_linear("bfloat16", 4, "quantized", bias=True).cuda(), X.gptq_checkpoint(case, v2=False, act_order=True,
                       scale_dtype=torch.float16, seed=77), False)
    cpu_bias.bias = cpu_bias.bias.cpu()
    _refused(RuntimeError, "bias must be a CUDA tensor", cpu_bias, A)
    # outputs of the wrong type or size
    _refused(TypeError, "output has dtype torch.float16", layer, A, output=torch.empty((4, N), dtype=torch.float16, device=DEV))
    _refused(ValueError, "output has 1536 elements", layer, A, output=torch.empty((3, N), dtype=torch.bfloat16, device=DEV))
    # buffers replaced after a successful call are checked again; the restored buffers run again
    good = {name: getattr(layer, name) for name in ("qweight", "scales", "zeros", "bias")}
    wrong = [("zeros", torch.zeros((K // G, N * 4 // 8 - 1), dtype=torch.int8, device=DEV), ValueError, "zeros has 4080 elements"),
             ("scales", good["scales"][:, :-1].contiguous(), ValueError, "scale has 7680 elements"),
             ("qweight", good["qweight"].view(torch.int16).clone(), TypeError, "W has dtype torch.int16"),
             ("bias", good["bias"].half(), TypeError, "bias has dtype torch.float16"),
             ("scales", good["scales"].cpu(), RuntimeError, "scale must be a CUDA tensor")]
    for name, t, exc, match in wrong:
        setattr(layer, name, t)
        _refused(exc, match, layer, A)
        _refused(exc, match, layer, A)   # a refused set is not remembered as checked
        setattr(layer, name, good[name])
        X.compare_exact(layer(A), ref, f"restored {name}")
