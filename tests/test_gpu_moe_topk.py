"""GPU: top-k gating (bb_moe_topk / moe_topk) against a float64 restatement of its semantics: the model presets at every token
count and logits dtype, exact ties, a binding group limit, the selection bias, NaN logits, determinism, and moe_topk -> MoEExperts
captured in one CUDA graph."""
import pytest
import torch

from test_gpu_moe import _make_block, _normwise, _oracle

pytestmark = pytest.mark.gpu

DEV = "cuda"
TORCH = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}
GAP = 1e-6   # relative gap between consecutive reference values above which the ids must match

# name -> (E, moe_topk keyword arguments); the last three stretch the limits (E = 256, k = 32, 32 groups, one expert)
PRESETS = {
    "mixtral-8x7b": (8, dict(top_k=2, renormalize=True)),
    "qwen3-30b-a3b": (128, dict(top_k=8, renormalize=True)),
    "qwen1.5-moe": (60, dict(top_k=4)),
    "deepseek-v2-lite": (64, dict(top_k=6, routed_scaling_factor=1.0)),
    "deepseek-v2": (160, dict(top_k=6, num_expert_group=8, topk_group=3, group_score="max", routed_scaling_factor=16.0)),
    "deepseek-v3": (256, dict(top_k=8, scoring="sigmoid", bias=True, num_expert_group=8, topk_group=4, group_score="top2_sum",
                              renormalize=True, routed_scaling_factor=2.5)),
    "e256-k32": (256, dict(top_k=32, renormalize=True)),
    "e256-k32-32groups": (256, dict(top_k=32, scoring="sigmoid", bias=True, num_expert_group=32, topk_group=4,
                                    group_score="top2_sum", routed_scaling_factor=0.5)),
    "e1-k1": (1, dict(top_k=1, scoring="sigmoid")),
}


# ---- the float64 reference ------------------------------------------------------------------------------------------------------
def _order(v, last=None):
    """indices along the last axis by the selection order: entries in `last` after all others, then NaN after every number, then
    descending value, ties to the lower index (three stable sorts, least significant key first)"""
    o = torch.sort(torch.where(torch.isnan(v), -torch.inf, v), dim=-1, descending=True, stable=True).indices
    o = o.gather(-1, torch.sort(torch.isnan(v).gather(-1, o).to(torch.int8), dim=-1, stable=True).indices)
    if last is not None:
        o = o.gather(-1, torch.sort(last.gather(-1, o).to(torch.int8), dim=-1, stable=True).indices)
    return o


def reference(logits, top_k, scoring="softmax", renormalize=False, correction_bias=None, num_expert_group=None, topk_group=None,
              group_score="max", routed_scaling_factor=1.0):
    """-> (ids [T, k], weights [T, k] float64, qualifies [T]): qualifies says that every gap between consecutive values that
    decide the result (the k + 1 best selection values, and the groups at the topk_group boundary) exceeds GAP relative"""
    l = logits.double()
    T, E = l.shape
    nan = torch.isnan(l)
    if scoring == "softmax":
        lm = torch.where(nan, -torch.inf, l)
        ex = torch.exp(lm - lm.max(dim=1, keepdim=True).values)
        s = torch.where(nan, torch.nan, ex / ex.sum(dim=1, keepdim=True))
    else:
        s = 1.0 / (1.0 + torch.exp(-l))
    v = s + correction_bias.double() if correction_bias is not None else s
    excluded = torch.zeros_like(v, dtype=torch.bool)
    ok = torch.ones(T, dtype=torch.bool)

    def gap_ok(a, b):   # a NaN ranks below every number and NaNs by index: no rounding can reorder them
        return ((a - b).abs() > GAP * torch.maximum(a.abs(), b.abs())) | torch.isnan(a) | torch.isnan(b)

    if num_expert_group is not None and num_expert_group > 1:
        n = num_expert_group
        vg = v.view(T, n, E // n)
        best = vg.gather(-1, _order(vg)[..., :2])
        score = best[..., 0] + best[..., 1] if group_score == "top2_sum" else best[..., 0]
        go = _order(score)
        keep = torch.zeros((T, n), dtype=torch.bool).scatter_(1, go[:, :topk_group], True)
        excluded = ~keep.repeat_interleave(E // n, dim=1)
        if topk_group < n:
            ranked = score.gather(1, go)
            ok &= gap_ok(ranked[:, topk_group - 1], ranked[:, topk_group])
    order = _order(v, excluded)
    ids = order[:, :top_k]
    sv = v.gather(1, order)
    allowed = int((~excluded[0]).sum())
    for j in range(min(top_k, allowed - 1)):
        ok &= gap_ok(sv[:, j], sv[:, j + 1])
    w = s.gather(1, ids)
    if renormalize:
        tot = w.sum(dim=1, keepdim=True)
        w = torch.where(tot != 0, w / tot, torch.zeros_like(w))
    return ids.to(torch.int32), w * routed_scaling_factor, ok


# ---- inputs ----------------------------------------------------------------------------------------------------------------------
def _distinct_logits(T, E, gen):
    """E distinct values per row from the 512 multiples of 1/64 in [-4, 4): exact in fp16, bf16 and fp32"""
    pick = torch.rand((T, 512), generator=gen).argsort(dim=1)[:, :E]
    return (pick - 256).double() / 64


def _preset(name, T, dtype, seed):
    """(logits on the device, k, moe_topk keyword arguments, reference ids and weights) with every row qualifying: rows that do
    not are drawn again"""
    E, kw = PRESETS[name]
    kw = dict(kw)
    gen = torch.Generator().manual_seed(seed)
    if kw.pop("bias", False):
        kw["correction_bias"] = (torch.rand(E, generator=gen) * 0.25).float()
    k = kw.pop("top_k")
    logits = _distinct_logits(T, E, gen).to(TORCH[dtype])
    for _ in range(20):
        ids, w, ok = reference(logits, k, **kw)
        if ok.all():
            break
        bad = (~ok).nonzero()[:, 0]
        logits[bad] = _distinct_logits(len(bad), E, gen).to(TORCH[dtype])
    assert ok.all(), f"{int((~ok).sum())} rows still within {GAP} of a tie"
    if "correction_bias" in kw:
        kw["correction_bias"] = kw["correction_bias"].to(DEV)
    return logits.to(DEV), k, kw, (ids, w)


def _run(logits_d, k, **kw):
    from bitblas_b200 import moe_topk
    ids, w = moe_topk(logits_d, k, **kw)
    assert ids.dtype == torch.int32 and w.dtype == torch.float32 and ids.shape == w.shape == (logits_d.shape[0], k)
    return ids.cpu(), w.cpu()


def _check_weights(w, ref_w):
    err = (w.double() - ref_w).abs()
    bad = ~(err <= 1e-5 * ref_w.abs())
    assert not bad.any(), f"{int(bad.sum())} weights outside 1e-5 relative; worst {float((err / ref_w.abs()).max()):.3g}"


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("T", [1, 7, 64, 2048, 16384])
@pytest.mark.parametrize("name", list(PRESETS))
def test_preset_matches_float64(name, T, dtype):
    seed = sum(map(ord, name)) * 1000 + T + list(TORCH).index(dtype)
    logits_d, k, kw, (ref_ids, ref_w) = _preset(name, T, dtype, seed)
    ids, w = _run(logits_d, k, **kw)
    assert torch.equal(ids, ref_ids), f"{int((ids != ref_ids).any(dim=1).sum())} rows differ"
    _check_weights(w, ref_w)


# ---- exact ties ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,k,kw", [(8, 2, {}), (64, 6, {}), (256, 32, dict(renormalize=True)), (60, 4, dict(scoring="sigmoid")),
                                    (160, 6, dict(num_expert_group=8, topk_group=3)),
                                    (256, 8, dict(scoring="sigmoid", num_expert_group=8, topk_group=4, group_score="top2_sum"))])
@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
def test_all_equal_logits_pick_the_lowest_ids(E, k, kw, dtype):
    logits = torch.full((5, E), 0.75, dtype=TORCH[dtype])
    logits[1] = -3.0
    ids, w = _run(logits.to(DEV), k, **kw)
    assert torch.equal(ids, torch.arange(k, dtype=torch.int32).expand(5, k))
    assert torch.equal(w[:, 1:], w[:, :1].expand(5, k - 1))   # equal scores, equal weights
    ref_ids, ref_w, _ = reference(logits, k, **kw)
    assert torch.equal(ids, ref_ids)
    _check_weights(w, ref_w)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("scoring", ["softmax", "sigmoid"])
def test_equal_pair_straddling_k_goes_to_the_lower_index(scoring, dtype):
    T, E, k = 256, 64, 6
    gen = torch.Generator().manual_seed(5)
    logits = _distinct_logits(T, E, gen)
    order = _order(logits)
    lo, hi = torch.minimum(order[:, k - 1], order[:, k]), torch.maximum(order[:, k - 1], order[:, k])
    r = torch.arange(T)
    logits[r, hi] = logits[r, lo]                        # the k-th and (k+1)-th values tie
    logits = logits.to(TORCH[dtype])
    ids, w = _run(logits.to(DEV), k, scoring=scoring)
    ref_ids, ref_w, _ = reference(logits, k, scoring=scoring)
    assert torch.equal(ids, ref_ids)
    assert torch.equal(ids[:, k - 1].long(), lo), "the lower index of the tied pair wins the last slot"
    assert not (ids.long() == hi[:, None]).any()
    _check_weights(w, ref_w)


def test_tied_pair_inside_the_top_k_keeps_index_order():
    E, k = 32, 4
    logits = torch.linspace(-2, 2, E).repeat(3, 1)
    logits[:, 5] = logits[:, 31]                         # experts 5 and 31 share the best value
    ids, _ = _run(logits.to(DEV), k)
    assert torch.equal(ids, torch.tensor([[5, 31, 30, 29]] * 3, dtype=torch.int32))


def test_tied_group_scores_keep_the_lower_group():
    E, n = 16, 4   # groups of 4
    x = torch.full((E,), -4.0)
    # max: groups 1 and 2 share the best max; topk_group = 1 keeps group 1
    a = x.clone()
    a[4:8] = torch.tensor([0.0, 3.0, 1.0, -1.0])
    a[8:12] = torch.tensor([3.0, 2.5, 2.0, 2.2])
    ids, _ = _run(a[None].to(DEV), 2, num_expert_group=n, topk_group=1)
    assert ids.tolist() == [[5, 6]]
    # top2_sum: groups 0 and 2 have the same two best values, group 3 a larger pair; topk_group = 2 keeps groups 3 and 0
    b = x.clone()
    b[0:4] = torch.tensor([2.0, 1.0, -1.0, -2.0])
    b[8:12] = torch.tensor([1.0, -1.0, -2.0, 2.0])
    b[12:16] = torch.tensor([3.0, 2.5, -3.0, -3.0])
    ids, _ = _run(b[None].to(DEV), 3, scoring="sigmoid", num_expert_group=n, topk_group=2, group_score="top2_sum")
    assert ids.tolist() == [[12, 13, 0]]
    for logits, kw in ((a, dict(top_k=2, num_expert_group=n, topk_group=1)),
                       (b, dict(top_k=3, scoring="sigmoid", num_expert_group=n, topk_group=2, group_score="top2_sum"))):
        k = kw.pop("top_k")
        assert torch.equal(_run(logits[None].to(DEV), k, **kw)[0], reference(logits[None], k, **kw)[0])


# ---- group limit, bias, NaN ------------------------------------------------------------------------------------------------------
def test_group_limit_binds():
    """top2_sum: in every row the k best experts overall are the stars of four groups with one strong expert each, and two groups
    with a pair of good experts outscore them; the result must come from those two groups"""
    T, E, n, k = 512, 64, 8, 4
    gs = E // n
    gen = torch.Generator().manual_seed(9)
    logits = -6.0 + (_distinct_logits(T, E, gen) + 4) / 16          # distinct background values in [-6, -5.5)
    groups = torch.stack([torch.randperm(n, generator=gen)[:6] for _ in range(T)])
    r = torch.arange(T)
    for j in range(4):
        logits[r, groups[:, j] * gs + j] = 6.0 + 0.25 * j
    for j in range(2):
        logits[r, groups[:, 4 + j] * gs + 1] = 1.0 + 0.1 * j
        logits[r, groups[:, 4 + j] * gs + 2] = 0.8 + 0.1 * j
    logits = logits.float()
    kw = dict(scoring="sigmoid", num_expert_group=n, topk_group=2, group_score="top2_sum")
    ids, w = _run(logits.to(DEV), k, **kw)
    ref_ids, ref_w, ok = reference(logits, k, **kw)
    assert ok.all()
    assert torch.equal(ids, ref_ids)
    _check_weights(w, ref_w)
    best = _order(logits)[:, :k]
    assert ((best // gs)[:, :, None] == groups[:, None, :4]).any(dim=2).all(), "the k best experts lie in the star groups"
    g = ids.long() // gs
    assert ((g == groups[:, 4:5]) | (g == groups[:, 5:6])).all()
    # group-limited max keeping 3 of the 4 star groups: the weakest star, one of the k best overall, is excluded
    kw = dict(num_expert_group=n, topk_group=3, group_score="max")
    ids, w = _run(logits.to(DEV), k, **kw)
    ref_ids, ref_w, ok = reference(logits, k, **kw)
    assert ok.all() and torch.equal(ids, ref_ids)
    _check_weights(w, ref_w)
    assert not (ids.long() == (groups[:, :1] * gs)).any() and (best[:, 3] == groups[:, 0] * gs).all()


def test_bias_steers_selection_only():
    T, E, k = 2048, 256, 8
    gen = torch.Generator().manual_seed(13)
    logits = _distinct_logits(T, E, gen).float()
    bias = (torch.rand(E, generator=gen) * 0.25).float()
    kw = dict(scoring="sigmoid", num_expert_group=8, topk_group=4, group_score="top2_sum")
    ids_b, w_b = _run(logits.to(DEV), k, correction_bias=bias.to(DEV), **kw)
    ids_0, w_0 = _run(logits.to(DEV), k, **kw)
    changed = (ids_b != ids_0).any(dim=1)
    assert changed.float().mean() > 0.5, "the bias changes the selection"
    ref_ids, ref_w, ok = reference(logits, k, correction_bias=bias, **kw)
    assert ok.float().mean() > 0.99
    assert torch.equal(ids_b[ok], ref_ids[ok])
    # the weight of an expert is its sigmoid score, bias or not: bit-identical wherever both runs chose it
    for t in range(T):
        common = {int(e): float(x) for e, x in zip(ids_0[t], w_0[t])}
        for e, x in zip(ids_b[t].tolist(), w_b[t].tolist()):
            if e in common:
                assert x == common[e], (t, e)
    sig = torch.sigmoid(logits.double()).gather(1, ids_b.long())
    _check_weights(w_b, sig)


@pytest.mark.parametrize("kw", [dict(scoring="softmax"), dict(scoring="softmax", renormalize=True), dict(scoring="sigmoid"),
                                dict(scoring="sigmoid", num_expert_group=8, topk_group=4, group_score="top2_sum"),
                                dict(scoring="softmax", num_expert_group=8, topk_group=3, group_score="max")])
def test_nan_logits_are_chosen_last(kw):
    T, E, k = 1024, 64, 6
    gen = torch.Generator().manual_seed(17)
    logits = _distinct_logits(T, E, gen)
    frac = torch.rand((T, 1), generator=gen)               # rows from no NaN to nearly all NaN
    logits[torch.rand((T, E), generator=gen) < frac] = torch.nan
    logits[0] = torch.nan
    logits[1, 1:] = torch.nan
    logits = logits.half()
    ids, w = _run(logits.to(DEV), k, **kw)
    ref_ids, ref_w, ok = reference(logits, k, **kw)   # top2_sum: sums of different groups may fall within GAP of each other
    assert ok.float().mean() > 0.95
    assert torch.equal(ids[ok], ref_ids[ok])
    picked_nan = torch.isnan(logits.gather(1, ids.long()))
    if "num_expert_group" not in kw:
        finite = (~torch.isnan(logits)).sum(dim=1)
        assert torch.equal(picked_nan.sum(dim=1), (k - finite).clamp(min=0)), "a NaN is chosen only when no finite logit is left"
    # the finite choices come first
    assert not (picked_nan[:, :-1] & ~picked_nan[:, 1:]).any()
    fin = ok & ~picked_nan.any(dim=1)
    _check_weights(w[fin], ref_w[fin])
    assert ids[0].tolist() == list(range(k))


# ---- determinism and the graph --------------------------------------------------------------------------------------------------
def test_repeated_calls_bit_identical_one_launch_each():
    from bitblas_b200 import _lib
    from bitblas_b200 import moe_topk
    for name in ("qwen3-30b-a3b", "deepseek-v3"):
        logits_d, k, kw, _ = _preset(name, 4096, "bfloat16", seed=3)
        lib = _lib.load()
        first = _run(logits_d, k, **kw)
        torch.cuda.synchronize()
        n0 = lib.bb_launch_count()
        for _ in range(5):
            again = _run(logits_d, k, **kw)
            assert torch.equal(again[0], first[0]) and torch.equal(again[1].view(torch.int32), first[1].view(torch.int32))
        torch.cuda.synchronize()
        assert lib.bb_launch_count() - n0 == 5
        n0 = lib.bb_launch_count()
        ids0, w0 = moe_topk(logits_d[:0], k, **kw)   # no tokens: no launch, still one step
        assert lib.bb_launch_count() == n0 + 1 and ids0.shape == w0.shape == (0, k)


@pytest.mark.parametrize("E,k", [(128, 8), (8, 2)])   # Qwen3-30B-A3B and Mixtral-8x7B routing, small dims
def test_graph_topk_then_block_matches_eager(E, k):
    import bitblas_b200 as bitblas
    from bitblas_b200 import moe_topk
    m, dq = _make_block(E=E, seed=E)
    T, H = 48, 512
    logits_d = torch.zeros((T, E), dtype=torch.float16, device=DEV)
    x_d = torch.zeros((T, H), dtype=torch.float16, device=DEV)
    out_d = torch.zeros((T, H), dtype=torch.float16, device=DEV)
    held = {}

    def layer():
        held["ids"], held["w"] = moe_topk(logits_d, k, renormalize=True)
        m(x_d, held["ids"], held["w"], output=out_d)

    step = bitblas.CapturedStep(layer)
    for trial in range(3):
        gen = torch.Generator().manual_seed(1000 * E + trial)
        logits = _distinct_logits(T, E, gen).half()
        x = (torch.rand((T, H), generator=gen) - 0.5).half()
        logits_d.copy_(logits)
        x_d.copy_(x)
        step()
        ids_e, w_e = moe_topk(logits.to(DEV), k, renormalize=True)
        out_e = m(x.to(DEV), ids_e, w_e)
        torch.cuda.synchronize()
        assert torch.equal(held["ids"], ids_e) and torch.equal(held["w"], w_e), trial
        assert torch.equal(out_d, out_e), trial
        ref_ids, ref_w, ok = reference(logits, k, renormalize=True)
        assert ok.all() and torch.equal(ids_e.cpu(), ref_ids)
        _check_weights(w_e.cpu(), ref_w)
        assert _normwise(out_d.cpu(), _oracle(dq, x, ref_ids, ref_w)) <= 1e-2, trial
