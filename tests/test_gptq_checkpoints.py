"""CPU: the synthetic GPTQ checkpoints of test_gpu_gptq_loading.py (exact_inputs.gptq_checkpoint) hold the exact cases they are built
from -- the oracle's qzeros unpacking (v1 wrap included) and the act-order loader's unpacking recover the fields, zero points and
scales, and perm_from_g_idx recovers the column order -- and every layer case the GPU file runs meets prove_exact.  Also the GPTQ
repack's argument checks that need no device."""
import pytest
import torch

import bitblas_b200 as bitblas
import bitblas_oracle as O
import exact_inputs as X
from bitblas_b200.act_order import _unpack, perm_from_g_idx
from test_gpu_gptq_loading import (DTYPES, G, GROUPED_CELLS, LINEAR_CELLS, MODES, N, K, TORCH, _cell_id, grouped_cases,
                                   linear_case)


def _check_recovers(case, ck, v2, act_order, scale_dtype):
    bits = case["bit"]
    g = case["K"] // case["qz"].shape[0]
    assert ck.qweight.dtype == ck.qzeros.dtype == torch.int32
    assert ck.qweight.shape == (case["K"] * bits // 32, case["N"]) and ck.qzeros.shape == (case["K"] // g, case["N"] * bits // 32)
    # zero points through the oracle (the reference's unpack_qzeros, with its `& mask` wrap for v1) and the raw stored values
    assert torch.equal(O.unpack_qzeros(ck.qzeros, bits, v2=v2).long(), case["qz"].long())
    stored = _unpack(ck.qzeros, bits, 1)
    assert torch.equal(stored, case["qz"].long() if v2 else (case["qz"].long() - 1) % 2 ** bits)
    # the weight: unpacked along K, in checkpoint column order; the sorted column j is checkpoint column perm[j]
    w = _unpack(ck.qweight, bits, 0)
    perm = perm_from_g_idx(ck.g_idx, case["K"], g)
    if act_order:
        assert torch.equal(perm.long(), ck.perm)
        assert not torch.equal(ck.perm, torch.arange(case["K"]))
        w = w[ck.perm]
        assert torch.equal(ck.A[:, ck.perm], case["A"])
    else:
        assert perm is None and ck.perm is None and ck.A is case["A"]
    assert torch.equal(w.T, case["fields"].long())
    assert ck.scales.dtype == scale_dtype and torch.equal(ck.scales.double().T, case["scale"].double())
    if case["bias"] is None:
        assert ck.bias is None
    else:
        assert ck.bias.dtype == scale_dtype and torch.equal(ck.bias.data.double(), case["bias"].double())


@pytest.mark.parametrize("c", LINEAR_CELLS, ids=_cell_id)
def test_linear_checkpoints(c):
    case, ck = linear_case(c)
    _check_recovers(case, ck, c["v2"], c["act"], TORCH[c["ckpt"]])
    # zero point 0 is present: v1 stores it as 2^bits - 1 and only the unpacking's wrap brings it back
    assert bool((case["qz"] == 0).any()) and bool((case["qz"] == 2 ** case["bit"] - 1).any())
    for mode in MODES:
        mc = X.zeros_mode_case(case, mode)
        assert torch.equal(X.dequantized(mc), X.dequantized(case)), mode
        X.prove_exact(mc)


@pytest.mark.parametrize("A_dtype,mode,v2", GROUPED_CELLS)
def test_grouped_checkpoints(A_dtype, mode, v2):
    from test_gpu_gptq_loading import ACT_EXPERTS
    for e, (case, ck) in enumerate(grouped_cases(A_dtype, v2)):
        _check_recovers(case, ck, v2, e in ACT_EXPERTS, torch.float16)
        X.prove_exact(X.zeros_mode_case(case, mode))


def test_cells_cover_every_toggle_per_dtype_pair():
    """act-order, bias and propagate_b each on and off for every (A_dtype, checkpoint dtype) pair; act-order with v1 and v2; one
    group (g = -1) in both bit widths"""
    for a in DTYPES:
        for s in DTYPES:
            cells = [c for c in LINEAR_CELLS if c["A"] == a and c["ckpt"] == s]
            assert len(cells) == 12
            for key in ("act", "bias", "tiled"):
                assert {c[key] for c in cells} == {False, True}, (a, s, key)
            assert {c["v2"] for c in cells if c["act"]} == {False, True}
    assert {c["bits"] for c in LINEAR_CELLS if c["g"] == -1} == {4, 2}
    assert not any(c["act"] for c in LINEAR_CELLS if c["g"] == -1)


def test_gptq_checkpoint_shares_g_idx_per_seed():
    """gate and up projections of an expert are built with one seed and must get one column order"""
    a = X.make_exact_case(1, 64, 512, W_dtype="uint4", group_size=128, mode="quantized", seed=1)
    b = X.make_exact_case(1, 64, 512, W_dtype="uint4", group_size=128, mode="quantized", seed=2)
    ca, cb = (X.gptq_checkpoint(x, v2=False, act_order=True, scale_dtype=torch.float16, seed=9) for x in (a, b))
    assert torch.equal(ca.g_idx, cb.g_idx)


# ---- repack argument checks ---------------------------------------------------------------------------------------------------------
def test_repack_without_module_bias_raises_value_error():
    case, ck = linear_case(LINEAR_CELLS[0])
    ck.bias = None
    layer = bitblas.Linear(K, N, bias=True, A_dtype="float16", W_dtype="uint4", group_size=G, with_scaling=True, with_zeros=True,
                           zeros_mode="quantized")
    with pytest.raises(ValueError, match="no bias"):
        layer.repack_from_gptq(ck)
    del ck.bias
    with pytest.raises(ValueError, match="no bias"):
        layer.repack_from_gptq_v2(ck)


def test_repack_int8_activations_raises_value_error():
    case, ck = linear_case(LINEAR_CELLS[0])
    layer = bitblas.Linear(K, N, A_dtype="int8", W_dtype="int4", accum_dtype="int32", out_dtype="int32")
    with pytest.raises(ValueError, match="float16 or bfloat16 activations"):
        layer.repack_from_gptq(ck)
