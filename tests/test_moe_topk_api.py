"""CPU: the top-k gating call's C ABI (bb_moe_topk) and moe_topk's argument checks (no compute calls)."""
import ctypes

import pytest
import torch

import bitblas_b200 as bitblas
from bitblas_b200 import _lib
from bitblas_b200.moe import moe_topk


def test_export_and_argtypes():
    lib = _lib.load()
    assert "bb_moe_topk" in _lib.EXPORTS and hasattr(lib, "bb_moe_topk")
    assert lib.bb_moe_topk.restype is ctypes.c_int and len(lib.bb_moe_topk.argtypes) == 15
    assert lib.bb_moe_topk.argtypes[11] is ctypes.c_float
    assert bitblas.moe_topk is moe_topk and lib.bb_version() == 100


# fake non-null, aligned device addresses: every call below is refused (or returns) before anything is dereferenced
def _topk(T=4, E=64, k=6, dtype=_lib.BB_F16, scoring=0, bias=None, n=0, topk_group=0, group_score=0, scale=1.0, logits=16,
          ids=16, w=16):
    return _lib.load().bb_moe_topk(logits, dtype, T, E, k, scoring, bias, n, topk_group, group_score, 1, scale, ids, w, 0)


@pytest.mark.parametrize("what,kw,msg", [
    ("int8 logits", dict(dtype=_lib.BB_I8), "float16, bfloat16 or float32"),
    ("E = 0", dict(E=0, k=1), "num_experts"),
    ("E = 257", dict(E=257), "num_experts"),
    ("top_k = 0", dict(k=0), "top_k"),
    ("top_k > 32", dict(E=256, k=33), "min(num_experts, 32) = 32"),
    ("top_k > E", dict(E=4, k=5), "min(num_experts, 32) = 4"),
    ("T < 0", dict(T=-1), "num_tokens"),
    ("T * k >= 2^31", dict(T=1 << 28, k=8), "2^31"),
    ("scoring", dict(scoring=2), "scoring"),
    ("n > 32", dict(E=128, n=64, topk_group=4), "<= 32"),
    ("n does not divide E", dict(E=60, n=8, topk_group=3), "divide"),
    ("topk_group = 0", dict(n=8, topk_group=0), "topk_group"),
    ("topk_group > n", dict(n=8, topk_group=9), "topk_group"),
    ("group_score", dict(n=8, topk_group=3, group_score=2), "group_score"),
    ("top2_sum of one expert", dict(E=16, k=2, n=16, topk_group=4, group_score=1), "top2_sum"),
    ("k above the kept experts", dict(E=64, k=9, n=8, topk_group=1), "kept groups"),
    ("scale inf", dict(scale=float("inf")), "routed_scaling_factor"),
    ("scale nan", dict(scale=float("nan")), "routed_scaling_factor"),
])
def test_rejects(what, kw, msg):
    assert _topk(**kw) == 1, what
    assert msg in _lib.last_error(), (what, _lib.last_error())
    if "T" not in kw:
        n0 = _lib.load().bb_launch_count()
        assert _topk(**dict(kw, T=0)) == 1, what   # the checks do not depend on the tokens
        assert _lib.load().bb_launch_count() == n0, "a rejected call is not counted"


def test_group_arguments_ignored_without_a_group_limit():
    n0 = _lib.load().bb_launch_count()
    for n in (0, 1, -3):
        assert _topk(T=0, n=n, topk_group=-1, group_score=7) == 0, n
    assert _topk(T=0, E=256, k=8, n=8, topk_group=4, group_score=1, scale=2.5) == 0
    assert _topk(T=0, E=160, k=6, n=8, topk_group=3, group_score=0, scale=16.0) == 0
    assert _topk(T=0, E=1, k=1, dtype=_lib.BB_F32, scoring=1) == 0
    assert _lib.load().bb_launch_count() == n0 + 6   # one step per accepted call


def test_zero_tokens_returns_without_touching_the_device_and_is_counted():
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    assert _topk(T=0, logits=None, ids=None, w=None) == 0   # null and unaligned pointers are never looked at
    assert _topk(T=0, logits=17, ids=18, w=18, bias=18) == 0
    assert lib.bb_launch_count() == n0 + 2


def test_rejects_null_and_unaligned():
    n0 = _lib.load().bb_launch_count()
    for kw, code, msg in [(dict(logits=None), 1, "logits must be non-null"), (dict(ids=None), 1, "topk_ids must be non-null"),
                          (dict(w=None), 1, "topk_weights must be non-null"),
                          (dict(logits=17), 5, "logits must be aligned to their element size (2 bytes)"),
                          (dict(logits=18, dtype=_lib.BB_F32), 5, "logits must be aligned to their element size (4 bytes)"),
                          (dict(ids=18), 5, "topk_ids must be 4-byte aligned"), (dict(w=18), 5, "topk_weights must be 4-byte aligned"),
                          (dict(bias=18), 5, "correction_bias must be 4-byte aligned")]:
        assert _topk(**kw) == code, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())
    assert _lib.load().bb_launch_count() == n0


# ---- moe_topk ------------------------------------------------------------------------------------------------------------------
def test_python_rejects_cpu_tensor():
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        moe_topk(torch.zeros(4, 8), 2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        moe_topk(torch.zeros(4, 8), 2, correction_bias=torch.zeros(8))


@pytest.mark.parametrize("logits,kw,err,msg", [
    (torch.zeros(4, 8, dtype=torch.float64), {}, TypeError, "float16, bfloat16 or float32"),
    (torch.zeros(4, 8, dtype=torch.int32), {}, TypeError, "float16, bfloat16 or float32"),
    ([[0.0] * 8] * 4, {}, TypeError, "torch.Tensor"),
    (torch.zeros(32), {}, TypeError, "2-D"),
    (torch.zeros(2, 4, 8), {}, TypeError, "2-D"),
    (torch.zeros(4, 8), dict(correction_bias=torch.zeros(8, dtype=torch.float16)), TypeError, "correction_bias"),
    (torch.zeros(4, 8), dict(correction_bias=torch.zeros(7)), TypeError, r"\[E=8\]"),
    (torch.zeros(4, 8), dict(correction_bias=torch.zeros(1, 8)), TypeError, r"\[E=8\]"),
    (torch.zeros(4, 8), dict(scoring="relu"), ValueError, "scoring"),
    (torch.zeros(4, 8), dict(group_score="sum"), ValueError, "group_score"),
    (torch.zeros(4, 8), dict(num_expert_group=4), ValueError, "topk_group"),
])
def test_python_rejects(logits, kw, err, msg):
    with pytest.raises(err, match=msg):
        moe_topk(logits, 2, **kw)


def test_python_rejects_mismatched_devices():
    with pytest.raises(ValueError, match="same device"):
        moe_topk(torch.zeros(4, 8), 2, correction_bias=torch.zeros(8, device="meta"))
