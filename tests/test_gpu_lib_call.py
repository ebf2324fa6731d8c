"""``matmul.lib.call(A, B, [LUT], [Scale], [Zeros], [Bias], C, [m], stream)``, the reference's positional FFI surface
(builder/wrapper/base.py:5-19): the same launch as ``Matmul.forward`` on the same buffers, bit for bit."""
from __future__ import annotations

import ctypes

import pytest
import torch

import helpers as H

pytestmark = pytest.mark.gpu

CASES = {
    "uint4": dict(N=256, K=1024, W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized",
                  with_bias=True),
    "nf4": dict(N=256, K=2048, W_dtype="nf4", group_size=128, with_scaling=True),
}


def _buffers(name, m):
    case = H.make_case(m, **CASES[name], seed=m)
    op = H.product_operator(case, M=[1, 16])
    A = case["A"].cuda()
    params = [H.product_weight(op, case)] + [case[k].cuda() for k in ("scale", "zeros", "bias") if case[k] is not None]
    return op, A, params


def _lib_call(op, A, params, m, lut=()):
    out = torch.empty((m, op.N), dtype=torch.float16, device="cuda")
    ptrs = [ctypes.c_void_p(t.data_ptr()) for t in (A, params[0], *lut, *params[1:], out)]
    op.lib.call(*ptrs, m, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return out


@pytest.mark.parametrize("m", [1, 16])
def test_lib_call_uint4_matches_forward(m):
    op, A, params = _buffers("uint4", m)
    W, scale, zeros, bias = params
    ref = op.forward(A, W, scale=scale, zeros=zeros, bias=bias)
    assert torch.equal(_lib_call(op, A, params, m), ref)
    with pytest.raises(TypeError, match="expected 6 buffers"):      # the bias is missing
        _lib_call(op, A, params[:-1], m)


@pytest.mark.parametrize("m", [1, 16])
def test_lib_call_nf4_matches_forward_with_and_without_table(m):
    op, A, params = _buffers("nf4", m)
    ref = op.forward(A, params[0], scale=params[1])
    assert torch.equal(_lib_call(op, A, params, m, lut=(op.lut,)), ref)
    assert torch.equal(_lib_call(op, A, params, m), ref)             # bitblas.Linear-style callers never pass the table
    with pytest.raises(TypeError, match="expected 5 buffers"):
        _lib_call(op, A, params, m, lut=(op.lut, op.lut))
