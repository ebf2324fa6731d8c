"""CPU: the restatement of the block-scaled FP8 GEMMs' fp32 order (fp8_restate) has power on the cases the GPU tests run.

  * every case list's inputs meet the precondition that makes the tensor core's block sum exact, and the split cases reach the
    factor they name under gemm_ts's rule (test_fp8_api.fp8_splits);
  * on each list, the header's order and each plausible wrong order -- an fma promotion, (P sa) sw, blocks descending, the
    splits reduced last to first or as a balanced tree, the bias added before the rounding -- give different outputs in a
    large share of the elements the GPU tests compare, so a kernel doing any of them fails there;
  * the restatement run on the device equals the one run on the CPU (skipped without a device).
"""
import pytest
import torch

import fp8_restate as R
from test_fp8_api import fp8_splits

SMS = 132   # the H100 SXM's SM count: the GPU tests' split factors at cap 0
MIN_SHARE = 0.05   # the least share of compared output elements each wrong order must change


class Tally:
    """per wrong order: output elements compared and elements it changes"""

    def __init__(self):
        self.seen, self.diff = {}, {}

    def add(self, variant, ref, wrong):
        self.seen[variant] = self.seen.get(variant, 0) + ref.numel()
        self.diff[variant] = self.diff.get(variant, 0) + int((ref != wrong).sum())

    def check(self, expected):
        assert set(self.seen) == set(expected)
        for v in expected:
            share = self.diff[v] / self.seen[v]
            assert share >= MIN_SHARE, f"{v}: {self.diff[v]} of {self.seen[v]} elements ({share:.2%})"
        return {v: self.diff[v] / self.seen[v] for v in expected}


def _fp8_case_outputs(qa, qw, sa, sw, splits, tally, bias_seed):
    """every output type with and without a bias, as the GPU test runs the case; each wrong order added to the tally"""
    R.prove_exact(qa, qw)
    P = R.block_sums(qa, qw)
    swn = R.scale_rows(sw, qw.shape[0])
    S = R.promote(P, sa, swn, splits)
    wrong = {v: R.promote(P, sa, swn, splits, v) for v in ("fma", "p_sa_sw", "descending")}
    if splits > 2:   # two splits reduce the same way in every order
        wrong.update({v: R.promote(P, sa, swn, splits, v) for v in ("reversed_splits", "pairwise_splits")})
    for out in R.OUT:
        for with_bias in (False, True):
            b = R.bias_for(qw.shape[0], out, bias_seed) if with_bias else None
            ref = R.round_out(S, out, b)
            for v, Sv in wrong.items():
                tally.add(v, ref, R.round_out(Sv, out, b))
            if with_bias and out != "float32":
                tally.add("bias_first", ref, R.round_out(S, out, b, bias_first=True))


def test_split_cases_reach_their_factor():
    assert sorted({c[0] for c in R.SPLIT_CASES}) == list(range(2, 9))
    for f, m, N, K, cap in R.SPLIT_CASES:
        assert fp8_splits(N, K, m, cap or SMS) == f, (f, m, N, K, cap)
        if cap:
            assert fp8_splits(N, K, m, SMS) != f    # the cap is what forces this factor


def test_fp8_cases_tell_the_orders_apart():
    tally = Tally()
    for m, N, K in R.FP8_CASES:
        qa, qw, sa, sw = R.fp8_case(m, N, K)
        _fp8_case_outputs(qa, qw, sa, sw, fp8_splits(N, K, m, SMS), tally, bias_seed=m + N)
    tally.check(("fma", "p_sa_sw", "descending", "reversed_splits", "pairwise_splits", "bias_first"))


def test_split_cases_tell_the_orders_apart():
    tally = Tally()
    for f, m, N, K, cap in R.SPLIT_CASES:
        qa, qw, sa, sw = R.split_case(f, m, N, K, cap)
        _fp8_case_outputs(qa, qw, sa, sw, f, tally, bias_seed=f)
        # and the same call run unsplit (no workspace) differs from the split one
        P, swn = R.block_sums(qa, qw), R.scale_rows(sw, N)
        tally.add("unsplit", R.promote(P, sa, swn, f), R.promote(P, sa, swn, 1))
    tally.check(("fma", "p_sa_sw", "descending", "reversed_splits", "pairwise_splits", "bias_first", "unsplit"))


@pytest.mark.parametrize("swiglu", [False, True], ids=["plain", "swiglu"])
def test_grouped_cases_tell_the_orders_apart(swiglu):
    tally = Tally()
    for counts, N, K, _, _ in R.GROUPED_CASES.values():
        off = R.offsets_of(counts)
        qa, sa, experts = R.grouped_case(counts, N, K, swiglu)
        for e, halves in enumerate(experts):
            r0, r1 = off[e], off[e + 1]
            if r1 == r0:
                continue
            for qw, _ in halves:
                R.prove_exact(qa[r0:r1], qw)
            Ps = [R.block_sums(qa[r0:r1], qw) for qw, _ in halves]
            swns = [R.scale_rows(sw, qw.shape[0]) for qw, sw in halves]
            for out in R.OUT:
                def y(variant):
                    Ss = [R.round_out(R.promote(P, sa[r0:r1], swn, 1, variant), out) for P, swn in zip(Ps, swns)]
                    return R.silu_mul(*Ss, out) if swiglu else Ss[0]
                ref = y(None)
                for v in ("fma", "p_sa_sw", "descending"):
                    tally.add(v, ref, y(v))
    tally.check(("fma", "p_sa_sw", "descending"))


@pytest.mark.gpu
def test_reference_device_equals_cpu():
    """the restatement on the device (as the GPU tests run it) and on the CPU, on a split case with every output type and a
    bias: identical bits"""
    m, N, K, splits = 5, 576, 3072, 3
    qa, qw, sa, sw = R.inexact_case(m, N, K, seed=17)
    S_cpu = R.restate(qa, qw, sa, sw, splits)
    S_dev = R.restate(qa.cuda(), qw.cuda(), sa.cuda(), sw.cuda(), splits)
    assert torch.equal(S_dev.cpu(), S_cpu)
    for out in R.OUT:
        b = R.bias_for(N, out, 3)
        assert torch.equal(R.round_out(S_dev, out, b.cuda()).cpu(), R.round_out(S_cpu, out, b))
