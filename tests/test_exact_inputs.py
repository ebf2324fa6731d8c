"""CPU: the exact-input checker of test_gpu_exact_shapes.py (proof, reference, comparison) and the work decompositions it relies
on -- the slab decode GEMV's stream-K fix-up protocol at every SM count of 1..132, its coverage at the tested shapes, and the
streaming GEMV's K split."""
import itertools

import pytest
import torch

import exact_inputs as X

SLAB_SHAPES = [(8192, 8192), (28672, 8192), (8192, 28672), (12288, 12288),      # bench.py
               (1024, 8192), (1024, 3584), (16, 4096), (48, 2304), (2064, 3840), (4112, 6144)]   # shards, padding, ragged, N % 32 = 16
SLAB_PROPERTIES = {"block_over_3_ranges", "range_inside_block", "owner_stops_mid_block", "one_unit_per_cta", "odd_NRB",
                   "padding_only_range", "ragged_last_unit_1_slices", "ragged_last_unit_2_slices", "ragged_last_unit_3_slices",
                   "N%32=16", "group_closes_2_blocks"}
SMALL_SM_PROPERTIES = {"group_closes_2_blocks"}   # at these shapes only below 120 SMs: tested at capped SM counts
# the SM counts test_gpu_sm_counts.py runs SLAB_SHAPES at, besides the device's own (1: R = 2 ranges; 114: H100 PCIe)
SLAB_CAPS = (1, 2, 3, 5, 33, 114)


def slab_cap_coverage(device_sms):
    """{property: the caps of SLAB_CAPS + (device_sms,) at which one of SLAB_SHAPES reaches it}"""
    hit = {}
    for cap in sorted(set(SLAB_CAPS) | {device_sms}):
        for p in set().union(*(X.slab_coverage(N, K, cap) for N, K in SLAB_SHAPES)):
            hit.setdefault(p, []).append(cap)
    return hit


# ---- the checker ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["none", "scale", "original", "rescale", "quantized"])
@pytest.mark.parametrize("A_dtype", ["float16", "bfloat16"])
def test_reference_is_exact_in_int64(mode, A_dtype):
    """the float64 reference equals an int64 recomputation on scaled integers, and the precondition holds"""
    for K, g in [(1024, 128), (3840, 384), (2048, -1)]:
        W = "int4" if mode in ("none", "scale") and g == 128 else "uint4"
        case = X.make_exact_case(3, 48, K, A_dtype=A_dtype, W_dtype=W, group_size=g, mode=mode, bias=True, seed=K + len(mode))
        X.prove_exact(case)
        Vi, e = X.int64_value(case)
        assert torch.equal(Vi.double() * 2.0 ** -e, X.exact_value(case))


@pytest.mark.parametrize("W_dtype", ["fp4_e2m1", "e4m3_float8", "e5m2_float8", "uint2", "int2"])
def test_reference_is_exact_other_formats(W_dtype):
    mode = "scale" if W_dtype != "uint2" else "quantized"
    case = X.make_exact_case(2, 32, 2048, W_dtype=W_dtype, group_size=128, mode=mode, seed=5)
    X.prove_exact(case, ("sum",))
    Vi, e = X.int64_value(case)
    assert torch.equal(Vi.double() * 2.0 ** -e, X.exact_value(case))


@pytest.mark.parametrize("K,group", [(28672, 28672), (28672, 128), (8192, 256), (3840, 384), (3840, 640), (12288, 12288)])
def test_activations_have_nonzero_block_group_and_row_sums(K, group):
    """every 32-block, every zero-point group and every row has a nonzero activation sum; the prefix stays small"""
    A = X.dyadic_activations(64, K, torch.Generator().manual_seed(K + group), 0.25, group)
    assert set(A.unique().tolist()) <= {-1.0, -0.5, 0.0, 0.5, 1.0}
    blk = A.reshape(64, -1, 32).sum(-1)
    assert bool((blk != 0).all()) and float(blk.abs().max()) <= 1.0
    assert float(blk.cumsum(1).abs().max()) <= 2.0
    assert bool((A.reshape(64, -1, group).sum(-1) != 0).all())
    assert bool((A.sum(1) != 0).all())


def test_exact_cases_have_nonzero_group_sums():
    """make_exact_case draws its activations with the case's group size, so prove_exact's nonzero-sum check holds for every
    zero-point mode and group size the GPU tests use"""
    for mode, g, K in itertools.product(["original", "rescale", "quantized", "scale"], [128, 256, 384, -1], [3840, 8192]):
        if K % (K if g == -1 else g):
            continue
        case = X.make_exact_case(8, 32, K, group_size=g, mode=mode, seed=K + (g if g > 0 else 0))
        X.prove_exact(case)


def test_precondition_rejects_zero_group_sums():
    case = X.make_exact_case(1, 32, 1024, mode="quantized", group_size=128, seed=4)
    A = case["A"].clone()
    A[0, :128] = 0.0
    with pytest.raises(AssertionError, match="group sums to zero"):
        X.prove_exact(dict(case, A=A))


def test_precondition_rejects_inexact_inputs():
    """activations of one sign at full density: the magic chains overflow the 2^22 budget and the proof must say so"""
    case = X.make_exact_case(1, 32, 28672, mode="original", group_size=-1, seed=1)
    case["A"] = torch.ones_like(case["A"])
    with pytest.raises(AssertionError, match="grid units"):
        X.prove_exact(case)
    # and a value off the dyadic grid of the activations breaks the fp32 exactness of V
    case = X.make_exact_case(1, 32, 1024, mode="scale", group_size=128, seed=2)
    case["A"] = case["A"].clone()
    case["A"][0, 0] = 1.0 + 2.0 ** -10
    case["A"][0, 1] = 3.0 * 2.0 ** 12
    with pytest.raises(AssertionError):
        X.prove_exact(case)


@pytest.mark.parametrize("out", ["float16", "bfloat16", "float32"])
def test_one_ulp_fails_the_comparison(out):
    case = X.make_exact_case(2, 64, 1024, mode="original", group_size=128, out_dtype=out, bias=True, seed=9)
    ref = X.exact_reference(case)
    X.compare_exact(ref.clone(), ref, "identical")
    for i, j in [(0, 0), (1, 63), (1, 17)]:
        bad = ref.clone()
        bad[i, j] = torch.nextafter(bad[i, j].float(), torch.tensor(float("inf"))).to(bad.dtype) if out == "float32" else \
            (bad[i, j].view(torch.int16) + 1).view(bad.dtype)
        with pytest.raises(AssertionError, match="1/128 elements differ"):
            X.compare_exact(bad, ref, "one ulp")


# ---- slab stream-K ----------------------------------------------------------------------------------------------------------------
PROTOCOL_SIZES = [(16, 256), (16, 4096), (48, 2304), (96, 11264), (272, 1024), (1024, 3584), (1024, 8192), (2064, 3840),
                  (4112, 6144), (8192, 8192), (8192, 28672), (28672, 8192), (12288, 12288)]


@pytest.mark.parametrize("N,K", PROTOCOL_SIZES, ids=lambda v: str(v))
def test_slab_fixup_protocol_every_sm_count(N, K):
    """at every SM count 1..132 (114: H100 PCIe): every parked partial collected exactly once by its block's owner, every awaited
    slot parked -- the protocol's only hang risk, checked without a GPU"""
    parked = 0
    for sms in range(1, 133):
        _, _, _, R = X.slab_geometry(N, K, sms)
        parked += X.check_fixup_protocol(N, K, R)
    assert parked > 0 or K <= X.UNIT_K   # one unit per row block: nothing to park


def test_slab_fixup_protocol_small_grid():
    """every N (multiple of 16) and K (multiple of 256) on a grid of small sizes, at every range count up to T"""
    for N, K in itertools.product(range(16, 272, 48), range(256, 5376, 768)):
        UPR, NRB, T, _ = X.slab_geometry(N, K, 132)
        for R in range(1, T + 1):
            X.check_fixup_protocol(N, K, R)


def test_slab_shapes_cover_every_stream_k_property():
    """the exact-shape GPU tests' slab shapes reach each property on a 132-SM H100 (the GPU test re-checks on its own device)"""
    hit = set()
    for N, K in SLAB_SHAPES:
        hit |= X.slab_coverage(N, K, 132)
    assert SLAB_PROPERTIES - SMALL_SM_PROPERTIES <= hit, SLAB_PROPERTIES - SMALL_SM_PROPERTIES - hit
    assert not SMALL_SM_PROPERTIES & hit, "reached on a full H100: not a small-SM-count property"


def test_slab_caps_cover_every_property_three_times():
    """the capped SM counts of test_gpu_sm_counts.py reach every property at three or more caps, one of them below 8"""
    hit = slab_cap_coverage(132)
    for p in sorted(SLAB_PROPERTIES):
        caps = hit.get(p, [])
        assert len(caps) >= 3 and min(caps) < 8, (p, caps)


def test_group_closes_2_blocks_property():
    """one group of one range closes two whole row blocks only when the range is long enough: two ranges over 896 row blocks
    do, 264 ranges do not, and a shape with one block per group never does"""
    N, K = 28672, 8192
    assert "group_closes_2_blocks" in X.slab_coverage(N, K, 1)           # R = 2: every group closes hundreds of blocks
    assert "group_closes_2_blocks" not in X.slab_coverage(N, K, 132)
    assert "group_closes_2_blocks" not in X.slab_coverage(48, 2304, 1)   # NRB = 2: one block per group


# ---- gemv_mma / gemv_i8 K split ---------------------------------------------------------------------------------------------------
def test_gemv_k_split_starts_mid_group():
    """K = 3840 (30 steps): for every K split ks = 2..8 one of g = 256, 384, 640 makes some warp start inside a group"""
    for ks in range(2, 9):
        assert any(X.mid_group_starts(3840, g, ks) for g in (256, 384, 640)), ks


def test_gemv_k_split_unequal_ranges():
    """29 and 31 steps: unequal warp ranges at every ks = 2..8 except the divisors"""
    for steps in (29, 31):
        for ks in range(2, 9):
            sizes = [e - b for b, e in (X.split_range(steps, ks, w) for w in range(ks))]
            assert sum(sizes) == steps and max(sizes) - min(sizes) == (0 if steps % ks == 0 else 1)
            assert steps % ks == 0 or len(set(sizes)) == 2
