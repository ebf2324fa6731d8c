"""The fp32 order of the block-scaled FP8 GEMMs (bb_matmul_fp8, bb_matmul_grouped_fp8[_swiglu]; include/bitblas_b200.h),
restated in torch, and inputs on which every bit of the result depends on that order.

    P[r, n, b] = sum_{k in block b} q_a[r, k] * q_w[n, k]           the tensor core's block sum: exact on inexact_case's inputs
    c = fl(a_scale[r, b] * w_scale[n / 128, b]),  t = fl(P * c),  S_j = fl(S_j + t)     split j's blocks, ascending, from 0
    S = ((0 + S_0) + S_1) + ... + S_{splits-1},   C = round_out(S)  (+ bias, added in out_dtype after the rounding)

How the tensor core sums a block's 128 products is not specified, so a test can pin the later steps only when P is exact in
every order.  inexact_case makes it so: activations are integers in [-4, 4] and weights integers in [-8, 8], all exact in e4m3,
so every product and every partial sum of a block is an integer of magnitude at most sum_k |a_k w_k| <= 128 * 32 = 2^12.  The
tensor core keeps 13 binades below the largest value of each k32 step (tools/fp8_accum_probe.py, DESIGN.md §3.2.6), i.e.
every unit down to 2^-1 here, and fp32 holds such integers exactly.  The scales are what a checkpoint and the activation
quantizer give -- a_scale = fl(amax / 448) for an amax of the activation type, 1e-10 / 448 for an all-zero block, w_scale
anywhere in 1e-4 .. 1e-2 -- so every product, sum and rounding after P is inexact, and an fma, another association of the
scales, another block or split order, or the bias added before the rounding changes the result (test_fp8_restate shows how
often, for every case list below).

Every step below is one torch elementwise op on float32 tensors -- one kernel, never contracted into an fma -- on the CPU or on
the device; the block sums are float32 matmuls of small integers, exact in any order.
"""
import torch

E4M3 = torch.float8_e4m3fn
OUT = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32}
P_MAX = 2.0 ** 12          # bound on sum_k |a_k w_k| over a block: the tensor core's block sum is exact below 2^13
ZERO_BLOCK_SCALE = torch.tensor(1e-10, dtype=torch.float32) / torch.tensor(448.0)


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def activation_scales(rows, KB, gen, zero_share=0.05):
    """a_scale [rows, KB] = fl(amax / 448) for amax a bfloat16 magnitude in [2^-4, 2^6]; a share of blocks all zero (a_scale =
    1e-10 / 448, bb_quantize_act_fp8's value for them).  Returns (a_scale, the all-zero mask)."""
    amax = torch.exp2(torch.rand(rows, KB, generator=gen) * 10 - 4).to(torch.bfloat16).float()
    sa = amax / torch.full_like(amax, 448.0)
    zero = torch.rand(rows, KB, generator=gen) < zero_share
    return torch.where(zero, ZERO_BLOCK_SCALE, sa), zero


def weight_scales(rows, KB, gen):
    """w_scale [rows, KB] fp32 spread log-uniformly over 1e-4 .. 1e-2, the range checkpoints' weight_scale_inv takes"""
    return torch.pow(10.0, torch.rand(rows, KB, generator=gen, dtype=torch.float64) * 2 - 4).float()


def inexact_activations(m, K, seed):
    """(qa [m, K], sa [m, K/128]) on the CPU: integers in [-4, 4] as float32 with bb_quantize_act_fp8-like scales; a block
    whose scale is the all-zero one holds zeros"""
    g = torch.Generator().manual_seed(seed)
    qa = torch.randint(-4, 5, (m, K), generator=g).float()
    sa, zero = activation_scales(m, K // 128, g)
    return qa.masked_fill(zero.repeat_interleave(128, 1), 0.0), sa


def inexact_weights(N, K, seed):
    """(qw [N, K], sw [ceil(N/128), K/128]) on the CPU: integers in [-8, 8] as float32 with checkpoint-like block scales"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-8, 9, (N, K), generator=g).float(), weight_scales((N + 127) // 128, K // 128, g)


def inexact_case(m, N, K, seed):
    """(qa, qw, sa, sw): integer operands (P exact, see the module doc) with inexact scales"""
    qa, sa = inexact_activations(m, K, seed)
    qw, sw = inexact_weights(N, K, seed + 1)
    return qa, qw, sa, sw


def bias_for(N, out, seed):
    """a bias [N] in out_dtype, of the outputs' magnitude"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(N, generator=g) * 0.5).to(OUT[out])


def grouped_case(counts, N, K, swiglu):
    """(qa [T, K], sa [T, K/128], per-expert weights): [(qw, sw)] for the plain form, [(gate, sg), (up, su)] for the SwiGLU
    form (N = 2I: gate and up [I, K] with [ceil(I/128), K/128] scales, as interleave_gate_up takes them)"""
    qa, sa = inexact_activations(sum(counts), K, seed=len(counts) + K)
    halves = (0, 1) if swiglu else (0,)
    rows = N // 2 if swiglu else N
    return qa, sa, [[inexact_weights(rows, K, seed=1000 * e + h) for h in halves] for e in range(len(counts))]


def fp8_case(m, N, K):
    return inexact_case(m, N, K, seed=m * 31 + N + K)


def split_case(f, m, N, K, cap):
    return inexact_case(m, N, K, seed=f * 1000 + m + cap)


def a_scale_view(sa, pad, device):
    """sa [m, KB] in bb_quantize_act_fp8's layout on the device: the [m, KB] view of a k-block-major [KB, ld] buffer with ld =
    round_up(m, 4) + pad; the gap between one block's m scales and the next block's is NaN, so a scale read from it shows"""
    m, KB = sa.shape
    buf = torch.full((KB, (m + 3) // 4 * 4 + pad), float("nan"))
    buf[:, :m] = sa.t()
    return buf.to(device).t()[:m]


def prove_exact(qa, qw):
    """the precondition under which P is exact in every order: integer operands exact in e4m3, every block's sum_k |a_k w_k| at
    most P_MAX (bounded by the row's sum_k |a_k| times max |w|)"""
    for q in (qa, qw):
        assert torch.equal(q, q.round()) and torch.equal(q.to(E4M3).float(), q)
    m, K = qa.shape
    bound = qa.abs().view(m, K // 128, 128).sum(-1).max() * qw.abs().max() if qa.numel() and qw.numel() else 0.0
    assert float(bound) <= P_MAX, float(bound)


def scale_rows(sw, N):
    """the [N, KB] weight scale of every weight row: row n reads block row n / 128"""
    return sw.repeat_interleave(128, 0)[:N]


def block_sums(qa, qw):
    """P [KB, m, N] float32, exact (prove_exact)"""
    m, K = qa.shape
    N = qw.shape[0]
    KB = K // 128
    return torch.bmm(qa.view(m, KB, 128).transpose(0, 1), qw.view(N, KB, 128).permute(1, 2, 0))


# ---- the header's order and the variants it must be told apart from ----------------------------------------------------------
def promote(P, sa, swn, splits=1, variant=None):
    """S [m, N] float32 from P [KB, m, N], a_scale [m, KB] and per-row weight scales swn [N, KB]: the header's order, or one
    plausible wrong one -- "fma" (fl(P c + S), one rounding), "p_sa_sw" ((P sa) sw), "descending" (blocks in descending
    order), "reversed_splits" (the splits reduced last to first), "pairwise_splits" (the splits reduced as a balanced tree)"""
    KB, m, N = P.shape
    assert KB % splits == 0
    per = KB // splits
    parts = []
    for j in range(splits):
        blocks = range(j * per, (j + 1) * per)
        if variant == "descending":
            blocks = reversed(blocks)
        S = torch.zeros(m, N, dtype=torch.float32, device=P.device)
        for b in blocks:
            sa_b, sw_b = sa[:, b, None], swn[None, :, b]
            if variant == "p_sa_sw":
                S = S + (P[b] * sa_b) * sw_b
            elif variant == "fma":
                # P c is exact in float64 (P has at most 13 significant bits) and the one rounding of P c + S is float64's,
                # then fp32's; the result is an fma's but in the rare double-rounding case
                S = (P[b].double() * (sa_b * sw_b).double() + S.double()).float()
            else:
                S = S + P[b] * (sa_b * sw_b)
        parts.append(S)
    if variant == "reversed_splits":
        parts = parts[::-1]
    if variant == "pairwise_splits":
        while len(parts) > 1:
            parts = [parts[i] + parts[i + 1] if i + 1 < len(parts) else parts[i] for i in range(0, len(parts), 2)]
        return parts[0]
    S = torch.zeros(m, N, dtype=torch.float32, device=P.device)
    for Sj in parts:
        S = S + Sj
    return S


def round_out(S, out, bias=None, bias_first=False):
    """C = round_out(S) (+ bias in out_dtype after the rounding; an fp32 output is one sum).  bias_first: the wrong order, the
    bias added to S in fp32 before the one rounding."""
    if bias is not None and bias_first and out != "float32":
        return (S + bias.float()).to(OUT[out])
    y = S.to(OUT[out])
    return y + bias if bias is not None else y


def restate(qa, qw, sa, sw, splits=1, variant=None):
    """S of bb_matmul_fp8 for host operands, computed on qa's device"""
    prove_exact(qa, qw)
    return promote(block_sums(qa, qw), sa, scale_rows(sw, qw.shape[0]), splits, variant)


def silu_mul(g, u, out):
    """the header's SwiGLU rule: g and u as stored (out_dtype), silu in fp32, one rounding"""
    gf, uf = g.float(), u.float()
    return (gf / (1 + torch.exp(-gf)) * uf).to(OUT[out])


def offsets_of(counts):
    out = [0]
    for c in counts:
        out.append(out[-1] + c)
    return out


# ---- the case lists the GPU tests run (and test_fp8_restate checks for power) ----------------------------------------------------
# bb_matmul_fp8: every BM instance (m <= 32, <= 64, > 64; one and several m-tiles), four N (N % 128 != 0 twice), K = 128, an odd
# block count (K = 1152) and DeepSeek-V3's K values; each m takes one of two sets that both hold every N.  Each case runs every
# output type, with and without a bias, the latter with a_scale_ld > m.
_NK = [[(576, 7168), (144, 128), (1040, 1152), (7168, 2048)],
       [(576, 18432), (144, 16384), (1040, 512), (7168, 1536)]]
FP8_MS = [1, 32, 33, 64, 65, 128, 129, 300]
FP8_CASES = [(m, N, K) for i, m in enumerate(FP8_MS) for N, K in _NK[i % 2]]

# split-K, (f, m, N, K, cap): every factor f = 2 .. 8 from K = 1024 f (8 blocks per split) at a tile count that leaves SMs
# idle on the full device (cap 0), and three factors an SM-count cap forces below the full device's
SPLIT_CASES = [(2, 1, 576, 2048, 0), (3, 20, 1040, 3072, 0), (4, 64, 576, 4096, 0), (5, 100, 144, 5120, 0),
               (6, 1, 2048, 6144, 0), (7, 33, 576, 7168, 0), (8, 128, 1040, 8192, 0),
               (2, 1, 576, 8192, 16), (3, 4, 1536, 6144, 40), (5, 1, 2048, 10240, 80)]

# grouped: (counts or offsets, N, K, SM-count cap); every BM bucket with experts starting at rows not = 0 mod 4, empty experts
# and T not a multiple of BM; E = 1; E = 256; and the BM buckets again under capped SM counts.  N is 2I for the SwiGLU form.
GROUPED_CASES = {   # name: (counts, N, K, SM-count cap or 0, the BM bucket launch_grouped_fp8_bm picks)
    "bm32": ([5, 0, 32, 17, 1, 40], 384, 7168, 0, 32),
    "bm64": ([50, 0, 64, 100, 33], 256, 2048, 0, 64),
    "bm128": ([300, 0, 129, 1, 200], 384, 1152, 0, 128),
    "e1": ([77], 256, 1536, 0, 128),
    "e256": ([(7 * e) % 6 if e % 9 else 0 for e in range(255)] + [3], 128, 512, 0, 32),
    "bm32_cap1": ([3, 9, 0, 30, 2], 256, 1024, 1, 32),
    "bm64_cap7": ([41, 0, 63, 70, 1, 60], 384, 2048, 7, 64),
    "bm128_cap114": ([200, 131, 0, 7, 300], 256, 1536, 114, 128),
}
