"""Inputs on which every kernel of the library must be exact, their proof, the exact reference, and the CPU mirrors of the
work decompositions (slab stream-K ranges and fix-up protocol, the GEMV K split).

Every value is a dyadic rational on a common grid 2^-E: activations in {0, +-1/2, +-1}, scales +-2^e (e in -2..0), zero points
that are integers, half-integers, negatives or the above-fold values (50 / 200 fp16, 120 / 200 bf16), "rescale" zeros j * s,
quantized zeros as stored.  `prove_exact` bounds every fp32 partial sum a kernel can form, in grid units, and requires it to stay
below 2^22: then products and sums are exact in fp32 in any order, split or K split, and every kernel must return the correctly
rounded exact result, round(V) (with bias round(round(V) + b) in the output type), bit for bit.

Bounds per family (values; times 2^E for grid units):
  * sum       gemm_ts, generic, grouped GEMM:  max sum_k |a_k| T_nk,  T = |s| (15 + |z|) (+ |z| for rescale), >= |dequantised w|
              and the slab's per-step fold c1 (partial - SM) + c2 S accumulated over K
  * slab      the magic chains inside one 128-k step:  (magic + 15) max sum_{k in step} |a_k|
  * gemv      gemv_mma / grouped GEMV: the weight chain and the fold chain run over a whole group (up to K), and a warp's K range can
              start anywhere:  (magic + 16 + max|z|) (2 max_k |prefix sum of a| + max 32-block sum |a|) + 15 sum_k |a_k|
"""
from __future__ import annotations

import torch

import bitblas_oracle as O

MAGIC = {"float16": 1024.0, "bfloat16": 128.0}
LIMIT_UNITS = 2 ** 22


# ---- inputs ------------------------------------------------------------------------------------------------------------------
def dyadic_activations(M, K, gen, density=0.25, group=None):
    """[M, K] float64 in {0, +-1/2, +-1}.  Every 32-element block has a nonzero sum tau in {+-1/2, +-1}, whose sign is normally
    chosen against the running prefix, so the prefix sum over blocks stays small.  The last block of each group of `group`
    elements (default K) and the last block of the row pick, among the four tau, the first that leaves the group's and the row's
    sum nonzero: every zero-point group and every row has a nonzero activation sum, so the magic and zero-point removal through
    the sums is exercised in every group, while the prefix stays within [-2, 2]."""
    assert K % 32 == 0
    group = K if group is None else group
    assert group % 32 == 0 and K % group == 0
    nb, gb = K // 32, group // 32
    B = M * nb
    mag = torch.where(torch.rand((B, 15), generator=gen) < 0.5, 0.5, 1.0)
    sign = torch.where(torch.rand((B, 15), generator=gen) < 0.5, -1.0, 1.0)
    x = (mag * sign * (torch.rand((B, 15), generator=gen) < density)).double()
    neg = -x.gather(1, torch.rand((B, 15), generator=gen).argsort(1))
    taum = torch.where(torch.rand((M, nb), generator=gen) < 0.5, 0.5, 1.0).double()
    coin = torch.where(torch.rand((M, nb), generator=gen) < 0.5, -1.0, 1.0).double()
    tau = torch.empty((M, nb), dtype=torch.float64)
    pre = torch.zeros(M, dtype=torch.float64)   # row prefix
    gsum = torch.zeros(M, dtype=torch.float64)  # sum of the current group so far
    for j in range(nb):
        sg = torch.where(pre > 0, -1.0, torch.where(pre < 0, 1.0, coin[:, j]))
        t = sg * taum[:, j]
        if (j + 1) % gb == 0:
            last_row = j == nb - 1
            # candidates in order of preference: the usual tau, the other magnitude, then the opposite sign
            cands = [t, sg * (1.5 - taum[:, j]), -sg * 0.5, -sg * 1.0]
            chosen = torch.full_like(t, float("nan"))
            for c in reversed(cands):
                ok = (gsum + c != 0) & ((pre + c != 0) | (not last_row))
                chosen = torch.where(ok, c, chosen)
            t = chosen
        tau[:, j] = t
        pre = pre + t
        gsum = torch.zeros_like(gsum) if (j + 1) % gb == 0 else gsum + t
    blk = torch.cat([x, neg, tau.reshape(B, 1), torch.zeros((B, 1), dtype=torch.float64)], 1)
    blk = blk.gather(1, torch.rand((B, 32), generator=gen).argsort(1))
    return blk.reshape(M, K)


def sharded_activations(M, K, shards, gen, density=0.25, group=None):
    """[M, K] activations of a row-parallel layer: dyadic_activations per K shard of K / shards columns, so every shard's row sum
    and every group sum inside a shard is nonzero (a shard is a problem of its own, and with whole-row groups its K range is one
    group); a row whose shard sums cancel has its last shard negated, which keeps the full row's sum nonzero as well"""
    per = K // shards
    assert per * shards == K
    group = K if group is None else group
    A = torch.cat([dyadic_activations(M, per, gen, density, min(group, per)) for _ in range(shards)], 1)
    A[A.sum(1) == 0, K - per:] *= -1
    return A


def _fp8_dyadic_codes(fmt):
    """8-bit float codes whose value is a multiple of 1/8 and at most 16 in magnitude"""
    u = torch.arange(256, dtype=torch.int32)
    v = O.decode_fields(u, fmt, 8, torch.float32).double()
    ok = torch.isfinite(v) & (v.abs() <= 16) & ((v * 8).round() == v * 8)
    return u[ok]


def _auto_density(K, mode, bit, scale, zeros, qz, fmt):
    """the activation density that keeps the sum family's bound near 0.7 x 2^22 grid units: sum_k |a_k| is about
    (K / 32) (22.5 d + 3/4) for dyadic_activations, the largest term T and the grid follow from the parameters alone"""
    u_max = 2.0 ** bit - 1 if fmt in ("uint", "int") else 16.0
    s = scale.double().abs() if scale is not None else torch.ones(1, dtype=torch.float64)
    gs = _grid_exp(s)
    if mode == "original":
        z = zeros.double()
        T, gz = float((s * (u_max + z.abs())).max()), gs + _grid_exp(z)
    elif mode == "rescale":
        z = zeros.double()
        T, gz = float((s * u_max + z.abs()).max()), max(gs, _grid_exp(z))
    else:
        T, gz = float(s.max()) * (u_max + 2.0 ** (bit - 1)), gs + (3 if fmt not in ("uint", "int") else 0)
    budget = 0.7 * LIMIT_UNITS / (T * 2.0 ** (1 + gz))
    return min(0.25, max(0.02, (budget / (K / 32) - 0.75) / 22.5))


def make_exact_case(M, N, K, *, A_dtype="float16", W_dtype="uint4", out_dtype="float16", group_size=-1, mode="none", bias=False,
                    fast_decoding=None, seed=0, A=None, density=None, propagate_b=False, shards=1):
    """one case in the layout of test_gpu_kernel_grid.make_case (so helpers.product_operator / run_product take it), built from
    the exact value sets of the module docstring.  A_dtype int8: integer activations, exact as before.  shards > 1: the
    activations of sharded_activations, so each of `shards` equal K ranges is an exact case of its own too."""
    g = torch.Generator().manual_seed(seed)
    fmt, bit = O.W_DTYPE_MAP[W_dtype]
    adt = O.TORCH_DTYPE[A_dtype]
    gs = K if group_size in (-1, None) else group_size
    assert K % gs == 0, (K, gs)
    G = K // gs
    if fmt in ("fp_e4m3", "fp_e5m2"):
        codes = _fp8_dyadic_codes(fmt)
        fields = codes[torch.randint(0, codes.numel(), (N, K), generator=g)].to(torch.uint8)
    else:
        fields = torch.randint(0, 2 ** bit, (N, K), generator=g, dtype=torch.uint8)
    with_scaling = mode != "none"
    with_zeros = mode in ("original", "rescale", "quantized")
    scale = zeros = qz = b = None
    if with_scaling:
        sign = torch.where(torch.rand((N, G), generator=g) < 0.3, -1.0, 1.0)
        scale = (sign * torch.pow(2.0, -torch.randint(0, 3, (N, G), generator=g).double())).to(adt)
    if mode == "original":
        big = (50.0, 200.0) if A_dtype == "float16" else (120.0, 200.0)
        choices = torch.stack([
            torch.randint(0, 2 ** bit, (N, G), generator=g).double(),                      # integer (folded by the GEMVs)
            torch.randint(0, 2 ** bit - 1, (N, G), generator=g).double() + 0.5,             # half-integer
            -torch.randint(1, 9, (N, G), generator=g).double() / 2,                         # negative, -1/2 .. -4
            torch.full((N, G), big[0], dtype=torch.float64), torch.full((N, G), big[1], dtype=torch.float64)])
        zeros = choices.gather(0, torch.randint(0, 5, (N, G), generator=g)[None]).squeeze(0).to(adt)
    elif mode == "rescale":
        j = torch.randint(-8, 2 ** bit, (N, G), generator=g).double()
        zeros = (j * scale.double()).to(adt)
    elif mode == "quantized":
        qz = torch.randint(0, 2 ** bit, (G, N), generator=g, dtype=torch.int32)
        zeros = torch.from_numpy(O.general_compress(qz.numpy(), bit))
    if bias:
        if A_dtype == "int8":
            b = torch.randint(-8, 8, (N,), generator=g, dtype=torch.int8)
        else:
            b = (torch.randint(-16, 17, (N,), generator=g).double() / 4).to(adt)
    if A is None:
        if A_dtype == "int8":
            A = torch.randint(-32, 32, (M, K), generator=g, dtype=torch.int8)
        else:
            if density is None:
                density = _auto_density(K, mode, bit, scale, zeros, qz, fmt)
            if shards > 1:
                A = sharded_activations(M, K, shards, g, density, gs).to(adt)
            else:
                A = dyadic_activations(M, K, g, density, gs).to(adt)
    cfg = dict(A_dtype=A_dtype, W_dtype=W_dtype, accum_dtype="int32" if A_dtype == "int8" else "float32",
               out_dtype=out_dtype, group_size=group_size, with_scaling=with_scaling, with_zeros=with_zeros,
               zeros_mode=mode if with_zeros else "original", with_bias=bias, fast_decoding=fast_decoding)
    return dict(M=M, N=N, K=K, A=A, fields=fields, scale=scale, zeros=zeros, qz=qz, bias=b, bit=bit, fmt=fmt, mode=mode,
                cfg=cfg, propagate_b=propagate_b)


def product_operator(case, M=None):
    """helpers.product_operator with the case's slab tiling (propagate_b)"""
    import bitblas_b200 as bitblas
    c = case["cfg"]
    cfg = bitblas.MatmulConfig(M=M if M is not None else case["M"], N=case["N"], K=case["K"], A_dtype=c["A_dtype"],
                               W_dtype=c["W_dtype"], accum_dtype=c["accum_dtype"], out_dtype=c["out_dtype"], layout="nt",
                               with_bias=c["with_bias"], group_size=c["group_size"], with_scaling=c["with_scaling"],
                               with_zeros=c["with_zeros"], zeros_mode=c["zeros_mode"], fast_decoding=c["fast_decoding"],
                               propagate_b=bool(case.get("propagate_b")))
    return bitblas.Matmul(cfg, enable_tuning=False)


def product_weight(op, case, device):
    """stored weight: the unsigned fields through the operator's own transform (and slab tiling), on the device"""
    w = case["fields"].to(device).view(torch.int8) if case["fields"].dtype == torch.uint8 else case["fields"].to(device, torch.int8)
    if op.weight_transform is not None:
        w = op.weight_transform(w).contiguous()
    if op.weight_tiled:
        w = op.tile_weight(w)
    return w


# ---- GPTQ checkpoints of exact cases ------------------------------------------------------------------------------------------------
def _pack_int32(vals, bits, dim):
    """int64 values in [0, 2^bits) -> int32 words along `dim`, element i of a word at bit bits * i (auto_gptq's packing)"""
    per = 32 // bits
    v = vals.to(torch.int64).movedim(dim, 0)
    word = torch.zeros((v.shape[0] // per, *v.shape[1:]), dtype=torch.int64)
    for i in range(per):
        word |= v[i::per] << (bits * i)
    word = torch.where(word >= 2 ** 31, word - 2 ** 32, word)
    return word.to(torch.int32).movedim(0, dim).contiguous()


def gptq_checkpoint(case, *, v2, act_order, scale_dtype, seed):
    """what an auto_gptq QuantLinear of the quantized-zeros case `case` (make_exact_case(..., mode="quantized")) holds, as a
    namespace: qweight int32 [K*bits/32, N], qzeros int32 [K/g, N*bits/32] (v1 stores z - 1 modulo 2^bits, so z = 0 is stored as
    2^bits - 1; v2 stores z), scales [K/g, N] and bias [N] in `scale_dtype` (+-2^e and quarter integers: exact in float16 and
    bfloat16), g_idx int32 [K].  The case's K axis is the sorted one: with act_order, GPTQ's desc_act assignment of the checkpoint's
    columns to groups (from `seed` alone, so modules built with one seed share a g_idx) puts sorted column j at checkpoint column
    perm[j], perm = stable_argsort(g_idx); without it g_idx = k // g and perm is None.  Also returns A, the case's activations in
    checkpoint column order (A[:, perm] is the case's), and perm."""
    from types import SimpleNamespace
    assert case["mode"] == "quantized" and case["fmt"] == "uint", (case["mode"], case["fmt"])
    N, K, bits = case["N"], case["K"], case["bit"]
    G = case["qz"].shape[0]
    g = K // G
    if act_order:
        gen = torch.Generator().manual_seed(seed)
        g_idx = torch.empty(K, dtype=torch.int32)
        g_idx[torch.randperm(K, generator=gen)] = torch.arange(K, dtype=torch.int32) // g
        perm = torch.sort(g_idx.long(), stable=True).indices
        A = torch.empty_like(case["A"])
        A[:, perm] = case["A"]
        intw = torch.empty((K, N), dtype=torch.int64)
        intw[perm] = case["fields"].T.to(torch.int64)
    else:
        g_idx = torch.arange(K, dtype=torch.int32) // g
        perm, A, intw = None, case["A"], case["fields"].T.to(torch.int64)
    z = case["qz"].to(torch.int64)
    stored_z = z if v2 else (z - 1) % 2 ** bits
    bias = None if case["bias"] is None else torch.nn.Parameter(case["bias"].double().to(scale_dtype), requires_grad=False)
    return SimpleNamespace(qweight=_pack_int32(intw, bits, 0), qzeros=_pack_int32(stored_z, bits, 1),
                           scales=case["scale"].double().T.contiguous().to(scale_dtype), bias=bias, g_idx=g_idx, A=A, perm=perm)


def zeros_mode_case(case, mode):
    """the quantized-zeros case with its integer zero points z expressed in `mode`: "original" zeros z, "rescale" zeros z s (exact:
    s = +-2^e), or the case itself; every mode dequantises to the same (w - z) s"""
    if mode == "quantized":
        return case
    adt = O.TORCH_DTYPE[case["cfg"]["A_dtype"]]
    z = case["qz"].double().T
    zeros = (z if mode == "original" else z * case["scale"].double()).to(adt)
    assert torch.equal(zeros.double(), z if mode == "original" else z * case["scale"].double())
    return dict(case, mode=mode, zeros=zeros, qz=None, cfg=dict(case["cfg"], zeros_mode=mode))


# ---- the operands as float64 ---------------------------------------------------------------------------------------------------
def _gidx(case, device):
    G = case["scale"].shape[1] if case["scale"] is not None else 1
    return torch.arange(case["K"], device=device) // (case["K"] // G)


def decoded(case, device="cpu"):
    """the decoded weight field values [N, K] (float64), before scale and zeros"""
    u = case["fields"].to(device).to(torch.int64)
    fmt, bit = case["fmt"], case["bit"]
    if fmt == "uint":
        return u.double()
    if fmt == "int":
        return (u - 2 ** (bit - 1)).double()
    adt = O.TORCH_DTYPE[case["cfg"]["A_dtype"]]
    return O.decode_fields(u.to(torch.int32).cpu(), fmt, bit, adt).double().to(device)


def zero_points(case, device="cpu"):
    """z [N, K] float64 of the mode: original / rescale zeros, quantized zeros (integers), or None"""
    mode = case["mode"]
    if mode in ("original", "rescale"):
        return case["zeros"].to(device).double()[:, _gidx(case, device)]
    if mode == "quantized":
        return case["qz"].to(device).double()[_gidx(case, device), :].T
    return None


def dequantized(case, device="cpu"):
    """W [N, K] float64: exactly (w - z) s, w s - z or w s (the inputs make every kernel's dequantisation order exact)"""
    w = decoded(case, device)
    mode = case["mode"]
    if mode == "none":
        return w
    s = case["scale"].to(device).double()[:, _gidx(case, device)]
    z = zero_points(case, device)
    if mode in ("original", "quantized"):
        return (w - z) * s
    if mode == "rescale":
        return w * s - z
    return w * s


def _grid_exp(x):
    """the least e >= 0 with x * 2^e integral everywhere"""
    for e in range(0, 40):
        y = x * 2.0 ** e
        if bool((y == y.round()).all()):
            return e
    raise AssertionError("values are not dyadic with fewer than 40 fractional bits")


# ---- the precondition ------------------------------------------------------------------------------------------------------------
def prove_exact(case, families=("sum", "slab", "gemv"), device="cpu"):
    """assert that every fp32 partial sum of the named kernel families is below 2^22 grid units, that each dequantisation step is
    exact in A_dtype, and that the result is finite in the output type.  Returns {family: worst bound in grid units}."""
    A_dtype = case["cfg"]["A_dtype"]
    if A_dtype == "int8":
        return {}
    adt = O.TORCH_DTYPE[A_dtype]
    A = case["A"].to(device).double()
    w = decoded(case, device)
    W = dequantized(case, device)
    z = zero_points(case, device)
    mode = case["mode"]
    # each step of the A_dtype dequantisation (gemm_ts / generic: w - z, then * s; w * s, then - z) is exact
    steps = [w, W]
    if z is not None and mode == "original":
        steps.append(w - z)
    if mode == "rescale":
        steps.append(w * case["scale"].to(device).double()[:, _gidx(case, device)])
    for t in steps:
        assert torch.equal(t.to(adt).double(), t), "a dequantisation step is not exact in " + A_dtype
    # the magic and zero-point removal act through activation sums: a group (or row) whose sum is zero would hide a wrong zero
    # point or magic there
    G = case["scale"].shape[1] if case["scale"] is not None else 1
    assert bool((A.sum(1) != 0).all()), "an activation row sums to zero"
    assert bool((A.reshape(A.shape[0], G, -1).sum(-1) != 0).all()), "an activation group sums to zero"
    ga, gd, gW = _grid_exp(A), _grid_exp(w), _grid_exp(W)
    gs = _grid_exp(case["scale"].to(device).double()) if case["scale"] is not None else 0
    gz = _grid_exp(z) if z is not None else 0
    # every term a kernel accumulates -- a w s, a z s, a (magic + u), a (magic + z), a z (rescale), a W -- lies on 2^-E
    E = ga + max(gs + gd, gz if mode == "rescale" else gs + gz, gW)
    Aa = A.abs()
    if case["fmt"] in ("uint", "int"):
        s_abs = case["scale"].to(device).double()[:, _gidx(case, device)].abs() if case["scale"] is not None else 1.0
        zp = 2.0 ** (case["bit"] - 1) if case["fmt"] == "int" else 0.0
        u_max = 2.0 ** case["bit"] - 1
        if mode == "rescale":
            T = s_abs * u_max + z.abs()
        else:
            T = s_abs * (u_max + (z.abs() if z is not None else zp))
        T = torch.maximum(T if torch.is_tensor(T) else torch.full_like(W, T), W.abs())
    else:
        T = W.abs()
    out = {}
    if "sum" in families:
        out["sum"] = float((Aa @ T.T).max())
    if case["fmt"] in ("uint", "int"):
        magic = MAGIC[A_dtype]
        zmax = float(z.abs().max()) if z is not None else 2.0 ** (case["bit"] - 1)
        if "slab" in families:
            step = Aa.reshape(A.shape[0], -1, 128).sum(-1) if case["K"] % 128 == 0 else Aa.sum(1, keepdim=True)
            out["slab"] = max(float(step.max()) * (magic + 15), out.get("sum", float((Aa @ T.T).max())))
        if "gemv" in families:
            pre = A.cumsum(1).abs().max()
            blk = Aa.reshape(A.shape[0], -1, 32).sum(-1).max()
            out["gemv"] = float((magic + 16 + zmax) * (2 * pre + blk) + 15 * Aa.sum(1).max())
    units = {k: v * 2.0 ** E for k, v in out.items()}
    for k, v in units.items():
        assert v < LIMIT_UNITS, f"{k}: a partial sum may reach {v:.3g} grid units (2^-{E}), not below 2^22"
    ref = exact_reference(case, device)
    assert torch.isfinite(ref.double()).all(), "the rounded reference is not finite in " + case["cfg"]["out_dtype"]
    return units


# ---- the reference -------------------------------------------------------------------------------------------------------------
def exact_value(case, device="cpu", rows=None):
    """V = A W^T in float64 (exact under prove_exact: every summation order gives the same value)"""
    A = case["A"] if rows is None else case["A"][rows]
    return A.to(device).double() @ dequantized(case, device).T


def round_out(V, case):
    """the output: round(V), with bias round(round(V) + round(b)) in the output type (fp32: V + b rounded once)"""
    odt = O.TORCH_DTYPE[case["cfg"]["out_dtype"]]
    v32 = V.float()
    assert torch.equal(v32.double(), V), "V is not exact in fp32"
    if case["bias"] is None:
        return v32.to(odt)
    b = case["bias"].to(V.device)
    if odt == torch.float32:
        return v32 + b.float()
    return v32.to(odt) + b.to(odt)


def exact_reference(case, device="cpu", rows=None):
    if case["cfg"]["A_dtype"] == "int8":
        from test_gpu_kernel_grid import int_reference
        c = dict(case, fields=case["fields"].to(torch.int32))
        return int_reference(c, rows).to(device)
    return round_out(exact_value(case, device, rows), case)


def int64_value(case):
    """V recomputed in int64 on scaled integers (CPU): A 2^ga, W 2^gw, V = (A_int W_int^T) 2^-(ga + gw)"""
    A = case["A"].double()
    W = dequantized(case)
    ga, gw = _grid_exp(A), _grid_exp(W)
    Ai = (A * 2.0 ** ga).to(torch.int64)
    Wi = (W * 2.0 ** gw).to(torch.int64)
    assert torch.equal(Ai.double(), A * 2.0 ** ga) and torch.equal(Wi.double(), W * 2.0 ** gw)
    Vi = (Ai[:, None, :] * Wi[None, :, :]).sum(-1)
    return Vi, ga + gw


def compare_exact(got, ref, what, context=None):
    """torch.equal; on a mismatch: how many differ, the first ones, and `context(row, col)` for each of them"""
    got = got.cpu()
    ref = ref.cpu()
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    if torch.equal(got, ref):
        return
    bad = got.double() != ref.double()
    if ref.is_floating_point():
        bad = bad & ~(got.isnan() & ref.isnan())
    idx = bad.nonzero()[:6].tolist()
    lines = [f"{what}: {int(bad.sum())}/{bad.numel()} elements differ"]
    for i in idx:
        i = tuple(i)
        extra = f"  {context(*i)}" if context is not None else ""
        lines.append(f"  at {list(i)}: got {got[i].item()!r} ref {ref[i].item()!r}{extra}")
    raise AssertionError("\n".join(lines))


# ---- slab stream-K: the partition (bb_gemv_slab.cu launch_gemv_slab / gemv_slab_kernel) ---------------------------------------------
NG, UNIT_K, ROWS = 2, 1024, 32


def slab_geometry(N, K, sms):
    """UPR, NRB, T, R of the launch on `sms` SMs (two CTAs per SM)"""
    UPR = -(-K // UNIT_K)
    NRB = -(-N // ROWS)
    T = -(-NRB // NG) * UPR * NG
    R = max(1, min(T, 2 * sms))
    return UPR, NRB, T, R


def slab_slot_bytes(sms):
    """bb_workspace_bytes of an m = 1 slab call on `sms` SMs: [2 CTAs per SM][NG groups][32 rows] 8-byte slots, + 256 for alignment"""
    return 2 * NG * ROWS * 8 * sms + 256


def range_begin(ri, T, R):
    return ri * T // R


def unit_of(t, UPR):
    g, rest = t % NG, t // NG
    q, ku = rest // UPR, rest % UPR
    return q * NG + g, ku


def slab_ranges_of_block(N, K, sms):
    """{row block: sorted list of the CTA ranges holding one of its units} (CTA index = R - 1 - range index)"""
    UPR, NRB, T, R = slab_geometry(N, K, sms)
    out = {}
    for ri in range(R):
        for t in range(range_begin(ri, T, R), range_begin(ri + 1, T, R)):
            rb, _ = unit_of(t, UPR)
            out.setdefault(rb, set()).add(ri)
    return {rb: sorted(v) for rb, v in out.items()}


def slab_coverage(N, K, sms):
    """the stream-K properties the shape reaches on `sms` SMs"""
    UPR, NRB, T, R = slab_geometry(N, K, sms)
    props = set()
    spans = slab_ranges_of_block(N, K, sms)
    if any(len(v) >= 3 for rb, v in spans.items() if rb < NRB):
        props.add("block_over_3_ranges")
    if T <= 2 * sms:
        props.add("one_unit_per_cta")
    if NRB % 2:
        props.add("odd_NRB")
    if N % 32 == 16:
        props.add("N%32=16")
    nsl = (K // 2 - (UPR - 1) * 512) // 128
    if nsl in (1, 2, 3):
        props.add(f"ragged_last_unit_{nsl}_slices")
    for ri in range(R):
        t0, t1 = range_begin(ri, T, R), range_begin(ri + 1, T, R)
        if t1 > t0 and all(unit_of(t, UPR)[0] >= NRB for t in range(t0, t1)):
            props.add("padding_only_range")
        for grp in range(NG):
            segs = _segments(t0, t1, grp, UPR)
            if sum(1 for rb, kus in segs if rb < NRB and kus == list(range(UPR))) >= 2:
                props.add("group_closes_2_blocks")   # several owner fix-ups of one group in one CTA (small SM counts only)
            for j, (rb, kus) in enumerate(segs):
                if rb >= NRB:
                    continue
                if kus[0] > 0 and kus[-1] < UPR - 1:
                    props.add("range_inside_block")
                if j > 0 and kus[0] == 0 and kus[-1] < UPR - 1 and segs[j - 1][1] == list(range(UPR)):
                    props.add("owner_stops_mid_block")
    return props


def _segments(t0, t1, grp, UPR):
    """the (row block, [ku...]) segments group `grp` of range [t0, t1) walks, in order"""
    segs = []
    for t in range(t0, t1):
        if t % NG != grp:
            continue
        rb, ku = unit_of(t, UPR)
        if segs and segs[-1][0] == rb:
            segs[-1][1].append(ku)
        else:
            segs.append((rb, [ku]))
    return segs


def slab_fixup_protocol(N, K, R):
    """the kernel's consumer-group loop (segments, seg_from0 / closes, park / collect), transcribed, over R ranges.  Returns
    (parks, collects): parks {(ri, grp): rb} of the slots written, collects [(owner ri, rj, grp, rb)] of the slots awaited."""
    UPR = -(-K // UNIT_K)
    NRB = -(-N // ROWS)
    T = -(-NRB // NG) * UPR * NG
    parks, collects = {}, []
    for ri in range(R):
        t0, t1 = range_begin(ri, T, R), range_begin(ri + 1, T, R)
        n_units = t1 - t0
        for grp in range(NG):
            i = (grp - t0 % NG + NG) % NG
            rb = ku = 0
            if i < n_units:
                rb, ku = unit_of(t0 + i, UPR)
            seg_from0 = seg_open = False
            while i < n_units:
                if not seg_open:
                    seg_from0, seg_open = ku == 0, True
                closes = ku == UPR - 1
                if closes or i + NG >= n_units:
                    if not seg_from0:
                        assert (ri, grp) not in parks, f"range {ri} group {grp} parks twice"
                        parks[(ri, grp)] = rb
                    elif not closes:
                        t_first = (t0 + i) - ku * NG
                        t_last = t_first + (UPR - 1) * NG
                        for rj in range(ri + 1, R):
                            bj, ej = range_begin(rj, T, R), range_begin(rj + 1, T, R)
                            if bj > t_last:
                                break
                            tf = bj + ((t_first - bj) % NG + NG) % NG
                            if tf >= ej or tf > t_last:
                                if ej > t_last:
                                    break
                                continue
                            collects.append((ri, rj, grp, rb))
                            if ej > t_last:
                                break
                    seg_open = False
                i += NG
                ku += 1
                if ku == UPR:
                    ku = 0
                    rb += NG
    return parks, collects


def check_fixup_protocol(N, K, R):
    """every parked partial is collected exactly once, by the owner of its row block; every awaited slot is parked with a
    partial of the same row block; owners wait only on later ranges (earlier CTAs); every unit of a block is summed once"""
    UPR = -(-K // UNIT_K)
    NRB = -(-N // ROWS)
    T = -(-NRB // NG) * UPR * NG
    parks, collects = slab_fixup_protocol(N, K, R)
    seen = {}
    for owner, rj, grp, rb in collects:
        assert rj > owner
        assert (rj, grp) in parks, f"N={N} K={K} R={R}: range {owner} waits on range {rj} group {grp}, which never parks"
        assert parks[(rj, grp)] == rb, f"N={N} K={K} R={R}: slot ({rj}, {grp}) holds block {parks[(rj, grp)]}, awaited for {rb}"
        assert (rj, grp) not in seen, f"N={N} K={K} R={R}: slot ({rj}, {grp}) collected twice"
        seen[(rj, grp)] = owner
    missing = set(parks) - set(seen)
    assert not missing, f"N={N} K={K} R={R}: parked but never collected: {sorted(missing)[:4]}"
    # every unit of a block belongs to the owner's segment or to exactly one collected parked segment
    owner_of = {}
    for ri in range(R):
        t0, t1 = range_begin(ri, T, R), range_begin(ri + 1, T, R)
        for grp in range(NG):
            for rb, kus in _segments(t0, t1, grp, UPR):
                if kus[0] == 0:
                    assert rb not in owner_of
                    owner_of[rb] = ri
    for rb in range(-(-NRB // NG) * NG):
        assert rb in owner_of, f"N={N} K={K} R={R}: block {rb} has no owner"
    for (rj, grp), rb in parks.items():
        assert seen[(rj, grp)] == owner_of[rb]
    return len(parks)


# ---- gemv_mma / gemv_i8 K split (bb_gemv_mma.cuh split_range) --------------------------------------------------------------------
def split_range(total, parts, idx):
    base, rem = divmod(total, parts)
    begin = idx * base + min(idx, rem)
    return begin, begin + base + (1 if idx < rem else 0)


def mid_group_starts(K, g, ks):
    """the warps whose K range of 128-k steps starts inside a group of g elements"""
    return [w for w in range(ks) if (split_range(K // 128, ks, w)[0] * 128) % g]
