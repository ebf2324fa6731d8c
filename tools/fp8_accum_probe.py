"""How the H100's FP8 tensor core sums the 128 products of one k-block, measured through bb_matmul_fp8 (K = 128, unit scales,
fp32 output, so C is the hardware's block sum P itself).

1. One large product 2^E (E = 8 or 16, at k = pos) and 127 equal small products 2^-j: the exact sum is 2^E + 127 * 2^-j.  The
   column "kept" is the fraction of the small products' sum that survives (1: all of it, 0: none), per distance d = E + j in
   binades below the large product.  The largest d with everything kept is the accumulator's effective width.
2. Random e4m3 blocks: max over elements of |P - exact| / sum_k |a_k w_k|, the relative bound the GPU tests assume (ACC_REL in
   tests/test_gpu_fp8.py).

    python tools/fp8_accum_probe.py [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bitblas_b200 import Matmul, MatmulConfig  # noqa: E402

E4M3 = torch.float8_e4m3fn


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def block_sums(a, w):
    """the kernel's P = a @ w.T for one k-block (a [m, 128], w [N, 128] exactly representable in e4m3), as fp32"""
    m, N = a.shape[0], w.shape[0]
    op = Matmul(MatmulConfig(N=N, K=128, A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32", out_dtype="float32"),
                enable_tuning=False)
    A = a.to(E4M3).cuda()
    W = w.to(E4M3).cuda()
    ld = (m + 3) // 4 * 4
    a_scale = torch.ones(1, ld, device="cuda").t()[:m]
    return op.forward_fp8(A, W, a_scale, torch.ones((N + 127) // 128, 1, device="cuda")).double().cpu()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_accum_probe needs a GPU")
    print(f"card: {card()}  (name, power limit, max SM clock)")
    rows = []
    print(f"{'pos':>4} {'E':>3} {'j':>3} {'d':>3} | {'exact':>22} {'got':>22} {'kept':>8}")
    for pos in (0, 31, 64, 127):
        js = list(range(0, 10))
        a = torch.stack([torch.full((128,), 2.0 ** -j) for j in js])
        a[:, pos] = 2.0 ** 8
        w = torch.zeros(16, 128)
        w[0] = 1.0                    # large product 2^8
        w[1] = 1.0
        w[1, pos] = 2.0 ** 8          # large product 2^16
        P = block_sums(a, w)
        exact = a.double() @ w.double().t()
        for i, j in enumerate(js):
            for n, E in ((0, 8), (1, 16)):
                small = 127 * 2.0 ** -j
                kept = (P[i, n] - 2.0 ** E) / small
                rows.append(dict(pos=pos, E=E, j=j, d=E + j, exact=float(exact[i, n]), got=float(P[i, n]), kept=float(kept)))
                print(f"{pos:>4} {E:>3} {j:>3} {E + j:>3} | {float(exact[i, n]):>22.12f} {float(P[i, n]):>22.12f} {float(kept):>8.4f}")
    full = [r["d"] for r in rows if r["kept"] == 1.0]
    lost = [r["d"] for r in rows if r["kept"] != 1.0]
    print(f"small products kept exactly up to d = {max(full) if full else None} binades below the large one; "
          f"first loss at d = {min(lost) if lost else None}")
    g = torch.Generator().manual_seed(0)
    worst = 0.0
    for scale in (1.0, 16.0, 0.05):
        a = (torch.randn(256, 128, generator=g) * scale).clamp(-448, 448).to(E4M3).double()
        w = (torch.randn(256, 128, generator=g) * scale).clamp(-448, 448).to(E4M3).double()
        P = block_sums(a, w)
        exact = a @ w.t()
        T = a.abs() @ w.abs().t()
        rel = ((P - exact).abs() / T.clamp(min=1e-300)).max().item()
        worst = max(worst, rel)
        print(f"random blocks (randn x {scale}): max |P - exact| / sum|a w| = {rel:.3e}  (2^{torch.tensor(rel).log2().item():.2f})")
    print(f"worst relative block error: {worst:.3e}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), rows=rows, worst_rel=worst), f, indent=1)


if __name__ == "__main__":
    main()
