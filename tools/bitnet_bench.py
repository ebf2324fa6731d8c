"""BitNet b1.58 linear layer: BitLinear (quantize_act_int8, then forward_scaled: 2 launches) against the torch glue integrations run.

    python tools/bitnet_bench.py [--iters 20] [--reps 3] [--shapes 2560x2560,...] [--rows 1,4,...] [--json PATH]

Variants, on the same ternary weights (int2 storage, one fp32 scale per output row), fp16 activations:
  layer    BitLinear.forward: bb_quantize_act_int8, then bb_matmul_scaled (its epilogue divides by both scales)
  glue     BitNet's activation_quant in torch, Matmul.forward with int32 output, then / s_a / s_w, the fp16 cast and the bias in
           torch (the integration's BitLinearBitBLAS)
  floor    Matmul.forward with int32 output on int8 activations: the matmul alone, nothing around it
  scaled   Matmul.forward_scaled on the same int8 activations: against floor, what the dequantizing epilogue costs
Shapes (N, K): the linears of a 2B-parameter BitNet b1.58 model (hidden 2560, intermediate 6912: q/o 2560x2560, k/v 640x2560,
gate/up 6912x2560, down 2560x6912) and 12288x12288, at m in {1, 4, 16, 128, 1024, 4096}.  Every variant is timed eager (CUDA events
around --iters calls) and as a CapturedStep replay (--iters calls captured in one CUDA graph), the variants alternated inside every
repetition; the table gives the median over --reps.  Also per point: library launches per call (torch's kernels are not counted)
and the quantization kernel alone in GB/s (rows * K * 3 + 4 * rows bytes over its time).  The 2B model's weights are 0.4-4.4 MB, so
they stay in the 50 MB L2 across calls: the m = 1 times are launch and L2 bound, as they are in a decode step that re-reads a
layer no more often than this loop does.  The card's name, power limit and maximum SM clock are printed with the results.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bitblas_b200 as bitblas  # noqa: E402
from mlp_bench import card, events_us, graph_us, launches  # noqa: E402

SHAPES = [(2560, 2560), (640, 2560), (6912, 2560), (2560, 6912), (12288, 12288)]
ROWS = [1, 4, 16, 128, 1024, 4096]


def build(N, K, gen):
    lin = bitblas.BitLinear(K, N, bias=True).cuda()
    q = torch.randint(-1, 2, (N, K), dtype=torch.int8, device="cuda", generator=gen)
    lin.load_quantized(q, torch.rand(N, device="cuda", generator=gen) + 0.5,
                       ((torch.rand(N, device="cuda", generator=gen) - 0.5)).half())
    op32 = bitblas.Matmul(bitblas.MatmulConfig(N=N, K=K, A_dtype="int8", W_dtype="int2", accum_dtype="int32", out_dtype="int32"),
                          enable_tuning=False)
    return lin, op32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(f"{n}x{k}" for n, k in SHAPES))
    ap.add_argument("--rows", default=",".join(map(str, ROWS)))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bitnet_bench measures on the GPU"
    print(card())
    gen = torch.Generator(device="cuda").manual_seed(0)
    results = []
    for shape in a.shapes.split(","):
        N, K = map(int, shape.split("x"))
        lin, op32 = build(N, K, gen)
        op = lin.bitblas_matmul
        print(f"\n{N}x{K}  (us per call, median of {a.reps}; launches = library launches per call)")
        print(f"{'m':>5} | {'variant':>7} | {'eager us':>9} | {'graph us':>9} | {'launches':>8}")
        for m in map(int, a.rows.split(",")):
            x = torch.randn((m, K), device="cuda", generator=gen).half()
            out = torch.empty((m, N), dtype=torch.float16, device="cuda")
            acc = torch.empty((m, N), dtype=torch.int32, device="cuda")
            q, s = bitblas.quantize_act_int8(x)

            def glue():
                xf = x.float()
                sa = 127.0 / xf.abs().amax(-1, keepdim=True).clamp(min=1e-5)
                qa = (xf * sa).round().clamp(-128, 127).to(torch.int8)
                y = op32.forward(qa, lin.qweight)
                return (y.float() / sa / lin.weight_scale).half() + lin.bias

            calls = {
                "layer": lambda: lin(x, output=out),
                "glue": glue,
                "floor": lambda: op32.forward(q, lin.qweight, output=acc),
                "scaled": lambda: op.forward_scaled(q, lin.qweight, s, lin.weight_scale, lin.bias, output=out),
            }
            for f in calls.values():   # warm-up: workspaces, kernel attributes
                f()
            torch.cuda.synchronize()
            assert torch.equal(lin(x), glue()), "layer and glue disagree"
            eager = {v: [] for v in calls}
            graph = {v: [] for v in calls}
            tq = []
            quant = lambda: bitblas.quantize_act_int8(x, q=q, scale=s)   # noqa: E731
            for _ in range(a.reps):
                for v, f in calls.items():
                    eager[v].append(events_us(f, a.iters))
                for v, f in calls.items():
                    graph[v].append(graph_us(f, a.iters))
                tq.append(events_us(quant, a.iters))
            row = dict(N=N, K=K, m=m, kernel=op.kernel_for(m))
            for v, f in calls.items():
                e, g = statistics.median(eager[v]), statistics.median(graph[v])
                n = launches(f)
                row[v] = dict(eager_us=e, graph_us=g, launches=n)
                print(f"{m:>5} | {v:>7} | {e:9.1f} | {g:9.1f} | {n:8d}")
            t = statistics.median(tq)
            row["quant_us"], row["quant_gbs"] = t, (m * K * 3 + 4 * m) / (t * 1e-6) / 1e9
            print(f"{m:>5} | layer/glue {row['layer']['eager_us'] / row['glue']['eager_us']:.3f}x eager, "
                  f"{row['layer']['graph_us'] / row['glue']['graph_us']:.3f}x graph; scaled/floor "
                  f"{row['scaled']['eager_us'] / row['floor']['eager_us']:.3f}x; quantization {t:.1f} us = {row['quant_gbs']:.0f} GB/s; "
                  f"kernel {row['kernel']}")
            results.append(row)
            del x, out, acc, q, s
        del lin, op32
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
