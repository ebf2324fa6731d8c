"""W4A8Linear (int8 activations, quantized on the device) against the W4A16 Linear built from the same GPTQ checkpoint (uint4,
g = 128, quantized zero points), at the Llama-2-70B and Llama-3-8B linear shapes.

For each (shape, m) both layers run eagerly and replayed from a CUDA graph, the variants alternated over several rounds; the
median over rounds is reported.  Columns: microseconds per layer call, the matmul's own time (replayed: W4A8's forward_w4a8 on
already quantized activations, with its split-K reduce when it splits; W4A16's Linear call, which is its matmul), TOPS =
2 m N K / (that matmul time), the quantization launch's share of the W4A8 layer call (its own replayed time over the call's),
and library launches per call.  The card's name, power limit and
maximum SM clock are printed first: a number is only worth something with them.

    python tools/w4a8_bench.py [--ms 1,4,16,128,512,1024,4096] [--shapes 70b,8b] [--iters 50] [--rounds 5] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bitblas  # noqa: E402
from bitblas_b200 import _lib  # noqa: E402

SHAPES = {"70b": [("qkv", 10240, 8192), ("o", 8192, 8192), ("gate_up", 57344, 8192), ("down", 8192, 28672)],
          "8b": [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336)]}


class GPTQ:
    """a random GPTQ v1 checkpoint module: qweight int32 [K/8, N], qzeros int32 [K/g, N/8] (z - 1), scales fp16 [K/g, N]"""

    def __init__(self, K, N, g, seed):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // 8, N), generator=gen, device="cuda", dtype=torch.int32)
        self.qzeros = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // g, N // 8), generator=gen, device="cuda", dtype=torch.int32)
        self.scales = (torch.rand(K // g, N, generator=gen, device="cuda") * 0.01 + 1e-3).half()
        self.bias = None


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def time_eager(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def time_graph(fn, iters):
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        fn()
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    g.replay()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def launches(fn):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    fn()
    return int(lib.bb_launch_count() - n0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", default="1,4,16,128,512,1024,4096")
    ap.add_argument("--shapes", default="70b,8b")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("w4a8_bench needs a GPU")
    print(f"card: {card()}  (name, power limit, max SM clock)")
    rows = []
    hdr = (f"{'model':>4} {'layer':>7} {'N':>6} {'K':>6} {'m':>5} | {'W4A8 us':>9} {'W4A16 us':>9} {'speedup':>7} | "
           f"{'graph W4A8':>10} {'graph W4A16':>11} {'speedup':>7} | {'mm W4A8':>8} {'TOPS a8':>7} {'TOPS a16':>8} {'quant %':>7} | "
           "launches")
    print(hdr)
    for model in a.shapes.split(","):
        for name, N, K in SHAPES[model]:
            mod = GPTQ(K, N, 128, seed=N + K)
            a8 = bitblas.W4A8Linear(K, N).cuda()
            a8.repack_from_gptq(mod)
            a16 = bitblas.Linear(K, N, A_dtype="float16", W_dtype="uint4", accum_dtype="float32", out_dtype="float16",
                                 group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized",
                                 enable_tuning=False).cuda()
            a16.repack_from_gptq(mod)
            for m in [int(v) for v in a.ms.split(",")]:
                x = torch.randn(m, K, device="cuda", dtype=torch.float16)
                out8 = torch.empty(m, N, device="cuda", dtype=torch.float16)
                out16 = torch.empty_like(out8)
                f8 = lambda: a8(x, out8)   # noqa: E731
                f16 = lambda: a16(x, out16)   # noqa: E731
                q = torch.empty(m, K, device="cuda", dtype=torch.int8)
                s = torch.empty(m, device="cuda", dtype=torch.float32)
                fq = lambda: bitblas.quantize_act_int8(x, q, s)   # noqa: E731
                fm = lambda: a8.bitblas_matmul.forward_w4a8(q, a8.qweight, s, a8.scales, a8.zeros, None, out8)   # noqa: E731
                for f in (f8, f16, fq, fm):
                    f()
                torch.cuda.synchronize()
                it = max(3, min(a.iters, int(a.iters * 4096 * 8192 / (m * N * K / 64 + 1)) or 3))
                res = {k: [] for k in ("e8", "e16", "g8", "g16", "gq", "gm")}
                for _ in range(a.rounds):   # the variants alternate
                    res["e8"].append(time_eager(f8, it))
                    res["e16"].append(time_eager(f16, it))
                    res["g8"].append(time_graph(f8, it))
                    res["g16"].append(time_graph(f16, it))
                    res["gq"].append(time_graph(fq, it))
                    res["gm"].append(time_graph(fm, it))
                med = {k: statistics.median(v) for k, v in res.items()}
                ops = 2.0 * m * N * K
                row = dict(model=model, layer=name, N=N, K=K, m=m, eager_w4a8_us=med["e8"], eager_w4a16_us=med["e16"],
                           graph_w4a8_us=med["g8"], graph_w4a16_us=med["g16"], quant_us=med["gq"], matmul_w4a8_us=med["gm"],
                           tops_w4a8=ops / med["gm"] / 1e6, tops_w4a16=ops / med["g16"] / 1e6,
                           quant_share=med["gq"] / med["g8"], launches_w4a8=launches(f8), launches_w4a16=launches(f16),
                           kernel_w4a8=a8.bitblas_matmul.kernel_for_w4a8(m), kernel_w4a16=a16.bitblas_matmul.kernel_for(m))
                rows.append(row)
                print(f"{model:>4} {name:>7} {N:>6} {K:>6} {m:>5} | {med['e8']:>9.1f} {med['e16']:>9.1f} "
                      f"{med['e16'] / med['e8']:>6.2f}x | {med['g8']:>10.1f} {med['g16']:>11.1f} {med['g16'] / med['g8']:>6.2f}x | "
                      f"{med['gm']:>8.1f} {row['tops_w4a8']:>7.1f} {row['tops_w4a16']:>8.1f} {100 * row['quant_share']:>6.1f}% | "
                      f"{row['launches_w4a8']} / {row['launches_w4a16']}  {row['kernel_w4a8']} / {row['kernel_w4a16']}", flush=True)
            del a8, a16, mod
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
