"""FP8Linear (128 x 128 block-scaled e4m3 weight, activations quantized on the device) against bf16 F.linear on the dequantized
weight (cuBLAS), the W4A16 Linear (uint4, g = 128, fp16 activations) and torch._scaled_mm with row-wise scales, at the
Llama-2-70B and DeepSeek-V3 dense linear shapes.

Every variant is captured in a CUDA graph and timed with CUDA events over replays; the variants alternate within each round and
the median over rounds is reported.  Every shape is warmed up first.  Columns (microseconds per call):
  fp8      FP8Linear: quantize_act_fp8 + forward_fp8 (2 launches, 3 with split-K)
  mm       forward_fp8 alone on already quantized activations, with TFLOP/s = 2 m N K / time and, at m <= 16, the weight bytes
           over that time in GB/s and as a share of the 3.35 TB/s data-sheet HBM3 rate
  bf16     F.linear(x, w_dequantized) in bfloat16
  w4a16    the W4A16 Linear on the same shape (its matmul)
  scaled   torch._scaled_mm, e4m3 x e4m3 with one scale per row of A and of W, bf16 out (reference only: it does less work and
           scales more coarsely; m is padded to 16 where it is smaller, as the call needs)
The card's name, power limit and maximum SM clock are printed first.

    python tools/fp8_bench.py [--ms 1,4,16,128,512,1024,4096] [--shapes 70b,dsv3] [--rounds 3] [--json PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bitblas  # noqa: E402
from bitblas_b200 import _lib  # noqa: E402
from bitblas_b200.fp8 import quantize_act_fp8  # noqa: E402

SHAPES = {"70b": [("qkv", 10240, 8192), ("o", 8192, 8192), ("gate_up", 57344, 8192), ("down", 8192, 28672)],
          "dsv3": [("q_a", 1536, 7168), ("q_b", 24576, 1536), ("kv_a", 576, 7168), ("kv_b", 32768, 512), ("o", 7168, 16384),
                   ("gate_up", 18432, 7168), ("down", 7168, 18432)]}
HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


class Timer:
    """one variant captured once as `iters` back-to-back calls; each measure() is one replay timed with CUDA events"""

    def __init__(self, fn, iters):
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            fn()
            fn()
        torch.cuda.current_stream().wait_stream(st)
        self.g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g):
            for _ in range(iters):
                fn()
        self.iters = iters
        self.g.replay()   # warm
        torch.cuda.synchronize()

    def measure(self):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        self.g.replay()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) * 1e3 / self.iters


class GPTQ:
    """a random GPTQ v1 checkpoint module: qweight int32 [K/8, N], qzeros int32 [K/g, N/8], scales fp16 [K/g, N]"""

    def __init__(self, K, N, g, seed):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.qweight = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // 8, N), generator=gen, device="cuda", dtype=torch.int32)
        self.qzeros = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // g, N // 8), generator=gen, device="cuda", dtype=torch.int32)
        self.scales = (torch.rand(K // g, N, generator=gen, device="cuda") * 0.01 + 1e-3).half()
        self.bias = None


def launches(fn):
    lib = _lib.load()
    n0 = lib.bb_launch_count()
    fn()
    return int(lib.bb_launch_count() - n0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", default="1,4,16,128,512,1024,4096")
    ap.add_argument("--shapes", default="70b,dsv3")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench needs a GPU")
    print(f"card: {card()}  (name, power limit, max SM clock)", flush=True)
    print(f"{'model':>5} {'layer':>7} {'N':>6} {'K':>6} {'m':>5} | {'fp8':>8} {'mm':>8} {'TFLOP/s':>7} {'GB/s':>6} {'HBM%':>5} | "
          f"{'bf16':>8} {'w4a16':>8} {'scaled':>8} | {'vs bf16':>7} {'vs w4a16':>8} | launches", flush=True)
    rows = []
    for model in a.shapes.split(","):
        for name, N, K in SHAPES[model]:
            torch.manual_seed(N + K)
            w = torch.randn(N, K, device="cuda") * 0.02
            lin = bitblas.FP8Linear(K, N).cuda()
            lin.load_float_weight(w)
            wdq = (lin.weight.float() * lin.weight_scale_inv.repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)).bfloat16()
            del w
            mod = GPTQ(K, N, 128, seed=N + K)
            a16 = bitblas.Linear(K, N, A_dtype="float16", W_dtype="uint4", accum_dtype="float32", out_dtype="float16",
                                 group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized",
                                 enable_tuning=False).cuda()
            a16.repack_from_gptq(mod)
            del mod
            wq_row = (wdq.float().abs().amax(1, keepdim=True).clamp(min=1e-10) / 448.0)
            w_rowq = (wdq.float() / wq_row).clamp(-448, 448).to(torch.float8_e4m3fn)
            for m in [int(v) for v in a.ms.split(",")]:
                x = torch.randn(m, K, device="cuda").bfloat16()
                xh = x.half()
                out = torch.empty(m, N, device="cuda", dtype=torch.bfloat16)
                out16 = torch.empty(m, N, device="cuda", dtype=torch.float16)
                q, s = quantize_act_fp8(x)
                mp = max(m, 16)
                xq = torch.zeros(mp, K, device="cuda", dtype=torch.float8_e4m3fn)
                xq[:m] = x.float().clamp(-448, 448).to(torch.float8_e4m3fn)
                sa = torch.ones(mp, 1, device="cuda")
                sb = wq_row.t().contiguous()
                fns = {
                    "fp8": lambda: lin(x, out),
                    "mm": lambda: lin.bitblas_matmul.forward_fp8(q, lin.weight, s, lin.weight_scale_inv, None, out),
                    "bf16": lambda: F.linear(x, wdq),
                    "w4a16": lambda: a16(xh, out16),
                    "scaled": lambda: torch._scaled_mm(xq, w_rowq.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16),
                }
                est = max(2.0 * m * N * K / 500e12, N * K * 2 / 2.5e12) * 1e6   # a rough µs per call, to size the graphs
                iters = max(3, min(200, int(4000 / est)))
                timers = {}
                for k, fn in fns.items():
                    try:
                        timers[k] = Timer(fn, iters)
                    except Exception as e:   # (torch._scaled_mm's support differs between builds; it is reference only)
                        print(f"  {k}: not measured ({type(e).__name__}: {str(e).splitlines()[0][:80]})")
                res = {k: [] for k in timers}
                for _ in range(a.rounds):   # the variants alternate
                    for k, t in timers.items():
                        res[k].append(t.measure())
                med = {k: statistics.median(v) for k, v in res.items()}
                del timers
                flops = 2.0 * m * N * K
                gbs = N * K / (med["mm"] * 1e-6) / 1e9
                row = dict(model=model, layer=name, N=N, K=K, m=m, iters=iters, **{f"{k}_us": v for k, v in med.items()},
                           mm_tflops=flops / med["mm"] / 1e6, mm_weight_gbs=gbs if m <= 16 else None,
                           launches_fp8=launches(fns["fp8"]))
                rows.append(row)
                fmt = lambda k: f"{med[k]:>8.1f}" if k in med else f"{'n/a':>8}"   # noqa: E731
                hbm = f"{gbs:>6.0f} {100 * gbs / 1e3 / HBM_TBS:>4.0f}%" if m <= 16 else f"{'':>6} {'':>5}"
                print(f"{model:>5} {name:>7} {N:>6} {K:>6} {m:>5} | {fmt('fp8')} {fmt('mm')} {row['mm_tflops']:>7.0f} {hbm} | "
                      f"{fmt('bf16')} {fmt('w4a16')} {fmt('scaled')} | {med['bf16'] / med['fp8']:>6.2f}x "
                      f"{med['w4a16'] / med['fp8']:>7.2f}x | {row['launches_fp8']}", flush=True)
                del x, xh, out, out16, q, s, xq
            del lin, wdq, a16, w_rowq
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
