"""Block-scaled FP8 mixture-of-experts expert blocks: FP8MoEExperts against what a caller can run without it.

    python tools/fp8_moe_bench.py [--models deepseek-v3,qwen3-235b-a22b,qwen3-30b-a3b] [--tokens 1,4,16,128,512,2048]
                                  [--rounds 7] [--reps 3] [--out PATH]

Shapes (every expert a 128 x 128 block-scaled e4m3 gate, up and down projection, bfloat16 activations):
    DeepSeek-V3      E=256, top-8, H=7168, I=2048
    Qwen3-235B-A22B  E=128, top-8, H=4096, I=1536
    Qwen3-30B-A3B    E=128, top-8, H=2048, I=768
Columns, each one expert block from router output (top-k ids and weights) to the [T, H] layer output:
    (a) fp8      FP8MoEExperts.forward: six library launches, replayed from a CUDA graph
    (b) bf16     library routing and combine around torch._grouped_mm for gate/up and down on the dequantized bfloat16 weights,
                 torch silu * mul, replayed from a CUDA graph
    (c) w4a16    MoEExperts with uint4 g128 quantized-zero weights on the same shapes (for information), replayed
    (d) loop     the per-expert FP8Linear path a caller has without the grouped GEMM: moe_route, offsets read on the host, then
                 per active expert quantize_act_fp8 + forward_fp8 for gate and up, torch silu * mul, quantize_act_fp8 + forward_fp8
                 for down, then moe_combine; eager (it synchronises, so it cannot be captured)
and the grouped FP8 GEMMs alone (gate/up with SwiGLU, and down, replayed on pre-quantized inputs): at T <= 16 the weight-stream
rate over the active experts' bytes as a share of 3.35 TB/s, at T >= 512 the TFLOP/s as a share of 1,979 (the H100 SXM data
sheet's HBM3 bandwidth and dense FP8 rate), and the two quantize launches' share of the replayed block.
Method: every timed window cycles through 16 seeded routings (so the active experts' weights do not stay in the 50 MB L2); a CUDA
graph holds one call per routing; the variants are replayed alternately, `reps` graph replays each per round, and the median over
`rounds` rounds is reported in microseconds per block.  The card's name, power limit and maximum SM clock are printed first.
"""
from __future__ import annotations

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
from bitblas_b200.fp8 import quantize_act_fp8  # noqa: E402
from bitblas_b200.moe import deinterleave_gate_up, moe_combine, moe_route  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP8_FLOPS = 1979e12
MODELS = {"deepseek-v3": dict(E=256, k=8, H=7168, I=2048), "qwen3-235b-a22b": dict(E=128, k=8, H=4096, I=1536),
          "qwen3-30b-a3b": dict(E=128, k=8, H=2048, I=768)}
N_ROUTINGS = 16
W4A16 = dict(A_dtype="bfloat16", out_dtype="bfloat16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True,
             zeros_mode="quantized")
E4M3 = torch.float8_e4m3fn


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        q = q[1 + torch.cuda.current_device()] if len(q) > 1 else "unknown"
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{torch.cuda.get_device_name()} (name, power.limit, clocks.max.sm: {q})"


class Blocks:
    """one model's expert weights, held once per variant: FP8MoEExperts (random e4m3 bytes and block scales), the bfloat16
    dequantized gate|up and down stacks, the de-interleaved e4m3 gate and up for the loop, and a W4A16 MoEExperts"""

    def __init__(self, E, H, I, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.E, self.H, self.I = E, H, I
        with torch.device("cuda"):
            self.fp8 = bitblas.FP8MoEExperts(E, H, I)
        m = self.fp8
        for e in range(E):   # |w| * scale ~ 0.02: e4m3 values of N(0, 64) clamped, scales 2^-12 .. 2^-11
            for buf in (m.gate_up_weight, m.down_weight):
                buf[e].copy_((torch.randn(buf.shape[1:], device="cuda", generator=g) * 64).clamp(-448, 448).to(E4M3))
        for buf in (m.gate_up_weight_scale_inv, m.down_weight_scale_inv):
            buf.copy_((torch.rand(buf.shape, device="cuda", generator=g) + 1) * 2.0 ** -12)
        u8 = torch.uint8
        gw, uw = deinterleave_gate_up(m.gate_up_weight.view(u8), "weight")
        gs, us = deinterleave_gate_up(m.gate_up_weight_scale_inv, "block_scale")
        self.gate, self.up = gw.view(E4M3), uw.view(E4M3)
        self.gate_s, self.up_s = gs, us

        def deq(q, s):
            return (q.float() * s.repeat_interleave(128, 0).repeat_interleave(128, 1)).to(torch.bfloat16)
        # (b): gate rows then up rows, [E, 2I, H], and down [E, H, I], bfloat16, filled expert by expert
        self.bf16_gate_up = torch.empty(E, 2 * I, H, dtype=torch.bfloat16, device="cuda")
        self.bf16_down = torch.empty(E, H, I, dtype=torch.bfloat16, device="cuda")
        for e in range(E):
            self.bf16_gate_up[e, :I] = deq(self.gate[e], gs[e])
            self.bf16_gate_up[e, I:] = deq(self.up[e], us[e])
            self.bf16_down[e] = deq(m.down_weight[e], m.down_weight_scale_inv[e])
        op = bitblas.Matmul
        cfg = dict(A_dtype="e4m3_float8", W_dtype="e4m3_float8", accum_dtype="float32", out_dtype="bfloat16")
        self.gate_op = op(bitblas.MatmulConfig(N=I, K=H, **cfg), enable_tuning=False)
        self.down_op = op(bitblas.MatmulConfig(N=H, K=I, **cfg), enable_tuning=False)
        with torch.device("cuda"):
            self.w4 = bitblas.MoEExperts(E, H, I, **W4A16).cuda()
        for gl in (self.w4.gate_up, self.w4.down):
            N, K = gl.out_features, gl.in_features
            G = K // 128
            gl.qweight = torch.randint(-128, 128, (E, N, K // 2), dtype=torch.int8, device="cuda", generator=g)
            gl.scales = (torch.rand((E, N, G), device="cuda", generator=g) * 0.01).to(torch.bfloat16)
            gl.zeros = torch.randint(-128, 128, (E, G, N // 2), dtype=torch.int8, device="cuda", generator=g)

    def bf16_block(self, x, ids, w, out):
        offsets, slot_rows, xs = moe_route(ids, x, self.E)
        offs = offsets[1:]
        h = torch._grouped_mm(xs, self.bf16_gate_up.transpose(-2, -1), offs=offs)
        a = F.silu(h[:, :self.I]) * h[:, self.I:]
        y = torch._grouped_mm(a, self.bf16_down.transpose(-2, -1), offs=offs)
        return moe_combine(y, slot_rows, w, out)

    def loop_block(self, x, ids, w, out):
        offsets, slot_rows, xs = moe_route(ids, x, self.E)
        off = offsets.cpu().tolist()
        y = torch.empty(xs.shape[0], self.H, dtype=x.dtype, device="cuda")
        for e in range(self.E):
            r0, r1 = off[e], off[e + 1]
            if r1 == r0:
                continue
            q, s = quantize_act_fp8(xs[r0:r1])
            g = self.gate_op.forward_fp8(q, self.gate[e], s, self.gate_s[e])
            u = self.gate_op.forward_fp8(q, self.up[e], s, self.up_s[e])
            q, s = quantize_act_fp8(F.silu(g) * u)
            self.down_op.forward_fp8(q, self.fp8.down_weight[e], s, self.fp8.down_weight_scale_inv[e], output=y[r0:r1])
        return moe_combine(y, slot_rows, w, out)


def routings(E, k, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(N_ROUTINGS):
        ids = torch.rand((T, E), device="cuda", generator=g).argsort(dim=1)[:, :k].to(torch.int32).contiguous()
        w = torch.softmax(torch.randn((T, k), device="cuda", generator=g), dim=1)
        out.append((ids, w))
    return out


def graph_of(fn):
    """a CUDA graph holding fn(0) .. fn(N_ROUTINGS - 1)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(N_ROUTINGS):
            fn(i)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(N_ROUTINGS):
            fn(i)
    return graph


def timed(run, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        run()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / (reps * N_ROUTINGS)   # us per block


def measure(variants, rounds, reps):
    """variants: name -> (run, reps multiplier); alternated within each round; median us per block"""
    for run, _ in variants.values():
        run()
    torch.cuda.synchronize()
    times = {name: [] for name in variants}
    for _ in range(rounds):
        for name, (run, mult) in variants.items():
            times[name].append(timed(run, max(1, reps * mult)))
    return {name: statistics.median(t) for name, t in times.items()}


def point(b, k, T, rounds, reps):
    E, H, I = b.E, b.H, b.I
    routes = routings(E, k, T, seed=T + E)
    x = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    x16 = x.clone()

    # the grouped GEMMs alone on each routing's pre-quantized inputs
    pre = []
    for ids, _ in routes:
        offsets, _, xs = moe_route(ids, x, E)
        q, s = quantize_act_fp8(xs)
        h = b.fp8.gate_up_matmul.forward_grouped_fp8_swiglu(q, b.fp8.gate_up_weight, offsets, s, b.fp8.gate_up_weight_scale_inv)
        qh, sh = quantize_act_fp8(h)
        pre.append((offsets, q, s, h, qh, sh, xs))
    y_buf = torch.empty(T * k, H, dtype=torch.bfloat16, device="cuda")

    def gate_up_only(i):
        offsets, q, s, h, _, _, _ = pre[i]
        b.fp8.gate_up_matmul.forward_grouped_fp8_swiglu(q, b.fp8.gate_up_weight, offsets, s, b.fp8.gate_up_weight_scale_inv,
                                                        output=h)

    def down_only(i):
        offsets, _, _, _, qh, sh, _ = pre[i]
        b.fp8.down_matmul.forward_grouped_fp8(qh, b.fp8.down_weight, offsets, sh, b.fp8.down_weight_scale_inv, output=y_buf)

    def quant_only(i):
        _, _, _, h, _, _, xs = pre[i]
        quantize_act_fp8(xs)
        quantize_act_fp8(h)

    graphs = {
        "fp8": graph_of(lambda i: b.fp8(x, *routes[i], output=out)),
        "bf16": graph_of(lambda i: b.bf16_block(x, *routes[i], out)),
        "w4a16": graph_of(lambda i: b.w4(x16, *routes[i], output=out)),
        "gemm_gate_up": graph_of(gate_up_only),
        "gemm_down": graph_of(down_only),
        "quantize": graph_of(quant_only),
    }
    variants = {name: (g.replay, 1) for name, g in graphs.items()}
    variants["loop"] = (lambda: [b.loop_block(x, *routes[i], out) for i in range(N_ROUTINGS)], 0)
    t = measure(variants, rounds, reps)

    # bytes and FLOP of the grouped GEMMs, averaged over the routings
    active = [int((torch.bincount(ids.reshape(-1).long(), minlength=E) > 0).sum()) for ids, _ in routes]
    act = statistics.mean(active)
    gu_bytes = act * (2 * I * H + 2 * (I // 128) * (H // 128) * 4)
    dn_bytes = act * (H * I + (H // 128) * (I // 128) * 4)
    flop_gu, flop_dn = 2.0 * T * k * 2 * I * H, 2.0 * T * k * H * I
    res = dict(T=T, active_experts=round(act, 1), us={n: round(v, 2) for n, v in t.items()},
               fp8_vs_bf16=round(t["bf16"] / t["fp8"], 3), fp8_vs_w4a16=round(t["w4a16"] / t["fp8"], 3),
               fp8_vs_loop=round(t["loop"] / t["fp8"], 2), quantize_share=round(t["quantize"] / t["fp8"], 3))
    if T <= 16:
        for name, nbytes in (("gemm_gate_up", gu_bytes), ("gemm_down", dn_bytes)):
            res[f"{name}_TBps"] = round(nbytes / t[name] * 1e-6, 3)
            res[f"{name}_hbm_share"] = round(nbytes / t[name] * 1e6 / HBM_BYTES_PER_S, 3)
    if T >= 512:
        for name, flop in (("gemm_gate_up", flop_gu), ("gemm_down", flop_dn)):
            res[f"{name}_TFLOPs"] = round(flop / t[name] * 1e-6, 1)
            res[f"{name}_fp8_share"] = round(flop / t[name] * 1e6 / FP8_FLOPS, 3)
    del graphs
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--tokens", default="1,4,16,128,512,2048")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_moe_bench needs a GPU")
    print(card(), flush=True)
    results = {"card": card(), "models": {}}
    for name in args.models.split(","):
        cfg = MODELS[name]
        b = Blocks(cfg["E"], cfg["H"], cfg["I"], seed=len(name))
        rows = []
        for T in [int(v) for v in args.tokens.split(",")]:
            r = point(b, cfg["k"], T, args.rounds, args.reps)
            print(json.dumps(dict(model=name, **r)), flush=True)
            rows.append(r)
        results["models"][name] = rows
        del b
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
