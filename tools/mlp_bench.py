"""Dense SwiGLU MLP: SwiGLUMLP (forward_swiglu, then down: 2 launches) against the two ways integrations run it today.

    python tools/mlp_bench.py [--iters 20] [--reps 3] [--json PATH]

Variants, on the same weights (uint4, group 128, quantized zeros, fp16 activations):
  fused    SwiGLUMLP: bb_matmul_swiglu forms silu(gate) * up in the gate/up kernel's epilogue, then the down projection
  merged   one gate/up Linear of 2I rows (the [m, 2I] output goes to memory), torch silu(g) * u, then down (vLLM's SiluAndMul)
  split    gate, up and down as three Linears, torch silu(g) * u
Shapes: Llama-2-70B (H 8192, I 28672) and Llama-3-8B (H 4096, I 14336) at m in {1, 4, 16, 128, 1024, 4096}.  Each variant is timed
eager (CUDA events around --iters calls) and as a CapturedStep replay (--iters calls captured in one CUDA graph), the variants
alternated inside every repetition; the table gives the median over --reps.  Also per point: library launches (torch's elementwise
kernels are not counted), the peak memory one call allocates beyond its inputs, and forward_swiglu alone against Matmul.forward on
the same gate/up weights, which isolates what the epilogue costs.  The Llama-3-8B gate/up weight (59 MB) is close to the 50 MB L2,
so its m = 1 times are partly L2 reads; the 70B weights are not.  The card's name, power limit and maximum SM clock are printed
with the results.
"""
from __future__ import annotations

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

CFG = dict(A_dtype="float16", W_dtype="uint4", out_dtype="float16", accum_dtype="float32", group_size=128, with_scaling=True,
           with_zeros=True, zeros_mode="quantized", opt_M=[1, 4, 16, 128, 1024, 4096])
MODELS = {"llama-2-70b": (8192, 28672), "llama-3-8b": (4096, 14336)}
ROWS = [1, 4, 16, 128, 1024, 4096]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        q = q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{torch.cuda.get_device_name()} (power.limit, clocks.max.sm: {q})"


def random_linear(lin, gen):
    """random stored buffers (the timing does not depend on the values; scales keep the outputs finite)"""
    lin.qweight = torch.randint(-128, 128, lin.qweight.shape, dtype=torch.int8, device="cuda", generator=gen)
    lin.scales = (torch.rand(lin.scales.shape, device="cuda", generator=gen) * 2e-3).half()
    lin.zeros = torch.randint(-128, 128, lin.zeros.shape, dtype=torch.int8, device="cuda", generator=gen)


def build(H, I, gen):
    mlp = bitblas.SwiGLUMLP(H, I, **CFG).cuda()
    random_linear(mlp.gate_up, gen)
    random_linear(mlp.down, gen)
    merged = bitblas.Linear(H, 2 * I, **CFG).cuda()   # the same buffers: only the layout's meaning differs
    merged.qweight, merged.scales, merged.zeros = mlp.gate_up.qweight, mlp.gate_up.scales, mlp.gate_up.zeros
    gate, up = bitblas.Linear(H, I, **CFG).cuda(), bitblas.Linear(H, I, **CFG).cuda()
    gate.qweight, up.qweight = (t.contiguous() for t in mlp.gate_up.qweight.chunk(2))
    gate.scales, up.scales = (t.contiguous() for t in mlp.gate_up.scales.chunk(2))
    gate.zeros, up.zeros = (t.contiguous() for t in mlp.gate_up.zeros.chunk(2, dim=1))
    down = mlp.down

    def fused(x, out):
        return mlp(x, output=out)

    def merged_fn(x, out):
        y = merged(x)
        return down(torch.nn.functional.silu(y[:, :I]) * y[:, I:], output=out)

    def split(x, out):
        return down(torch.nn.functional.silu(gate(x)) * up(x), output=out)

    return mlp, {"fused": fused, "merged": merged_fn, "split": split}


def events_us(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1e3


def graph_us(fn, iters):
    step = bitblas.CapturedStep(lambda: [fn() for _ in range(iters)], warmup=1)
    step()
    with torch.cuda.stream(step.stream):   # the replays run on the step's stream: time them there
        return events_us(step.graph.replay, 3) / iters


def launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    fn()
    torch.cuda.synchronize()
    return lib.bb_launch_count() - n0


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--rows", default=",".join(map(str, ROWS)))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "mlp_bench measures on the GPU"
    print(card())
    gen = torch.Generator(device="cuda").manual_seed(0)
    results = []
    for name in a.models.split(","):
        H, I = MODELS[name]
        mlp, variants = build(H, I, gen)
        gu = mlp.gate_up
        op = gu.bitblas_matmul
        print(f"\n{name}: H={H} I={I}  (us per MLP call, median of {a.reps}; launches = library launches; peak = MB one call "
              f"allocates)")
        print(f"{'m':>5} | {'variant':>7} | {'eager us':>9} | {'graph us':>9} | {'launches':>8} | {'peak MB':>8}")
        for m in map(int, a.rows.split(",")):
            x = (torch.rand((m, H), device="cuda", generator=gen) - 0.5).half()
            out = torch.empty((m, H), dtype=torch.float16, device="cuda")
            calls = {v: (lambda f=f: f(x, out)) for v, f in variants.items()}
            for f in calls.values():   # warm-up: workspaces, kernel attributes
                f()
            torch.cuda.synchronize()
            eager = {v: [] for v in calls}
            graph = {v: [] for v in calls}
            for _ in range(a.reps):
                for v, f in calls.items():
                    eager[v].append(events_us(f, a.iters))
                for v, f in calls.items():
                    graph[v].append(graph_us(f, a.iters))
            row = dict(model=name, m=m)
            for v, f in calls.items():
                e, g = statistics.median(eager[v]), statistics.median(graph[v])
                n, p = launches(f), peak_mb(f)
                row[v] = dict(eager_us=e, graph_us=g, launches=n, peak_mb=p)
                print(f"{m:>5} | {v:>7} | {e:9.1f} | {g:9.1f} | {n:8d} | {p:8.1f}")
            # the epilogue alone: forward_swiglu against the plain gate/up matmul on the same weights
            h = torch.empty((m, I), dtype=torch.float16, device="cuda")
            pre = torch.empty((m, 2 * I), dtype=torch.float16, device="cuda")
            sw = lambda: op.forward_swiglu(x, gu.qweight, gu.scales, gu.zeros, output=h)   # noqa: E731
            pl = lambda: op.forward(x, gu.qweight, gu.scales, gu.zeros, output=pre)   # noqa: E731
            t_sw, t_pl = [], []
            for _ in range(a.reps):
                t_sw.append(events_us(sw, a.iters))
                t_pl.append(events_us(pl, a.iters))
            row["forward_swiglu_us"], row["forward_us"] = statistics.median(t_sw), statistics.median(t_pl)
            print(f"{m:>5} | gate/up alone: forward_swiglu {row['forward_swiglu_us']:.1f} us, forward {row['forward_us']:.1f} us "
                  f"({row['forward_swiglu_us'] / row['forward_us']:.3f}x), kernel {op.kernel_for(m)}")
            results.append(row)
            del x, out, h, pre
        del mlp, variants
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
