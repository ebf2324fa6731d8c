"""Mixture-of-experts projections: the grouped matmul (Matmul.forward_grouped, one launch) against what a caller does without it
(one bitblas.Linear per active expert, counts known on the host).

    python tools/moe_bench.py [--iters 200] [--sweep-only | --no-sweep] [--no-layer]

Expert shapes (uint4, group 128, quantized zeros, fp16), gate/up (fused) and down as separate cases:
    Mixtral-8x7B      E=8,   top-2, gate/up 28672 x 4096, down 4096 x 14336
    Qwen3-30B-A3B     E=128, top-8, gate/up  1536 x 2048, down 2048 x   768
    DeepSeek-V2-Lite  E=64,  top-6, gate/up  2816 x 2048, down 2048 x  1408
Routing: seeded uniform top-k per token.  Every timed window cycles through 16 routings, so successive calls mostly read other
experts' weights and the active weight set does not stay in the 50 MB L2.  Device time: CUDA events around `--iters` calls.
Bytes: the active experts' weights, scales and zeros, plus activations and outputs; FLOP: 2 T N K.  The sweep times, for every
shape up to a few thousand tokens, forward_grouped(capturable=True) (the grouped GEMV up to
GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP rows per expert, the grouped wgmma GEMM above it) against both sides of the default
forward_grouped: the single grouped GEMV launch and the per-group bb_matmul path.  The layer section times one prefill MoE layer
(device routing, gate/up, SiLU gating, down) eager and replayed from one CUDA graph.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bitblas_b200 as bitblas  # noqa: E402
from bitblas_b200 import _lib  # noqa: E402
from bitblas_b200.ops import general_matmul as GM  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
MODELS = {
    "mixtral-8x7b": dict(E=8, topk=2, gate_up=(28672, 4096), down=(4096, 14336)),
    "qwen3-30b-a3b": dict(E=128, topk=8, gate_up=(1536, 2048), down=(2048, 768)),
    "deepseek-v2-lite": dict(E=64, topk=6, gate_up=(2816, 2048), down=(2048, 1408)),
}
CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
N_ROUTINGS = 16
SWEEP_PATHS = ("capturable", "single", "per_group")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        q = q[1 + torch.cuda.current_device()] if len(q) > 1 else "unknown"
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{torch.cuda.get_device_name()} (power.limit, clocks.max.sm: {q})"


class Layer:
    """one projection of E experts: stacked buffers for the grouped call, per-expert Linear views of them for the loop"""

    def __init__(self, E, N, K, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.E, self.N, self.K = E, N, K
        self.gl = bitblas.GroupedLinear(E, K, N, **CFG)
        G = K // 128
        self.gl.qweight = torch.randint(-128, 128, (E, N, K // 2), dtype=torch.int8, device="cuda", generator=g)
        self.gl.scales = (torch.rand((E, N, G), device="cuda", generator=g) * 0.01).half()
        self.gl.zeros = torch.randint(-128, 128, (E, G, N // 2), dtype=torch.int8, device="cuda", generator=g)
        self.lins = []
        for e in range(E):
            lin = bitblas.Linear(K, N, **CFG)
            lin.qweight, lin.scales, lin.zeros = self.gl.qweight[e], self.gl.scales[e], self.gl.zeros[e]
            self.lins.append(lin)
        self.expert_bytes = N * K // 2 + N * G * 2 + G * N // 2

    def bytes(self, counts):
        active = sum(1 for c in counts if c)
        T = sum(counts)
        return active * self.expert_bytes + T * self.K * 2 + T * self.N * 2


def routings(E, topk, tokens, seed):
    """N_ROUTINGS seeded uniform top-k routings: (host counts, host offsets, device offsets)"""
    out = []
    g = torch.Generator().manual_seed(seed)
    for _ in range(N_ROUTINGS):
        ids = torch.rand((tokens, E), generator=g).argsort(dim=1)[:, :topk].reshape(-1)
        counts = torch.bincount(ids, minlength=E).tolist()
        offsets = [0]
        for c in counts:
            offsets.append(offsets[-1] + c)
        out.append((counts, offsets, torch.tensor(offsets, dtype=torch.int32, device="cuda")))
    return out


def time_calls(fn, iters):
    for i in range(min(iters, 2 * N_ROUTINGS)):
        fn(i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(iters):
        fn(i)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1e3   # us per call


def launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    fn(0)
    return lib.bb_launch_count() - n0


def point(layer, routes, iters, paths):
    T = sum(routes[0][0])
    A = (torch.rand((T, layer.K), device="cuda") - 0.5).half()
    C = torch.empty((T, layer.N), dtype=torch.float16, device="cuda")

    def grouped(i):
        layer.gl(A, routes[i % N_ROUTINGS][2], output=C)

    def capturable(i):
        layer.gl(A, routes[i % N_ROUTINGS][2], output=C, capturable=True)

    def loop(i):
        _, offs, _ = routes[i % N_ROUTINGS]
        for e, lin in enumerate(layer.lins):
            if offs[e + 1] > offs[e]:
                lin(A[offs[e]:offs[e + 1]], output=C[offs[e]:offs[e + 1]])

    def with_threshold(rows_per_group):   # one side of forward_grouped whatever the row count
        def fn(i):
            old = GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP
            GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = rows_per_group
            try:
                grouped(i)
            finally:
                GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = old
        return fn

    fns = dict(grouped=grouped, loop=loop, capturable=capturable, single=with_threshold(1 << 30), per_group=with_threshold(-1))
    nbytes = sum(layer.bytes(r[0]) for r in routes) / len(routes)
    flop = 2.0 * T * layer.N * layer.K
    res = dict(T=T, active=sum(1 for c in routes[0][0] if c), bytes=int(nbytes), flop=flop)
    for p in paths:
        us = time_calls(fns[p], iters)
        res[p] = dict(us=round(us, 2), TFLOPs=round(flop / us * 1e-6, 2), GBps=round(nbytes / us * 1e-3, 1),
                      hbm=round(nbytes / us * 1e6 / HBM_BYTES_PER_S, 3), launches=launches(fns[p]))
    return res


def moe_layer(name, tokens, iters):
    """one prefill MoE layer: routing on the device (top-k ids -> counts -> offsets, rows gathered by expert), gate/up, SiLU
    gating, down; eager (default forward_grouped, and capturable=True) and as one CapturedStep replay (capturable=True)"""
    m = MODELS[name]
    E, topk = m["E"], m["topk"]
    (N1, K1), (N2, K2) = m["gate_up"], m["down"]
    up, down = Layer(E, N1, K1, seed=3).gl, Layer(E, N2, K2, seed=4).gl
    g = torch.Generator(device="cuda").manual_seed(tokens)
    x = (torch.rand((tokens, K1), device="cuda", generator=g) - 0.5).half()
    ids = torch.rand((tokens, E), device="cuda", generator=g).argsort(dim=1)[:, :topk].reshape(-1)
    off = torch.zeros(E + 1, dtype=torch.int32, device="cuda")

    def fwd(capturable):
        counts = torch.zeros(E, dtype=torch.int64, device="cuda").scatter_add_(0, ids, torch.ones_like(ids))
        off[1:] = torch.cumsum(counts, 0).to(torch.int32)
        rows = x[torch.argsort(ids, stable=True) // topk]
        h = up(rows, off, capturable=capturable)
        a = torch.nn.functional.silu(h[:, :K2]) * h[:, K2:]
        return down(a.contiguous(), off, capturable=capturable)

    def host_time(run, sync):
        for _ in range(3):
            run()
        sync()
        t0 = time.perf_counter()
        for _ in range(iters):
            run()
        sync()
        return (time.perf_counter() - t0) / iters * 1e6

    ref = fwd(False).clone()
    step = bitblas.CapturedStep(lambda: fwd(True))
    step()
    res = dict(model=name, tokens=tokens, rows=tokens * topk,
               eager_default_us=host_time(lambda: fwd(False), torch.cuda.synchronize),
               eager_capturable_us=host_time(lambda: fwd(True), torch.cuda.synchronize),
               graph_us=host_time(step.run, step.wait))
    out = fwd(True)
    res["max_abs_diff_vs_default"] = float((out.float() - ref.float()).abs().max())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tokens", default="1,4,16,64")
    ap.add_argument("--sweep-tokens", default="1,2,4,8,16,32,64,128,256,512,1024,2048,4096")
    ap.add_argument("--sweep-only", action="store_true")
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--no-layer", action="store_true")
    ap.add_argument("--layer-tokens", default="512,2048")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "moe_bench measures on the GPU; there is no CPU fallback"
    print(f"# {card()}")
    print(f"# GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = {GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP}")
    results = []
    if not args.sweep_only:
        print(f"{'model':18s} {'proj':8s} {'tok':>5s} {'T':>6s} {'act':>4s} {'MB':>8s} | "
              f"{'grouped us':>10s} {'GB/s':>7s} {'HBM':>6s} {'L':>3s} | {'loop us':>9s} {'GB/s':>7s} {'HBM':>6s} {'L':>4s} | speedup | "
              f"{'capt us':>9s} {'TFLOP/s':>7s} {'GB/s':>7s} {'L':>2s}")
        for name, m in MODELS.items():
            for proj in ("gate_up", "down"):
                N, K = m[proj]
                layer = Layer(m["E"], N, K, seed=1)
                for tok in map(int, args.tokens.split(",")):
                    routes = routings(m["E"], m["topk"], tok, seed=tok)
                    r = point(layer, routes, args.iters, ("grouped", "loop", "capturable"))
                    r.update(model=name, proj=proj, tokens=tok)
                    results.append(r)
                    g, lp, cp = r["grouped"], r["loop"], r["capturable"]
                    print(f"{name:18s} {proj:8s} {tok:5d} {r['T']:6d} {r['active']:4d} {r['bytes'] / 1e6:8.2f} | "
                          f"{g['us']:10.2f} {g['GBps']:7.1f} {g['hbm']:6.3f} {g['launches']:3d} | "
                          f"{lp['us']:9.2f} {lp['GBps']:7.1f} {lp['hbm']:6.3f} {lp['launches']:4d} | {lp['us'] / g['us']:6.2f}x | "
                          f"{cp['us']:9.2f} {cp['TFLOPs']:7.2f} {cp['GBps']:7.1f} {cp['launches']:2d}", flush=True)
                del layer
                torch.cuda.empty_cache()
    if not args.no_sweep:
        print("\n# sweep: forward_grouped(capturable=True) vs the single grouped GEMV launch and one bb_matmul per non-empty group")
        print(f"{'model':18s} {'proj':8s} {'tok':>5s} {'T':>6s} {'rows/exp':>8s} | "
              + " | ".join(f"{p + ' us':>14s} {'TFLOP/s':>7s} {'GB/s':>7s} {'L':>3s}" for p in SWEEP_PATHS)
              + " | single/capt per_group/capt")
        for name, m in MODELS.items():
            for proj in ("gate_up", "down"):
                N, K = m[proj]
                layer = Layer(m["E"], N, K, seed=2)
                for tok in map(int, args.sweep_tokens.split(",")):
                    routes = routings(m["E"], m["topk"], tok, seed=tok)
                    iters = max(10, min(args.iters, 20000 // tok))
                    r = point(layer, routes, iters, SWEEP_PATHS)
                    r.update(model=name, proj=proj, tokens=tok, sweep=True)
                    results.append(r)
                    cp = r["capturable"]["us"]
                    print(f"{name:18s} {proj:8s} {tok:5d} {r['T']:6d} {r['T'] / max(1, r['active']):8.1f} | "
                          + " | ".join(f"{r[p]['us']:14.2f} {r[p]['TFLOPs']:7.2f} {r[p]['GBps']:7.1f} {r[p]['launches']:3d}"
                                       for p in SWEEP_PATHS)
                          + f" | {r['single']['us'] / cp:11.2f} {r['per_group']['us'] / cp:13.2f}", flush=True)
                del layer
                torch.cuda.empty_cache()
    if not args.no_layer:
        print("\n# one prefill MoE layer (device routing, gate/up, SiLU gating, down): eager vs one CUDA-graph replay")
        print(f"{'model':18s} {'tok':>5s} {'rows':>6s} | {'eager default us':>16s} {'eager capt us':>13s} {'graph us':>9s} | "
              f"max |graph - default|")
        for name in MODELS:
            for tok in map(int, args.layer_tokens.split(",")):
                r = moe_layer(name, tok, max(5, min(args.iters, 20000 // tok)))
                results.append(r)
                print(f"{name:18s} {tok:5d} {r['rows']:6d} | {r['eager_default_us']:16.1f} {r['eager_capturable_us']:13.1f} "
                      f"{r['graph_us']:9.1f} | {r['max_abs_diff_vs_default']:.3g}", flush=True)
                torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
