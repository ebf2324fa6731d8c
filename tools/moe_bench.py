"""Mixture-of-experts projections: the grouped matmul (Matmul.forward_grouped, one launch) against what a caller does without it
(one bitblas.Linear per active expert, counts known on the host).

    python tools/moe_bench.py [--iters 200] [--sweep-only | --no-sweep]

Expert shapes (uint4, group 128, quantized zeros, fp16), gate/up (fused) and down as separate cases:
    Mixtral-8x7B      E=8,   top-2, gate/up 28672 x 4096, down 4096 x 14336
    Qwen3-30B-A3B     E=128, top-8, gate/up  1536 x 2048, down 2048 x   768
    DeepSeek-V2-Lite  E=64,  top-6, gate/up  2816 x 2048, down 2048 x  1408
Routing: seeded uniform top-k per token.  Every timed window cycles through 16 routings, so successive calls mostly read other
experts' weights and the active weight set does not stay in the 50 MB L2.  Device time: CUDA events around `--iters` calls.
Bytes: the active experts' weights, scales and zeros, plus activations and outputs.  The sweep times both sides of
Matmul.forward_grouped (the single launch and the per-group bb_matmul path) up to a few thousand tokens to place
GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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

    fns = dict(grouped=grouped, loop=loop, single=with_threshold(1 << 30), per_group=with_threshold(-1))
    nbytes = sum(layer.bytes(r[0]) for r in routes) / len(routes)
    res = dict(T=T, active=sum(1 for c in routes[0][0] if c), bytes=int(nbytes))
    for p in paths:
        us = time_calls(fns[p], iters)
        res[p] = dict(us=round(us, 2), GBps=round(nbytes / us * 1e-3, 1), hbm=round(nbytes / us * 1e6 / HBM_BYTES_PER_S, 3),
                      launches=launches(fns[p]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tokens", default="1,4,16,64")
    ap.add_argument("--sweep-tokens", default="1,2,4,8,16,32,64,128,256,512,1024,2048,4096")
    ap.add_argument("--sweep-only", action="store_true")
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "moe_bench measures on the GPU; there is no CPU fallback"
    print(f"# {card()}")
    print(f"# GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = {GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP}")
    results = []
    if not args.sweep_only:
        print(f"{'model':18s} {'proj':8s} {'tok':>5s} {'T':>6s} {'act':>4s} {'MB':>8s} | "
              f"{'grouped us':>10s} {'GB/s':>7s} {'HBM':>6s} {'L':>3s} | {'loop us':>9s} {'GB/s':>7s} {'HBM':>6s} {'L':>4s} | speedup")
        for name, m in MODELS.items():
            for proj in ("gate_up", "down"):
                N, K = m[proj]
                layer = Layer(m["E"], N, K, seed=1)
                for tok in map(int, args.tokens.split(",")):
                    routes = routings(m["E"], m["topk"], tok, seed=tok)
                    r = point(layer, routes, args.iters, ("grouped", "loop"))
                    r.update(model=name, proj=proj, tokens=tok)
                    results.append(r)
                    g, lp = r["grouped"], r["loop"]
                    print(f"{name:18s} {proj:8s} {tok:5d} {r['T']:6d} {r['active']:4d} {r['bytes'] / 1e6:8.2f} | "
                          f"{g['us']:10.2f} {g['GBps']:7.1f} {g['hbm']:6.3f} {g['launches']:3d} | "
                          f"{lp['us']:9.2f} {lp['GBps']:7.1f} {lp['hbm']:6.3f} {lp['launches']:4d} | {lp['us'] / g['us']:6.2f}x", flush=True)
                del layer
                torch.cuda.empty_cache()
    if not args.no_sweep:
        print("\n# sweep: single grouped launch vs one bb_matmul per non-empty group (both sides of forward_grouped)")
        print(f"{'model':18s} {'proj':8s} {'tok':>5s} {'T':>6s} {'rows/exp':>8s} | {'single us':>10s} {'per-group us':>12s} | ratio")
        for name, proj in (("qwen3-30b-a3b", "gate_up"), ("mixtral-8x7b", "down")):
            m = MODELS[name]
            N, K = m[proj]
            layer = Layer(m["E"], N, K, seed=2)
            for tok in map(int, args.sweep_tokens.split(",")):
                routes = routings(m["E"], m["topk"], tok, seed=tok)
                iters = max(10, min(args.iters, 20000 // tok))
                r = point(layer, routes, iters, ("single", "per_group"))
                r.update(model=name, proj=proj, tokens=tok, sweep=True)
                results.append(r)
                print(f"{name:18s} {proj:8s} {tok:5d} {r['T']:6d} {r['T'] / max(1, r['active']):8.1f} | "
                      f"{r['single']['us']:10.2f} {r['per_group']['us']:12.2f} | {r['per_group']['us'] / r['single']['us']:5.2f}",
                      flush=True)
            del layer
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
