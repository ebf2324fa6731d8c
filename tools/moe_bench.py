"""Mixture-of-experts projections: the grouped matmul (Matmul.forward_grouped, one launch) against what a caller does without it
(one bitblas.Linear per active expert, counts known on the host).

    python tools/moe_bench.py [--iters 200] [--sweep-only | --no-sweep] [--no-layer | --layer-only]

Expert shapes (uint4, group 128, quantized zeros, fp16), gate/up (fused) and down as separate cases:
    Mixtral-8x7B      E=8,   top-2, gate/up 28672 x 4096, down 4096 x 14336
    Qwen3-30B-A3B     E=128, top-8, gate/up  1536 x 2048, down 2048 x   768
    DeepSeek-V2-Lite  E=64,  top-6, gate/up  2816 x 2048, down 2048 x  1408
Routing: seeded uniform top-k per token.  Every timed window cycles through 16 routings, so successive calls mostly read other
experts' weights and the active weight set does not stay in the 50 MB L2.  Device time: CUDA events around `--iters` calls.
Bytes: the active experts' weights, scales and zeros, plus activations and outputs; FLOP: 2 T N K.  The sweep times, for every
shape up to a few thousand tokens, forward_grouped(capturable=True) (the grouped GEMV up to
GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP rows per expert, the grouped wgmma GEMM above it) against both sides of the default
forward_grouped: the single grouped GEMV launch and the per-group bb_matmul path.  The layer section times one MoE expert block
from router output to layer output, MoEExperts.forward against the torch glue around the two grouped calls (both with the top-k
weighted combine), eager and replayed from one CUDA graph.  Above 8 rows per expert it also times the copy-free block
(moe_route_index -> forward_grouped_swiglu(x, row_index=row_token) -> down -> combine), which gives MoEExperts' bits without
moe_route's [T*k, H] copy of x, eager and replayed, with each block's routing launch (bb_moe_route / bb_moe_route_index) and its
share of the replayed block, the peak memory each block allocates, and the gate/up call alone: the gathering GEMM on x against
the plain GEMM on the pre-gathered rows, at the BM the launch picks.
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
    """one MoE expert block, router output (top-k ids and weights) in, [T, H] layer output out: MoEExperts.forward (device routing,
    gate/up with SwiGLU in the epilogue, down, weighted combine: 4 library launches) against the torch glue around the two grouped
    calls (counts, cumsum, argsort, gather, slice + silu + mul, scatter of the slot rows, weighted sum), eager and as one CapturedStep
    replay each"""
    m = MODELS[name]
    E, topk = m["E"], m["topk"]
    (N1, H), (_, I) = m["gate_up"], m["down"]
    moe = bitblas.MoEExperts(E, H, I, **CFG).cuda()
    for gl, seed in ((moe.gate_up, 3), (moe.down, 4)):
        src = Layer(E, gl.out_features, gl.in_features, seed=seed).gl
        gl.qweight, gl.scales, gl.zeros = src.qweight, src.scales, src.zeros
    g = torch.Generator(device="cuda").manual_seed(tokens)
    x = (torch.rand((tokens, H), device="cuda", generator=g) - 0.5).half()
    ids = torch.rand((tokens, E), device="cuda", generator=g).argsort(dim=1)[:, :topk].to(torch.int32).contiguous()
    w = torch.softmax(torch.randn((tokens, topk), device="cuda", generator=g), dim=1)
    off = torch.zeros(E + 1, dtype=torch.int32, device="cuda")
    out = torch.empty((tokens, H), dtype=torch.float16, device="cuda")

    def glue():
        flat = ids.reshape(-1).long()
        counts = torch.zeros(E, dtype=torch.int64, device="cuda").scatter_add_(0, flat, torch.ones_like(flat))
        off[1:] = torch.cumsum(counts, 0).to(torch.int32)
        order = torch.argsort(flat, stable=True)
        h = moe.gate_up(x[order // topk], off, capturable=True).view(-1, I // 8, 2, 8)   # gate/up interleave
        a = (torch.nn.functional.silu(h[:, :, 0]) * h[:, :, 1]).reshape(-1, I)
        y = moe.down(a, off, capturable=True)
        rows = torch.empty_like(order).scatter_(0, order, torch.arange(order.numel(), device="cuda"))
        out.copy_((w[..., None] * y[rows].view(tokens, topk, H).float()).sum(1))
        return out

    def fused():
        return moe(x, ids, w, output=out)

    mm, gu = moe.gate_up.bitblas_matmul, moe.gate_up

    def gathering():   # MoEExperts.forward without moe_route's copy of x: the gate/up GEMM reads x through row_token
        offsets, slot_rows, row_token = bitblas.moe.moe_route_index(ids, E)
        h = mm.forward_grouped_swiglu(x, gu.qweight, offsets, gu.scales, gu.zeros, row_index=row_token)
        return bitblas.moe.moe_combine(moe.down(h, offsets, capturable=True), slot_rows, w, out)

    def peak_bytes(fn):   # allocated by one block beyond what is live before it
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def host_time(run, sync, n):
        for _ in range(3):
            run()
        sync()
        t0 = time.perf_counter()
        for _ in range(n):
            run()
        sync()
        return (time.perf_counter() - t0) / n * 1e6

    def device_ops(fn):
        try:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        except Exception:   # the count is informative only
            return -1

    ref = glue().float().clone()
    got = fused().float()
    lib_launches = launches(lambda i: fused())
    res = dict(model=name, tokens=tokens, rows=tokens * topk, launches_fused=lib_launches,
               ops_fused=device_ops(fused), ops_glue=device_ops(glue),
               max_abs_diff=float((got - ref).abs().max()), max_abs_ref=float(ref.abs().max()))
    # the gathering gate/up call is the grouped GEMM at every T; MoEExperts' is the GEMM (same bits) above 8 rows per expert
    gathers = tokens * topk > GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP * E
    res["gathers"] = gathers
    g_glue, g_fused = bitblas.CapturedStep(glue), bitblas.CapturedStep(fused)
    g_gath = bitblas.CapturedStep(gathering) if gathers else None
    res["peak_fused_MB"] = peak_bytes(fused) / 2**20
    for _ in range(2):    # alternate the sides so drift on a shared host hits all of them
        res["glue_eager_us"] = host_time(glue, torch.cuda.synchronize, iters)
        res["fused_eager_us"] = host_time(fused, torch.cuda.synchronize, iters)
        res["glue_graph_us"] = host_time(g_glue.run, g_glue.wait, iters)
        res["fused_graph_us"] = host_time(g_fused.run, g_fused.wait, iters)
        if gathers:
            res["gath_eager_us"] = host_time(gathering, torch.cuda.synchronize, iters)
            res["gath_graph_us"] = host_time(g_gath.run, g_gath.wait, iters)
    res["route_us"] = time_calls(lambda i: bitblas.moe.moe_route(ids, x, E), iters)
    if gathers:   # the gate/up call alone: gathering GEMM on x vs the plain GEMM on the pre-gathered rows
        res["gath_equal"] = bool(torch.equal(gathering().float(), got))
        res["peak_gath_MB"] = peak_bytes(gathering) / 2**20
        res["route_index_us"] = time_calls(lambda i: bitblas.moe.moe_route_index(ids, E), iters)
        offsets, _, row_token = bitblas.moe.moe_route_index(ids, E)
        xs = x[row_token.long()]
        rows = tokens * topk
        mean = -(-rows // min(E, rows))
        res["bm"] = 32 if mean <= 32 else (64 if mean <= 64 else 128)
        for _ in range(2):
            res["gemm_gather_us"] = time_calls(
                lambda i: mm.forward_grouped_swiglu(x, gu.qweight, offsets, gu.scales, gu.zeros, row_index=row_token), iters)
            res["gemm_plain_us"] = time_calls(lambda i: mm.forward_grouped_swiglu(xs, gu.qweight, offsets, gu.scales, gu.zeros),
                                              iters)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tokens", default="1,4,16,64")
    ap.add_argument("--sweep-tokens", default="1,2,4,8,16,32,64,128,256,512,1024,2048,4096")
    ap.add_argument("--sweep-only", action="store_true")
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--no-layer", action="store_true")
    ap.add_argument("--layer-only", action="store_true", help="only the MoE expert block section")
    ap.add_argument("--layer-tokens", default="1,4,16,64,256,512,1024,2048")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "moe_bench measures on the GPU; there is no CPU fallback"
    print(f"# {card()}")
    print(f"# GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP = {GM.GROUPED_SINGLE_LAUNCH_MAX_ROWS_PER_GROUP}")
    results = []
    if args.layer_only:
        args.sweep_only = args.no_sweep = True
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
        print("\n# one MoE expert block (router output in, [T, H] out): MoEExperts.forward vs torch glue around the grouped calls")
        print("# fused = MoEExperts.forward (moe_route's copy of x); gath = the copy-free block (moe_route_index + the gathering "
              "gate/up GEMM), above 8 rows per expert;\n# route = the routing launch alone (its share of the replayed block); "
              "peak = MB allocated by one block; gather/plain = the gate/up GEMM alone; = fused: bit-identical")
        print(f"{'model':18s} {'tok':>5s} {'rows':>6s} | {'glue eager':>10s} {'fused eager':>11s} {'gath eager':>10s} "
              f"{'glue graph':>10s} {'fused graph':>11s} {'gath graph':>10s} {'fused/gath':>10s} | {'route us':>8s} {'share':>6s} "
              f"{'idx rt':>7s} {'share':>6s} | {'peak MB':>7s} {'gath MB':>7s} | {'BM':>3s} {'gather us':>9s} {'plain us':>8s} | "
              f"{'L':>2s} {'ops glue':>8s} {'ops fused':>9s} | = fused | max |fused - glue| (max |ref|)")
        for name in MODELS:
            for tok in map(int, args.layer_tokens.split(",")):
                r = moe_layer(name, tok, max(5, min(args.iters, 20000 // tok)))
                results.append(r)
                if r["gathers"]:
                    gath = (f"{r['gath_eager_us']:10.1f}", f"{r['gath_graph_us']:10.1f}",
                            f"{r['fused_graph_us'] / r['gath_graph_us']:9.3f}x",
                            f"{r['route_index_us']:7.1f} {r['route_index_us'] / r['gath_graph_us']:6.1%}", f"{r['peak_gath_MB']:7.1f}",
                            f"{r['bm']:3d} {r['gemm_gather_us']:9.1f} {r['gemm_plain_us']:8.1f}", "y" if r["gath_equal"] else "N")
                else:
                    gath = (f"{'-':>10s}", f"{'-':>10s}", f"{'-':>10s}", f"{'-':>7s} {'-':>6s}", f"{'-':>7s}",
                            f"{'-':>3s} {'-':>9s} {'-':>8s}", "-")
                print(f"{name:18s} {tok:5d} {r['rows']:6d} | {r['glue_eager_us']:10.1f} {r['fused_eager_us']:11.1f} {gath[0]} "
                      f"{r['glue_graph_us']:10.1f} {r['fused_graph_us']:11.1f} {gath[1]} {gath[2]} | "
                      f"{r['route_us']:8.1f} {r['route_us'] / r['fused_graph_us']:6.1%} {gath[3]} | {r['peak_fused_MB']:7.1f} {gath[4]} | "
                      f"{gath[5]} | {r['launches_fused']:2d} {r['ops_glue']:8d} {r['ops_fused']:9d} | {gath[6]:>7s} "
                      f"| {r['max_abs_diff']:.3g} ({r['max_abs_ref']:.3g})", flush=True)
                torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
