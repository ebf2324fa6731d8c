"""GPTQ act-order: what the activation column gather (bb_permute_cols) costs on top of the matmul.

    python tools/act_order_bench.py [--iters 200] [--dense-only | --moe-only] [--json PATH]

Dense layers: the Llama-2-70B linears (N x K = 8192 x 8192, 28672 x 8192, 8192 x 28672; uint4, group 128, quantized zeros, fp16)
at m in {1, 4, 16, 128, 4096}: an act-order Linear (permute_cols, then the matmul: 2 launches) against the same layer without
act-order (1 launch), and the gather alone, whose time over the act-order layer's is its share.  Each timed window cycles through
enough copies of the weight that it does not stay in the 50 MB L2.  The same comparison runs again in a child process with BB_PDL=0
(the library reads it once per process), which shows what the programmatic-dependent-launch overlap of the gather and the matmul
buys: with PDL the m <= 8 GEMVs stream their weights while the gather runs.

Expert block: MoEExperts with and without act-order experts (route -> gather of x_sorted -> gate/up -> down -> combine, 5 launches,
against 4) on the Qwen3-30B-A3B and Mixtral-8x7B shapes of tools/moe_bench.py at 1-2048 tokens, eager and replayed from one CUDA
graph, and the grouped gather of x_sorted alone.

Device time: CUDA events around --iters calls (dense), host time around --iters block calls ended by a synchronise (block).
The card's name, power limit and maximum SM clock are printed with the results.
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

CFG = dict(A_dtype="float16", W_dtype="uint4", group_size=128, with_scaling=True, with_zeros=True, zeros_mode="quantized")
DENSE = [(8192, 8192), (28672, 8192), (8192, 28672)]
DENSE_M = [1, 4, 16, 128, 4096]
MODELS = {   # tools/moe_bench.py
    "qwen3-30b-a3b": dict(E=128, topk=8, H=2048, I=768),
    "mixtral-8x7b": dict(E=8, topk=2, H=4096, I=14336),
}
BLOCK_TOKENS = [1, 4, 16, 64, 256, 512, 1024, 2048]
L2_FLUSH_BYTES = 150e6


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        q = q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return f"{torch.cuda.get_device_name()} (power.limit, clocks.max.sm: {q})"


def launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    fn(0)
    torch.cuda.synchronize()
    return lib.bb_launch_count() - n0


def device_us(fn, iters):
    for i in range(min(iters, 20)):
        fn(i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(iters):
        fn(i)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1e3


def graph_us(fn, reps, loops=5):
    """device time per call of `reps` calls fn(0..reps-1) captured into one CUDA graph: no host overhead between the launches,
    so the PDL overlap of consecutive kernels shows"""
    step = bitblas.CapturedStep(lambda: [fn(i) for i in range(reps)])
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(step.stream):
        step.graph.replay()
        start.record()
        for _ in range(loops):
            step.graph.replay()
        end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / (loops * reps) * 1e3


def host_us(run, sync, iters):
    for _ in range(3):
        run()
    sync()
    t0 = time.perf_counter()
    for _ in range(iters):
        run()
    sync()
    return (time.perf_counter() - t0) / iters * 1e6


def random_perm(n, gen, device="cuda"):
    return torch.randperm(n, generator=gen).to(torch.int32).to(device)


def randomize(layer, gen):
    """random stored weights, scales and quantized zeros (generated on the device)"""
    for name in ("qweight", "zeros"):
        setattr(layer, name, torch.randint(-128, 128, tuple(getattr(layer, name).shape), dtype=torch.int8, device="cuda",
                                           generator=gen))
    layer.scales = (torch.rand(tuple(layer.scales.shape), device="cuda", generator=gen) * 0.01).half()


def random_linear(N, K, gen):
    lin = bitblas.Linear(K, N, **CFG).cuda()
    randomize(lin, gen)
    return lin


def dense(iters):
    rows = []
    gen, gen_d = torch.Generator().manual_seed(0), torch.Generator(device="cuda").manual_seed(0)
    for N, K in DENSE:
        wbytes = N * K // 2
        copies = max(2, int(-(-L2_FLUSH_BYTES // wbytes)))
        plain = [random_linear(N, K, gen_d) for _ in range(copies)]
        act = []
        for p in plain:   # the same buffers with a column order
            a = bitblas.Linear(K, N, **CFG).cuda()
            a.qweight, a.scales, a.zeros = p.qweight, p.scales, p.zeros
            a.perm = random_perm(K, gen)
            act.append(a)
        for m in DENSE_M:
            A = (torch.rand((m, K), generator=gen) - 0.5).half().cuda()
            C = torch.empty((m, N), dtype=torch.float16, device="cuda")
            P = torch.empty_like(A)
            n = max(10, min(iters, 40000 // m))
            f_plain = lambda i: plain[i % copies](A, output=C)                      # noqa: E731
            f_act = lambda i: act[i % copies](A, output=C)                          # noqa: E731
            f_perm = lambda i: bitblas.permute_cols(A, act[i % copies].perm, output=P)   # noqa: E731
            assert torch.equal(act[0](A), plain[0](A[:, act[0].perm.long()]))
            r = dict(N=N, K=K, m=m, launches_plain=launches(f_plain), launches_act=launches(f_act))
            reps = max(2 * copies, min(40, 4000 // m)) // copies * copies
            for _ in range(2):   # alternate the sides so drift on a shared host hits both
                for tag, f in (("plain", f_plain), ("act", f_act), ("perm", f_perm)):
                    r[f"{tag}_us"] = device_us(f, n)
                    r[f"{tag}_graph_us"] = graph_us(f, reps)
            r["overhead"] = r["act_us"] / r["plain_us"] - 1
            r["overhead_graph"] = r["act_graph_us"] / r["plain_graph_us"] - 1
            r["perm_share"] = r["perm_graph_us"] / r["act_graph_us"]
            r["perm_GBps"] = 2 * m * K * 2 / r["perm_graph_us"] * 1e-3
            rows.append(r)
        del plain, act
        torch.cuda.empty_cache()
    return rows


def print_dense(rows, title):
    print(f"\n# dense, {title}: act-order Linear (gather + matmul) vs the same layer without act-order; perm = the gather alone.\n"
          "# eager: back-to-back Python calls (host-bound at small m); graph: the calls replayed from one CUDA graph; share and GB/s "
          "(bytes read + written) from the graph times")
    print(f"{'N':>6s} {'K':>6s} {'m':>5s} | {'plain eager':>11s} {'act eager':>9s} {'overhead':>8s} | {'plain graph':>11s} "
          f"{'act graph':>9s} {'overhead':>8s} | {'perm eager':>10s} {'perm graph':>10s} {'share':>6s} {'GB/s':>7s} | L")
    for r in rows:
        print(f"{r['N']:6d} {r['K']:6d} {r['m']:5d} | {r['plain_us']:11.2f} {r['act_us']:9.2f} {r['overhead']:8.1%} | "
              f"{r['plain_graph_us']:11.2f} {r['act_graph_us']:9.2f} {r['overhead_graph']:8.1%} | {r['perm_us']:10.2f} "
              f"{r['perm_graph_us']:10.2f} {r['perm_share']:6.1%} {r['perm_GBps']:7.1f} | {r['launches_plain']}/{r['launches_act']}",
              flush=True)


def moe_block(name, tokens, iters):
    m = MODELS[name]
    E, k, H, I = m["E"], m["topk"], m["H"], m["I"]
    gen, gen_d = torch.Generator().manual_seed(tokens), torch.Generator(device="cuda").manual_seed(tokens)
    blocks = []
    for act_order in (False, True):
        b = bitblas.MoEExperts(E, H, I, **CFG).cuda()
        for gl in (b.gate_up, b.down):
            randomize(gl, gen_d)
        if act_order:   # the down projection's order is absorbed into the gate/up rows at load time: no run-time cost
            b.gate_up.perm = torch.stack([random_perm(H, gen, "cpu") for _ in range(E)]).cuda()
        blocks.append(b)
    x = (torch.rand((tokens, H), generator=gen) - 0.5).half().cuda()
    ids = torch.rand((tokens, E), generator=gen).argsort(dim=1)[:, :k].to(torch.int32).cuda()
    w = torch.softmax(torch.randn((tokens, k), generator=gen), dim=1).cuda()
    out = torch.empty((tokens, H), dtype=torch.float16, device="cuda")
    fns = [lambda b=b: b(x, ids, w, output=out) for b in blocks]
    r = dict(model=name, tokens=tokens, rows=tokens * k, launches=[launches(lambda i, f=f: f()) for f in fns])
    graphs = [bitblas.CapturedStep(f) for f in fns]
    for _ in range(2):
        for tag, f, g in zip(("plain", "act"), fns, graphs):
            r[f"{tag}_eager_us"] = host_us(f, torch.cuda.synchronize, iters)
            r[f"{tag}_graph_us"] = host_us(g.run, g.wait, iters)
    offsets, _, xs = bitblas.moe.moe_route(ids, x, E)
    P = torch.empty_like(xs)
    perm = blocks[1].gate_up.perm
    r["perm_us"] = device_us(lambda i: bitblas.permute_cols(xs, perm, offsets, output=P), iters)
    r["perm_share"] = r["perm_us"] / r["act_graph_us"]
    r["overhead_graph"] = r["act_graph_us"] / r["plain_graph_us"] - 1
    del blocks, graphs
    torch.cuda.empty_cache()
    return r


def print_moe(rows):
    print("\n# expert block: MoEExperts without / with act-order experts, eager and replayed; perm = the grouped gather of x_sorted "
          "alone (device time) and its share of the replayed act-order block")
    print(f"{'model':14s} {'tok':>5s} {'rows':>6s} | {'plain eager':>11s} {'act eager':>10s} | {'plain graph':>11s} {'act graph':>10s} "
          f"{'overhead':>8s} | {'perm us':>8s} {'share':>6s} | L")
    for r in rows:
        print(f"{r['model']:14s} {r['tokens']:5d} {r['rows']:6d} | {r['plain_eager_us']:11.1f} {r['act_eager_us']:10.1f} | "
              f"{r['plain_graph_us']:11.1f} {r['act_graph_us']:10.1f} {r['overhead_graph']:8.1%} | {r['perm_us']:8.1f} "
              f"{r['perm_share']:6.1%} | {r['launches'][0]}/{r['launches'][1]}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--dense-only", action="store_true")
    ap.add_argument("--moe-only", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)   # the BB_PDL=0 dense run: JSON on the last line
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "act_order_bench measures on the GPU; there is no CPU fallback"
    if args.child:
        print(json.dumps(dense(args.iters)))
        return
    print(f"# {card()}")
    results = {"card": card()}
    if not args.moe_only:
        results["dense_pdl"] = dense(args.iters)
        print_dense(results["dense_pdl"], "BB_PDL=1 (default)")
        env = dict(os.environ, BB_PDL="0")
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(args.iters)], env=env,
                           capture_output=True, text=True)
        if p.returncode:
            sys.stderr.write(p.stderr[-4000:])
            raise SystemExit("the BB_PDL=0 run failed")
        results["dense_nopdl"] = json.loads(p.stdout.strip().splitlines()[-1])
        print_dense(results["dense_nopdl"], "BB_PDL=0")
        print("\n# PDL: act-order cost over the plain layer, graph-replayed, with / without programmatic dependent launch")
        for a, b in zip(results["dense_pdl"], results["dense_nopdl"]):
            print(f"{a['N']:6d} {a['K']:6d} {a['m']:5d} | PDL {a['overhead_graph']:7.1%} ({a['act_graph_us'] - a['plain_graph_us']:7.2f} us)"
                  f" | no PDL {b['overhead_graph']:7.1%} ({b['act_graph_us'] - b['plain_graph_us']:7.2f} us) | gather alone "
                  f"{a['perm_graph_us']:6.2f} us")
    if not args.dense_only:
        results["moe"] = []
        for name in MODELS:
            for tok in BLOCK_TOKENS:
                results["moe"].append(moe_block(name, tok, max(5, min(args.iters, 20000 // tok))))
        print_moe(results["moe"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
