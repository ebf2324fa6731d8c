"""Mixture-of-experts top-k gating: moe_topk (bb_moe_topk, one launch) against the torch gating it replaces, alone and in front of
the expert block.

    python tools/moe_topk_bench.py [--iters 200] [--tokens 1,8,64,512,2048] [--no-layer] [--json PATH]

Models (router logits fp16 [T, E]; expert shapes of tools/moe_bench.py, uint4, group 128, quantized zeros, fp16):
    Mixtral-8x7B      E=8,   top-2, renormalize                                      H=4096, I=14336
    Qwen3-30B-A3B     E=128, top-8, renormalize                                      H=2048, I=768
    DeepSeek-V2-Lite  E=64,  top-6, scale 1.0                                        H=2048, I=1408
    DeepSeek-V2       E=160, top-6, 8 groups, 3 kept by max, scale 16                (gating only)
    DeepSeek-V3       E=256, top-8, sigmoid, bias, 8 groups, 4 kept by top2_sum,     (gating only)
                      renormalize, scale 2.5
The torch gating is what a caller writes without the library: softmax (or sigmoid) in fp32, for the group-limited models the
biased selection values, the group scores, a top-k over the groups and the mask of the other groups' experts, torch.topk, the
gather of the unbiased scores, the renormalisation where the model has one, the scale, and the int32 cast of the ids (the
weights are already fp32).  Each side is captured in one CUDA graph
(CapturedStep); the torch and the library graph are replayed alternately, --iters times each, on one stream with a CUDA event
after every replay, and each side's time is the sum of its replays' event intervals.  Alternating replay by replay keeps clock
and power drift (the card may be power-limited) from favouring the side timed later.  The gating graphs hold GATE_REPS calls
each, so the time per call is what the gating adds inside a captured layer, without the launch of the graph itself.  The layer
section captures gating followed by MoEExperts.forward (route -> gate/up with SwiGLU -> down -> combine) both ways, one layer per
graph.  The torch gating's kernel count comes from torch.profiler in an untimed call.  Printed with the card's name, power limit
and maximum SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bitblas_b200 as bitblas  # noqa: E402
from bitblas_b200 import _lib  # noqa: E402
from moe_bench import CFG, Layer, card  # noqa: E402

# gate: moe_topk's keyword arguments ("correction_bias": True draws a seeded fp32 bias); H, I: the expert block's shapes
MODELS = {
    "mixtral-8x7b": dict(E=8, topk=2, gate=dict(renormalize=True), H=4096, I=14336),
    "qwen3-30b-a3b": dict(E=128, topk=8, gate=dict(renormalize=True), H=2048, I=768),
    "deepseek-v2-lite": dict(E=64, topk=6, gate=dict(routed_scaling_factor=1.0), H=2048, I=1408),
    "deepseek-v2": dict(E=160, topk=6, gate=dict(num_expert_group=8, topk_group=3, group_score="max",
                                                 routed_scaling_factor=16.0)),
    "deepseek-v3": dict(E=256, topk=8, gate=dict(scoring="sigmoid", correction_bias=True, num_expert_group=8, topk_group=4,
                                                 group_score="top2_sum", renormalize=True, routed_scaling_factor=2.5)),
}
GATE_REPS = 20


def torch_gating(logits, k, scoring="softmax", renormalize=False, correction_bias=None, num_expert_group=None, topk_group=None,
                 group_score="max", routed_scaling_factor=1.0):
    x = logits.float()
    s = torch.softmax(x, dim=-1) if scoring == "softmax" else torch.sigmoid(x)
    v = s if correction_bias is None else s + correction_bias
    if num_expert_group:
        T, E = v.shape
        vg = v.view(T, num_expert_group, E // num_expert_group)
        gscore = vg.max(dim=-1).values if group_score == "max" else vg.topk(2, dim=-1).values.sum(dim=-1)
        keep = torch.zeros_like(gscore).scatter_(1, gscore.topk(topk_group, dim=-1).indices, 1.0)
        v = v.masked_fill(keep.repeat_interleave(E // num_expert_group, dim=1) == 0, float("-inf"))
    w, ids = torch.topk(v, k, dim=-1)
    if v is not s:
        w = s.gather(1, ids)
    if renormalize:
        w = w / w.sum(dim=-1, keepdim=True)
    if routed_scaling_factor != 1.0:
        w = w * routed_scaling_factor
    return ids.to(torch.int32), w


def lib_gating(logits, k, **gate):
    return bitblas.moe_topk(logits, k, **gate)


def interleaved_us(graphs, iters):
    """device time (us) of one replay of each graph: the graphs are replayed in turn, `iters` rounds, on one stream with a CUDA
    event after every replay"""
    n = len(graphs)
    events = [torch.cuda.Event(enable_timing=True) for _ in range(n * iters + 1)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(3):
            for g in graphs:
                g.replay()
        events[0].record()
        for i in range(iters):
            for j, g in enumerate(graphs):
                g.replay()
                events[i * n + j + 1].record()
    stream.synchronize()
    return [sum(events[i * n + j].elapsed_time(events[i * n + j + 1]) for i in range(iters)) / iters * 1e3 for j in range(n)]


def kernels(fn):
    """device kernels one call launches (torch.profiler; informative only)"""
    try:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    except Exception:
        return -1


def block(m):
    moe = bitblas.MoEExperts(m["E"], m["H"], m["I"], **CFG).cuda()
    for gl, seed in ((moe.gate_up, 3), (moe.down, 4)):
        src = Layer(m["E"], gl.out_features, gl.in_features, seed=seed).gl
        gl.qweight, gl.scales, gl.zeros = src.qweight, src.scales, src.zeros
    return moe


def point(name, m, T, iters, moe):
    g = torch.Generator(device="cuda").manual_seed(T)
    logits = torch.randn((T, m["E"]), device="cuda", generator=g).half()
    k, gate = m["topk"], dict(m["gate"])
    if gate.get("correction_bias"):
        gate["correction_bias"] = torch.rand(m["E"], device="cuda", generator=g) * 0.25
    ids_t, w_t = torch_gating(logits, k, **gate)
    ids_l, w_l = lib_gating(logits, k, **gate)
    res = dict(model=name, tokens=T, ids_equal=bool(torch.equal(ids_t, ids_l)),
               max_w_diff=float((w_t - w_l).abs().max()), kernels_torch=kernels(lambda: torch_gating(logits, k, **gate)))
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.bb_launch_count()
    lib_gating(logits, k, **gate)
    res["launches_lib"] = int(lib.bb_launch_count() - n0)
    sides = (torch_gating, lib_gating)
    gating = [bitblas.CapturedStep(lambda fn=fn: [fn(logits, k, **gate) for _ in range(GATE_REPS)]) for fn in sides]
    t_us, l_us = interleaved_us([s.graph for s in gating], iters)
    res.update(torch_us=round(t_us / GATE_REPS, 2), lib_us=round(l_us / GATE_REPS, 2))
    if moe is not None:
        x = (torch.rand((T, m["H"]), device="cuda", generator=g) - 0.5).half()
        out = torch.empty_like(x)
        layers = [bitblas.CapturedStep(lambda fn=fn: moe(x, *fn(logits, k, **gate), output=out)) for fn in sides]
        t_us, l_us = interleaved_us([s.graph for s in layers], iters)
        res.update(layer_torch_us=round(t_us, 2), layer_lib_us=round(l_us, 2))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tokens", default="1,8,64,512,2048")
    ap.add_argument("--no-layer", action="store_true", help="time the gating alone")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "moe_topk_bench measures on the GPU; there is no CPU fallback"
    print(f"# {card()}")
    print("# CUDA-graph replays, device time (us): gating = scores -> [group limit] -> top-k -> [renormalise] -> int32 ids, fp32 weights,"
          f" per call of {GATE_REPS} in one graph;\n# layer = gating + MoEExperts.forward, per replay of one layer; K = torch gating "
          "kernels, L = library launches; = ids: torch and library agree")
    print(f"{'model':18s} {'tok':>5s} | {'torch us':>8s} {'lib us':>7s} {'speedup':>7s} {'K':>3s} {'L':>2s} | "
          f"{'layer torch':>11s} {'layer lib':>9s} {'saved us':>8s} {'saved':>6s} | = ids  max |dw|")
    results = []
    for name, m in MODELS.items():
        moe = None if args.no_layer or "H" not in m else block(m)
        for T in map(int, args.tokens.split(",")):
            iters = max(20, min(args.iters, 40000 // T)) if moe is not None else args.iters
            r = point(name, m, T, iters, moe)
            results.append(r)
            if moe is not None:
                saved = r["layer_torch_us"] - r["layer_lib_us"]
                layer = f"{r['layer_torch_us']:11.1f} {r['layer_lib_us']:9.1f} {saved:8.1f} {saved / r['layer_torch_us']:6.1%}"
            else:
                layer = f"{'-':>11s} {'-':>9s} {'-':>8s} {'-':>6s}"
            print(f"{name:18s} {T:5d} | {r['torch_us']:8.2f} {r['lib_us']:7.2f} {r['torch_us'] / r['lib_us']:6.2f}x "
                  f"{r['kernels_torch']:3d} {r['launches_lib']:2d} | {layer} | {'y' if r['ids_equal'] else 'N':>5s}  "
                  f"{r['max_w_diff']:.2g}", flush=True)
        del moe
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
