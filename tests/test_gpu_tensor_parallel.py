"""GPU, one device: the tensor-parallel layers of bitblas_b200.parallel with every rank of a world in one process, bit for bit.

Each rank runs in a Python thread of its own on the one device.  A fake process group (FakeGroup, below) stands in for
torch.distributed: the names parallel.py reads -- is_initialized, get_world_size and get_rank at construction, all_reduce (SUM
and MIN) and all_gather_into_tensor in forward -- are monkeypatched.  Every collective waits on a threading.Barrier for all
ranks, synchronises the device, combines the deposited tensors in rank order (the fp32 sum for SUM) and releases the ranks.
The fused column-parallel path gets W ordinary device buffers per ring slot in place of symmetric memory (every rank sees the
same slot index and the same peer pointer array) and the thread barrier plus a device synchronise in place of PeerBarrier, so
each rank's scatter epilogue really stores its column slice into every rank's buffer.  No NCCL, no second GPU.

The inputs are exact (exact_inputs.py): every shard's partial product is exact in fp32, and so is their sum, so every rank's
output must equal the float64 reference of the FULL layer, round(V) (with bias round(round(V) + b)), under torch.equal.
prove_exact runs on the full problem and on each shard's own sub-problem: with whole-row groups at world > 1 a K shard is a group
of its own, so the full problem's nonzero group sums say nothing about it (exact_inputs.sharded_activations builds them per shard).
Every test asserts the kernel each shard dispatches to (Matmul.kernel_for) for every row count it runs.
"""
import ctypes
import threading

import pytest
import torch
import torch.distributed as dist

import exact_inputs as X
from test_gpu_kernel_grid import _check_split

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODES = ["none", "scale", "original", "rescale", "quantized"]
OUTS = ["float16", "bfloat16", "float32"]
# (weight format, zero-point mode) pairs the formats allow: a signed integer weight has its zero point built in
FORMATS = [("uint4", m) for m in MODES] + [("uint2", m) for m in MODES] + [("int4", "none"), ("int4", "scale")]
# K of the Llama-70B row-parallel projections (both have N = 8192, cut down here: N does not change a K shard's storage or kernel)
LLAMA70B_K = {"o_proj": 8192, "down_proj": 28672}
# the slab GEMV (4-bit) or gemv_mma, gemv_mma, the wgmma GEMM with split-K, the wgmma GEMM without it
M_SET = (1, 4, 16, 300)


class FakeGroup:
    """One process group of `world` ranks, each a thread of this process on the one device (see the module docstring)."""

    def __init__(self, world, monkeypatch):
        from bitblas_b200 import parallel as P
        self.world = world
        self.local = threading.local()
        self.lock = threading.Lock()
        self.barrier = threading.Barrier(world, action=self._combine, timeout=120)
        self.deposits = [None] * world
        self.completed = 0   # collectives combined so far
        self.counts = {"all_reduce": 0, "all_gather": 0, "peer_barrier": 0}
        self.rings = {}   # (rows capacity, dtype) -> ring of (one buffer per rank, peer pointer array)
        self.streams = [torch.cuda.Stream() for _ in range(world)]
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: self.local.rank)
        monkeypatch.setattr(dist, "all_reduce", self.all_reduce)
        monkeypatch.setattr(dist, "all_gather_into_tensor", self.all_gather_into_tensor)
        monkeypatch.setattr(P.ColumnParallelLinear, "_symm_buffers",
                            lambda layer, m, dtype, device: self._symm_buffers(layer, m, dtype, device))
        monkeypatch.setattr(P, "PeerBarrier", lambda device, group=None: self._peer_barrier)

    # ---- collectives ---------------------------------------------------------------------------------------------------------
    def all_reduce(self, tensor, op=dist.ReduceOp.SUM, group=None, async_op=False):
        self._collective("all_reduce", (tensor, op))

    def all_gather_into_tensor(self, output_tensor, input_tensor, group=None, async_op=False):
        self._collective("all_gather", (output_tensor, input_tensor))

    def _peer_barrier(self, stream=None):
        self._collective("peer_barrier", self.local.slot)

    def _collective(self, kind, payload):
        self.deposits[self.local.rank] = (kind, payload)
        done = self.completed
        try:
            self.barrier.wait()
        except threading.BrokenBarrierError:
            if self.completed == done:   # broken by a rank that failed (run), not a rank leaving after this collective
                raise

    def _combine(self):
        """runs once, when every rank has arrived"""
        kinds = {d[0] for d in self.deposits}
        assert len(kinds) == 1, f"the ranks are in different collectives: {[d[0] for d in self.deposits]}"
        kind = kinds.pop()
        self.counts[kind] += 1
        payloads = [d[1] for d in self.deposits]
        torch.cuda.synchronize()
        if kind == "all_reduce":
            op = payloads[0][1]
            assert all(p[1] == op for p in payloads)
            acc = payloads[0][0].clone()
            for t, _ in payloads[1:]:
                if op == dist.ReduceOp.SUM:
                    acc += t
                elif op == dist.ReduceOp.MIN:
                    acc = torch.minimum(acc, t)
                else:
                    raise AssertionError(f"unexpected reduction {op}")
            for t, _ in payloads:
                t.copy_(acc)
        elif kind == "all_gather":
            full = torch.cat([inp for _, inp in payloads])
            for out, _ in payloads:
                out.copy_(full.view_as(out))
        else:
            assert len(set(payloads)) == 1, f"the ranks wrote different ring slots: {payloads}"
        torch.cuda.synchronize()
        self.deposits = [None] * self.world
        self.completed += 1

    def _symm_buffers(self, layer, m, dtype, device):
        """ColumnParallelLinear._symm_buffers on plain device memory: the ring is shared by the ranks' layers, each rank gets its
        own buffer of the slot and the pointers of all of them"""
        cap = 1
        while cap < m:
            cap *= 2
        key = (cap, dtype)
        if key not in layer._symm:
            with self.lock:
                if key not in self.rings:
                    ring = []
                    for _ in range(layer.fused_ring):
                        bufs = [torch.full((cap, layer.out_features), float("nan"), dtype=dtype, device=device)
                                for _ in range(self.world)]
                        ring.append((bufs, (ctypes.c_void_p * self.world)(*[ctypes.c_void_p(b.data_ptr()) for b in bufs])))
                    self.rings[key] = ring
            layer._symm[key] = [self.rings[key], 0]
        entry = layer._symm[key]
        slot = entry[1]
        entry[1] = (slot + 1) % layer.fused_ring
        self.local.slot = (key, slot)
        bufs, arr = entry[0][slot]
        return bufs[layer.rank], None, arr

    # ---- ranks -----------------------------------------------------------------------------------------------------------------
    def build(self, make):
        """make() once per rank, with that rank's get_rank"""
        layers = []
        for r in range(self.world):
            self.local.rank = r
            layers.append(make())
        return layers

    def run(self, fn, raise_errors=True):
        """fn(rank) on one thread per rank; returns the results in rank order (and with raise_errors=False the exceptions)"""
        out, err = [None] * self.world, [None] * self.world

        def body(r):
            self.local.rank = r
            try:
                # a new thread has no CUDA context current until its first runtime call that needs one; the library's
                # tensor-map encoding (a driver call, made before the slab GEMV or wgmma GEMM launch) requires it, as it would
                # in the process's main thread
                torch.cuda.synchronize()
                # one stream per rank, as every real rank has its own device: the ranks' layers share one Matmul (the operator
                # cache) and its scratch per (device, stream), so two threads on one stream could put another rank's split-K
                # GEMM between this rank's GEMM and its reduction of the partials
                with torch.cuda.stream(self.streams[r]):
                    out[r] = fn(r)
            except BaseException as e:   # noqa: B036 -- reported below; the barrier is broken so no rank waits forever
                err[r] = e
                self.barrier.abort()

        threads = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if not raise_errors:
            return out, err
        first = [e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)]
        first = first or [e for e in err if e is not None]
        if first:
            raise first[0]
        return out


# ---- cases, sub-problems, layers ----------------------------------------------------------------------------------------------
def _groups(case):
    G = case["scale"].shape[1] if case["scale"] is not None else 1
    return G, case["K"] // G


def k_shard(case, lo, hi):
    """a row-parallel rank's own problem: columns [lo, hi) of A and W with their groups (the one group of whole-row groups
    belongs to every shard), fp32 output, no bias (it is added once, after the reduction)"""
    G, g = _groups(case)
    gs = slice(0, 1) if G == 1 else slice(lo // g, hi // g)
    sub = dict(case, K=hi - lo, A=case["A"][:, lo:hi], fields=case["fields"][:, lo:hi], bias=None,
               cfg=dict(case["cfg"], out_dtype="float32"))
    if case["scale"] is not None:
        sub["scale"] = case["scale"][:, gs]
    if case["mode"] in ("original", "rescale"):
        sub["zeros"] = case["zeros"][:, gs]
    if case["qz"] is not None:
        sub["qz"] = case["qz"][gs]
    return sub


def n_shard(case, lo, hi):
    """a column-parallel rank's own problem: rows [lo, hi) of W and their parameters"""
    sub = dict(case, N=hi - lo, fields=case["fields"][lo:hi])
    for k in ("scale", "bias"):
        if case[k] is not None:
            sub[k] = case[k][lo:hi]
    if case["mode"] in ("original", "rescale"):
        sub["zeros"] = case["zeros"][lo:hi]
    if case["qz"] is not None:
        sub["qz"] = case["qz"][:, lo:hi]
    return sub


def prove(case, shards):
    """the precondition for the full problem (its partial sums bound the reduction of the shards' partials) and for each shard"""
    X.prove_exact(case, ("sum",), device=DEV)
    for sub in shards:
        X.prove_exact(sub, device=DEV)


def linear_kwargs(case):
    c = case["cfg"]
    return dict(A_dtype=c["A_dtype"], W_dtype=c["W_dtype"], accum_dtype=c["accum_dtype"], group_size=c["group_size"],
                with_scaling=c["with_scaling"], with_zeros=c["with_zeros"], zeros_mode=c["zeros_mode"],
                fast_decoding=c["fast_decoding"], propagate_b=bool(case["propagate_b"]), enable_tuning=False)


def full_params(case):
    """the full layer's parameters on the device, the weight in the full layer's own storage (its legalised propagate_b)"""
    full_op = X.product_operator(case)
    dev = lambda k: case[k].to(DEV) if case[k] is not None else None   # noqa: E731
    return full_op, (X.product_weight(full_op, case, DEV), dev("scale"), dev("zeros"), dev("bias"))


def expected_kernel(op, m):
    """the dispatcher's pick (bb_api.cu select) for the shard operators of this file: m = 1 with 4-bit weights on the slab GEMV;
    other m <= 8 on gemv_mma from row-major storage; the wgmma GEMM where N % 128 == 0; gemv_mma up to m = 32 from row-major
    storage; generic_simt otherwise"""
    if m == 1 and op.bit == 4:
        return "gemv_slab"
    if m <= 8 and not op.weight_tiled:
        return "gemv_mma"
    if op.N % 128 == 0:
        return "gemm_ts_wgmma"
    if m <= 32 and not op.weight_tiled:
        return "gemv_mma"
    return "generic_simt"


def assert_kernel(op, m):
    want = expected_kernel(op, m)
    assert op.kernel_for(m) == want, (m, op.kernel_for(m), want, op.config)
    if want == "gemm_ts_wgmma":   # split-K exactly where the host rule splits (every m <= 128 of this file, at these shard shapes)
        _check_split(op, m, m <= 128, 64)
    return want


def compare_ranks(outs, ref, what):
    for r, got in enumerate(outs):
        X.compare_exact(got, ref, f"{what}, rank {r}")


# ---- row-parallel ---------------------------------------------------------------------------------------------------------------
def _row_cells():
    """24 cells: every (world, group size) pair four times, every format / zeros mode pair twice (both group sizes and both
    shapes), both activation types, all output types, bias, fast decoding, propagate_b and input_is_parallel on and off"""
    cells = []
    for j in range(24):
        W_dtype, mode = FORMATS[(j // 2) % 12]
        cells.append(dict(world=(2, 4, 8)[j % 3], W=W_dtype, mode=mode, g=(128, -1)[j % 2],
                          shape=("o_proj", "down_proj")[(j // 2 + j) % 2], T=("float16", "bfloat16")[(j // 3) % 2],
                          out=OUTS[(j // 3) % 3], bias=(j // 4) % 2 == 0, il=(j // 5) % 2 == 0, tiled=(j // 6) % 2 == 1,
                          parallel_input=j % 4 < 2, seed=j))
    return cells


def run_row_parallel(monkeypatch, case, world, parallel_input=True, full_tiled=None, shard_tiled=None):
    """the case through `world` RowParallelLinear ranks at every m of M_SET (the first m rows of the case's activations)"""
    from bitblas_b200.parallel import RowParallelLinear
    K, N = case["K"], case["N"]
    per = K // world
    prove(case, [k_shard(case, r * per, (r + 1) * per) for r in range(world)])
    full_op, params = full_params(case)
    if full_tiled is not None:
        assert full_op.weight_tiled == full_tiled
    fg = FakeGroup(world, monkeypatch)
    layers = fg.build(lambda: RowParallelLinear(K, N, bias=case["bias"] is not None, out_dtype=case["cfg"]["out_dtype"],
                                                input_is_parallel=parallel_input, **linear_kwargs(case)).cuda())
    for layer in layers:
        layer.load_full_params(*params)
    op = layers[0].local.bitblas_matmul
    assert op.K == per and op.out_dtype == "float32", "the partial products leave the kernel in fp32"
    if case["cfg"]["group_size"] == -1:
        assert op.config.group_size == per, "whole-row groups: one group per shard"
    if shard_tiled is not None:
        assert op.weight_tiled == shard_tiled
    A = case["A"].to(DEV)
    ref = X.exact_reference(case, DEV).cpu()
    for m in M_SET:
        kernel = assert_kernel(op, m)

        def rank(r, m=m):
            x = A[:m, r * per:(r + 1) * per] if parallel_input else A[:m]
            return layers[r](x).cpu()

        n0 = fg.counts["all_reduce"]
        outs = fg.run(rank)
        assert fg.counts["all_reduce"] == n0 + 1
        compare_ranks(outs, ref[:m], f"row-parallel world={world} m={m} ({kernel})")


@pytest.mark.parametrize("c", _row_cells(), ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_row_parallel(monkeypatch, c):
    K = LLAMA70B_K[c["shape"]]
    case = X.make_exact_case(max(M_SET), 256, K, A_dtype=c["T"], W_dtype=c["W"], out_dtype=c["out"],
                             group_size=c["g"], mode=c["mode"], bias=c["bias"],
                             fast_decoding=c["il"], seed=c["seed"], propagate_b=c["tiled"], shards=c["world"])
    run_row_parallel(monkeypatch, case, c["world"], parallel_input=c["parallel_input"])


@pytest.mark.parametrize("W_dtype", ["uint4", "int4"])
def test_row_parallel_whole_row_groups_without_scale(monkeypatch, W_dtype):
    """whole-row groups (the default group_size) with no scale at all: each shard still takes its K range of the weight"""
    case = X.make_exact_case(max(M_SET), 256, 8192, W_dtype=W_dtype, mode="none", bias=True, seed=31, shards=8)
    run_row_parallel(monkeypatch, case, 8)


@pytest.mark.parametrize("shape,full_tiled,shard_tiled", [("down_proj", True, False), ("o_proj", True, True)])
@pytest.mark.parametrize("W_dtype", ["uint4", "uint2"])
def test_row_parallel_shard_tiling(monkeypatch, shape, full_tiled, shard_tiled, W_dtype):
    """propagate_b at world 8: the full Llama-70B projection is slab-tiled; the down_proj shard (K = 3584: 1792 bytes per 4-bit
    row) is not, the o_proj shard (K = 1024) is at 4 bits.  The loader un-tiles the full weight and tiles the shard only where
    the shard operator does"""
    K = LLAMA70B_K[shape]
    if W_dtype == "uint2" and shape == "o_proj":
        shard_tiled = False   # 256 bytes per shard row
    case = X.make_exact_case(max(M_SET), 512, K, W_dtype=W_dtype, group_size=128, mode="quantized", bias=True, fast_decoding=True,
                             seed=K, propagate_b=True, shards=8)
    run_row_parallel(monkeypatch, case, 8, full_tiled=full_tiled, shard_tiled=shard_tiled)


# ---- column-parallel ------------------------------------------------------------------------------------------------------------
def column_case(M, N, K, i, **kw):
    """a column-parallel case; `i` picks the format, zeros mode and activation type"""
    W_dtype, mode = FORMATS[i % 12]
    args = dict(A_dtype=("float16", "bfloat16")[i % 2], W_dtype=W_dtype, out_dtype=OUTS[i % 3],
                group_size=128 if mode != "none" else -1, mode=mode, bias=i % 2 == 0, fast_decoding=i % 4 < 2, seed=100 + i)
    args.update(kw)
    return X.make_exact_case(M, N, K, **args)


def column_layers(monkeypatch, case, world, full_tiled=None, shard_tiled=None, **layer_kw):
    from bitblas_b200.parallel import ColumnParallelLinear
    N, K = case["N"], case["K"]
    per = N // world
    prove(case, [n_shard(case, r * per, (r + 1) * per) for r in range(world)])
    full_op, params = full_params(case)
    if full_tiled is not None:
        assert full_op.weight_tiled == full_tiled
    fg = FakeGroup(world, monkeypatch)
    layers = fg.build(lambda: ColumnParallelLinear(K, N, bias=case["bias"] is not None, out_dtype=case["cfg"]["out_dtype"],
                                                   **linear_kwargs(case), **layer_kw).cuda())
    for layer in layers:
        layer.load_full_params(*params)
    op = layers[0].local.bitblas_matmul
    assert op.N == per
    if shard_tiled is not None:
        assert op.weight_tiled == shard_tiled
    return fg, layers, op


def chunk_rows(layer, m):
    """the row counts of ColumnParallelLinear.forward's all-gather chunks"""
    n = layer._chunks_for(m)
    b = [(i * m) // n for i in range(n + 1)]
    return [b[i + 1] - b[i] for i in range(n) if b[i + 1] > b[i]]


@pytest.mark.parametrize("chunks", [None, 3])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_column_parallel_all_gather(monkeypatch, world, chunks):
    """fused_gather=False: the all-gather path, one collective per chunk of rows; the largest m comes as a 3-D input"""
    big, lead = (1100, (11, 100)) if chunks is None else (300, (3, 100))
    i = world + (chunks or 0)
    case = column_case(big, 1024, 2048, i, propagate_b=i % 2 == 1)
    fg, layers, op = column_layers(monkeypatch, case, world, fused_gather=False, pipeline_chunks=chunks)
    A = case["A"].to(DEV)
    ref = X.exact_reference(case, DEV).cpu()
    for m in (1, 4, 16, big):
        rows = chunk_rows(layers[0], m)
        assert (len(rows) > 1) == (m > 1 if chunks else m >= 1024), rows
        kernels = {assert_kernel(op, r) for r in rows}
        x = A[:m].reshape(*lead, case["K"]) if m == big else A[:m]
        n0 = fg.counts["all_gather"]
        outs = fg.run(lambda r: layers[r](x).cpu())
        assert fg.counts["all_gather"] == n0 + len(rows) and fg.counts["peer_barrier"] == 0
        compare_ranks([o.reshape(m, case["N"]) for o in outs], ref[:m],
                      f"column-parallel all-gather world={world} chunks={rows} m={m} ({sorted(kernels)})")
        assert outs[0].shape == (*x.shape[:-1], case["N"])


def _read_schedule(calls, ring, clone):
    """the call after which each result is read: a fused result stays valid until ring - 1 further calls have been issued
    (ColumnParallelLinear), with clone_output every result is kept to the end"""
    return {c: (calls - 1 if clone else min(calls - 1, c + ring - 2)) for c in range(calls)}


@pytest.mark.parametrize("ring,clone", [(2, False), (3, False), (2, True)], ids=["ring2", "ring3", "ring2-clone"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_column_parallel_fused(monkeypatch, world, ring, clone):
    """the fused path (scatter epilogue into every rank's buffer, then the barrier) at every m of M_SET, three calls per m with
    different rows, so the ring of buffers wraps at each m"""
    reps = 3
    i = 3 * world + ring + int(clone)
    case = column_case(reps * max(M_SET), 1024, 2048, i)
    fg, layers, op = column_layers(monkeypatch, case, world, fused_ring=ring, clone_output=clone)
    A = case["A"].to(DEV)
    ref = X.exact_reference(case, DEV).cpu()
    calls = [(m, slice(k * max(M_SET), k * max(M_SET) + m)) for m in M_SET for k in range(reps)]
    for m in M_SET:
        assert_kernel(op, m)
    read_after = _read_schedule(len(calls), ring, clone)

    def rank(r):
        got, live = {}, {}
        for c, (m, rows) in enumerate(calls):
            live[c] = layers[r](A[rows])
            for d in [d for d in live if read_after[d] == c]:
                got[d] = live.pop(d).cpu()
        return got

    outs = fg.run(rank)
    assert all(layer.fused_gather is True for layer in layers)
    assert fg.counts == {"all_reduce": 1, "all_gather": 0, "peer_barrier": len(calls)}, fg.counts
    for c, (m, rows) in enumerate(calls):
        compare_ranks([o[c] for o in outs], ref[rows], f"column-parallel fused world={world} ring={ring} clone={clone} call {c} "
                                                       f"m={m} ({expected_kernel(op, m)})")


def test_column_parallel_fused_generic_fallback(monkeypatch):
    """N / world = 192 rows: m > 32 dispatches the shard to generic_simt, which has no scatter epilogue, so that call (and only
    that call) takes the all-gather path on every rank"""
    world = 8
    case = column_case(64, 1536, 2048, 4)   # uint4, quantized zeros
    fg, layers, op = column_layers(monkeypatch, case, world, shard_tiled=False)
    A = case["A"].to(DEV)
    ref = X.exact_reference(case, DEV).cpu()
    for m, path in ((1, "peer_barrier"), (40, "all_gather"), (16, "peer_barrier"), (64, "all_gather"), (4, "peer_barrier")):
        kernel = assert_kernel(op, m)
        assert (kernel == "generic_simt") == (path == "all_gather")
        before = dict(fg.counts)
        outs = fg.run(lambda r: layers[r](A[:m]).cpu())
        assert layers[0].fused_gather is True
        assert fg.counts[path] == before[path] + 1, (m, before, fg.counts)
        compare_ranks(outs, ref[:m], f"column-parallel N=1536 world=8 m={m} ({kernel}, {path})")


@pytest.mark.parametrize("requested", [True, None])
def test_column_parallel_fused_decision(monkeypatch, requested):
    """one rank unable to fuse: the MIN over ranks turns the path off everywhere -- fused_gather=True raises on every rank,
    None falls back to the all-gather on every rank"""
    world = 4
    case = column_case(16, 1024, 2048, 2)
    fg, layers, op = column_layers(monkeypatch, case, world, fused_gather=requested)
    layers[2]._fused_supported_here = lambda x2: False
    A = case["A"].to(DEV)
    outs, errs = fg.run(lambda r: layers[r](A).cpu(), raise_errors=False)
    assert fg.counts["all_reduce"] == 1 and fg.counts["peer_barrier"] == 0 and not fg.rings
    if requested:
        assert all(isinstance(e, RuntimeError) and "cannot use it" in str(e) for e in errs), errs
        return
    assert errs == [None] * world, errs
    assert all(layer.fused_gather is False for layer in layers)
    assert fg.counts["all_gather"] == 1
    assert_kernel(op, 16)
    compare_ranks(outs, X.exact_reference(case, DEV).cpu(), "column-parallel, fused path declined by one rank")


@pytest.mark.parametrize("N,full_tiled,shard_tiled", [(1536, True, False), (1024, True, True)], ids=["shard_row_major", "shard_tiled"])
def test_column_parallel_shard_tiling(monkeypatch, N, full_tiled, shard_tiled):
    """propagate_b at world 8 with 1024 bytes per row: the full weight is slab-tiled; a 192-row shard is not, a 128-row shard is.
    The loader un-tiles the full weight and tiles the shard only where the shard operator does.  Fused path where the shard's
    kernel has the scatter epilogue, the all-gather otherwise"""
    world = 8
    case = X.make_exact_case(max(M_SET), N, 2048, group_size=128, mode="quantized", bias=True, fast_decoding=True, seed=N,
                             propagate_b=True)
    fg, layers, op = column_layers(monkeypatch, case, world, full_tiled=full_tiled, shard_tiled=shard_tiled)
    A = case["A"].to(DEV)
    ref = X.exact_reference(case, DEV).cpu()
    for m in M_SET + (40,):
        kernel = assert_kernel(op, m)
        before = dict(fg.counts)
        outs = fg.run(lambda r: layers[r](A[:m]).cpu())
        path = "all_gather" if kernel == "generic_simt" else "peer_barrier"
        assert fg.counts[path] > before[path], (m, kernel, before, fg.counts)
        compare_ranks(outs, ref[:m], f"column-parallel N={N} world=8 m={m} ({kernel})")
