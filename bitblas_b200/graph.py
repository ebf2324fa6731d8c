"""CUDA-graph capture of a fixed sequence of operator calls (a decode step).

The reference removes per-call host overhead with a tracing compiler around its generated kernels; on H100 the idiomatic tool is a
CUDA graph: the operators of this package never allocate, synchronise or read host state inside ``forward`` once their workspace
exists (include/bitblas_b200.h), the decode kernel's launch parameters do not change between replays (its stream-K nonce lives in
slots that every replay resets), and the programmatic-dependent-launch edges between consecutive matmuls survive capture.  A
decode step -- host activations in, a chain of ``Matmul`` / ``Linear`` calls on static device buffers, results out -- then costs ONE
``cudaGraphLaunch`` instead of one Python call, one ctypes call and one launch per projection.

    step = CapturedStep(lambda: [op(a_dev, W, scale=s, zeros=z, output=c_dev) for ...],
                        h2d=[(a_dev, a_host_pinned)], d2h=[(c_host_pinned, c_dev)])
    a_host_pinned.copy_(new_activations); step.run(); step.wait()      # results are in c_host_pinned
"""
from __future__ import annotations

from typing import Callable, Iterable, Optional, Tuple

import torch


class CapturedStep:
    """Captures ``[h2d copies] -> fn() -> [d2h copies]`` on a private stream into one CUDA graph.

    ``fn`` must only touch pre-allocated tensors (the usual CUDA-graph contract); host buffers in ``h2d`` / ``d2h`` must be pinned.
    ``warmup`` un-captured runs come first so that every operator has its per-stream workspace and its kernels their attributes."""

    def __init__(self, fn: Callable[[], object], *, h2d: Iterable[Tuple[torch.Tensor, torch.Tensor]] = (),
                 d2h: Iterable[Tuple[torch.Tensor, torch.Tensor]] = (), device: Optional[torch.device] = None, warmup: int = 2):
        self.h2d = list(h2d)
        self.d2h = list(d2h)
        for dst, src in self.h2d:
            if not (dst.is_cuda and not src.is_cuda and src.is_pinned()):
                raise ValueError("h2d pairs are (device tensor, pinned host tensor)")
        for dst, src in self.d2h:
            if not (src.is_cuda and not dst.is_cuda and dst.is_pinned()):
                raise ValueError("d2h pairs are (pinned host tensor, device tensor)")
        dev = device
        if dev is None:
            cand = [t for t, _ in self.h2d] + [s for _, s in self.d2h]
            dev = cand[0].device if cand else torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.stream = torch.cuda.Stream(device=dev)
        self._fn = fn

        def body():
            for dst, src in self.h2d:
                dst.copy_(src, non_blocking=True)
            fn()
            for dst, src in self.d2h:
                dst.copy_(src, non_blocking=True)

        self.stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(self.stream):
            for _ in range(max(1, warmup)):
                body()
            self.stream.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                body()
        self.stream.synchronize()

    def run(self):
        """enqueue one replay on the step's stream (asynchronous)"""
        with torch.cuda.stream(self.stream):
            self.graph.replay()

    def wait(self):
        """block the host until the last replay's d2h copies have landed"""
        self.stream.synchronize()

    def __call__(self):
        self.run()
        self.wait()


__all__ = ["CapturedStep"]
