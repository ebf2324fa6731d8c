"""Operator base: what survives of bitblas/ops/operator.py once TVM is gone.

Keeps the attributes callers touch (``lib``, ``profile_latency``, ``hardware_aware_finetune``, ``get_source``,
``cleanup``; reference: bitblas/ops/operator.py:133,347-382,442-463) -- there is nothing to compile or tune at
construction time, every configuration is served by the prebuilt sm_90a library.
"""
from __future__ import annotations

from dataclasses import dataclass
from enum import IntEnum


class TransformKind(IntEnum):  # bitblas/base/operator_common.py
    NonTransform = 0
    InterWarpTransform = 1
    IntraWarpTransform = 2
    LDMatrixTransform = 3


class OptimizeStrategy(IntEnum):  # bitblas/base/operator_common.py
    SingleBatchDecodeOnly = 0
    ContigousBatching = 1


@dataclass(frozen=True)
class OperatorConfig:
    """Base class for operator configurations (bitblas/ops/operator.py:38-41)."""
    pass


class Operator:
    def __init__(self, name: str, config: OperatorConfig, target=None, backend: str = "b200"):
        self.name = name
        self.config = config
        self.target = target
        self.backend = backend
        self.lib = None
        self.profile_tensors = None

    def hardware_aware_finetune(self, topk: int = 20, target=None, parallel_build: bool = True):
        """No-op: kernels are hand-written for sm_90a; selection is a run-time dispatch on m."""
        return None

    def get_source(self, target=None, kenrel_only: bool = False) -> str:
        raise NotImplementedError

    def cleanup(self):
        pass

    def is_tir_backend(self):
        return False

    def is_tilelang_backend(self):
        return False
