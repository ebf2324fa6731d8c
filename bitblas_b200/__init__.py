"""bitblas_b200 -- a H100-native (sm_90a) implementation of the BitBLAS low-bit-weight matmul operator API.

Public surface mirrors ``bitblas/__init__.py:169-175``: ``Matmul``, ``MatmulConfig``, ``Linear``,
``auto_detect_nvidia_target``, ``set_log_level``, ``__version__`` (+ ``bitblas.cache``, ``bitblas.quantization``,
``bitblas.testing``).  ``import bitblas`` resolves to this package through the ``bitblas/`` alias at the repo root.
"""
import logging

__version__ = "0.1.0"

logger = logging.getLogger("bitblas")


def set_log_level(level):
    """bitblas/__init__.py:39-55."""
    if isinstance(level, str):
        level = getattr(logging, level.upper(), logging.INFO)
    logging.getLogger("bitblas").setLevel(level)
    logging.getLogger(__name__).setLevel(level)


from .ops.operator import OperatorConfig, Operator, TransformKind, OptimizeStrategy  # noqa: E402,F401
from .ops.general_matmul import Matmul, MatmulConfig  # noqa: E402,F401
from .module import Linear  # noqa: E402,F401
from .utils import auto_detect_nvidia_target  # noqa: E402,F401
from . import cache, quantization, testing  # noqa: E402,F401
from .parallel import ColumnParallelLinear  # noqa: E402,F401
from .graph import CapturedStep  # noqa: E402,F401
