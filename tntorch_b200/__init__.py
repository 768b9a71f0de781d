"""tntorch_b200 — H100-native (sm_90a) decomposition / rounding hot path of rballester/tntorch.

Drop-in surface for that path: ``Tensor(data, ranks_tt=/eps=)``, ``Tensor.round_tt``, ``round_tt``,
``round``, ``truncated_svd``, ``relative_error``, ``Tensor(data, ranks_cp=)`` (CP-ALS), ``cross`` (TT-cross).  Importing does not need a GPU; every compute call does.
"""
from .round import reduce, relative_error, round, round_tt, round_tucker, truncated_svd  # noqa: F401
from .tensor import Tensor  # noqa: F401
from .cross import cross, cross_forward, meshgrid  # noqa: F401
from .cross_batch import cross_batch  # noqa: F401
from .callers import TTMatrix, dot, hadamard_sum, shift_mode  # noqa: F401
from . import ops  # noqa: F401

__version__ = "0.1.0"
