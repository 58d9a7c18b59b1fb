"""dfgpu — H100-native (sm_90a) engine for DataFusion 0.6.0's Arrow-batch hot path:
FilterRelation / ProjectRelation / AggregateRelation behind the reference's operator API.

Layout: csrc/ (CUDA kernels + C ABI of include/dfgpu.h + the C++ host mirror of the reference's
Relation / ExecutionContext API), engine.py (ctypes view of the C ABI for tests and bench.py),
expr.py (Python mirror of the reference's Expr IR for writing tests)."""
from . import _abi  # noqa: F401

__all__ = ["_abi", "engine", "expr"]
