"""vectordb_b200 — H100-native (sm_90a) vector-search hot path of Epsilla behind a C ABI.

The product is ``libepsilla_b200.so`` (hand-written CUDA, ``csrc/``) declared in
``include/epsilla_b200.h``.  This package is the thin Python host layer used by the tests and
``bench.py``: a ctypes loader that FAILS LOUDLY when the library is missing (there is no CPU
fallback) and an ``Index`` class (and ``SparseIndex`` for sparse-vector fields) that mirrors the C ABI one-to-one.
"""
from .lib import load_library, library_path, EpsError  # noqa: F401
from .index import Index, SparseIndex, Stats, METRICS, filter_nodes_array  # noqa: F401

__all__ = ["load_library", "library_path", "EpsError", "Index", "SparseIndex", "Stats", "METRICS", "filter_nodes_array"]
