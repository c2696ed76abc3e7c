"""H100-native WVA optimization hot path (queueing sizer, allocator, saturation model, limiter).

The compute lives in csrc/ (hand-written sm_90a CUDA behind the C-ABI of
include/wva_b200.h).  This package is the Python binding used by tests/ and
bench.py; the Go binding a maintainer would add is shown in INTEGRATION.md.
There is no CPU fallback: constructing an Engine without the built CUDA library
or without a GPU raises.
"""
from . import _abi, sharding, synth  # noqa: F401
from . import engine, manager, pipeline  # noqa: F401
from .engine import Engine, Group, Ingest, IngestV2, K2History, WvaError, comm_unique_id, lib_path, load_library, pinned_copy, pinned_empty  # noqa: F401
from .manager import Manager, flatten_spec  # noqa: F401
from .pipeline import (CapacityKnowledgeStore, CostAwareOptimizer, Enforcer, Limiter, SaturationAnalyzer,  # noqa: F401
                       SaturationAnalyzerV2, ingest_v2_decisions, optimize_v2)
