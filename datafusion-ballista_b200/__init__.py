"""CUDA-native (H100, sm_90a) execution engine for Apache DataFusion Ballista's executor hot path.

Host-side mirror (Python harness) of the reference plug-in interface
``ExecutionEngine`` / ``QueryStageExecutor`` (ballista/executor/src/execution_engine.rs:45-81) on
top of the C-ABI library ``libb200exec.so`` (include/b200exec.h).  All compute happens in the CUDA
library; this package only marshals Arrow C Data Interface structs and plan JSON.
"""
from . import plan, tpch, driver, engine  # noqa: F401
from .engine import GpuExecutionEngine, QueryStageExecutor, ShuffleWritePartition, B200Error  # noqa: F401

__all__ = ["plan", "tpch", "driver", "engine", "GpuExecutionEngine", "QueryStageExecutor", "ShuffleWritePartition", "B200Error"]
