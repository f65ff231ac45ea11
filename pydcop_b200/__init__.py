"""pydcop_b200 — batched factor-graph message passing on the H100 for pyDcop's MaxSum / DSA hot path.

Public API:
    build_layout / layout_from_instance   host packing of a factor graph (pydcop_b200.layout)
    MaxSumEngine / DsaEngine              GPU engines over the C-ABI (pydcop_b200.engine)
    pydcop_b200.algorithms.{maxsum_gpu,dsa_gpu}   drop-in pyDcop algorithm modules
    pydcop_b200.ingest                    YAML / pyDcop objects / binary container -> arrays
    pydcop_b200.solve                     file or arrays -> engine -> pyDcop's result dict
"""
from .layout import FactorGraphLayout, build_layout, layout_from_instance  # noqa: F401

__all__ = ["FactorGraphLayout", "build_layout", "layout_from_instance", "MaxSumEngine", "DsaEngine"]


def __getattr__(name):  # lazy: importing the package must not require torch / the .so
    if name in ("MaxSumEngine", "DsaEngine", "EngineError"):
        from . import engine
        return getattr(engine, name) if name != "EngineError" else engine.EngineError
    raise AttributeError(name)
