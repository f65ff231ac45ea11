"""syncbb_gpu through the UNMODIFIED reference orchestrator (thread mode), with the SyncBB oracle behind the engine
seam: module surface, registration, value reporting and the run's metrics against the reference's own `syncbb` run,
without a GPU."""
import os

import numpy as np
import pytest

import ref_shim
from _syncbb_oracle import SyncbbOracle
from test_syncbb_cpu import load

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


class SyncbbOracleEngine:
    """SyncbbEngine's driving API (init / step / finished / values / bounds) over the oracle.  The session packs
    the variables in name order, so the chain is the canonical order."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "syncbb"
        self.o = SyncbbOracle(inst, np.float64, params["mode"])

    def init(self):
        self.o.init()
        return self

    def step(self, n=1):
        self.o.run(n)
        return self

    @property
    def finished(self):
        return self.o.finished

    def values(self):
        return self.o.values()

    @property
    def cycle(self):
        return int(self.o.cycle_counts().max())

    def cycle_counts(self):
        return self.o.cycle_counts()

    def bounds(self):
        return self.o.bounds()


@pytest.fixture(scope="module")
def pydcop_ready():
    ref_shim.install()
    import logging
    logging.disable(logging.CRITICAL)
    from pydcop_b200 import launcher
    launcher.install()
    yield
    logging.disable(logging.NOTSET)


@pytest.fixture
def oracle_seam(pydcop_ready):
    from pydcop_b200.algorithms._session import GpuSession
    GpuSession.reset()
    GpuSession.engine_factory = SyncbbOracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


def orchestrated(algo_name, dcop):
    from pydcop.algorithms import AlgorithmDef
    from pydcop.computations_graph import ordered_graph
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    algo = AlgorithmDef.build_with_default_param(algo_name, {}, mode=dcop.objective)
    cg = ordered_graph.build_computation_graph(dcop)
    orchestrator = run_local_thread_dcop(algo, cg, oneagent.distribute(cg, dcop.agents.values()), dcop, 1e9)
    try:
        orchestrator.deploy_computations()
        orchestrator.run(timeout=60)
        metrics = orchestrator.end_metrics()
        status = orchestrator.status
    finally:
        orchestrator.stop_agents(5)
        orchestrator.stop()
    return status, metrics


def load_yaml(instance):
    from pydcop.dcop.yamldcop import load_dcop_from_file
    return load_dcop_from_file([os.path.join(ref_shim.INSTANCES, instance)])


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    assert "syncbb_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("syncbb"), load_algorithm_module("syncbb_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "ordered_graph"
    assert {p.name for p in gpu.algo_params} == {"precision", "seed", "session"}
    assert not getattr(ref, "algo_params", [])


@needs_ref
@pytest.mark.parametrize("instance,fixture", [("graph_coloring_tuto.yaml", "syncbb_tuto"),
                                              ("graph_coloring_csp.yaml", "syncbb_gc_csp")])
def test_orchestrated_run_matches_the_reference_run(oracle_seam, instance, fixture):
    """syncbb_gpu gives the fixture's assignment, and the status and cycle of the reference's own orchestrated
    `syncbb` run (the largest per-variable new_cycle count).  Its msg_count leaves out the SyncBB messages, which
    the proxies do not post: the reference's exceeds it by at least their number."""
    ref_status, ref_metrics = orchestrated("syncbb", load_yaml(instance))
    dcop = load_yaml(instance)
    status, metrics = orchestrated("syncbb_gpu", dcop)
    assert status == ref_status and status not in ("TIMEOUT", "STOPPED"), (status, ref_status)
    inst, _ = load(fixture)
    assert metrics["cycle"] == ref_metrics["cycle"] == int(inst["cycle_count"].max()) > 0
    assert metrics["assignment"] == ref_metrics["assignment"]
    assert ref_metrics["msg_count"] - metrics["msg_count"] >= int(inst["msg_count"])
    names = [str(n) for n in inst["var_names"]]
    doms = [list(dcop.variables[n].domain) for n in names]
    assert [doms[i].index(metrics["assignment"][n]) for i, n in enumerate(names)] == inst["final_sel"].tolist()
    assert metrics["cost"] == ref_metrics["cost"] and metrics["violation"] == ref_metrics["violation"]


@needs_ref
def test_orchestrated_infeasible_run_reports_no_values(oracle_seam):
    """Every full assignment costs inf: no variable ever selects a value, with the reference as with the proxies,
    and the orchestrator reports an incomplete assignment."""
    import sys
    from pydcop.dcop.dcop import DCOP
    from pydcop.dcop.objects import AgentDef
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import make_golden_syncbb as M

    def build():
        vs, cs = M.infeasible()
        dcop = DCOP("infeasible", "min")
        for c in cs:
            dcop.add_constraint(c)
        dcop.add_agents([AgentDef(f"a{i}") for i in range(len(vs))])
        return dcop
    ref_status, ref_metrics = orchestrated("syncbb", build())
    status, metrics = orchestrated("syncbb_gpu", build())
    assert status == ref_status and status not in ("TIMEOUT", "STOPPED"), (status, ref_status)
    assert metrics["assignment"] == ref_metrics["assignment"] == {}
    assert metrics["cost"] is ref_metrics["cost"] is None


@needs_ref
def test_arity3_refused_when_built(pydcop_ready):
    from pydcop.algorithms import AlgorithmDef, ComputationDef
    from pydcop.computations_graph import ordered_graph
    from pydcop_b200.algorithms import syncbb_gpu
    from test_syncbb_cpu import _golden_driver
    vs, cs = _golden_driver().arity3()
    g = ordered_graph.build_computation_graph(None, variables=vs, constraints=cs)
    algo = AlgorithmDef.build_with_default_param("syncbb_gpu", {}, mode="min")
    with pytest.raises(ValueError, match="constraint abc has arity 3"):
        for node in g.nodes:
            syncbb_gpu.build_computation(ComputationDef(node, algo))
