"""mgm2_gpu through the UNMODIFIED reference orchestrator (thread mode) and `solve(..., "mgm2")`, with
the MGM-2 oracle behind the engine seam: the plugin plumbing (module surface, registration, value
reporting, cycle counting, FINISHED status) without a GPU.  The kernels are the GPU tests' job."""
import os

import numpy as np
import pytest

import ref_shim
from _mgm2_oracle import Mgm2Oracle

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


class Mgm2OracleEngine:
    """Mgm2Engine's driving API (init / step / finished / values) over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "mgm2"
        keys = ("threshold", "favor", "stop_cycle", "seed")
        self.o = Mgm2Oracle(dict(inst), np.float64, mode=params["mode"], **{k: params[k] for k in keys if k in params})

    def init(self):
        self.o.init()
        return self

    def step(self, n=1):
        self.o.step(n)
        return self

    @property
    def finished(self):
        return self.o.finished

    def values(self):
        return self.o.values()


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
    GpuSession.engine_factory = Mgm2OracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


def two_opt(dcop, assignment):
    """No single variable and no pair of neighbours can lower the cost (min mode)."""
    _, cost = dcop.solution_cost(assignment, 1e9)
    variables = list(dcop.variables.values())
    for v in variables:
        for x in v.domain:
            assert dcop.solution_cost(dict(assignment, **{v.name: x}), 1e9)[1] >= cost - 1e-9, (v.name, x)
    for c in dcop.constraints.values():
        names = [v.name for v in c.dimensions]
        for i, a in enumerate(names):
            for b in names[i + 1:]:
                for x in dcop.variable(a).domain:
                    for y in dcop.variable(b).domain:
                        _, c2 = dcop.solution_cost(dict(assignment, **{a: x, b: y}), 1e9)
                        assert c2 >= cost - 1e-9, (a, x, b, y)
    return cost


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    assert "mgm2_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("mgm2"), load_algorithm_module("mgm2_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "constraints_hypergraph"
    params = {p.name: p for p in gpu.algo_params}
    for p in ref.algo_params:
        assert params[p.name] == p
    assert {"precision", "seed", "session"} <= set(params)
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    for node in constraints_hypergraph.build_computation_graph(dcop).nodes:
        assert gpu.computation_memory(node) == ref.computation_memory(node)
        for nb in node.neighbors:
            assert gpu.communication_load(node, nb) == ref.communication_load(node, nb)
        with pytest.raises(ValueError):
            gpu.communication_load(node, "no_such_variable")


@needs_ref
def test_orchestrated_run_finishes_at_stop_cycle_on_a_2opt_point(oracle_seam):
    from pydcop.algorithms import AlgorithmDef, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    module = load_algorithm_module("mgm2_gpu")
    algo = AlgorithmDef.build_with_default_param("mgm2_gpu", {"stop_cycle": 30, "seed": 5, "favor": "coordinated"},
                                                 mode=dcop.objective)
    cg = constraints_hypergraph.build_computation_graph(dcop)
    dist = oneagent.distribute(cg, dcop.agents.values(), computation_memory=module.computation_memory,
                               communication_load=module.communication_load)
    orchestrator = run_local_thread_dcop(algo, cg, dist, dcop, 1e9)
    try:
        orchestrator.deploy_computations()
        orchestrator.run(timeout=60)
        metrics = orchestrator.end_metrics()
        status = orchestrator.status
    finally:
        orchestrator.stop_agents(5)
        orchestrator.stop()
    assert status not in ("TIMEOUT", "STOPPED"), status
    assert metrics["cycle"] == 30            # the session's cycle count, as for mgm_gpu
    assert set(metrics["assignment"]) == {f"v{i}" for i in range(10)}
    cost = two_opt(dcop, metrics["assignment"])
    assert metrics["cost"] == pytest.approx(cost)


def test_solve_through_the_seam():
    from pydcop_b200 import solve as S
    from pydcop_b200.ingest import load_yaml
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instances", "graph_coloring1.yaml")
    res = S.solve(path, "mgm2", {"stop_cycle": 20, "threshold": "0.7"}, seed=3, engine_factory=Mgm2OracleEngine)
    assert res["status"] == "FINISHED" and res["cycle"] == 20 and res["algo"] == "mgm2"
    assert res["assignment"] in ({"v1": "R", "v2": "G", "v3": "R"}, {"v1": "G", "v2": "R", "v3": "G"})
    d = load_yaml(path)
    assert S.check_params("mgm2", {"favor": "no"})["favor"] == "no"
    with pytest.raises(ValueError):
        S.check_params("mgm2", {"favor": "sometimes"})
    with pytest.raises(ValueError):
        S.check_params("mgm2", {"break_mode": "lexic"})
    assert S.check_params("mgm2", None) == {"threshold": 0.5, "favor": "unilateral", "stop_cycle": 0}
    assert d.n_vars == 3
    assert S.ALGOS["mgm2_gpu"] == "mgm2"


def test_engine_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pydcop_b200 import EngineError
    from pydcop_b200.engine import Mgm2Engine
    from pydcop_b200.generators import random_factor_graph
    from pydcop_b200.layout import layout_from_instance
    with pytest.raises(EngineError):
        Mgm2Engine(layout_from_instance(random_factor_graph(50, 3, 60, 2, seed=1)))
