"""gdba_gpu through the UNMODIFIED reference orchestrator (thread mode) and `solve(..., "gdba")`, with
the GDBA oracle behind the engine seam: the plugin plumbing (module surface, registration, value
reporting, cycle counting, FINISHED status at stop_cycle) without a GPU.  The kernels are the GPU tests' job."""
import os

import numpy as np
import pytest

import ref_shim
from _gdba_oracle import GdbaOracle

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


class GdbaOracleEngine:
    """GdbaEngine's driving API (init / step / finished / values) over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "gdba"
        keys = ("modifier", "violation", "increase_mode", "stop_cycle", "seed")
        self.o = GdbaOracle(dict(inst), np.float64, mode=params["mode"], **{k: params[k] for k in keys if k in params})

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
    GpuSession.engine_factory = GdbaOracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    assert "gdba_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("gdba"), load_algorithm_module("gdba_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "constraints_hypergraph"
    params = {p.name: p for p in gpu.algo_params}
    for p in ref.algo_params:
        assert params[p.name] == p
    assert {"stop_cycle", "precision", "seed", "session"} <= set(params)
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    for node in constraints_hypergraph.build_computation_graph(dcop).nodes:
        nbrs = {v.name for c in node.constraints for v in c.dimensions} - {node.name}
        assert gpu.computation_memory(node) == len(nbrs) * ref.UNIT_SIZE
        with pytest.raises(AttributeError):       # the reference reads `.nodes` on neighbour names
            ref.computation_memory(node)
        for nb in node.neighbors:
            assert gpu.communication_load(node, nb) == ref.communication_load(node, nb)


@needs_ref
def test_orchestrated_run_finishes_at_stop_cycle(oracle_seam):
    from pydcop.algorithms import AlgorithmDef, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    module = load_algorithm_module("gdba_gpu")
    algo = AlgorithmDef.build_with_default_param("gdba_gpu", {"stop_cycle": 30, "seed": 5, "increase_mode": "T"},
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
    _, cost = dcop.solution_cost(metrics["assignment"], 1e9)
    assert metrics["cost"] == pytest.approx(cost)


def test_solve_through_the_seam():
    from pydcop_b200 import solve as S
    from pydcop_b200.ingest import load_yaml
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instances", "graph_coloring1.yaml")
    res = S.solve(path, "gdba", {"stop_cycle": 20, "increase_mode": "R", "modifier": "M"}, seed=3,
                  engine_factory=GdbaOracleEngine)
    assert res["status"] == "FINISHED" and res["cycle"] == 20 and res["algo"] == "gdba"
    d = load_yaml(path)
    assert d.n_vars == 3 and set(res["assignment"]) == {"v1", "v2", "v3"}
    assert S.check_params("gdba", None) == {"modifier": "A", "violation": "NZ", "increase_mode": "E", "stop_cycle": 0}
    assert S.check_params("gdba", {"violation": "MX"})["violation"] == "MX"
    for bad in ({"modifier": "B"}, {"violation": "NN"}, {"increase_mode": "X"}, {"favor": "no"}):
        with pytest.raises(ValueError):
            S.check_params("gdba", bad)
    assert S.ALGOS["gdba_gpu"] == "gdba"


@needs_ref
def test_solve_parameters_are_the_reference_algo_params(pydcop_ready):
    """`solve` accepts exactly the reference's parameters (plus stop_cycle) with the same choices and defaults."""
    from pydcop.algorithms import load_algorithm_module
    from pydcop_b200 import solve as S
    ref = load_algorithm_module("gdba")
    assert set(S.GDBA_DEFAULTS) == {p.name for p in ref.algo_params} | {"stop_cycle"}
    for p in ref.algo_params:
        assert S.GDBA_DEFAULTS[p.name] == p.default_value
        assert tuple(S._CHOICES[p.name]) == tuple(p.values)


def test_not_sharded():
    """Under torchrun, gdba is refused as mgm is (a one-rank gloo group stands in for torchrun)."""
    import socket

    import torch.distributed as dist
    from pydcop_b200 import solve as S
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instances", "graph_coloring1.yaml")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        with pytest.raises(ValueError, match="gdba is not sharded"):
            S.solve(path, "gdba", {"stop_cycle": 5}, distributed=True, sharded_kwargs={"engine_factory": object})
    finally:
        dist.destroy_process_group()


def test_engine_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from pydcop_b200 import EngineError
    from pydcop_b200.engine import GdbaEngine
    from pydcop_b200.generators import random_factor_graph
    from pydcop_b200.layout import layout_from_instance
    with pytest.raises(EngineError):
        GdbaEngine(layout_from_instance(random_factor_graph(50, 3, 60, 2, seed=1)))
