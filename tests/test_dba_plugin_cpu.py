"""dba_gpu through the UNMODIFIED reference orchestrator (thread mode) and `solve(..., "dba")`, with the DBA oracle
behind the engine seam: the plugin plumbing (module surface, registration, value reporting, per-variable finish,
early FINISHED status) without a GPU.  The kernels are the GPU tests' job."""
import os

import numpy as np
import pytest

import ref_shim
from _dba_oracle import LIVE, DbaOracle

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
CSP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instances", "graph_coloring_csp.yaml")


class DbaOracleEngine:
    """DbaEngine's driving API (init / step / finished / cycle / values / finished_vars) over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "dba"
        keys = ("infinity", "max_distance", "stop_cycle", "seed")
        self.o = DbaOracle(dict(inst), np.float64, mode=params["mode"], **{k: params[k] for k in keys if k in params})

    def init(self):
        self.o.init()
        return self

    def step(self, n=1):
        self.o.step(n)
        return self

    @property
    def finished(self):
        return self.o.finished

    @property
    def cycle(self):
        return self.o.cycle

    def values(self):
        return self.o.values()

    def finished_vars(self):
        return np.array(self.o.finish) != LIVE


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
    GpuSession.engine_factory = DbaOracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    assert "dba_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("dba"), load_algorithm_module("dba_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "constraints_hypergraph"
    params = {p.name: p for p in gpu.algo_params}
    for p in ref.algo_params:
        assert params[p.name] == p
    assert set(params) == {p.name for p in ref.algo_params} | {"stop_cycle", "precision", "seed", "session"}
    for path in (CSP, os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")):
        dcop = load_dcop_from_file([path])
        for node in constraints_hypergraph.build_computation_graph(dcop).nodes:
            assert gpu.computation_memory(node) == ref.computation_memory(node)
            for nb in node.neighbors:
                assert gpu.communication_load(node, nb) == ref.communication_load(node, nb)


@needs_ref
def test_computation_memory_substring_test(pydcop_ready):
    """The reference drops every neighbour whose name is a substring of the variable's own name."""
    from pydcop.algorithms import load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.objects import Domain, Variable
    from pydcop.dcop.relations import NAryMatrixRelation
    ref, gpu = load_algorithm_module("dba"), load_algorithm_module("dba_gpu")
    d = Domain("d", "", [0, 1])
    v1, v12, v2 = Variable("v1", d), Variable("v12", d), Variable("v2", d)
    cs = [NAryMatrixRelation([v12, v1], np.zeros((2, 2)), name="a"),
          NAryMatrixRelation([v12, v2], np.zeros((2, 2)), name="b")]
    g = constraints_hypergraph.build_computation_graph(None, variables=[v1, v12, v2], constraints=cs)
    node = next(n for n in g.nodes if n.name == "v12")
    assert gpu.computation_memory(node) == ref.computation_memory(node) == 5   # v1 is dropped, v2 counted


def orchestrated_run(params, timeout=60):
    """dba_gpu on graph_coloring_csp.yaml through the unmodified thread-mode orchestrator: (status, end metrics)."""
    from pydcop.algorithms import AlgorithmDef, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    dcop = load_dcop_from_file([CSP])
    module = load_algorithm_module("dba_gpu")
    algo = AlgorithmDef.build_with_default_param("dba_gpu", params, mode=dcop.objective)
    cg = constraints_hypergraph.build_computation_graph(dcop)
    dist = oneagent.distribute(cg, dcop.agents.values(), computation_memory=module.computation_memory,
                               communication_load=module.communication_load)
    orchestrator = run_local_thread_dcop(algo, cg, dist, dcop, 1e9)
    try:
        orchestrator.deploy_computations()
        orchestrator.run(timeout=timeout)
        return orchestrator.status, orchestrator.end_metrics()
    finally:
        orchestrator.stop_agents(5)
        orchestrator.stop()


@needs_ref
def test_orchestrated_run_finishes_with_the_flood(oracle_seam):
    """graph_coloring_csp.yaml: every variable has a neighbour, so every proxy finishes when its variable does and
    the orchestrator ends before its timeout, with a consistent colouring."""
    status, metrics = orchestrated_run({"max_distance": 3, "seed": 5})
    assert status not in ("TIMEOUT", "STOPPED"), status
    assert set(metrics["assignment"]) == {"v1", "v2", "v3"}
    a = metrics["assignment"]
    assert a["v1"] != a["v2"] and a["v2"] != a["v3"]
    from pydcop_b200.algorithms._session import GpuSession
    snap = GpuSession.last("dba:default").snapshot
    assert snap.done == {"v1", "v2", "v3"} and not snap.finished and snap.cycle > 0


@needs_ref
@pytest.mark.parametrize("stop_cycle", [11, 12, 21, 25])
def test_orchestrated_run_finishes_at_stop_cycle(oracle_seam, stop_cycle):
    """max_distance 0: no variable ever stops, so only stop_cycle ends the run.  The engine runs stop_cycle - 1
    rounds; every proxy finishes then, whether or not that count is a multiple of the session's chunk of rounds."""
    from pydcop_b200.algorithms._session import GpuSession
    assert GpuSession("probe", "dba").cycles_per_poll == 10      # 11 and 21: the engine ends on a chunk boundary
    status, metrics = orchestrated_run({"max_distance": 0, "seed": 5, "stop_cycle": stop_cycle}, timeout=30)
    assert status not in ("TIMEOUT", "STOPPED"), status
    snap = GpuSession.last("dba:default").snapshot
    assert snap.finished and snap.cycle == stop_cycle - 1 and not snap.done
    assert metrics["cycle"] == stop_cycle - 1 and set(metrics["assignment"]) == {"v1", "v2", "v3"}


def test_solve_through_the_seam():
    from pydcop_b200 import solve as S
    res = S.solve(CSP, "dba", {"max_distance": 3, "stop_cycle": 100}, seed=3, engine_factory=DbaOracleEngine)
    assert res["status"] == "FINISHED" and 0 < res["cycle"] < 99 and res["algo"] == "dba"
    assert res["violation"] == 0 and res["cost"] == 0
    res = S.solve(CSP, "dba", {"max_distance": 0, "stop_cycle": 20}, seed=3, engine_factory=DbaOracleEngine)
    assert res["status"] == "FINISHED" and res["cycle"] == 19          # rounds run = stop_cycle - 1
    assert S.check_params("dba", None) == {"infinity": 10000, "max_distance": 50, "stop_cycle": 0}
    for bad in ({"max_distance": "x"}, {"modifier": "A"}):
        with pytest.raises(ValueError):
            S.check_params("dba", bad)
    assert S.ALGOS["dba_gpu"] == "dba"


def test_solve_refuses_max_mode():
    from pydcop_b200 import solve as S
    path = os.path.join(os.path.dirname(CSP), "graph_coloring_tuto_max.yaml")
    with pytest.raises(ValueError, match="only support minimization"):
        S.solve(path, "dba", {"stop_cycle": 5}, engine_factory=DbaOracleEngine)


@needs_ref
def test_solve_parameters_are_the_reference_algo_params(pydcop_ready):
    from pydcop.algorithms import load_algorithm_module
    from pydcop_b200 import solve as S
    ref = load_algorithm_module("dba")
    assert set(S.DBA_DEFAULTS) == {p.name for p in ref.algo_params} | {"stop_cycle"}
    for p in ref.algo_params:
        assert S.DBA_DEFAULTS[p.name] == p.default_value


def test_not_sharded():
    import socket

    import torch.distributed as dist
    from pydcop_b200 import solve as S
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        with pytest.raises(ValueError, match="dba is not sharded"):
            S.solve(CSP, "dba", {"stop_cycle": 5}, distributed=True, sharded_kwargs={"engine_factory": object})
    finally:
        dist.destroy_process_group()


def test_engine_refuses_max_mode_and_fails_loudly_without_gpu():
    import torch
    from pydcop_b200 import EngineError
    from pydcop_b200.engine import DbaEngine
    from pydcop_b200.generators import random_factor_graph
    from pydcop_b200.layout import layout_from_instance
    L = layout_from_instance(random_factor_graph(50, 3, 60, 2, seed=1))
    with pytest.raises(ValueError, match="only support minimization"):
        DbaEngine(L, mode="max")
    if not torch.cuda.is_available():
        with pytest.raises(EngineError):
            DbaEngine(L)
