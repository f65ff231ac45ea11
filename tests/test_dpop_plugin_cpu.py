"""dpop_gpu through the UNMODIFIED reference orchestrator (thread mode) and `solve(..., "dpop")`, with the
DPOP oracle behind the engine seam: module surface, registration, the tree taken from the nodes' links,
value reporting and the run's metrics against the reference's own `dpop` run, without a GPU."""
import contextlib
import os

import numpy as np
import pytest

import ref_shim
from _dpop_oracle import DpopOracle
from test_dpop_cpu import load

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")


class DpopOracleEngine:
    """DpopEngine's driving API (init / step / finished / values) over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "dpop"
        self.o = DpopOracle(inst, inst["tree"], np.float64, params["mode"])
        self.finished = False

    def init(self):
        return self

    def step(self, n=1):
        if not self.finished:
            self.o.run()
            self.finished = True
        return self

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
    GpuSession.engine_factory = DpopOracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


@contextlib.contextmanager
def numpy2_set_value():
    """NumPy 2 removed `ndarray.itemset`, which the reference's NAryMatrixRelation.set_value_for_assignment
    calls with a dict assignment (relations.py:857): an item assignment that converts the value the same way."""
    from pydcop.dcop.relations import NAryMatrixRelation
    orig = NAryMatrixRelation.set_value_for_assignment

    def set_value(self, var_values, rel_value):
        if not isinstance(var_values, dict):
            return orig(self, var_values, rel_value)
        _, s = self._slice_matrix([v.name for v in self._variables], [var_values[v.name] for v in self._variables])
        m = np.copy(self._m)
        m[s] = rel_value
        return NAryMatrixRelation(self._variables, m, name=self.name)
    NAryMatrixRelation.set_value_for_assignment = set_value
    try:
        yield
    finally:
        NAryMatrixRelation.set_value_for_assignment = orig


def orchestrated(algo_name, path, params=None):
    from pydcop.algorithms import AlgorithmDef
    from pydcop.computations_graph import pseudotree
    from pydcop.dcop.yamldcop import load_dcop_from_file
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    dcop = load_dcop_from_file([path])
    algo = AlgorithmDef.build_with_default_param(algo_name, params or {}, mode=dcop.objective)
    cg = pseudotree.build_computation_graph(dcop)
    orchestrator = run_local_thread_dcop(algo, cg, oneagent.distribute(cg, dcop.agents.values()), dcop, 1e9)
    try:
        orchestrator.deploy_computations()
        orchestrator.run(timeout=60)
        metrics = orchestrator.end_metrics()
        status = orchestrator.status
    finally:
        orchestrator.stop_agents(5)
        orchestrator.stop()
    return dcop, status, metrics


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    assert "dpop_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("dpop"), load_algorithm_module("dpop_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "pseudotree"
    assert {p.name for p in gpu.algo_params} == {"precision", "seed", "session"}
    assert not getattr(ref, "algo_params", [])
    for mod in (ref, gpu):
        with pytest.raises(NotImplementedError):
            mod.computation_memory(None)
        with pytest.raises(NotImplementedError):
            mod.communication_load(None, "x")


@needs_ref
@pytest.mark.parametrize("instance,fixture", [
    ("graph_coloring_10_4_15_0.1.yml", "dpop_ref_gc_10_4_15_0_1"),
    ("graph_coloring_tuto_max.yaml", "dpop_ref_gc_tuto_max"),
    ("graph_coloring_seperate_costs.yaml", "dpop_ref_gc_seperate_costs"),
])
def test_orchestrated_run_matches_the_reference_run(oracle_seam, instance, fixture):
    """dpop_gpu with the tree from the nodes' links: the fixture's assignment, and the same status, cycle
    and msg_count as the reference's own orchestrated `dpop` run on the same instance."""
    path = os.path.join(ref_shim.INSTANCES, instance)
    with numpy2_set_value():
        _, ref_status, ref_metrics = orchestrated("dpop", path)
    dcop, status, metrics = orchestrated("dpop_gpu", path)
    assert status == ref_status and status not in ("TIMEOUT", "STOPPED"), status
    assert metrics["cycle"] == ref_metrics["cycle"] == 0
    assert metrics["msg_count"] == ref_metrics["msg_count"]
    assert metrics["assignment"] == ref_metrics["assignment"]
    inst, _ = load(fixture)
    names = [str(n) for n in inst["var_names"]]
    doms = [list(dcop.variables[n].domain) for n in names]
    assert [doms[i].index(metrics["assignment"][n]) for i, n in enumerate(names)] == inst["value"].tolist()
    _, cost = dcop.solution_cost(metrics["assignment"], 1e9)
    assert metrics["cost"] == pytest.approx(cost)


def test_solve_through_the_seam():
    from pydcop_b200 import solve as S
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instances",
                        "graph_coloring_10_4_15_0.1.yml")
    res = S.solve(path, "dpop", engine_factory=DpopSeam)
    assert res["status"] == "FINISHED" and res["cycle"] == 0 and res["algo"] == "dpop"
    inst, _ = load("dpop_ref_gc_10_4_15_0_1")
    d = S.load(path)
    assert [d.values_of(i).index(res["assignment"][str(n)]) for i, n in enumerate(inst["var_names"])] == \
        inst["value"].tolist()
    assert S.ALGOS["dpop_gpu"] == "dpop" and S.check_params("dpop", None) == {}
    with pytest.raises(ValueError, match="takes no parameters"):
        S.check_params("dpop", {"stop_cycle": 3})


class DpopSeam(DpopOracleEngine):
    """solve()'s engine seam: the tree is built from the packed arrays, as solve() does."""

    def __init__(self, kind, layout, inst, params):
        from pydcop_b200.pseudotree import build_tree
        inst = dict(inst, tree=build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"]))
        super().__init__(kind, layout, inst, params)


def test_not_sharded():
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
        with pytest.raises(ValueError, match="dpop is not sharded"):
            S.solve(path, "dpop", distributed=True, sharded_kwargs={"engine_factory": object})
    finally:
        dist.destroy_process_group()
