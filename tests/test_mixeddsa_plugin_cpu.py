"""mixeddsa_gpu through the UNMODIFIED reference orchestrator (thread mode) and `solve(..., "mixeddsa")`, with the
MixedDSA oracle behind the engine seam: the plugin plumbing (module surface, registration, value reporting, cycle
counting, FINISHED status at stop_cycle, parameter validation) without a GPU.  The kernels are the GPU tests' job."""
import os

import numpy as np
import pytest

import ref_shim
from _mixeddsa_oracle import MixedDsaOracle

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")

HARD_YAML = """name: hard colouring with soft preferences
objective: min
domains:
  colors:
    values: [R, G, B]
variables:
  v1: {domain: colors}
  v2: {domain: colors}
  v3: {domain: colors}
  v4: {domain: colors}
constraints:
  d12: {type: intention, function: 1e400 if v1 == v2 else 0}
  d23: {type: intention, function: 1e400 if v2 == v3 else 0}
  d34: {type: intention, function: 1e400 if v3 == v4 else 0}
  d41: {type: intention, function: 1e400 if v4 == v1 else 0}
  d13: {type: intention, function: 1e400 if v1 == v3 else 0}
  p1: {type: intention, function: 0 if v1 == 'R' else 1}
  p4: {type: intention, function: 2 if v4 == 'B' else 0}
agents: [a1, a2, a3, a4]
"""


def hard_yaml(tmp_path):
    p = tmp_path / "hard.yaml"
    p.write_text(HARD_YAML)
    return str(p)


class MixedDsaOracleEngine:
    """MixedDsaEngine's driving API (init / step / finished / values) over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "mixeddsa"
        keys = ("proba_hard", "proba_soft", "variant", "stop_cycle", "seed")
        inst = dict(inst)
        if inst.get("var_ptr") is None:
            from pydcop_b200.layout import default_var_csr
            inst["var_ptr"], inst["var_edge"] = default_var_csr(len(inst["dom_size"]), inst["edge_var"])
        self.o = MixedDsaOracle(inst, np.float64, mode=params["mode"], **{k: params[k] for k in keys if k in params})

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
    GpuSession.engine_factory = MixedDsaOracleEngine
    yield GpuSession
    GpuSession.engine_factory = None
    GpuSession.reset()


@needs_ref
def test_module_surface_matches_reference(pydcop_ready):
    from pydcop.algorithms import list_available_algorithms, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.dcop.yamldcop import load_dcop_from_file
    assert "mixeddsa_gpu" in list_available_algorithms()
    ref, gpu = load_algorithm_module("mixeddsa"), load_algorithm_module("mixeddsa_gpu")
    assert gpu.GRAPH_TYPE == ref.GRAPH_TYPE == "constraints_hypergraph"
    params = {p.name: p for p in gpu.algo_params}
    for p in ref.algo_params:
        assert params[p.name] == p
    assert [p.default_value for p in ref.algo_params] == [0.7, 0.5, "B", 0]
    assert {"precision", "seed", "session"} <= set(params)
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    for node in constraints_hypergraph.build_computation_graph(dcop).nodes:
        assert gpu.computation_memory(node) == ref.computation_memory(node)
        for nb in node.neighbors:
            assert gpu.communication_load(node, nb) == ref.communication_load(node, nb)


def run_orchestrated(dcop, params, timeout=60):
    from pydcop.algorithms import AlgorithmDef, load_algorithm_module
    from pydcop.computations_graph import constraints_hypergraph
    from pydcop.distribution import oneagent
    from pydcop.infrastructure.run import run_local_thread_dcop
    module = load_algorithm_module("mixeddsa_gpu")
    algo = AlgorithmDef.build_with_default_param("mixeddsa_gpu", params, mode=dcop.objective)
    cg = constraints_hypergraph.build_computation_graph(dcop)
    dist = oneagent.distribute(cg, dcop.agents.values(), computation_memory=module.computation_memory,
                               communication_load=module.communication_load)
    orchestrator = run_local_thread_dcop(algo, cg, dist, dcop, 1e9)
    try:
        orchestrator.deploy_computations()
        orchestrator.run(timeout=timeout)
        return orchestrator.end_metrics(), orchestrator.status
    finally:
        orchestrator.stop_agents(5)
        orchestrator.stop()


@needs_ref
@pytest.mark.parametrize("stop_cycle", [30, 17])
def test_orchestrated_run_finishes_at_stop_cycle(oracle_seam, stop_cycle):
    """Runs ended by stop_cycle, on and off the session's chunk of 10 rounds."""
    from pydcop.dcop.yamldcop import load_dcop_from_file
    dcop = load_dcop_from_file([os.path.join(ref_shim.INSTANCES, "graph_coloring_10_4_15_0.1.yml")])
    metrics, status = run_orchestrated(dcop, {"stop_cycle": stop_cycle, "seed": 5, "variant": "A"})
    assert status not in ("TIMEOUT", "STOPPED"), status
    assert metrics["cycle"] == stop_cycle         # dsa_gpu's convention: stop_cycle rounds
    assert set(metrics["assignment"]) == {f"v{i}" for i in range(10)}
    _, cost = dcop.solution_cost(metrics["assignment"], 1e9)
    assert metrics["cost"] == pytest.approx(cost)


@needs_ref
def test_orchestrated_hard_problem(oracle_seam, tmp_path):
    from pydcop.dcop.yamldcop import load_dcop_from_file
    dcop = load_dcop_from_file([hard_yaml(tmp_path)])
    metrics, status = run_orchestrated(dcop, {"stop_cycle": 20, "seed": 2})
    assert status not in ("TIMEOUT", "STOPPED"), status
    assert metrics["cycle"] == 20 and len(metrics["assignment"]) == 4


def test_solve_through_the_seam(tmp_path):
    from pydcop_b200 import solve as S
    path = hard_yaml(tmp_path)
    res = S.solve(path, "mixeddsa", {"stop_cycle": 50, "proba_hard": "0.9"}, seed=3,
                  engine_factory=MixedDsaOracleEngine)
    assert res["status"] == "FINISHED" and res["cycle"] == 50 and res["algo"] == "mixeddsa"
    assert set(res) >= {"status", "assignment", "cost", "violation", "time", "cycle", "msg_count", "msg_size"}
    assert set(res["assignment"]) == {"v1", "v2", "v3", "v4"}
    assert S.ALGOS["mixeddsa_gpu"] == S.ALGOS["mixeddsa"] == "mixeddsa"


def test_solve_parameter_validation(tmp_path):
    from pydcop_b200 import solve as S
    path = hard_yaml(tmp_path)
    assert S.check_params("mixeddsa", None) == {"proba_hard": 0.7, "proba_soft": 0.5, "variant": "B", "stop_cycle": 0}
    for bad in ({"variant": "D"}, {"proba_soft": "x"}, {"stop_cycle": "many"}, {"probability": 0.5}):
        with pytest.raises(ValueError):
            S.solve(path, "mixeddsa", dict(bad, stop_cycle=bad.get("stop_cycle", 5)), engine_factory=MixedDsaOracleEngine)
    with pytest.raises(ValueError, match="does not stop"):
        S.solve(path, "mixeddsa", {}, engine_factory=MixedDsaOracleEngine)
    with pytest.raises(ValueError, match="not sharded"):
        S._sharded_engine("mixeddsa", None, None, {}, "min", "f32", None, 0, "auto", "auto", None)


def test_plan_passes_every_create_check():
    """mixeddsa_plan's descriptor passes every check of fg_mixeddsa_create up to the device: without one the call
    fails with FG_ERR_CUDA, never FG_ERR_ARG."""
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("checked on the device by the GPU tests")
    from pydcop_b200 import _cabi
    from test_mixeddsa_hostshim import HostMixedDsa, limits_instance, random_mixed
    from pydcop_b200.layout import layout_from_instance
    lib = _cabi.load()
    for inst in (random_mixed(80, seed=4), limits_instance("no_factors"), limits_instance("d256")):
        for precision in ("f32", "f64"):
            for variant in "ABC":
                d = HostMixedDsa(layout_from_instance(inst), precision=precision, variant=variant,
                                 mode="max", stop_cycle=3).d
                h = C.c_void_p()
                rc = lib.fg_mixeddsa_create(C.byref(d), C.byref(h))
                msg = (lib.fg_mixeddsa_last_error(h) or b"").decode()
                lib.fg_mixeddsa_destroy(h)
                assert rc == _cabi.FG_ERR_CUDA and "no CUDA device" in msg, msg

