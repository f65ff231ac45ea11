"""dsa_gpu — drop-in pyDcop algorithm module: DSA-A/B/C on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/dsa.py` (GRAPH_TYPE :114, algo_params
:130-135, computation_memory :138-160, communication_load :163-184; build_computation is what
load_algorithm_module would inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable
of the constraints hypergraph; the per-process GpuSession evaluates every variable's
`evaluate_cycle` (dsa.py:320-357) in one CUDA kernel per cycle.  Random decisions use the
counter-based Philox draws keyed by (seed, variable, cycle) (oracle/philox.py): unlike the
reference's thread-arrival-ordered stdlib stream they are reproducible.

Extra parameters: precision ('f64' default | 'f32'), seed (int), session (str).
"""
from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import VariableComputation

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "constraints_hypergraph"
HEADER_SIZE = 0
UNIT_SIZE = 1
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("probability", "float", None, 0.7),
    AlgoParameterDef("p_mode", "str", ["fixed", "arity"], "fixed"),
    AlgoParameterDef("variant", "str", ["A", "B", "C"], "B"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour, as in the reference (dsa.py:138-160)."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """A DSA message carries one value (dsa.py:163-184)."""
    return UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return DsaGpuComputation(comp_def)


class DsaGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "dsa_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = comp_def.node.constraints      # node.constraints order, dsa.py:255
        self.stop_cycle = comp_def.algo.param_value("stop_cycle")
        params = comp_def.algo.params
        self._session = GpuSession.get("dsa:" + str(params.get("session", "default")), "dsa")
        self._session.add_variable(self.name, self.variable, [c.name for c in self.constraints],
                                   self.constraints, params, self.mode)
        self._seen_cycle = -1

    def on_start(self):
        self._session.notify_started(self.name)
        self.add_periodic_action(POLL_PERIOD, self._poll)

    def on_stop(self):
        self._session.notify_stopped(self.name)

    def on_pause(self, paused):
        pass

    def _poll(self):
        snap = self._session.poll()
        if snap is None or snap.cycle == self._seen_cycle:
            return
        self._seen_cycle = snap.cycle
        value, cost = snap.values[self.name]
        self.value_selection(value, cost)      # before new_cycle(): the cycle notification carries it
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
