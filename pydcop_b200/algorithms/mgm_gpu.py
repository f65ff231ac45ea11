"""mgm_gpu — drop-in pyDcop algorithm module: MGM on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/mgm.py` (GRAPH_TYPE :68, algo_params
:78-81, computation_memory :84-110, communication_load :113-133; build_computation is what
load_algorithm_module would inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable
of the constraints hypergraph; the per-process GpuSession runs every variable's value phase
(mgm.py:343-397) and gain phase (:497-537) as two CUDA kernels per cycle.  The initial values and
the choice among equally good values use Philox draws keyed by (seed, variable, cycle)
(oracle/philox.py) instead of the reference's thread-arrival-ordered stdlib stream.

Extra parameters: precision ('f64' default | 'f32'), seed (int), session (str).
"""
import math

from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import VariableComputation

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "constraints_hypergraph"
HEADER_SIZE = 100
UNIT_SIZE = 5
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("break_mode", "str", ["lexic", "random"], "lexic"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour (mgm.py:84-110)."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """Value and gain messages carry one number each (mgm.py:113-133)."""
    return UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return MgmGpuComputation(comp_def)


class MgmGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "mgm_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = list(comp_def.node.constraints)   # node.constraints order, mgm.py:233
        self.stop_cycle = comp_def.algo.param_value("stop_cycle")
        params = comp_def.algo.params
        self._session = GpuSession.get("mgm:" + str(params.get("session", "default")), "mgm")
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
        # current_cost stays None until the first round (mgm.py:349); value before new_cycle(): the
        # cycle notification carries it
        self.value_selection(value, None if cost is None or math.isnan(cost) else cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
