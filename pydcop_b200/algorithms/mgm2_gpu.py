"""mgm2_gpu — drop-in pyDcop algorithm module: MGM-2 on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/mgm2.py` (GRAPH_TYPE :60, algo_params
:139-143, computation_memory :66-88, communication_load :91-124; build_computation is what
load_algorithm_module would inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable
of the constraints hypergraph; the per-process GpuSession runs every variable's cycle — value phase
and offers, answers, commits, gain phase and coordinated moves (mgm2.py:742-1001) — as five CUDA
kernels per cycle.  The random decisions use Philox draws keyed by (seed, variable, cycle, purpose)
instead of the reference's thread-arrival-ordered stdlib stream.

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
    AlgoParameterDef("threshold", "float", None, 0.5),
    AlgoParameterDef("favor", "str", ["unilateral", "no", "coordinated"], "unilateral"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """A value and a gain per neighbour (mgm2.py:66-88)."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * 2 * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """The largest message is the offer: two values and a gain for every pair of values of the two
    variables (mgm2.py:91-124)."""
    target_domain = None
    for c in src.constraints:
        for v in c.dimensions:
            if v.name == target:
                target_domain = v.domain
    if target_domain is None:
        raise ValueError(f"target variable {target} not found in constraints for {src}")
    return len(target_domain) * len(src.variable.domain) * UNIT_SIZE * 3 + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return Mgm2GpuComputation(comp_def)


class Mgm2GpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "mgm2_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = list(comp_def.node.constraints)   # node.constraints order, mgm2.py:433
        self.stop_cycle = comp_def.algo.param_value("stop_cycle")
        params = comp_def.algo.params
        self._session = GpuSession.get("mgm2:" + str(params.get("session", "default")), "mgm2")
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
        # current_cost stays None until the first round (mgm2.py:480-490)
        self.value_selection(value, None if cost is None or math.isnan(cost) else cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
