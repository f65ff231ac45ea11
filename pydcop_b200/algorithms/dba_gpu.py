"""dba_gpu — drop-in pyDcop algorithm module: DBA on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/dba.py` (GRAPH_TYPE :120, algo_params :265-268,
computation_memory :130-151, communication_load :154-176; build_computation is what load_algorithm_module would
inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable of the constraints hypergraph; the
per-process GpuSession runs every variable's ok phase (dba.py:366-420) and improve phase (:504-562) as two CUDA
kernels per round.  The start values and the choice among equally good values use Philox draws keyed by (seed,
variable, cycle), as mgm_gpu's, instead of the reference's thread-arrival-ordered stdlib stream.

A proxy reports `finished()` when its own variable finished on the device (its termination counter reached
max_distance, or the End flood reached it).  A variable without neighbours never finishes, as in the reference, so a
run that has one ends at the orchestrator's timeout unless stop_cycle ends it first.

Extra parameters: stop_cycle (int, 0 = never; rounds stop when round + 1 >= stop_cycle, as for gdba_gpu — the
reference has none), precision ('f64' default | 'f32'), seed (int), session (str).
"""
import math

from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import VariableComputation

from pydcop_b200.algorithms._session import GpuSession
from pydcop_b200.engine import DBA_MODE_ERROR

GRAPH_TYPE = "constraints_hypergraph"
HEADER_SIZE = 100
UNIT_SIZE = 5
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("infinity", "int", None, 10000),
    AlgoParameterDef("max_distance", "int", None, 50),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour's value (dba.py:130-151), counted as the reference counts it: the names of the
    nodes of the computation's links that are not a substring of its own name."""
    neighbors = set((n for l in computation.links for n in l.nodes if n not in computation.name))
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """The ok and improve messages carry one value or one improvement (dba.py:154-176)."""
    return 2 * UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return DbaGpuComputation(comp_def)


class DbaGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "dba_gpu"
        super().__init__(comp_def.node.variable, comp_def)
        if comp_def.algo.mode != "min":
            raise ValueError(DBA_MODE_ERROR)
        self.constraints = list(comp_def.node.constraints)   # node.constraints order, dba.py:310
        params = comp_def.algo.params
        self._session = GpuSession.get("dba:" + str(params.get("session", "default")), "dba")
        self._session.add_variable(self.name, self.variable, [c.name for c in self.constraints],
                                   self.constraints, params, "min")
        self._seen = None

    def on_start(self):
        self._session.notify_started(self.name)
        self.add_periodic_action(POLL_PERIOD, self._poll)

    def on_stop(self):
        self._session.notify_stopped(self.name)

    def on_pause(self, paused):
        pass

    def _poll(self):
        snap = self._session.poll()
        if snap is None or snap is self._seen:
            return
        self._seen = snap
        value, cost = snap.values[self.name]
        # current_cost stays None until the first ok phase (dba.py:385)
        self.value_selection(value, None if cost is None or math.isnan(cost) else cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished or self.name in snap.done:
            self.finished()
            self.stop()
