"""gdba_gpu — drop-in pyDcop algorithm module: GDBA on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/gdba.py` (GRAPH_TYPE :59, algo_params
:181-185, computation_memory :75-97, communication_load :100-123; build_computation is what
load_algorithm_module would inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable
of the constraints hypergraph; the per-process GpuSession runs every variable's ok phase
(gdba.py:352-387) and improve phase with its breakouts (:493-541) as two CUDA kernels per round.  The
start values and the choice among equally good values use Philox draws keyed by (seed, variable,
cycle), as mgm_gpu's, instead of the reference's thread-arrival-ordered stdlib stream.

Extra parameters: stop_cycle (int, 0 = never; rounds stop when round + 1 >= stop_cycle, as for
mgm_gpu — the reference has no stop condition), precision ('f64' default | 'f32'), seed (int),
session (str).
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
    AlgoParameterDef("modifier", "str", ["A", "M"], "A"),
    AlgoParameterDef("violation", "str", ["NZ", "NM", "MX"], "NZ"),
    AlgoParameterDef("increase_mode", "str", ["E", "R", "C", "T"], "E"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour's value (gdba.py:75-97).  The reference iterates `computation.neighbors`,
    which are names, and reads `.nodes` on them, so it raises for every variable that has a neighbour;
    this counts the distinct neighbours through the node's links, as its docstring describes."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """The ok and improve messages carry one value or one improvement (gdba.py:100-123)."""
    return 2 * UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return GdbaGpuComputation(comp_def)


class GdbaGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "gdba_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = list(comp_def.node.constraints)   # node.constraints order, gdba.py:252
        self.stop_cycle = comp_def.algo.param_value("stop_cycle")
        params = comp_def.algo.params
        self._session = GpuSession.get("gdba:" + str(params.get("session", "default")), "gdba")
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
        # current_cost stays None until the first round (gdba.py:319, :366)
        self.value_selection(value, None if cost is None or math.isnan(cost) else cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
