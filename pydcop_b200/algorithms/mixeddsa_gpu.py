"""mixeddsa_gpu — drop-in pyDcop algorithm module: MixedDSA on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/mixeddsa.py` (GRAPH_TYPE :51, algo_params :119-124,
computation_memory :67-92, communication_load :95-116; build_computation is what load_algorithm_module would
inject, pydcop/algorithms/__init__.py:556-564).  One proxy per variable of the constraints hypergraph; the
per-process GpuSession runs every variable's round (_on_neighbors_values :272-373) as one CUDA kernel.  The start
values, the probability tests and the choice among the best values use Philox draws keyed by (seed, variable,
cycle), as dsa_gpu's, instead of the reference's thread-arrival-ordered stdlib stream.

The reference module cannot be run as such: its build_computation forwards `stop_cycle`, which
MixedDsaComputation.__init__ does not accept.  Here stop_cycle (int, 0 = never) ends the run after stop_cycle
rounds, dsa_gpu's convention (dsa.py:352).  Extra parameters: precision ('f64' default | 'f32'), seed (int),
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
    AlgoParameterDef("proba_hard", "float", None, 0.7),
    AlgoParameterDef("proba_soft", "float", None, 0.5),
    AlgoParameterDef("variant", "str", ["A", "B", "C"], "B"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour's value (mixeddsa.py:67-92), with the reference's test of a neighbour's name against
    the computation's name (`in`, a substring test)."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """The value message carries one value (mixeddsa.py:95-116)."""
    return UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return MixedDsaGpuComputation(comp_def)


class MixedDsaGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "mixeddsa_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = list(comp_def.node.constraints)   # node.constraints order, mixeddsa.py:205
        self.stop_cycle = comp_def.algo.param_value("stop_cycle")
        params = comp_def.algo.params
        self._session = GpuSession.get("mixeddsa:" + str(params.get("session", "default")), "mixeddsa")
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
        # current_cost stays None until the variable's first move (mixeddsa.py:233, :302)
        self.value_selection(value, None if cost is None or math.isnan(cost) else cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
