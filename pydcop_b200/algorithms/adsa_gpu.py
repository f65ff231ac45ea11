"""adsa_gpu — drop-in pyDcop algorithm module: A-DSA on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/adsa.py` (GRAPH_TYPE :100, algo_params :121-125:
period 0.5, probability 0.7, variant B; memory / load models as DSA's).  The reference's computation is
timer-driven: every `period` seconds a variable re-evaluates its value against the LAST values it received
(adsa.py:255-300), so its trajectory depends on how the timers of the agents interleave.  The engine runs the
execution in which all periods are aligned: one engine cycle = one tick of every variable on the values of the
previous tick — the schedule the reference trajectories of oracle/make_golden_adsa.py were recorded with.
The decision is DSA's with ONE difference (adsa.py:344-377): every candidate value carries the variable's own
cost, the current cost does not; `DsaEngine(var_costs=True)`.  Variables without neighbours take the argopt of
their own cost (the evident intent of adsa.py:236-253, which unpacks optimal_cost_value's pair the wrong way round).

`period` is kept for the signature: it paces how often the proxies poll, not the engine.  Extra parameters:
stop_cycle (ticks; 0 = run until the orchestrator's timeout, as the reference does), precision, seed, session.
"""
from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import VariableComputation

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "constraints_hypergraph"
HEADER_SIZE = 0
UNIT_SIZE = 1
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("period", "float", None, 0.5),
    AlgoParameterDef("probability", "float", None, 0.7),
    AlgoParameterDef("variant", "str", ["A", "B", "C"], "B"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """One unit per neighbour, as for DSA (adsa.py reuses dsa's model)."""
    neighbors = set(n for l in computation.links for n in l.nodes if n not in computation.name)
    return len(neighbors) * UNIT_SIZE


def communication_load(src, target: str) -> float:
    """An A-DSA message carries one value."""
    return UNIT_SIZE + HEADER_SIZE


def build_computation(comp_def: ComputationDef):
    return ADsaGpuComputation(comp_def)


class ADsaGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "adsa_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.constraints = comp_def.node.constraints
        params = comp_def.algo.params
        self._session = GpuSession.get("adsa:" + str(params.get("session", "default")), "adsa")
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
        self.value_selection(value, cost)
        while self.cycle_count < snap.cycle:
            self.new_cycle()
        if snap.finished:
            self.finished()
            self.stop()
