"""syncbb_gpu — drop-in pyDcop algorithm module: SyncBB on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/syncbb.py` (GRAPH_TYPE "ordered_graph" :160, no algorithm
parameters of its own; build_computation is what load_algorithm_module would inject,
pydcop/algorithms/__init__.py:556-564).  One proxy per variable of the ordered graph; the per-process GpuSession packs
the variables in name order, which is the chain the reference walks (ordered_graph.py:173), runs the whole
branch-and-bound search on the device (DESIGN.md §18) and each proxy then reports its variable's LAST value
selection and finishes, as SyncBBComputation does when its terminate message arrives (syncbb.py:213-232).  A
variable that never selected a value reports none, so the orchestrator sees an incomplete assignment, as with the
reference.  Each proxy takes its variable's cycle count from the device, so the run's `cycle` is the reference's;
the proxies post no SyncBB messages, so its msg_count is not (DESIGN.md §18).

Parameters: precision ('f64' default | 'f32'), session (str), seed (int, accepted for uniformity with the other
modules; SyncBB draws nothing).  Constraints of arity > 2 are refused when the computation is built: the reference
fails on them inside assignment_cost (syncbb.py:456).
"""
from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import VariableComputation

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "ordered_graph"
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def build_computation(comp_def: ComputationDef):
    return SyncbbGpuComputation(comp_def)


class SyncbbGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "syncbb_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        constraints = list(comp_def.node.constraints)          # node.constraints order, syncbb.py:186
        for c in constraints:
            if len(c.dimensions) > 2:
                raise ValueError(f"constraint {c.name} has arity {len(c.dimensions)}: SyncBB supports binary "
                                 "constraints only (syncbb.py:456)")
        params = comp_def.algo.params
        self._session = GpuSession.get("syncbb:" + str(params.get("session", "default")), "syncbb")
        self._session.add_variable(self.name, self.variable, [c.name for c in constraints], constraints,
                                   params, self.mode)
        self._done = False

    def on_start(self):
        self._session.notify_started(self.name)
        self.add_periodic_action(POLL_PERIOD, self._poll)

    def on_stop(self):
        self._session.notify_stopped(self.name)

    def on_pause(self, paused):
        pass

    def _poll(self):
        snap = self._session.poll()
        if self._done or snap is None or not snap.finished:
            return
        self._done = True
        value, bound = snap.values[self.name]
        # the variable's new_cycle count (one per message it handled, :211-412): set at once rather than by as many
        # new_cycle() calls, so the orchestrator's `cycle` (the largest count) is the reference run's
        n = snap.cycles[self.name]
        if n > 0:
            self.__cycle_count__ = n - 1
            self.new_cycle()
        if value is not None:
            self.value_selection(value, bound)    # syncbb.py:314, 364: the value with the variable's bound
        self.stop()
        self.finished()
