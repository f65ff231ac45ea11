"""dpop_gpu — drop-in pyDcop algorithm module: DPOP on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/dpop.py` (GRAPH_TYPE :71, no algo_params,
computation_memory and communication_load raise NotImplementedError as :78-83; build_computation is what
load_algorithm_module would inject, pydcop/algorithms/__init__.py:556-564).  One proxy per node of the
pseudo-tree the orchestrator built; the per-process GpuSession takes the tree from the nodes' links,
runs the UTIL and VALUE phases of every node as one fixed sequence of CUDA launches (DESIGN.md §16) and
each proxy then selects its value and finishes, as DpopAlgo.select_value_and_finish (dpop.py:292-311).
Before it finishes, a proxy posts what its DpopAlgo would have posted: one UTIL message to its parent and
one VALUE message to each child (dpop.py:250, :363-365, :377, :438-439), each naming the separator or the
values chosen, so a run's message count is the reference's.

Parameters: precision ('f64' default | 'f32'), session (str), seed (int, accepted for uniformity with
the other modules; DPOP draws nothing).
"""
from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.computations_graph.pseudotree import get_dfs_relations
from pydcop.infrastructure.computations import Message, VariableComputation, register

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "pseudotree"
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(*args):
    raise NotImplementedError("DPOP has no computation memory implementation (yet)")


def communication_load(*args):
    raise NotImplementedError("DPOP has no communication_load implementation (yet)")


def build_computation(comp_def: ComputationDef):
    return DpopGpuComputation(comp_def)


class DpopGpuComputation(VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "dpop_gpu"
        assert comp_def.algo.mode in ("min", "max")
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        node = comp_def.node
        constraints = list(node.constraints)          # node.constraints order, dpop.py:191
        params = comp_def.algo.params
        self._session = GpuSession.get("dpop:" + str(params.get("session", "default")), "dpop")
        self._session.add_variable(self.name, self.variable, [c.name for c in constraints], constraints,
                                   params, self.mode)
        self._session.add_tree_links(self.name, node.links)
        self._parent, _, self._children, _ = get_dfs_relations(node)
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
        value, cost = snap.values[self.name]
        if self._parent is not None:
            self.post_msg(self._parent, Message("UTIL", self.name))
        for c in self._children:
            self.post_msg(c, Message("VALUE", (self.name, value)))
        self.value_selection(value, cost)
        self.stop()
        self.finished()

    @register("UTIL")
    def _on_util(self, sender, msg, t):
        pass

    @register("VALUE")
    def _on_value(self, sender, msg, t):
        pass
