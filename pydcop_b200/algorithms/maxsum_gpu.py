"""maxsum_gpu — drop-in pyDcop algorithm module: synchronous MaxSum on the GPU engine.

Same module surface as the reference's `pydcop/algorithms/maxsum.py` (GRAPH_TYPE :103,
algo_params :212-220, build_computation :118-124, computation_memory :127-171,
communication_load :174-209).  `pydcop solve --algo maxsum_gpu ...` deploys one proxy computation
per factor-graph node exactly like `--algo maxsum`; the proxies hand their nodes to a per-process
GpuSession (pydcop_b200/algorithms/_session.py) which runs ALL factor->variable and
variable->factor updates of a cycle in CUDA kernels and feeds values back through the reference's
own `value_selection` / `new_cycle` / `finished` hooks.

Extra parameters (the reference's MaxSum has no stop condition, maxsum.py:62):
  stop_cycle  int, 0 = run until the orchestrator's timeout (like the reference)
  precision   'f64' (default: the reference's own arithmetic, assignments bit-exact) | 'f32'
  seed        int, 0 = unseeded noise draws (like the reference's random.uniform)
  session     str, separates independent graphs solved concurrently in one process
"""
from pydcop.algorithms import AlgoParameterDef, ComputationDef
from pydcop.infrastructure.computations import DcopComputation, VariableComputation

from pydcop_b200.algorithms._session import GpuSession

GRAPH_TYPE = "factor_graph"

HEADER_SIZE = 0
UNIT_SIZE = 1
FACTOR_UNIT_SIZE = 1
VARIABLE_UNIT_SIZE = 1
POLL_PERIOD = 0.02

algo_params = [
    AlgoParameterDef("damping", "float", None, 0.5),
    AlgoParameterDef("damping_nodes", "str", ["vars", "factors", "both", "none"], "both"),
    AlgoParameterDef("stability", "float", None, 0.1),
    AlgoParameterDef("noise", "float", None, 0.01),
    AlgoParameterDef("start_messages", "str", ["leafs", "leafs_vars", "all"], "leafs"),
    AlgoParameterDef("stop_cycle", "int", None, 0),
    AlgoParameterDef("precision", "str", ["f32", "f64"], "f64"),
    AlgoParameterDef("seed", "int", None, 0),
    AlgoParameterDef("session", "str", None, "default"),
]


def computation_memory(computation) -> float:
    """Same footprint model as the reference (maxsum.py:127-171)."""
    if computation.type == "FactorComputation":
        return sum(len(v.domain) * FACTOR_UNIT_SIZE for v in computation.variables)
    if computation.type == "VariableComputation":
        return len(list(computation.links)) * len(computation.variable.domain) * VARIABLE_UNIT_SIZE
    raise ValueError(f"Invalid computation node type {computation}, maxsum_gpu only defines "
                     "VariableComputationNode and FactorComputationNode")


def communication_load(src, target: str) -> float:
    """Same edge load model as the reference (maxsum.py:174-209)."""
    if src.type == "VariableComputation":
        return UNIT_SIZE * len(src.variable.domain) + HEADER_SIZE
    if src.type == "FactorComputation":
        for v in src.variables:
            if v.name == target:
                return UNIT_SIZE * len(v.domain) + HEADER_SIZE
        raise ValueError(f"Could not find variable {target} in constraint of factor {src}")
    raise ValueError("maxsum_gpu communication_load only supports VariableComputationNode and "
                     f"FactorComputationNode, invalid computation: {src}")


def build_computation(comp_def: ComputationDef):
    if comp_def.node.type == "VariableComputation":
        return MaxSumGpuVariableComputation(comp_def)
    if comp_def.node.type == "FactorComputation":
        return MaxSumGpuFactorComputation(comp_def)
    raise ValueError(f"maxsum_gpu cannot build a computation for node type {comp_def.node.type}")


class _ProxyMixin:
    """Polls the session from the hosting agent's own thread."""

    def _attach(self, comp_def):
        params = comp_def.algo.params
        self._session = GpuSession.get("maxsum:" + str(params.get("session", "default")), "maxsum")
        self._seen_cycle = -1
        self._poll_handle = None

    def on_start(self):
        self._session.notify_started(self.name)
        self._poll_handle = self.add_periodic_action(POLL_PERIOD, self._poll)

    def on_stop(self):
        self._session.notify_stopped(self.name)

    def on_pause(self, paused):
        pass

    def _advance_cycle(self, cycle):
        # the reference's MaxSum counts cycles in the synchronous mixin (computations.py:790-792);
        # here the engine's cycle is mirrored through new_cycle so cycle metrics keep working
        while self.cycle_count < cycle:
            self.new_cycle()


class MaxSumGpuFactorComputation(_ProxyMixin, DcopComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "maxsum_gpu"
        super().__init__(comp_def.node.factor.name, comp_def)
        self.mode = comp_def.algo.mode
        self.factor = comp_def.node.factor
        self.variables = self.factor.dimensions
        self._attach(comp_def)
        self._session.add_factor(self.name, self.factor, comp_def.algo.params, self.mode)

    def footprint(self) -> float:
        return computation_memory(self.computation_def.node)

    def _poll(self):
        snap = self._session.poll()
        if snap is None or snap.cycle == self._seen_cycle:
            return
        self._seen_cycle = snap.cycle
        self._advance_cycle(snap.cycle)
        if snap.finished:
            self.finished()
            self.stop()


class MaxSumGpuVariableComputation(_ProxyMixin, VariableComputation):
    def __init__(self, comp_def: ComputationDef):
        assert comp_def.algo.algo == "maxsum_gpu"
        super().__init__(comp_def.node.variable, comp_def)
        self.mode = comp_def.algo.mode
        self.factors = [link.factor_node for link in comp_def.node.links]  # `links` order, maxsum.py:466
        self._attach(comp_def)
        self._session.add_variable(self.name, self.variable, self.factors, None,
                                   comp_def.algo.params, self.mode)

    def _poll(self):
        snap = self._session.poll()
        if snap is None or snap.cycle == self._seen_cycle:
            return
        self._seen_cycle = snap.cycle
        # value first, then the cycle counter: the reference's cycle-change notification carries the
        # value selected IN that cycle (computations.py:915-928), `--collect_on cycle_change` reads it
        value, cost = snap.values[self.name]
        self.value_selection(value, cost)
        self._advance_cycle(snap.cycle)
        if snap.finished:
            self.finished()
            self.stop()
