"""Per-process GPU session behind the `maxsum_gpu` / `dsa_gpu` proxy computations.

pyDcop builds ONE computation object per graph node and hosts them on agent threads
(pydcop/infrastructure/orchestratedagents.py:265-290, agents.py:175-225).  The GPU engine wants
the WHOLE graph at once.  Each proxy therefore registers its node here; when the registered nodes
form a closed graph (every referenced factor / variable is present) and all of them have been
started, a worker thread packs the graph (pydcop_b200.layout), runs the engine in chunks of
cycles and publishes (cycle, values, costs) snapshots.  Proxies poll the snapshots from their
own agent thread (periodic action) and report through the reference's own hooks
(`value_selection`, `new_cycle`, `finished`), so the orchestrator, metrics and CLI output work
unchanged.

Everything here is duck-typed on the reference's node / constraint / variable objects
(`.name`, `.dimensions`, `.domain`, `__call__`, `.cost_for_val`, `.initial_value`): no pydcop
import is needed, which keeps this module testable without the reference.
"""
import random
import threading
import time
from typing import Any, Callable, Dict, List, Optional

import numpy as np


def domain_values(variable) -> list:
    return list(variable.domain)


def tabulate(constraint, cache=None) -> np.ndarray:
    """Dense row-major cost table, axis i <-> constraint.dimensions[i]
    (layout of NAryMatrixRelation._m, pydcop/dcop/relations.py:716-733).  Expression constraints
    are evaluated on broadcast numpy axes and shared between identical functions
    (pydcop_b200.ingest.tabulate_constraint)."""
    from ..ingest import tabulate_constraint
    shape = tuple(len(v.domain) for v in constraint.dimensions)
    return tabulate_constraint(constraint, cache).reshape(shape)


class Snapshot:
    """`finished`: every proxy reports finished; `done`: the variables that finished on their own (DBA);
    `cycles`: name -> the variable's own cycle count (SyncBB)."""
    __slots__ = ("cycle", "values", "costs", "finished", "done", "cycles")

    def __init__(self, cycle, values, costs, finished, done=frozenset(), cycles=None):
        self.cycle, self.values, self.costs, self.finished = cycle, values, costs, finished
        self.done, self.cycles = done, cycles


class GpuSession:
    """Collects the nodes of one DCOP run and drives one engine for all of them."""

    _lock = threading.Lock()
    _sessions: Dict[str, "GpuSession"] = {}
    _retired: Dict[str, "GpuSession"] = {}    # most recent finished session per key (introspection / tests)

    #: engine factory, replaceable by tests: (kind, layout, params) -> engine with
    #: init() / step(n) / values()  (values() -> value indices, or (indices, costs))
    engine_factory: Optional[Callable] = None

    def __init__(self, key: str, kind: str):
        self.key, self.kind = key, kind
        self.lock = threading.RLock()
        self.variables: Dict[str, Any] = {}       # name -> variable object
        self.var_links: Dict[str, List[str]] = {}  # name -> constraint names in `links` order
        self.tree_links: Dict[str, list] = {}      # dpop: name -> (type, target) of its PseudoTreeLinks
        self.constraints: Dict[str, Any] = {}     # name -> constraint object
        self.needed_factors: set = set()
        self.needed_vars: set = set()
        self.started: set = set()
        self.stopped: set = set()
        self.members: set = set()
        self.params: Dict[str, Any] = {}
        self.mode = "min"
        self.snapshot: Optional[Snapshot] = None
        self.error: Optional[BaseException] = None
        self.thread: Optional[threading.Thread] = None
        self.closed = False
        self.var_order: List[str] = []
        self.cycles_per_poll = 10
        self._first_start: Optional[float] = None

    # -- registry ---------------------------------------------------------------------------
    @classmethod
    def get(cls, key: str, kind: str) -> "GpuSession":
        """The session collecting the nodes of the CURRENT run under `key`.  A session that already runs
        (worker started), has published a result, failed or was closed belongs to a PREVIOUS run — e.g.
        pydcop.infrastructure.run.solve called twice in one process with the default session name — and
        is replaced: all nodes of a run are built before any of them is started
        (orchestrator.py:745-761, 932-944)."""
        with cls._lock:
            s = cls._sessions.get(key)
            if (s is None or s.closed or s.thread is not None or s.snapshot is not None
                    or s.error is not None):
                s = cls._sessions[key] = GpuSession(key, kind)
            return s

    def _retire(self):
        """The worker is done (finished, failed, or every member stopped): the proxies keep their
        reference and the last snapshot, the registry forgets the session."""
        self.closed = True
        with type(self)._lock:
            if type(self)._sessions.get(self.key) is self:
                del type(self)._sessions[self.key]
            type(self)._retired[self.key] = self

    @classmethod
    def last(cls, key: str) -> Optional["GpuSession"]:
        """The running session under `key`, else the most recent finished one (None if there was none)."""
        with cls._lock:
            return cls._sessions.get(key) or cls._retired.get(key)

    @classmethod
    def reset(cls):
        with cls._lock:
            for s in cls._sessions.values():
                s.closed = True
            cls._sessions.clear()
            cls._retired.clear()

    # -- registration (called from build_computation, any thread) ------------------------------
    def add_variable(self, name, variable, constraint_names, constraints=None, params=None, mode="min"):
        with self.lock:
            self.variables[name] = variable
            self.var_links[name] = list(constraint_names)
            self.needed_factors.update(constraint_names)
            for c in constraints or ():
                self.constraints[c.name] = c
                self.needed_vars.update(v.name for v in c.dimensions)
            self.members.add(name)
            self._set_params(params, mode)

    def add_tree_links(self, name, links):
        """The node's pseudo-tree links (parent, children, pseudo_parent, pseudo_children), in order."""
        with self.lock:
            self.tree_links[name] = [(l.type, l.target) for l in links if l.source == name]

    def add_factor(self, name, constraint, params=None, mode="min"):
        with self.lock:
            self.constraints[name] = constraint
            self.needed_vars.update(v.name for v in constraint.dimensions)
            self.members.add(name)
            self._set_params(params, mode)

    def _set_params(self, params, mode):
        if params:
            self.params = dict(params)
        self.mode = mode

    def is_complete(self) -> bool:
        return (self.needed_factors <= set(self.constraints)
                and self.needed_vars <= set(self.variables) and bool(self.members))

    # -- lifecycle --------------------------------------------------------------------------
    #: seconds a started but incomplete session waits before it reports itself as stuck
    incomplete_grace = 5.0

    def notify_started(self, name):
        with self.lock:
            self.started.add(name)
            if self._first_start is None:
                self._first_start = time.monotonic()
            if (self.thread is None and self.error is None and self.is_complete()
                    and self.members <= self.started):
                self.thread = threading.Thread(target=self._run, name=f"gpu-session-{self.key}",
                                               daemon=True)
                self.thread.start()

    def notify_stopped(self, name):
        with self.lock:
            self.stopped.add(name)

    def all_stopped(self) -> bool:
        with self.lock:
            return self.members <= self.stopped

    def poll(self) -> Optional[Snapshot]:
        if self.error is not None:
            raise self.error
        if (self.thread is None and self._first_start is not None and not self.is_complete()
                and time.monotonic() - self._first_start > self.incomplete_grace):
            # every computation of the graph must live in THIS process (thread mode): with
            # `pydcop solve -m process` each agent process only ever sees its own nodes
            missing = sorted((self.needed_factors - set(self.constraints))
                             | (self.needed_vars - set(self.variables)))
            self.error = RuntimeError(
                f"pydcop_b200: {self.kind}_gpu session '{self.key}' never saw the whole graph in this process "
                f"(missing {missing[:5]}{'...' if len(missing) > 5 else ''}): the GPU modules need thread mode "
                "(`pydcop solve -m thread`), one process cannot share a device session with another")
            import logging
            import sys
            logging.getLogger("pydcop_b200").critical(str(self.error))
            print(str(self.error), file=sys.stderr, flush=True)
            raise self.error
        return self.snapshot

    # -- packing ----------------------------------------------------------------------------
    def build_instance(self):
        """Flat arrays of the registered graph.  Variables and constraints are taken in NAME order,
        not in the (thread-dependent) order the proxies registered in, so the instance — and with
        a `seed` the noise / random draws — is identical from run to run; every variable keeps the
        `links` order pyDcop gave it."""
        var_names = sorted(self.variables)
        vidx = {n: i for i, n in enumerate(var_names)}
        cons_names = sorted(self.constraints)
        cidx = {n: i for i, n in enumerate(cons_names)}
        dom_size = np.array([len(self.variables[n].domain) for n in var_names], dtype=np.int32)
        factor_ptr, edge_var, tables, edge_of = [0], [], [], {}
        from ..ingest import TableCache
        cache = TableCache()
        for cn in cons_names:
            c = self.constraints[cn]
            for v in c.dimensions:
                edge_of[(cn, v.name)] = len(edge_var)
                edge_var.append(vidx[v.name])
            factor_ptr.append(len(edge_var))
            tables.append(tabulate(c, cache).reshape(-1))
        var_ptr, var_edge = [0], []
        for n in var_names:
            for cn in self.var_links[n]:
                var_edge.append(edge_of[(cn, n)])
            var_ptr.append(len(var_edge))
        unary, init_value = [], []
        for n in var_names:
            v = self.variables[n]
            dom = domain_values(v)
            cost = getattr(v, "cost_for_val", None)
            unary.extend(float(cost(x)) if cost else 0.0 for x in dom)
            iv = getattr(v, "initial_value", None)
            init_value.append(dom.index(iv) if iv is not None else -1)
        self.var_order = var_names
        return dict(dom_size=dom_size, factor_ptr=np.array(factor_ptr, dtype=np.int64),
                    edge_var=np.array(edge_var, dtype=np.int32),
                    tables=np.concatenate(tables) if tables else np.zeros(0),
                    unary=np.array(unary, dtype=np.float64), var_ptr=np.array(var_ptr, dtype=np.int32),
                    var_edge=np.array(var_edge, dtype=np.int32),
                    init_value=np.array(init_value, dtype=np.int32))

    # -- worker -----------------------------------------------------------------------------
    def _make_engine(self, layout, inst):
        factory = type(self).engine_factory
        p = dict(self.params)
        if factory is not None:
            return factory(self.kind, layout, inst, dict(p, mode=self.mode))
        from ..engine import make_engine
        # variables are packed in name order: the name rank equals the index (no var_rank)
        return make_engine(self.kind, layout, p, mode=self.mode, precision=p.get("precision", "f64"),
                           seed=p.get("seed", 0), isolated_value=inst.get("isolated_value"), tree=inst.get("tree"))

    def _run(self):
        try:
            from ..layout import build_layout
            inst = self.build_instance()
            if self.kind == "maxsum":
                noise = float(self.params.get("noise", 0.01))
                if noise != 0:  # VariableNoisyCostFunc: cost + U(0, noise) per value (objects.py:566)
                    seed = int(self.params.get("seed", 0))
                    rnd = random.Random(seed) if seed else random
                    inst["unary"] = inst["unary"] + np.array(
                        [rnd.uniform(0, noise) for _ in range(len(inst["unary"]))])
            elif self.kind == "dpop":
                inst["tree"] = self._pseudo_tree(inst)
            elif self.kind == "syncbb":   # name order is the chain: no start values to work out
                pass
            else:
                inst["isolated_value"] = self._isolated_values(inst)
            layout = build_layout(**{k: v for k, v in inst.items() if k not in ("isolated_value", "tree")})
            engine = self._make_engine(layout, inst)
            engine.init()
            stop_cycle = int(self.params.get("stop_cycle", 0) or 0)
            cycle = 0
            self._publish(engine, cycle, False)
            while not self.closed and not self.all_stopped():
                if self.kind == "syncbb":   # a message per step: launches of SYNCBB_CHUNK until the search ends
                    from ..solve import SYNCBB_CHUNK
                    engine.step(SYNCBB_CHUNK)
                    done = bool(engine.finished)
                    self._publish(engine, engine.cycle, done)
                    if done:
                        break
                    time.sleep(0)
                    continue
                n = self.cycles_per_poll
                if stop_cycle:
                    n = min(n, stop_cycle - cycle)
                if n <= 0:
                    break
                engine.step(n)
                cycle += n
                if self.kind == "dba":   # each proxy finishes with its own variable; the rounds that changed state
                    # the engine stops at stop_cycle - 1 rounds (gdba_gpu's convention): then every proxy finishes
                    stopped = bool(stop_cycle and cycle + 1 >= stop_cycle)
                    self._publish(engine, engine.cycle, stopped)
                    if stopped or engine.finished:
                        break
                    time.sleep(0)
                    continue
                done = bool(stop_cycle and cycle >= stop_cycle) or bool(getattr(engine, "finished", False))
                self._publish(engine, cycle, done)
                if done:
                    break
                time.sleep(0)  # let the agent threads poll
        except BaseException as e:  # noqa: BLE001 — surfaced to every proxy (fail loudly)
            self.error = e
            import logging
            import sys
            msg = f"pydcop_b200: {self.kind}_gpu session '{self.key}' failed: {e!r} (no CPU fallback)"
            logging.getLogger("pydcop_b200").critical(msg)
            print(msg, file=sys.stderr, flush=True)
        finally:
            self._retire()

    def _publish(self, engine, cycle, finished):
        out = engine.values()
        if isinstance(out, tuple):
            idx, costs = out
        else:
            idx, costs = out, None
        vals = {}
        if self.kind == "syncbb":      # last value selection and the bound it came with; (None, None): never selected
            costs = engine.bounds()
        for i, n in enumerate(self.var_order):
            dom = domain_values(self.variables[n])
            if idx[i] < 0:
                vals[n] = (None, None)
                continue
            vals[n] = (dom[int(idx[i])], float(costs[i]) if costs is not None else 0.0)
        done = frozenset()
        if self.kind == "dba":
            fin = engine.finished_vars()
            done = frozenset(n for i, n in enumerate(self.var_order) if fin[i])
        cycles = None
        if self.kind == "syncbb":
            cycles = dict(zip(self.var_order, (int(c) for c in engine.cycle_counts())))
        self.snapshot = Snapshot(cycle, vals, None, finished, done, cycles)

    def _pseudo_tree(self, inst):
        """The orchestrator's pseudo-tree over the packed arrays; each node joins the constraints it owns
        in its node.constraints order (dpop.py:191-199)."""
        from ..pseudotree import tree_from_links
        cidx = {n: i for i, n in enumerate(sorted(self.constraints))}
        con_order = [[cidx[c] for c in self.var_links[n]] for n in self.var_order]
        return tree_from_links(self.var_order, self.tree_links, inst["dom_size"], inst["factor_ptr"],
                               inst["edge_var"], con_order)

    def _isolated_values(self, inst):
        """DSA on_start for a variable without neighbours (dsa.py:278-289): argopt of
        (own cost, value) with Python's tuple ordering on the real domain values."""
        out = np.zeros(len(self.var_order), dtype=np.int32)
        for i, n in enumerate(self.var_order):
            v = self.variables[n]
            dom = domain_values(v)
            cost = getattr(v, "cost_for_val", None)
            pairs = [((float(cost(x)) if cost else 0.0), x) for x in dom]
            try:
                best = min(pairs) if self.mode == "min" else max(pairs)
                out[i] = dom.index(best[1])
            except TypeError:  # unorderable domain values: first optimum
                cs = [p[0] for p in pairs]
                out[i] = int(np.argmin(cs) if self.mode == "min" else np.argmax(cs))
        return out
