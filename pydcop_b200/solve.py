"""Direct solve: a DCOP file (or arrays, or a pyDcop DCOP object) -> GPU engine -> result dict
(algorithms: maxsum, dsa, adsa, mgm, mgm2, gdba, dpop, dba, syncbb, mixeddsa).

The plugin modules (pydcop_b200/algorithms/) keep pyDcop's orchestrator, agents and one Python
computation object per graph node around the engine — that is the drop-in path, and it is what
bounds instance size (10^6 proxy objects and agent threads do not fit).  This entry skips the
control plane for large instances: ingestion (pydcop_b200.ingest) -> layout -> engine, and returns
the same result keys `pydcop solve` prints (pydcop/infrastructure/orchestrator.py:1262-1272,
pydcop/commands/solve.py:611-624): status, assignment, cost, violation, time, cycle, msg_count,
msg_size.

Parameters and defaults are the reference algorithms' own (maxsum.py:212-220, dsa.py:130-135,
mgm.py:78-81, mgm2.py:139-143, gdba.py:181-185; GDBA adds `stop_cycle` with MGM's convention).
MaxSum has no termination test of its own (maxsum.py: it runs until `stop_cycle` or the
orchestrator's timeout), so one of `stop_cycle` / `timeout` is required here as well; status is
FINISHED when `stop_cycle` was reached and TIMEOUT otherwise, as in the reference
(orchestrator.py:1262, commands/solve.py:560-580).  DPOP is exact and not iterative: it needs neither,
runs its UTIL and VALUE phases once on the pseudo-tree pydcop_b200.pseudotree builds, and is FINISHED at
cycle 0.
DBA (dba.py:265-268, plus `stop_cycle` with GDBA's convention) stops by itself once every variable with
neighbours has finished (its termination counter reached `max_distance`, or an End message arrived): the loop
then leaves early and reports the engine's cycle with status FINISHED.  DBA minimises only.
SyncBB (syncbb.py) takes no parameters and stops by itself: the loop enqueues launches of SYNCBB_CHUNK messages until
the last terminate message is delivered (FINISHED), or until the timeout (TIMEOUT, with the bounds and selections
reached so far).  `cycle` is the largest per-variable new_cycle count (messages a variable handled, plus one for the
first variable's start), which is what the reference's orchestrated run reports; `msg_count` is the number of SyncBB
messages posted (forward, backward, terminate and the start message).  The orchestrated run's msg_count also counts
the orchestrator's own traffic, which a direct run has none of.  A
variable that never selected a value is left out of the assignment and cost / violation are then None, as the
orchestrator reports an incomplete assignment (orchestrator.py:1226-1240).
MixedDSA (mixeddsa.py:119-124) runs `stop_cycle` rounds, DSA's convention (dsa.py:352); its cost and violation
count come from the same device reduction as every other algorithm's, so runs on a hard-constrained problem compare
directly with DBA's and GDBA's.

No CPU path: the engines raise EngineError without a CUDA device.  `engine_factory` exists so
the host logic can be tested without one.
"""
import json
import os
import time
from typing import Any, Callable, Dict, List, Optional, Sequence, Union

import numpy as np

from . import batch, ingest
from .layout import build_layout

MAXSUM_DEFAULTS = {"damping": 0.5, "damping_nodes": "both", "stability": 0.1, "noise": 0.01,
                   "start_messages": "leafs", "stop_cycle": 0}
DSA_DEFAULTS = {"probability": 0.7, "p_mode": "fixed", "variant": "B", "stop_cycle": 0}
ADSA_DEFAULTS = {"period": 0.5, "probability": 0.7, "variant": "B", "stop_cycle": 0}   # adsa.py:121-125 + stop_cycle
MGM_DEFAULTS = {"break_mode": "lexic", "stop_cycle": 0}
MGM2_DEFAULTS = {"threshold": 0.5, "favor": "unilateral", "stop_cycle": 0}
GDBA_DEFAULTS = {"modifier": "A", "violation": "NZ", "increase_mode": "E", "stop_cycle": 0}
DBA_DEFAULTS = {"infinity": 10000, "max_distance": 50, "stop_cycle": 0}
MIXEDDSA_DEFAULTS = {"proba_hard": 0.7, "proba_soft": 0.5, "variant": "B", "stop_cycle": 0}   # mixeddsa.py:119-124
DEFAULTS = {"maxsum": MAXSUM_DEFAULTS, "dsa": DSA_DEFAULTS, "mgm": MGM_DEFAULTS, "adsa": ADSA_DEFAULTS,
            "mgm2": MGM2_DEFAULTS, "gdba": GDBA_DEFAULTS, "dpop": {}, "dba": DBA_DEFAULTS, "syncbb": {},
            "mixeddsa": MIXEDDSA_DEFAULTS}
_CHOICES = {"damping_nodes": ("vars", "factors", "both", "none"),
            "start_messages": ("leafs", "leafs_vars", "all"),
            "p_mode": ("fixed", "arity"), "variant": ("A", "B", "C"),
            "break_mode": ("lexic", "random"), "favor": ("unilateral", "no", "coordinated"),
            "modifier": ("A", "M"), "violation": ("NZ", "NM", "MX"), "increase_mode": ("E", "R", "C", "T")}
ALGOS = {"maxsum": "maxsum", "maxsum_gpu": "maxsum", "dsa": "dsa", "dsa_gpu": "dsa",
         "mgm": "mgm", "mgm_gpu": "mgm", "adsa": "adsa", "adsa_gpu": "adsa", "mgm2": "mgm2", "mgm2_gpu": "mgm2",
         "gdba": "gdba", "gdba_gpu": "gdba", "dpop": "dpop", "dpop_gpu": "dpop", "dba": "dba", "dba_gpu": "dba",
         "syncbb": "syncbb", "syncbb_gpu": "syncbb", "mixeddsa": "mixeddsa", "mixeddsa_gpu": "mixeddsa"}
SYNCBB_CHUNK = 1 << 16   # SyncBB messages per launch: the timeout is checked between launches


def check_params(kind: str, params: Optional[Dict[str, Any]]) -> Dict[str, Any]:
    """Defaults + type / choice validation, the job of AlgoParameterDef
    (pydcop/algorithms/__init__.py:180-290): unknown names and invalid values raise ValueError."""
    defaults = DEFAULTS[kind]
    if not defaults and params:   # DPOP: exact and not iterative, so no stop_cycle either
        raise ValueError(f"{kind} takes no parameters: unknown algorithm parameter(s) {sorted(params)}")
    out = dict(defaults)
    for k, v in (params or {}).items():
        if k not in defaults:
            raise ValueError(f"Unknown parameter for algorithm {kind}: {k}")
        want = type(defaults[k])
        try:
            v = want(v) if want is not str else str(v)
        except (TypeError, ValueError):
            raise ValueError(f"Invalid value for parameter {k}: {v!r}") from None
        if k in _CHOICES and v not in _CHOICES[k]:
            raise ValueError(f"Invalid value for parameter {k}: {v!r} not in {_CHOICES[k]}")
        out[k] = v
    return out


def load(problem, seed: Optional[int] = None) -> ingest.DcopArrays:
    """DcopArrays from: a DcopArrays, a path / list of paths (YAML, or the binary container by its
    magic), a dict of front-door arrays, or a pyDcop DCOP object."""
    if isinstance(problem, ingest.DcopArrays):
        return problem
    if isinstance(problem, dict):
        return ingest.from_arrays(problem)
    if isinstance(problem, (str, os.PathLike)):
        with open(problem, "rb") as f:
            magic = f.read(len(ingest.MAGIC))
        if magic == ingest.MAGIC:
            return ingest.load_instance(problem)
        return ingest.load_yaml(problem, seed)
    if isinstance(problem, (list, tuple)):
        return ingest.load_yaml(problem, seed)
    if hasattr(problem, "variables") and hasattr(problem, "constraints"):
        return ingest.from_dcop(problem)
    raise TypeError(f"cannot load a DCOP from {type(problem).__name__}")


def isolated_values(dcop: ingest.DcopArrays, mode: str) -> np.ndarray:
    """DSA start value of a variable without NEIGHBOURS — no constraint at all, or only unary ones (the engines
    treat both as isolated and take this value verbatim): argopt of (own cost, value) in Python tuple order over
    the real domain values (dsa.py:278-289, relations.py:1641-1669)."""
    a = dcop.arrays
    out = np.zeros(dcop.n_vars, dtype=np.int32)
    uoff = np.concatenate([[0], np.cumsum(a["dom_size"].astype(np.int64))])
    fp, ev = np.asarray(a["factor_ptr"], dtype=np.int64), np.asarray(a["edge_var"], dtype=np.int64)
    n_nbr = np.zeros(dcop.n_vars, dtype=np.int64)
    if len(ev):
        np.add.at(n_nbr, ev, np.repeat(np.diff(fp) - 1, np.diff(fp)))
    for i in np.nonzero(n_nbr == 0)[0]:
        dom = dcop.values_of(int(i))
        pairs = [(float(a["unary"][uoff[i] + k]), x) for k, x in enumerate(dom)]
        try:
            best = min(pairs) if mode == "min" else max(pairs)
            out[i] = dom.index(best[1])
        except TypeError:  # unorderable values: first optimum
            cs = [p[0] for p in pairs]
            out[i] = int(np.argmin(cs) if mode == "min" else np.argmax(cs))
    return out


def solution_cost(dcop: ingest.DcopArrays, value_index, infinity: float = float("inf")):
    """(violation, cost): constraints and variable costs equal to `infinity` are counted, the
    others summed (pydcop/dcop/dcop.py:319-367; `infinity` default as commands/solve.py `-i`: float("inf"))."""
    a = dcop.arrays
    idx = np.asarray(value_index, dtype=np.int64)
    fp, ev = a["factor_ptr"].astype(np.int64), a["edge_var"].astype(np.int64)
    dom = a["dom_size"].astype(np.int64)
    lin = np.zeros(len(fp) - 1, dtype=np.int64)
    arity = np.diff(fp)
    for j in range(int(arity.max(initial=0))):
        m = arity > j
        e = fp[:-1][m] + j
        lin[m] = lin[m] * dom[ev[e]] + idx[ev[e]]
    costs = np.concatenate([
        np.asarray(a["tables"])[np.asarray(a["table_off"][:-1], dtype=np.int64) + lin].astype(np.float64),
        np.asarray(a["unary"], dtype=np.float64)[np.concatenate([[0], np.cumsum(dom)])[:-1] + idx]])
    hard = costs == infinity
    return int(hard.sum()), float(costs[~hard].sum())


def name_rank(dcop: ingest.DcopArrays) -> np.ndarray:
    """Position of every variable's name in sorted order: MGM's tie break (mgm.py:574-583)."""
    order = sorted(range(dcop.n_vars), key=lambda i: dcop.var_names[i])
    rank = np.zeros(dcop.n_vars, dtype=np.int32)
    rank[order] = np.arange(dcop.n_vars, dtype=np.int32)
    return rank


def _var_inputs(kind, dcop, mode):
    """(var_rank, isolated_value) of `dcop` as the engine of `kind` takes them, canonical order; None where it takes
    none."""
    if kind == "dpop":
        return None, None
    return (name_rank(dcop) if kind in ("mgm", "mgm2", "gdba", "dba", "syncbb") else None,
            isolated_values(dcop, mode) if kind not in ("mgm2", "dba", "mixeddsa") else None)


def _default_engine(kind, layout, dcop, params, mode, precision, device, seed):
    from .engine import make_engine
    tree = None
    if kind == "dpop":
        from .pseudotree import build_tree
        a = dcop.arrays
        tree = build_tree(a["dom_size"], a["factor_ptr"], a["edge_var"])
    var_rank, isolated_value = _var_inputs(kind, dcop, mode)
    return make_engine(kind, layout, params, mode=mode, precision=precision, device=device, seed=seed or 0,
                       var_rank=var_rank, isolated_value=isolated_value, tree=tree)


def _sharded_engine(kind, inst, dcop, params, mode, precision, device, seed, partition, halo, sharded_kwargs):
    """One rank's engine of a multi-process run (torch.distributed is initialised): the variables
    are split over the ranks (rank 0 computes the partition and broadcasts it), boundary rows /
    values are exchanged every cycle (pydcop_b200.multigpu, multigpu_dsa, multigpu_mgm2)."""
    import torch
    import torch.distributed as dist
    from .multigpu import ShardedMaxSum, broadcast_owner
    from .multigpu_dsa import ShardedDsa
    from .multigpu_mgm2 import ShardedMgm2
    if kind in ("mgm", "gdba", "dpop", "dba", "syncbb", "mixeddsa"):
        raise ValueError(f"{kind} is not sharded: run it on one GPU")
    rank, world = dist.get_rank(), dist.get_world_size()
    kw = dict(sharded_kwargs or {})
    dev = device if device is not None else (torch.device("cuda", torch.cuda.current_device())
                                             if torch.cuda.is_available() and "engine_factory" not in kw
                                             else torch.device("cpu"))
    if isinstance(partition, str):
        owner, err = broadcast_owner(inst, world, rank, dev, partition)
    else:                                  # an owner array every rank already holds
        owner, err = np.asarray(partition, dtype=np.int32), None
    if kind == "maxsum":
        eng = ShardedMaxSum(inst, rank, world, dev, precision=precision, halo=halo, partition=owner, mode=mode,
                            damping=params["damping"], damping_nodes=params["damping_nodes"],
                            stability=params["stability"], start_messages=params["start_messages"],
                            **dict({"record_sent": False} if "engine_factory" not in kw else {}, **kw))
    elif kind == "mgm2":
        eng = ShardedMgm2(inst, rank, world, dev, precision=precision, halo=halo, partition=owner, mode=mode,
                          threshold=params["threshold"], favor=params["favor"], stop_cycle=params["stop_cycle"],
                          seed=seed or 0, var_rank=name_rank(dcop), **kw)
    else:
        eng = ShardedDsa(inst, rank, world, dev, precision=precision, halo=halo, partition=owner, mode=mode,
                         probability=params["probability"], p_mode=params.get("p_mode", "fixed"),
                         variant=params["variant"], stop_cycle=params["stop_cycle"], seed=seed or 0,
                         isolated_value=isolated_values(dcop, mode), var_costs=(kind == "adsa"), **kw)
    eng.partition_error = err
    return eng


def solve(problem, algo: str = "maxsum", algo_params: Optional[Dict[str, Any]] = None,
          timeout: Optional[float] = None, precision: str = "f32", device=None,
          seed: Optional[int] = None, infinity: float = float("inf"), chunk: int = 50,
          on_cycle: Optional[Callable[[int, np.ndarray], None]] = None,
          engine_factory: Optional[Callable] = None, distributed: Optional[bool] = None,
          partition="auto", halo: str = "auto", sharded_kwargs: Optional[Dict[str, Any]] = None,
          trace: bool = False, best: bool = False) -> Dict[str, Any]:
    """Run `algo` on `problem` and return pyDcop's result dict.

    Under `torchrun` (torch.distributed initialised, world size > 1; `distributed` None = detect)
    every rank calls solve() with the same arguments: the variables are partitioned over the
    ranks (`partition`: auto | blocks | multilevel | an owner array), each rank runs its shard on
    its GPU and boundary messages / values are exchanged every cycle (`halo`: auto | p2p | nccl);
    every rank returns the same result.  `seed` defaults to 0 there (all ranks must draw the same
    noise).

    problem      see `load`
    algo         maxsum | dsa | adsa | mgm | mgm2 | gdba | dpop | dba | syncbb | mixeddsa (the *_gpu spellings of the plugin
                 modules are accepted)
    algo_params  the reference's parameter names; `stop_cycle` bounds the run in cycles
    timeout      wall-clock bound in seconds (checked every `chunk` cycles; SyncBB: between launches of
                 SYNCBB_CHUNK messages)
    precision    f32 | f64 (f64 reproduces the reference's double arithmetic bit for bit)
    seed         MaxSum: the U(0, noise) draws; DSA: the Philox stream of the random choices
    on_cycle     callback(cycle, value_index) after every chunk (metrics collection)
    trace        the result gains "trace": {"cycle", "time", "cost", "violation"}, one entry per cycle the engine ran
                 (pydcop solve --collect_on cycle_change): each cycle's solution cost recorded on the device inside
                 the step loop, without a host round trip; "time" is seconds on the device timer since the first
                 cycle was enqueued.  The last entry's cost and violation are the result's.  Single-GPU iterative
                 algorithms only (not dpop, syncbb or torchrun).
    best         the result gains "best": {"cycle", "cost", "violation", "assignment"}, the run's best cycle (the
                 anytime result): of the cycles the trace numbers, the first with the fewest violations and, among
                 those, the strictly best cost in the problem's objective; later ties do not replace it.  Kept on the
                 device inside the step loop with or without `trace`; None when no cycle ran.  The same algorithms
                 as `trace`.
    SyncBB has no cycles to chunk: it ignores `chunk` and never calls `on_cycle` (a variable may have no value
    until the search ends).
    """
    kind, params, stop_cycle = _algorithm(algo, algo_params, timeout)
    if distributed is None:
        distributed = _under_torchrun()
    if trace:
        _check_trace(kind, distributed)
    if best:
        _check_trace(kind, distributed, "best")
    if distributed and seed is None:
        seed = 0
    t0 = time.perf_counter()
    dcop = load(problem, seed)
    mode = dcop.objective
    if kind == "dba" and mode != "min":
        from .engine import DBA_MODE_ERROR
        raise ValueError(DBA_MODE_ERROR)
    if kind == "syncbb":                   # before any device work: assignment_cost raises on such a constraint
        arity = np.diff(np.asarray(dcop.arrays["factor_ptr"], dtype=np.int64))
        big = np.nonzero(arity > 2)[0]
        if len(big):
            raise ValueError(f"constraint {dcop.con_names[int(big[0])]} has arity {int(arity[big[0]])}: SyncBB "
                             "supports binary constraints only (syncbb.py:456)")
    inst = dcop.instance()
    if kind == "maxsum":
        inst["unary"] = ingest.add_noise(inst["unary"], params["noise"], seed)
    n_gpus = 1
    if distributed:
        import torch.distributed as dist
        engine = _sharded_engine(kind, inst, dcop, params, mode, precision, device, seed, partition, halo,
                                 sharded_kwargs)
        n_gpus = dist.get_world_size()
    else:
        layout = build_layout(**inst)
        if engine_factory is not None:
            engine = engine_factory(kind, layout, dict(inst, var_rank=name_rank(dcop)),
                                    dict(params, mode=mode, seed=seed or 0))
        else:
            engine = _default_engine(kind, layout, dcop, params, mode, precision, device, seed)
    t_packed = time.perf_counter()
    engine.init()
    deadline = None if timeout is None else t0 + float(timeout)
    if kind == "syncbb":
        return _finish_syncbb(engine, dcop, deadline, infinity, precision, t0, t_packed)
    tracer = _Trace(engine, stop_cycle, infinity, dcop.arrays["unary"], None,
                    lambda idx: [solution_cost(dcop, idx, infinity)], best, trace, mode) if trace or best else None
    cycle, status = _run_cycles(engine, stop_cycle, chunk, deadline, distributed, on_cycle, kind == "dba",
                                tracer.after_cycle if tracer else None)
    if kind == "dba":                      # the rounds that changed the state
        cycle = engine.cycle
    idx = _indices(engine)
    if hasattr(getattr(engine, "engine", engine), "_solution_cost"):   # reduced on the device(s); sharded engines all-reduce over NCCL
        cost, violation = engine.solution_cost(infinity, dcop.arrays["unary"])
    else:                                  # engine seam of the CPU tests
        violation, cost = solution_cost(dcop, idx, infinity)
    out = {"status": status, "assignment": dcop.assignment(idx), "cost": cost,
           "violation": violation, "time": time.perf_counter() - t0, "cycle": 0 if kind == "dpop" else cycle,
           "msg_count": 0, "msg_size": 0,  # nothing crosses an agent boundary
           "algo": kind, "precision": precision, "n_gpus": n_gpus,
           "ingest_time": t_packed - t0,
           # bytes this process moved host -> device (problem arrays) and device -> host (assignment, costs)
           "h2d_bytes": int(getattr(getattr(engine, "engine", engine), "h2d_bytes", 0)),
           "d2h_bytes": int(len(idx) * 12 + 16)}
    if tracer is not None:
        traces, kept = tracer.finish(cycle if kind == "dba" else None)
        if trace:
            out["trace"] = traces[0]
        if best:
            out["best"] = _best_entry(dcop, kept[0][0], kept[1])
    return out


def _algorithm(algo, algo_params, timeout):
    """(kind, checked parameters, stop_cycle) of `algo`, or ValueError."""
    if algo not in ALGOS:
        raise ValueError(f"unknown algorithm {algo!r}: expected one of {sorted(ALGOS)}")
    kind = ALGOS[algo]
    params = check_params(kind, algo_params)
    stop_cycle = 1 if kind == "dpop" else 0 if kind == "syncbb" else int(params["stop_cycle"])   # DPOP: both phases in one step
    if not stop_cycle and timeout is None and kind != "syncbb":
        raise ValueError(f"{kind} does not stop by itself: give algo_params['stop_cycle'] or a timeout")
    return kind, params, stop_cycle


def _under_torchrun():
    try:
        import torch.distributed as dist
        return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    except ImportError:
        return False


def _run_cycles(engine, stop_cycle, chunk, deadline, distributed=False, on_cycle=None, stops_itself=False,
                after_cycle=None):
    """Step an initialised engine `chunk` cycles at a time until stop_cycle (0: none) or the deadline (checked before
    every chunk; under torchrun every rank leaves in the same round), or, with `stops_itself`, until engine.finished.
    `after_cycle`: called after every single step(1) of a chunk stepped one cycle at a time (the host trace of the
    engine seam).  Returns (cycles run, FINISHED | TIMEOUT)."""
    cycle, status = 0, "FINISHED"
    while True:
        n = chunk if not stop_cycle else min(chunk, stop_cycle - cycle)
        if n <= 0:
            break
        expired = deadline is not None and time.perf_counter() >= deadline
        if distributed and deadline is not None:   # every rank must leave the loop in the same round
            import torch
            import torch.distributed as dist
            flag = torch.tensor([int(expired)], dtype=torch.int32, device=engine.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MAX)
            expired = bool(flag.item())
        if expired:
            status = "TIMEOUT"
            break
        if after_cycle is None:
            engine.step(n)
        else:
            for _ in range(n):
                engine.step(1)
                after_cycle()
        cycle += n
        if on_cycle is not None:
            on_cycle(cycle, _indices(engine))
        if stops_itself and engine.finished:   # DBA: every variable with neighbours finished, or stop_cycle
            break
    return cycle, status


TRACE_BYTES = 64 << 20   # device rows of one trace block, at most: a block of n_seg problems holds fewer cycles


def _check_trace(kind, distributed, what="trace"):
    if kind in ("dpop", "syncbb"):
        raise ValueError(f"{what}: {kind} has no cycles to trace")
    if distributed:
        raise ValueError(f"{what}: traces are recorded on one GPU: start the run without torchrun")


def best_better(cost, viol, best_cost, best_viol, mode_max):
    """csrc/cost.cuh's best_better, the rule the device keeps a trace's best row by, for the host trace of the
    engine seam: strictly fewer violations, or equal ones and a strictly better cost (a NaN cost never better)."""
    if viol != best_viol:
        return viol < best_viol
    if cost != cost:
        return False
    if best_cost != best_cost:
        return True
    return cost > best_cost if mode_max else cost < best_cost


class _Trace:
    """The cost of every cycle of one engine run: recorded on the device (engine.start_trace), or for an engine
    without one (the CPU tests' engine seam) on the host after every single cycle: host_costs(value_index) ->
    [(violation, cost)] per segment, with solution_cost.  best: each segment's best cycle and its values are kept too
    (var_start: the segments' variable ranges, canonical order); rows=False: the rows serve the best only."""

    def __init__(self, engine, stop_cycle, infinity, unary, seg, host_costs, best=False, rows=True, mode="min",
                 var_start=None):
        self.engine, self.rows, self.t0 = engine, [], time.perf_counter()
        self.n_seg = 1 if seg is None else seg[2]
        self.keep_best, self.keep_rows = best, rows
        self.device = hasattr(engine, "start_trace")
        if self.device:
            want = stop_cycle or 1024
            engine.start_trace(max(1, min(want, TRACE_BYTES // (16 * self.n_seg))), infinity, unary, seg, best=best,
                               rows=rows)
        else:
            self.host_costs, self.cycle = host_costs, getattr(engine, "cycle", 0)
            self.mode_max, self.var_start = mode == "max", var_start
            self.best_row = [(0, 0.0, 0)] * self.n_seg   # (cycle, cost, violation); cycle 0 = none
            self.best_value = None
        # what _run_cycles calls after every single cycle: nothing when the device records inside the step loop
        self.after_cycle = None if self.device else self._host_row

    def _host_row(self):
        c = getattr(self.engine, "cycle", None)
        if c is not None and c == self.cycle:   # the engine stopped: no cycle ran
            return
        self.cycle = c
        t = time.perf_counter() - self.t0
        idx = _indices(self.engine)
        costs = self.host_costs(idx)
        self.rows.append((t, costs))
        if not self.keep_best:
            return
        n = len(self.rows)
        if self.best_value is None:
            self.best_value = np.zeros_like(idx)
        for k, (v, cost) in enumerate(costs):
            b = self.best_row[k]
            if b[0] == 0 or best_better(float(cost), float(v), b[1], float(b[2]), self.mode_max):
                self.best_row[k] = (n, float(cost), int(v))
                lo, hi = (0, len(idx)) if self.var_start is None else (self.var_start[k], self.var_start[k + 1])
                self.best_value[lo:hi] = idx[lo:hi]

    def best(self):
        """(cycle, cost, violation) of every segment's best cycle (cycle 0: none ran) and the values of the best
        cycles, canonical order."""
        if self.device:
            b = self.engine.best()
            return [(int(c), float(x), int(v)) for c, x, v in zip(b["cycle"], b["cost"], b["violation"])], b["value"]
        return self.best_row, _indices(self.engine) if self.best_value is None else self.best_value

    def result(self, n_cycles=None):
        """One trace dict per segment; `n_cycles`: keep the first n (DBA: the rounds that changed the state)."""
        if self.device:
            tr = self.engine.trace()
            t, cost, viol = tr["time"], tr["cost"], tr["violation"]
        else:
            t = np.array([r[0] for r in self.rows], dtype=np.float64)
            cost = np.array([[c for _, c in r[1]] for r in self.rows], dtype=np.float64).reshape(-1, self.n_seg)
            viol = np.array([[v for v, _ in r[1]] for r in self.rows], dtype=np.int64).reshape(-1, self.n_seg)
        n = len(t) if n_cycles is None else min(len(t), int(n_cycles))
        return [{"cycle": list(range(1, n + 1)), "time": [float(x) for x in t[:n]],
                 "cost": [float(x) for x in cost[:n, k]], "violation": [int(x) for x in viol[:n, k]]}
                for k in range(self.n_seg)]

    def finish(self, n_cycles=None):
        """(result(n_cycles) or None without rows, best() or None without a best), the device trace stopped."""
        out = (self.result(n_cycles) if self.keep_rows else None, self.best() if self.keep_best else None)
        if self.device:
            self.engine.stop_trace()
        return out


def _best_entry(dcop, row, value):
    """A result's "best": its cycle, cost, violation and assignment (value: the problem's slice); None when no cycle
    ran."""
    cycle, cost, violation = row
    if not cycle:
        return None
    return {"cycle": cycle, "cost": cost, "violation": violation, "assignment": dcop.assignment(value)}


BATCHED = ("maxsum", "dsa", "adsa", "mgm", "mgm2", "gdba", "mixeddsa")
# the parameters problems of one engine may differ in: read per variable through a parameter set (DSA, A-DSA, MGM-2,
# GDBA, MixedDSA), drawn per problem when the union is built (MaxSum's noise), or never read by the engine (A-DSA's
# period, MGM's break_mode); every other parameter is one scalar per engine and splits groups
IN_UNION = {"dsa": ("probability", "p_mode", "variant"), "adsa": ("period", "probability", "variant"),
            "mgm": ("break_mode",), "mgm2": ("threshold", "favor"), "gdba": ("modifier", "violation"),
            "mixeddsa": ("proba_hard", "proba_soft", "variant"), "maxsum": ("noise",)}
ENGINE_PSETS = ("dsa", "adsa", "mgm2", "gdba", "mixeddsa")   # the families whose engines take parameter sets
NOT_BATCHED = {"dba": "it stops per problem by itself, so each problem would need its own finish cycle",
               "dpop": "it computes over a pseudo-tree of the whole problem",
               "syncbb": "it searches over an order of the whole problem"}


def solve_batch(problems, algo: str, algo_params: Union[None, Dict[str, Any], Sequence] = None,
                timeout: Optional[float] = None,
                precision: str = "f32", device=None, seed: Union[None, int, Sequence[int]] = None,
                infinity: float = float("inf"),
                chunk: int = 50, max_vars: int = batch.MAX_BATCH_VARS,
                engine_factory: Optional[Callable] = None, trace: bool = False,
                best: bool = False) -> List[Dict[str, Any]]:
    """Run `algo` on every problem of `problems` and return one result dict per problem, in input order, with
    solve()'s keys.

    problems  a list of anything `load` accepts, ONE problem per entry (a list of paths inside it is one DCOP split
              over files, as in solve())
    The problems run as disjoint unions, one engine per group: problems of one objective (min or max), cut in input
    order so that no engine exceeds `max_vars` variables or an int32 index range; the groups run one after the other.
    Every problem keeps its own Philox counters, name ranks and start values, so `assignment`, `status` and `cycle`
    equal those of solve(problem, algo, algo_params, precision=precision, seed=seed) and `cost` / `violation` equal
    them up to the order of the device reduction (per problem, fg_solution_cost_segmented).
    seed      None or an int: one seed for every problem (solve()'s default draws with 0); or a sequence of ints, one
              per problem: problem i's result is then solve(problems[i], ..., seed=seed[i])'s.  With it the same
              problem can appear many times, once per seed, to compare runs of a stochastic algorithm (pydcop
              batch's iterations); a DcopArrays entry is not re-parsed.
    algo_params  None or a dict: one set of parameters for every problem; or a sequence with one dict (or None) per
              problem: problem i's result is then solve(problems[i], algo, algo_params[i], ...)'s (pydcop batch's
              parameter combinations).  The parameters IN_UNION names run in one engine, each variable reading its
              problem's set; problems that differ in another parameter (stop_cycle, MaxSum's damping, GDBA's
              increase_mode, ...) run in separate groups.
    `timeout` bounds the whole batch: a problem whose group has not reached stop_cycle when it expires reports
    TIMEOUT at the cycle its group reached (0 for groups that had not started).
    `time` and `ingest_time` are the whole batch's (loading, unions, layouts and engines for ingest_time);
    `h2d_bytes` is the problem's engine's.  `n_gpus` is 1: a batch runs on one device, never under torchrun.
    algo: maxsum | dsa | adsa | mgm | mgm2 | gdba | mixeddsa (the fixed-length families; dba, dpop and syncbb are
    refused).  engine_factory(kind, layout, inst, params): as in solve(), `inst` with var_rank, var_global_id,
    var_seed (None when the group's problems share one seed, params["seed"]) and var_pset (None when they share one
    parameter set; else the group's sets are params["psets"]).
    trace: every result gains solve()'s "trace", cut out of its group's per-problem record (its times are the
    group's); the trace of a problem whose group never started is empty.
    best: every result gains solve()'s "best", kept per problem on the device (its cycle in the trace's numbering);
    None for a problem whose group never started.
    """
    kind = ALGOS.get(algo)
    if kind in NOT_BATCHED:
        raise ValueError(f"{kind} is not batched: {NOT_BATCHED[kind]}")
    problems = list(problems)
    if kind is None:
        _algorithm(algo, None, timeout)   # unknown algorithm
    if algo_params is None or isinstance(algo_params, dict):
        kind, params, stop_cycle = _algorithm(algo, algo_params, timeout)
        per_problem = None
    else:
        per_problem = _batch_params(algo, algo_params, timeout, len(problems))
        kind, params, stop_cycle = per_problem[0] if per_problem else _algorithm(algo, None, timeout)
    if not problems:
        raise ValueError("solve_batch needs at least one problem")
    seeds = _batch_seeds(seed, len(problems))
    if _under_torchrun():
        raise ValueError("solve_batch runs on one GPU: start it without torchrun")
    t0 = time.perf_counter()
    deadline = None if timeout is None else t0 + float(timeout)
    dcops = []
    for i, p in enumerate(problems):
        try:
            dcops.append(load(p, seeds[i]))
        except (ValueError, TypeError) as e:
            raise ValueError(f"problem {i}: {e}") from e
        batch.check_problem(i, dcops[-1])
    results: List[Optional[Dict[str, Any]]] = [None] * len(dcops)
    ingest_time = time.perf_counter() - t0
    keys = sets = None
    if per_problem is not None:
        checked = [p for _, p, _ in per_problem]
        keys = [batch.pset_key({k: v for k, v in p.items() if k not in IN_UNION[kind]}) for p in checked]
        sets = [batch.pset_key(p) for p in checked]
    for members in batch.groups(dcops, max_vars, keys, sets):
        t_group = time.perf_counter()
        mode = dcops[members[0]].objective
        group_params = None if per_problem is None else [per_problem[i][1] for i in members]
        if group_params is not None:
            params, stop_cycle = group_params[0], per_problem[members[0]][2]
        noise = ([p["noise"] for p in group_params] if group_params is not None else params["noise"]) \
            if kind == "maxsum" else 0.0
        if engine_factory is not None:
            var_inputs = lambda d: (name_rank(d), None)  # noqa: E731
        else:
            var_inputs = lambda d: _var_inputs(kind, d, mode)  # noqa: E731
        u = batch.build_union(dcops, members, var_inputs, noise, [seeds[i] for i in members], group_params)
        layout = batch.union_layout(u, dcops)
        # one seed for the whole group: the scalar key, as solve() runs; else each variable's own (u.var_seed)
        group_seed = seeds[members[0]] or 0
        var_seed = None if kind == "maxsum" else u.var_seed   # MaxSum draws nothing on the device: its noise is in u
        # one parameter set for the whole group: the scalars; else each variable's own set (u.var_pset)
        var_pset = u.var_pset if kind in ENGINE_PSETS else None
        psets = u.psets if var_pset is not None else None
        if engine_factory is not None:
            engine = engine_factory(kind, layout, dict(u.inst, var_rank=u.var_rank, var_global_id=u.var_global_id,
                                                       var_seed=var_seed, var_pset=var_pset),
                                    dict(params, mode=mode, seed=group_seed, **({"psets": psets} if psets else {})))
        else:
            from .engine import make_engine
            engine = make_engine(kind, layout, params, mode=mode, precision=precision, device=device, seed=group_seed,
                                 var_rank=u.var_rank, isolated_value=u.isolated_value, var_global_id=u.var_global_id,
                                 var_seed=var_seed, var_pset=var_pset, psets=psets)
        ingest_time += time.perf_counter() - t_group
        engine.init()
        tracer = None
        if trace or best:
            tracer = _Trace(engine, stop_cycle, infinity, u.unary, (u.seg_factor, u.seg_var, len(members)),
                            lambda idx: [solution_cost(dcops[i], idx[u.var_start[k]:u.var_start[k + 1]], infinity)
                                         for k, i in enumerate(members)], best, trace, mode, u.var_start)
        cycle, status = _run_cycles(engine, stop_cycle, chunk, deadline,
                                    after_cycle=tracer.after_cycle if tracer else None)
        traces, kept = tracer.finish() if tracer is not None else (None, None)
        idx = _indices(engine)
        if hasattr(engine, "solution_costs_segmented"):   # reduced per problem on the device
            costs, violations = engine.solution_costs_segmented(u.seg_factor, u.seg_var, len(members), infinity,
                                                                u.unary)
        else:                                  # engine seam of the CPU tests
            violations, costs = zip(*(solution_cost(dcops[i], idx[u.var_start[k]:u.var_start[k + 1]], infinity)
                                      for k, i in enumerate(members)))
        h2d = int(getattr(engine, "h2d_bytes", 0))
        for k, i in enumerate(members):
            v = idx[u.var_start[k]:u.var_start[k + 1]]
            results[i] = {"status": status, "assignment": dcops[i].assignment(v), "cost": float(costs[k]),
                          "violation": int(violations[k]), "cycle": cycle, "msg_count": 0, "msg_size": 0,
                          "algo": kind, "precision": precision, "n_gpus": 1, "h2d_bytes": h2d,
                          "d2h_bytes": int(len(v) * 12 + 16)}
            if traces is not None:
                results[i]["trace"] = traces[k]
            if kept is not None:
                results[i]["best"] = _best_entry(dcops[i], kept[0][k], kept[1][u.var_start[k]:u.var_start[k + 1]])
    total = time.perf_counter() - t0
    for r in results:
        r.update(time=total, ingest_time=ingest_time)
    return results


def _batch_params(algo, algo_params, timeout, n: int) -> list:
    """solve_batch's per-problem `algo_params`: (kind, checked parameters, stop_cycle) of every problem, each dict
    through _algorithm, errors prefixed with the problem's index."""
    try:
        entries = list(algo_params)
    except TypeError:
        raise ValueError(f"algo_params must be a dict or a sequence of dicts, got {type(algo_params).__name__}") \
            from None
    if len(entries) != n:
        raise ValueError(f"algo_params: {len(entries)} parameter dicts for {n} problems")
    out = []
    for i, p in enumerate(entries):
        if p is not None and not isinstance(p, dict):
            raise ValueError(f"problem {i}: algo_params must be a dict or None, got {type(p).__name__}")
        try:
            out.append(_algorithm(algo, p, timeout))
        except ValueError as e:
            raise ValueError(f"problem {i}: {e}") from e
    return out


def _batch_seeds(seed, n: int) -> list:
    """solve_batch's `seed` as one seed per problem: None or an int serves all `n`, a sequence must hold n ints."""
    if seed is None or isinstance(seed, (int, np.integer)):
        return [seed] * n
    try:
        seeds = list(seed)
    except TypeError:
        raise ValueError(f"seed must be an int or a sequence of ints, got {type(seed).__name__}") from None
    if len(seeds) != n:
        raise ValueError(f"seed: {len(seeds)} seeds for {n} problems")
    for i, s in enumerate(seeds):
        if isinstance(s, bool) or not isinstance(s, (int, np.integer)):
            raise ValueError(f"seed {i}: expected an int, got {s!r}")
    return [int(s) for s in seeds]


def _finish_syncbb(engine, dcop, deadline, infinity, precision, t0, t_packed):
    status = "FINISHED"
    while not engine.finished:
        if deadline is not None and time.perf_counter() >= deadline:
            status = "TIMEOUT"
            break
        engine.step(SYNCBB_CHUNK)
    idx = _indices(engine)
    has = idx >= 0
    if has.all():
        if hasattr(engine, "_solution_cost"):
            cost, violation = engine.solution_cost(infinity, dcop.arrays["unary"])
        else:                              # engine seam of the CPU tests
            violation, cost = solution_cost(dcop, idx, infinity)
    else:                                  # incomplete assignment (orchestrator.py:1226-1240)
        cost = violation = None
    full = dcop.assignment(np.maximum(idx, 0))
    names = list(full)
    assignment = {names[i]: full[names[i]] for i in range(len(names)) if has[i]}
    return {"status": status, "assignment": assignment, "cost": cost, "violation": violation,
            "time": time.perf_counter() - t0, "cycle": engine.cycle, "msg_count": int(engine.messages),
            "msg_size": 0, "algo": "syncbb", "precision": precision, "n_gpus": 1, "ingest_time": t_packed - t0,
            "h2d_bytes": int(getattr(engine, "h2d_bytes", 0)), "d2h_bytes": int(len(idx) * 12 + 16)}


def _indices(engine) -> np.ndarray:
    out = engine.values()
    return np.asarray(out[0] if isinstance(out, tuple) else out)


def main(argv=None):
    """`python -m pydcop_b200.solve --algo maxsum -p stop_cycle:100 problem.yaml` — argument names
    follow `pydcop solve` (commands/solve.py:380-470): -a/--algo, -p/--algo_params name:value,
    -t/--timeout; prints the result as JSON.  With --batch every file is one problem (solve_batch) and the output
    is a JSON list in file order, each entry with "problem": its path."""
    import argparse
    ap = argparse.ArgumentParser(prog="pydcop_b200.solve")
    ap.add_argument("dcop_files", nargs="+")
    ap.add_argument("-a", "--algo", default="maxsum", choices=sorted(ALGOS))
    ap.add_argument("-p", "--algo_params", action="append", default=[], metavar="name:value")
    ap.add_argument("-t", "--timeout", type=float, default=None)
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("-i", "--infinity", type=float, default=float("inf"),
                    help="cost that marks a violated hard constraint; like `pydcop solve -i` it defaults to inf "
                         "(commands/solve.py:315-324: the help text there says 10 000, the default is float('inf'))")
    ap.add_argument("--no-assignment", action="store_true",
                    help="omit the assignment from the output (10^6 variables)")
    ap.add_argument("--save", metavar="FILE", help="also write the instance as a binary container")
    ap.add_argument("--run_metrics", metavar="FILE",
                    help="CSV of cycle,time,cost,violation,msg_count,msg_size,status every --metrics_every "
                         "cycles (the columns of `pydcop solve --run_metrics`, commands/solve.py:356-375)")
    ap.add_argument("--metrics_every", type=int, default=10, metavar="CYCLES")
    ap.add_argument("--collect_on", choices=["cycle_change"], default=None,
                    help="cycle_change: the solution cost of EVERY cycle, recorded on the device inside the step loop "
                         "(solve(trace=True)): --run_metrics gets one row per cycle, --batch entries a \"trace\"")
    ap.add_argument("--best", action="store_true",
                    help="add the run's best cycle (solve(best=True)): \"best\" with its cycle, cost, violation and "
                         "assignment, kept on the device; in every --batch entry too")
    ap.add_argument("--partition", default="auto", choices=["auto", "blocks", "multilevel"],
                    help="under torchrun: how the variables are split over the GPUs")
    ap.add_argument("--batch", action="store_true",
                    help="every file is one problem, all solved in one engine run per objective (solve_batch); "
                         "prints a JSON list in file order")
    ap.add_argument("--iterations", type=int, default=None, metavar="N",
                    help="with --batch: solve every file N times, with seeds --seed + r for r = 0..N-1 (--seed "
                         "defaults to 0 here), as `pydcop batch` iterations; the list is file-major and every entry "
                         "carries \"iteration\" and \"seed\"")
    ap.add_argument("--sweep", action="append", default=[], metavar="name:v1,v2,...",
                    help="with --batch: solve every file once per combination of the swept parameters' values, as "
                         "`pydcop batch` expands its algo_params lists (names sorted, each value list sorted as "
                         "strings); the list is file-major, then combination, then iteration, and every entry carries "
                         "its checked \"algo_params\"")
    args = ap.parse_args(argv)
    if args.iterations is not None and not args.batch:
        ap.error("--iterations needs --batch")
    if args.sweep and not args.batch:
        ap.error("--sweep needs --batch")
    if args.iterations is not None and args.iterations < 1:
        ap.error("--iterations must be >= 1")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if args.batch:
        if args.run_metrics or args.save or world > 1:
            ap.error("--batch runs on one GPU and takes neither --run_metrics, --save nor torchrun")
        return _main_batch(args, _algo_params(ap, args), _sweeps(ap, args))
    trace = args.collect_on == "cycle_change"
    if world > 1:   # launched by torchrun: one process per GPU over NCCL
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    params = _algo_params(ap, args)
    files = args.dcop_files if len(args.dcop_files) > 1 else args.dcop_files[0]
    dcop = load(files, args.seed)
    if args.save and rank == 0:
        ingest.save_instance(args.save, dcop)
    rows, t_start = [], time.perf_counter()

    def collect(cycle, idx):
        violation, cost = solution_cost(dcop, idx, args.infinity)
        rows.append((cycle, time.perf_counter() - t_start, cost, violation, 0, 0, "RUNNING"))

    host_rows = args.run_metrics and not trace
    res = solve(dcop, args.algo, params, args.timeout, args.precision, seed=args.seed,
                infinity=args.infinity, partition=args.partition,
                chunk=max(1, args.metrics_every) if host_rows else 50,
                on_cycle=collect if host_rows else None, trace=trace, best=args.best)
    if trace and args.run_metrics:
        tr = res.pop("trace")
        rows = [(c, t, cost, v, 0, 0, "RUNNING")
                for c, t, cost, v in zip(tr["cycle"], tr["time"], tr["cost"], tr["violation"])]
    if args.run_metrics and rank == 0:
        import csv
        with open(args.run_metrics, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["cycle", "time", "cost", "violation", "msg_count", "msg_size", "status"])
            w.writerows(rows)
            w.writerow([res["cycle"], res["time"], res["cost"], res["violation"], 0, 0, res["status"]])
    if args.no_assignment:
        _drop_assignment(res)
    if rank == 0:
        print(json.dumps(res, indent=2, sort_keys=True, default=str))
    if world > 1:
        dist.destroy_process_group()
    return 0


def _drop_assignment(res):
    """--no-assignment: the result without its assignments, the best cycle's included."""
    res.pop("assignment")
    if res.get("best"):
        res["best"].pop("assignment")


def _algo_params(ap, args):
    params = {}
    for p in args.algo_params:
        if ":" not in p:
            ap.error(f"algo_params must be name:value, got {p!r}")
        k, v = p.split(":", 1)
        params[k] = v
    return params


def _sweeps(ap, args):
    """--sweep name:v1,v2,... as [(name, [values])], names sorted and every value list sorted as strings (pydcop
    batch's parameters_configuration); a name also given to -p, twice, or without values is an argparse error."""
    fixed = {p.split(":", 1)[0] for p in args.algo_params}
    out = {}
    for s in args.sweep:
        if ":" not in s:
            ap.error(f"--sweep must be name:v1,v2,..., got {s!r}")
        k, vs = s.split(":", 1)
        values = [v for v in vs.split(",") if v != ""]
        if not values:
            ap.error(f"--sweep {k}: no values")
        if k in fixed:
            ap.error(f"parameter {k} is given to both -p and --sweep")
        if k in out:
            ap.error(f"--sweep {k} is given twice")
        out[k] = sorted(values)
    return sorted(out.items())


def _main_batch(args, params, sweeps=()):
    if sweeps:
        return _main_sweep(args, params, sweeps)
    if args.iterations is None:
        res = solve_batch(args.dcop_files, args.algo, params, args.timeout, args.precision, seed=args.seed,
                          infinity=args.infinity, trace=args.collect_on == "cycle_change", best=args.best)
        for path, r in zip(args.dcop_files, res):
            r["problem"] = path
    else:
        # every file is read once; a YAML file's own noise_level draws are made then, with the first seed
        base, n = args.seed or 0, args.iterations
        dcops = [load(path, base) for path in args.dcop_files]
        res = solve_batch([d for d in dcops for _ in range(n)], args.algo, params, args.timeout, args.precision,
                          seed=[base + r for _ in dcops for r in range(n)], infinity=args.infinity,
                          trace=args.collect_on == "cycle_change", best=args.best)
        for k, r in enumerate(res):
            r.update(problem=args.dcop_files[k // n], iteration=k % n, seed=base + k % n)
    for r in res:
        if args.no_assignment:
            _drop_assignment(r)
    print(json.dumps(res, indent=2, sort_keys=True, default=str))
    return 0


def _main_sweep(args, params, sweeps):
    """--batch --sweep: every file x every combination x every iteration (--iterations, default 1) in one
    solve_batch call, each problem with its own parameters and seed."""
    import itertools
    names = [k for k, _ in sweeps]
    combos = [dict(params, **dict(zip(names, vs))) for vs in itertools.product(*(v for _, v in sweeps))]
    n = args.iterations or 1
    base = (args.seed or 0) if args.iterations else args.seed
    dcops = [load(path, base) for path in args.dcop_files]
    entries = [(f, c, r) for f in range(len(dcops)) for c in range(len(combos)) for r in range(n)]
    seeds = [base + r for _, _, r in entries] if args.iterations else args.seed
    res = solve_batch([dcops[f] for f, _, _ in entries], args.algo, [combos[c] for _, c, _ in entries],
                      args.timeout, args.precision, seed=seeds, infinity=args.infinity,
                      trace=args.collect_on == "cycle_change", best=args.best)
    checked = [check_params(ALGOS[args.algo], c) for c in combos]
    for (f, c, r), out in zip(entries, res):
        out.update(problem=args.dcop_files[f], algo_params=checked[c])
        if args.iterations:
            out.update(iteration=r, seed=base + r)
        if args.no_assignment:
            _drop_assignment(out)
    print(json.dumps(res, indent=2, sort_keys=True, default=str))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
