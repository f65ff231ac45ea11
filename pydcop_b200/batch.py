"""Many problems in one engine run (solve.solve_batch): the disjoint union of their front-door arrays.

Every kernel computes a variable or a factor from its own neighbourhood, in `node.constraints` order, so packing
several problems into one layout changes nothing any problem computes, as long as every per-variable input a kernel
reads is the problem's own: the Philox counter (`var_global_id`: the variable's index in its own problem, the
mechanism the sharded engines use the other way round, DESIGN.md §6), the name rank (only ever compared between
neighbours) and the start value of a variable without neighbours.  The union's canonical variable order is the
concatenation of the problems', so problem k's values are one slice of the result.  Problems with seeds of their own
also carry their own Philox key (`var_seed`: the problem's seed on each of its variables), so one problem can run many
times in one union, once per seed.  Problems with algorithm parameters of their own carry the index of their parameter
set (`var_pset`) on each of their variables, for the parameters the kernels read per variable; the others split
groups (`groups`' keys).
"""
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Union as AnyOf

import numpy as np

from . import ingest
from .layout import FactorGraphLayout, build_layout

INDEX_LIMIT = 2 ** 31 - 1      # variables, factors and edges of one engine are int32 indices
MAX_BATCH_VARS = 1 << 20       # default bound on the variables of one engine: C4's size
MAX_PSETS = 65535              # parameter sets of one engine: uint16 indices (FG_MAX_PSETS)


def _front_door_consistent(a: Dict[str, np.ndarray]) -> bool:
    """The array sizes and ranges a union could hide: with them right, every other check build_layout makes on the
    union is local to one problem's factors or variables."""
    V, E = len(a["dom_size"]), len(a["edge_var"])
    fp, to, vp = a["factor_ptr"], a["table_off"], a["var_ptr"]
    ev = np.asarray(a["edge_var"])
    return (len(fp) >= 1 and fp[0] == 0 and fp[-1] == E and len(to) == len(fp) and to[0] == 0
            and to[-1] == len(a["tables"]) and len(vp) == V + 1 and vp[0] == 0 and vp[-1] == E
            and len(a["var_edge"]) == E and len(a["unary"]) == int(np.sum(a["dom_size"], dtype=np.int64))
            and len(a["init_value"]) == V and (not E or (ev.min() >= 0 and ev.max() < V)))


def check_problem(index: int, dcop: ingest.DcopArrays):
    """Raise what solve() raises on problem `index`'s arrays, with its index, if a union could hide it."""
    if not _front_door_consistent(dcop.arrays):
        layout_of(index, dcop.arrays)
        raise ValueError(f"problem {index}: inconsistent front-door arrays")


def layout_of(index: int, inst) -> FactorGraphLayout:
    try:
        return build_layout(**inst)
    except ValueError as e:
        raise ValueError(f"problem {index}: {e}") from e


def groups(dcops: List[ingest.DcopArrays], max_vars: int = MAX_BATCH_VARS, keys: Optional[Sequence] = None,
           sets: Optional[Sequence] = None) -> List[List[int]]:
    """Problem indices per engine: one objective and one group key per group (mode_max and the parameters the kernels
    cannot take per variable are one scalar per engine; keys: one hashable per problem, None: one for all), groups in
    order of first appearance, input order inside; a group is cut before it would exceed `max_vars` variables, an
    int32 index range (a problem larger than that runs alone) or MAX_PSETS distinct parameter sets (sets: one hashable
    per problem, None: one for all)."""
    keys = [None] * len(dcops) if keys is None else list(keys)
    sets = [None] * len(dcops) if sets is None else list(sets)
    out = []
    for group in dict.fromkeys(zip((d.objective for d in dcops), keys)):
        cur, size, seen = [], np.zeros(3, dtype=np.int64), set()
        for i, d in enumerate(dcops):
            if (d.objective, keys[i]) != group:
                continue
            a = d.arrays
            s = np.array([d.n_vars, len(a["factor_ptr"]) - 1, len(a["edge_var"])], dtype=np.int64)
            t = size + s
            new_set = sets[i] not in seen
            if cur and (t[0] > max_vars or (t > INDEX_LIMIT).any() or (new_set and len(seen) >= MAX_PSETS)):
                out.append(cur)
                cur, t, seen = [], s, set()
            cur.append(i)
            seen.add(sets[i])
            size = t
        out.append(cur)
    return out


@dataclass
class Union:
    """The front-door arrays of problems `members` as one problem, and the per-problem inputs the engines take."""
    members: List[int]
    inst: Dict[str, np.ndarray]          # front-door arrays (MaxSum: unary with each problem's noise)
    unary: np.ndarray                    # the variables' own costs, without noise: what the solution cost adds
    var_start: np.ndarray                # [n + 1] first variable of every problem, then the total
    var_global_id: np.ndarray            # each variable's index in its own problem
    var_seed: Optional[np.ndarray]       # each variable's problem's seed (uint64), None when all problems share one
    var_pset: Optional[np.ndarray]       # each variable's problem's parameter set, None when all problems share one
    psets: List[dict]                    # the distinct parameter sets, in order of first appearance
    var_rank: Optional[np.ndarray]       # each variable's name rank in its own problem
    isolated_value: Optional[np.ndarray]  # start value of the variables without neighbours, per problem
    seg_factor: np.ndarray               # problem (0..n-1) of every canonical factor
    seg_var: np.ndarray                  # problem of every canonical variable


def build_union(dcops: List[ingest.DcopArrays], members: List[int], var_inputs,
                noise: AnyOf[float, Sequence[float]] = 0.0, seed: AnyOf[None, int, Sequence[int]] = None,
                params: Optional[Sequence[dict]] = None) -> Union:
    """Concatenate the problems `members` of `dcops`: variable, edge and table indices are offset by the problems
    before.  var_inputs(dcop) -> (var_rank or None, isolated_value or None), each problem's own; `seed`: one for every
    member, or a sequence with one per member; `noise`: MaxSum's, one for every member or one per member, drawn per
    problem with its seed exactly as solve() draws it; `params`: one parameter dict per member (None: one set for
    all), whose distinct dicts become `psets`."""
    parts = [dcops[i].arrays for i in members]
    seeds = [seed] * len(members) if seed is None or isinstance(seed, (int, np.integer)) else list(seed)
    if len(seeds) != len(members):
        raise ValueError(f"{len(seeds)} seeds for {len(members)} problems")
    noises = list(noise) if isinstance(noise, (list, tuple, np.ndarray)) else [noise] * len(members)
    if len(noises) != len(members):
        raise ValueError(f"{len(noises)} noise levels for {len(members)} problems")
    ids = {}
    member_set = [ids.setdefault(pset_key(p), len(ids)) for p in params] if params is not None else [0] * len(members)
    psets = [dict(params[member_set.index(k)]) for k in range(len(ids))] if params is not None else []
    n_var = np.array([len(a["dom_size"]) for a in parts], dtype=np.int64)
    n_fac = np.array([len(a["factor_ptr"]) - 1 for a in parts], dtype=np.int64)
    n_edge = np.array([len(a["edge_var"]) for a in parts], dtype=np.int64)
    n_tab = np.array([len(a["tables"]) for a in parts], dtype=np.int64)
    v0, e0, t0 = (np.concatenate([[0], np.cumsum(x)]) for x in (n_var, n_edge, n_tab))

    def ptr(key, off):
        return np.concatenate([np.asarray(a[key][:-1], dtype=np.int64) + o for a, o in zip(parts, off[:-1])]
                              + [[off[-1]]]).astype(np.int64)

    cat = lambda key, dt=None: np.concatenate([np.asarray(a[key], dtype=dt) for a in parts])  # noqa: E731
    unary = cat("unary", np.float64)
    inst = dict(dom_size=cat("dom_size", np.int32), factor_ptr=ptr("factor_ptr", e0),
                edge_var=np.concatenate([np.asarray(a["edge_var"], dtype=np.int64) + o
                                         for a, o in zip(parts, v0[:-1])]).astype(np.int32),
                table_off=ptr("table_off", t0), tables=np.concatenate([np.asarray(a["tables"]) for a in parts]),
                unary=(np.concatenate([ingest.add_noise(a["unary"], nz, s) for a, nz, s in zip(parts, noises, seeds)])
                       if any(noises) else unary),
                var_ptr=ptr("var_ptr", e0).astype(np.int32),
                var_edge=np.concatenate([np.asarray(a["var_edge"], dtype=np.int64) + o
                                         for a, o in zip(parts, e0[:-1])]).astype(np.int32),
                init_value=cat("init_value", np.int32))
    ranks, isos = zip(*(var_inputs(dcops[i]) for i in members))
    seg = np.arange(len(members), dtype=np.int32)
    return Union(members=list(members), inst=inst, unary=unary, var_start=v0,
                 var_global_id=np.concatenate([np.arange(n, dtype=np.int32) for n in n_var]),
                 var_seed=(None if len(set(seeds)) == 1 else
                           np.repeat(np.array([int(s) & (2 ** 64 - 1) for s in seeds], dtype=np.uint64), n_var)),
                 var_pset=None if len(psets) <= 1 else np.repeat(np.array(member_set, dtype=np.int32), n_var),
                 psets=psets,
                 var_rank=None if ranks[0] is None else np.concatenate(ranks).astype(np.int32),
                 isolated_value=None if isos[0] is None else np.concatenate(isos).astype(np.int32),
                 seg_factor=np.repeat(seg, n_fac), seg_var=np.repeat(seg, n_var))


def pset_key(params: dict):
    """A hashable identity of one parameter dict."""
    return tuple(sorted(params.items()))


def union_layout(u: Union, dcops: List[ingest.DcopArrays]) -> FactorGraphLayout:
    """build_layout of the union; a problem it refuses is named by its index in the batch, with solve()'s message."""
    try:
        return build_layout(**u.inst)
    except ValueError:
        for i in u.members:
            layout_of(i, dcops[i].arrays)
        raise
