"""All-binary unions over one domain size: the batches that run DSA's oriented-table and active-row kernels
(k_dsa_step_bin, k_dsa_step_cached) and MGM's fast and active-row value phases (k_mgm_gain_bin, k_mgm_gain_cached)
with a Philox key (var_seed) and, for DSA and A-DSA, a parameter set (var_pset) per problem, and the CPU oracle of
every member run alone.  These kernels never run through the host shims, so the oracle is what pins them.

Shared by tests/test_binary_unions_cpu.py (the instances and the oracle trajectories, without a GPU) and
tests/test_gpu_zz_binary_paths.py (the device kernels against those trajectories).

Every union has seven problems in this order: the same instance three times (COPIES), a hub problem in the middle
(HUB, when asked for), and one problem that runs with probability 0 in the mixed-set runs (FROZEN)."""
import functools

import numpy as np

import oracle as orc
from bench import oracle_instance
from pydcop_b200 import batch, ingest
from pydcop_b200.engine import make_engine
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import check_params, name_rank

FAST_DOMS = (2, 3, 4, 5, 6, 8, 10, 16, 20)   # FG_FAST_DOMS (csrc/maxsum_fast.cuh): the compiled domain sizes
MGM_DOMS = (4, 8, 10, 16, 20)                # k_mgm_gain_bin / k_mgm_gain_cached
HUB_DEGREE = 1100       # above the largest active-row chunk, CH = 128 * SPT <= 1024 slots (DsaCachedCfg, MgmCachedCfg)
CTA = 128               # variables per block of both DSA kernels and of k_mgm_gain_cached
COPIES, HUB, FROZEN = (1, 4, 6), 3, 5
# variables per problem: none a multiple of 128, so blocks hold variables of several problems (the layout also
# groups variables by degree across problems); the copies are one instance
SIZES = (333, 517, 201, 645, 517, 419, 517)
ISOLATED = (9, 0, 0, 0, 0, 13, 0)             # variables without constraints (has_nbr = 0)


def _problem(n, D, seed, levels, n_isolated=0, hub=False, var_costs=False, mode="min", name="p"):
    """n variables over domain size D, 1.5 n binary constraints with integer tables of `levels` values (ties
    everywhere), `n_isolated` of the variables in no constraint; hub: one variable in HUB_DEGREE of them, each with a
    different neighbour; var_costs: integer variable costs in [0, 2] (A-DSA's decisive own costs, with ties)."""
    rng = np.random.default_rng(seed)
    core = n - n_isolated
    inst = random_factor_graph(core, D, 3 * n // 2 + (HUB_DEGREE if hub else 0), 2, seed=seed, noise=0)
    ev = inst["edge_var"].reshape(-1, 2)
    if hub:
        ev[:HUB_DEGREE, 0] = 0
        ev[:HUB_DEGREE, 1] = rng.choice(np.arange(1, core), HUB_DEGREE, replace=False)
    perm = rng.permutation(n)                 # the isolated variables (ids core..n-1) spread over the problem
    inst["edge_var"] = perm[ev.reshape(-1)].astype(np.int32)
    inst["dom_size"] = np.full(n, D, np.int32)
    inst["tables"] = rng.integers(0, levels, len(inst["tables"])).astype(np.float32)
    inst["unary"] = rng.integers(0, 3, n * D).astype(np.float64) if var_costs else np.zeros(n * D)
    return ingest.from_arrays(inst, name=name, objective=mode)


def uniform_union(D, seed, *, hub=False, levels=3, var_costs=False, mode="min"):
    """The seven problems of one union (module docstring), every one all-binary over domain size D.  The copies
    start from one given assignment (init_value: MGM starts there, DSA draws its own), so under MGM only the
    value-phase draws can tell them apart."""
    out = []
    for i, (n, iso) in enumerate(zip(SIZES, ISOLATED)):
        if i in COPIES[1:]:
            out.append(out[COPIES[0]])
            continue
        is_hub = hub and i == HUB
        out.append(_problem(n + (HUB_DEGREE if is_hub else 0), D, seed * 101 + i, levels, iso, is_hub, var_costs, mode,
                            f"p{i}"))
        if i == COPIES[0]:
            a = out[-1].arrays
            a["init_value"] = np.random.default_rng(seed).integers(0, D, n).astype(np.int32)
    return out


def dsa_params(kind, mixed, variant="B"):
    """One parameter dict per problem.  mixed: variants A, C and B on the copies (same probability), probability 1.0
    and 0.0 (FROZEN), p_mode arity (DSA) and a hub in variant B; else `variant` at 0.7 for all."""
    if not mixed:
        return [dict(variant=variant, probability=0.7)] * len(SIZES)
    arity = dict(variant="B", p_mode="arity", probability=0.5) if kind == "dsa" else dict(variant="B", probability=0.5,
                                                                                          period=2.0)
    return [dict(variant="C", probability=1.0), dict(variant="A", probability=0.6), arity,
            dict(variant="B", probability=0.8), dict(variant="C", probability=0.6), dict(variant="A", probability=0.0),
            dict(variant="B", probability=0.6)]


def seeds_for(D, shared_copies):
    """One seed per problem: 0, -1 (keyed as 2**64 - 1) and 2**63 among them; shared_copies: the copies share one."""
    s = [0, -1, 2 ** 63, 1000 + D, 2000 + D, 3000 + D, 4000 + D]
    if shared_copies:
        for i in COPIES:
            s[i] = s[COPIES[0]]
    return s


UNION_SEED = 12345      # the engine's scalar seed: none of the members', so every draw must take its variable's key
# DSA and A-DSA unions run in mode max at these domain sizes, in mode min at the others.  MGM's run in mode min: in
# mode max these instances settle within two cycles, which leaves nothing for the late cycles to test
MAX_DOMS = (3, 5, 8, 20)
HUB_DOMS = (2, 10, 20)     # DSA and A-DSA unions with a hub; MGM's have one at every domain size


@functools.lru_cache(maxsize=None)
def case(kind, D, mixed):
    """(dcops, params, seeds) of one case.  mixed: DSA / A-DSA with a parameter set per problem (dsa_params), the
    copies sharing one seed; else one set (variant A, B or C by D) and a seed per problem.  MGM: mixed is False."""
    dcops = uniform_union(D, D, hub=kind == "mgm" or D in HUB_DOMS, var_costs=kind == "adsa",
                          mode="max" if D in MAX_DOMS and kind != "mgm" else "min")
    params = None if kind == "mgm" else dsa_params(kind, mixed, "ABC"[D % 3])
    return dcops, params, seeds_for(D, mixed)


@functools.lru_cache(maxsize=None)
def case_trajectories(kind, D, mixed, precision, n_cycles):
    """trajectories() of case(kind, D, mixed) in `precision` ("f32" | "f64")."""
    dcops, params, seeds = case(kind, D, mixed)
    return trajectories(kind, dcops, params, seeds, np.float64 if precision == "f64" else np.float32, n_cycles)


def union_engine(kind, dcops, params, seeds, precision):
    """make_engine over the union of `dcops` with one parameter dict (params, None for MGM) and one seed per problem:
    (engine, Union).  DSA and A-DSA get var_pset / psets when the dicts differ."""
    checked = None if params is None else [check_params(kind, p) for p in params]
    rank = kind == "mgm"
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d) if rank else None, None),
                          seed=seeds, params=checked)
    L = batch.union_layout(u, dcops)
    sets = dict(var_pset=u.var_pset, psets=u.psets) if u.var_pset is not None else {}
    eng = make_engine(kind, L, checked[0] if checked else {}, mode=dcops[0].objective, precision=precision,
                      seed=UNION_SEED, var_rank=u.var_rank, var_global_id=u.var_global_id, var_seed=u.var_seed, **sets)
    return eng, u


def oracle_for(kind, dcop, params, seed, dt):
    """The CPU oracle of `dcop` alone in precision `dt`, with its scalar parameters and its own seed, initialised."""
    inst = dcop.instance()
    ref = oracle_instance(inst, build_layout(**inst))
    key = int(seed) & (2 ** 64 - 1)
    if kind == "mgm":
        return orc.MgmOracle(dict(ref, var_rank=name_rank(dcop)), dt, mode=dcop.objective, seed=key).init()
    p = check_params(kind, params)
    return orc.DsaOracle(ref, dt, mode=dcop.objective, variant=p["variant"], probability=p["probability"],
                         p_mode=p.get("p_mode", "fixed"), seed=key, var_costs=kind == "adsa").init()


def oracle_state(kind, o):
    """What the engine must equal after each cycle: (values,) for DSA; (values, costs with NaN where none is known yet,
    gains, intended values) for MGM."""
    if kind != "mgm":
        return (o.val.copy(),)
    return (o.val.copy(), np.where(o.has_cost == 1, o.cost, np.nan), o.gain.copy(), o.new_val.copy())


def trajectories(kind, dcops, params, seeds, dt, n_cycles):
    """Per problem, the oracle states (oracle_state) after init and after each of `n_cycles` cycles."""
    out, threads = [], orc.threads()
    orc.threads(1)      # a few hundred variables per problem: one thread beats OpenMP's fork and join
    try:
        for i, d in enumerate(dcops):
            out.append(_trajectory(kind, d, None if params is None else params[i], seeds[i], dt, n_cycles))
    finally:
        orc.threads(threads)
    return out


def _trajectory(kind, dcop, params, seed, dt, n_cycles):
    o = oracle_for(kind, dcop, params, seed, dt)
    t = [oracle_state(kind, o)]
    for _ in range(n_cycles):
        o.step()
        t.append(oracle_state(kind, o))
    return t


def values_of(traj):
    """[cycles + 1, n] values of one problem's trajectory."""
    return np.stack([s[0] for s in traj])


def check_non_vacuous(kind, traj, mixed):
    """What shows that the inputs under test took effect, on the trajectories alone: the copies diverge (keys-only:
    different seeds, and under MGM one start, so the value-phase draws split them; mixed: one seed, variants A, C and
    B), the FROZEN problem keeps its start (mixed), many variables move in cycle 1 and some problem still moves after
    cycle 10, so the active-row kernels run both regimes: most rows fetched, and almost none.  MGM moves only the
    best gain of each neighbourhood, about one variable in 1 + degree, so its bar for cycle 1 is 10 % (DSA: 20 %)."""
    vals = [values_of(t) for t in traj]
    a, c, b = (vals[i] for i in COPIES)
    assert not np.array_equal(a, c) and not np.array_equal(a, b), "the copies follow one trajectory"
    if mixed or kind == "mgm":
        assert np.array_equal(a[0], c[0]) and np.array_equal(a[0], b[0]), "the copies start apart"
    if mixed:
        assert (vals[FROZEN] == vals[FROZEN][0]).all(), "a problem with probability 0 moved"
    moved = np.concatenate([v[1] != v[0] for v in vals])
    assert moved.mean() > (0.1 if kind == "mgm" else 0.2), moved.mean()
    assert any((v[11:] != v[10:-1]).any() for v in vals), "nothing moves after cycle 10"
