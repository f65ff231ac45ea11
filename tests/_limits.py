"""Instances at the shape limits of the C-ABI (FG_MAX_DOM = 256, FG_MAX_ARITY = 8, FG_DPOP_MAX_SEP = 32) and
the other edges the device dispatch branches on: domain size 1, hubs far above the degree classes, unary-only
and factor-free graphs.  Shared by the host-shim tests of every family and tests/test_gpu_limits.py, so each
shape runs through the kernel source on the CPU and through the device kernels on the GPU.

Every builder returns the flat instance arrays (dom_size, factor_ptr, edge_var, tables, unary) plus, for the
local-search families, var_ptr / var_edge, var_rank and init_value.  Tables are float32 values (exact in
both precisions' uploads), uniform in [-3, 3), or integers in [0, levels) where ties matter."""
import numpy as np

from pydcop_b200.generators import _distinct_scopes, bounded_separator_instance
from pydcop_b200.layout import default_var_csr


def from_scopes(dom, scopes, seed, levels=0, const=None):
    """Instance over variables of domain sizes `dom` and the factors `scopes` (a list of 1-D int arrays, in
    factor order): tables and variable costs drawn from `seed` (floats, integers in [0, levels), or every
    entry `const`)."""
    rng = np.random.default_rng(seed)
    dom = np.asarray(dom, dtype=np.int32)
    sizes = [int(np.prod(dom[s].astype(np.int64))) for s in scopes]

    def draw(n):
        if const is not None:
            return np.full(n, const, dtype=np.float32)
        if levels:
            return rng.integers(0, levels, n).astype(np.float32)
        return rng.uniform(-3, 3, n).astype(np.float32)
    ptr = np.zeros(len(scopes) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in scopes], out=ptr[1:])
    return dict(dom_size=dom, factor_ptr=ptr,
                edge_var=(np.concatenate(scopes) if scopes else np.zeros(0)).astype(np.int32),
                tables=draw(int(sum(sizes))), unary=draw(int(dom.sum())).astype(np.float64))


def random_graph(n, doms, shapes, seed, levels=0, const=None):
    """Variables with domain sizes drawn from `doms`; shapes: list of (arity, count) with scopes of distinct
    variables, uniform over all variables."""
    rng = np.random.default_rng(seed)
    dom = rng.choice(np.asarray(doms, dtype=np.int32), size=n).astype(np.int32)
    scopes = []
    for arity, count in shapes:
        scopes.extend(_distinct_scopes(rng, n, count, arity) if arity > 1 else rng.integers(0, n, (count, 1)))
    return from_scopes(dom, [np.asarray(s) for s in scopes], seed + 1, levels, const)


def hub_graph(d, hub_degree, extra, seed, n_isolated=0, n_unary=0, levels=0):
    """Variable 0 in `hub_degree` binary constraints, one with each of variables 1..hub_degree; each of those
    is in `extra` = (lo, hi) more binary constraints among themselves (self pairs dropped, so at least lo - 2),
    then `n_isolated` variables without constraints and `n_unary` unary constraints.  One domain size `d`."""
    rng = np.random.default_rng(seed)
    others = np.arange(1, hub_degree + 1)
    stubs = np.repeat(others, rng.integers(extra[0], extra[1] + 1, hub_degree))
    rng.shuffle(stubs)
    pairs = stubs[:len(stubs) // 2 * 2].reshape(-1, 2)
    pairs = pairs[pairs[:, 0] != pairs[:, 1]]
    n = hub_degree + 1 + n_isolated
    scopes = [np.array([0, u]) for u in others] + list(pairs)
    scopes += [np.array([u]) for u in rng.integers(0, hub_degree + 1, n_unary)]
    return from_scopes(np.full(n, d), scopes, seed + 1, levels)


def with_local_search_arrays(inst, seed):
    """The arrays MGM, MGM-2 and GDBA take beyond the factor graph: canonical var_ptr / var_edge, random name
    ranks and an initial value on about a third of the variables."""
    rng = np.random.default_rng(seed)
    n = len(inst["dom_size"])
    out = dict(inst)
    out["var_ptr"], out["var_edge"] = default_var_csr(n, inst["edge_var"])
    out["var_rank"] = rng.permutation(n).astype(np.int32)
    out["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, 1 << 30, n) % inst["dom_size"], -1).astype(np.int32)
    return out


# ----------------------------------------------------------------------------------------------------------------
# MaxSum: name -> instance.  The factor side of every non-compiled shape runs k_f2v_tiled_rt (binary 256 x 256
# tables are 256 KB in f32 and 512 KB in f64: larger than its 72 KB of shared memory, so read in place); the
# variable side of domains outside FG_FAST_DOMS and of degrees above 32 runs k_v2f_generic.
MAXSUM = {
    "d1": lambda: random_graph(1500, [1], [(2, 2500), (1, 200)], seed=1),
    "d256": lambda: random_graph(160, [256], [(2, 200), (1, 40)], seed=2),
    "doms_1_3_256": lambda: random_graph(600, [1, 3, 256], [(2, 900), (1, 150)], seed=3),
    "arity8_d3": lambda: random_graph(400, [3], [(8, 120), (2, 300), (1, 50)], seed=4),
    "arity5_6_mixed": lambda: random_graph(400, [2, 3, 4], [(5, 80), (6, 40), (2, 300)], seed=5),
    "hub2400": lambda: hub_graph(3, 2400, (18, 31), seed=6, n_isolated=20, n_unary=100),
    "unary_only": lambda: random_graph(500, [1, 3, 256], [(1, 350)], seed=7),
    "no_factors": lambda: random_graph(50, [1, 3, 256], [], seed=8),
}

# DSA / A-DSA: the generic kernel (a unary constraint keeps every instance off the binary fast path)
DSA = {
    "d1": lambda: random_graph(2000, [1], [(2, 3000), (1, 100)], seed=11),
    "d256": lambda: random_graph(300, [256], [(2, 450), (1, 30)], seed=12, levels=3),
    "d256_all_tie": lambda: random_graph(300, [256], [(2, 450), (1, 30)], seed=13, const=1.0),
    "arity8_d2": lambda: random_graph(500, [2], [(8, 300), (2, 400), (1, 20)], seed=14, levels=3),
    "hub2400": lambda: hub_graph(3, 2400, (18, 31), seed=15, n_isolated=20, n_unary=100, levels=3),
}

# (case, variant, mode, var_costs): variants A, B and C at d = 1 and 256; all 256 values tied (C's drop_cur draws
# among 255); A-DSA's variable costs at d = 256
DSA_RUNS = ([("d1", v, "min", False) for v in "ABC"] + [("d256", v, m, False) for v, m in zip("ABC", ("min", "max", "min"))]
             + [("d256_all_tie", "C", "min", False), ("d256_all_tie", "B", "max", False),
                ("arity8_d2", "B", "min", False), ("hub2400", "A", "max", False), ("d256", "B", "min", True)])

# MGM's generic gain kernel (k_mgm_gain): all-tie tables, so every value ties for the best
MGM = {
    "d1": lambda: with_local_search_arrays(random_graph(2000, [1], [(2, 3000), (1, 100)], seed=21, const=1.0), 1),
    "d256_all_tie": lambda: with_local_search_arrays(
        random_graph(300, [256], [(2, 450), (1, 30)], seed=22, const=2.0), 2),
}


def mgm_hub(d):
    """MGM's active-row kernel (k_mgm_gain_cached, binary constraints over one domain size in {4, 8, 10, 16,
    20}): a hub of degree 3100, above three chunks of CH = 128 * SPT <= 1024 slots, plus isolated variables."""
    return with_local_search_arrays(hub_graph(d, 3100, (2, 6), seed=30 + d, n_isolated=40, levels=4), d)


# MGM-2 and GDBA (one generic kernel set): binary and unary constraints, integer costs with few levels.  Small at
# d = 256: the MGM-2 oracle evaluates every one of an offer's 65 536 value pairs in Python.
LOCAL = {
    "d1": lambda: with_local_search_arrays(random_graph(1200, [1], [(2, 1500), (1, 100)], seed=41, levels=2), 1),
    "d256": lambda: with_local_search_arrays(random_graph(24, [256], [(2, 22), (1, 6)], seed=42, levels=2), 2),
    "doms_1_2_256": lambda: with_local_search_arrays(
        random_graph(90, [1, 2, 256], [(2, 80), (1, 12)], seed=43, levels=2), 3),
}


# GDBA: one modifier per increase mode
GDBA_MODES = [("A", "E"), ("M", "R"), ("A", "C"), ("M", "T")]


def gdba_instance(case):
    """LOCAL[case] with every cost raised by 1: no entry is 0, so under violation NZ every constraint stays
    violated, local minima are quasi-local minima and breakouts raise the modifiers."""
    inst = LOCAL[case]()
    inst["tables"] = inst["tables"] + 1
    return inst


# ----------------------------------------------------------------------------------------------------------------
# DPOP
def dpop_d256(seed=51):
    """A DFS tree at d = 256 whose separators have two variables: UTIL tables of 65 536 entries (grid-wide
    nodes) and a VALUE walk with 8 values per lane; integer costs in [0, 3), so the argopt meets ties."""
    inst = bounded_separator_instance(9, 256, back=1, span=1, seed=seed)
    inst["tables"] = np.random.default_rng(seed).integers(0, 3, len(inst["tables"])).astype(np.float64)
    return inst


def dpop_with_domain_one(seed=52):
    """A d = 10 tree with about a quarter of its variables reduced to a single value."""
    inst = bounded_separator_instance(300, 10, back=2, span=3, p_back=0.5, seed=seed)
    dom = inst["dom_size"].copy()
    dom[np.random.default_rng(seed).random(len(dom)) < 0.25] = 1
    ev, fp = inst["edge_var"], inst["factor_ptr"]
    return from_scopes(dom, [ev[fp[f]:fp[f + 1]] for f in range(len(fp) - 1)], seed, levels=4)


def clique(n, d=1):
    """Every pair of n variables constrained: the deepest separator has n - 1 variables."""
    pairs = [np.array([i, j]) for i in range(n) for j in range(i + 1, n)]
    return from_scopes(np.full(n, d), pairs, n, levels=5)


# ----------------------------------------------------------------------------------------------------------------
# Solution cost
def big_float_instance(n_factors=1_000_000, seed=61, infinity=1000.0):
    """n_factors binary float constraints with mixed-sign costs over d = 3, and a few entries equal to
    `infinity` (violations when the assignment meets them)."""
    inst = random_graph(n_factors // 4, [3], [(2, n_factors)], seed=seed)
    rng = np.random.default_rng(seed)
    inst["tables"] = (rng.standard_normal(len(inst["tables"])) * 10.0 ** rng.integers(-3, 4, len(inst["tables"])))\
        .astype(np.float32)
    inst["tables"][rng.random(len(inst["tables"])) < 1e-3] = infinity
    return inst


def cost_terms(inst, value):
    """Every constraint's table entry and every variable's own cost at `value` (canonical order), float64."""
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    fp, ev = np.asarray(inst["factor_ptr"], np.int64), np.asarray(inst["edge_var"], np.int64)
    arity = np.diff(fp)
    sizes = np.ones(len(arity), dtype=np.int64)
    lin = np.zeros(len(arity), dtype=np.int64)
    for j in range(int(arity.max(initial=0))):
        m = arity > j
        e = fp[:-1][m] + j
        lin[m] = lin[m] * dom[ev[e]] + np.asarray(value, np.int64)[ev[e]]
        sizes[m] *= dom[ev[e]]
    toff = np.concatenate([[0], np.cumsum(sizes)])[:-1]
    uoff = np.concatenate([[0], np.cumsum(dom)])[:-1]
    return (np.asarray(inst["tables"])[toff + lin].astype(np.float64),
            np.asarray(inst["unary"], dtype=np.float64)[uoff + np.asarray(value, np.int64)])
