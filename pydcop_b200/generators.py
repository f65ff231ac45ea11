"""Synthetic instance generators for the BASELINE.json configs, as flat arrays (array front door).

They restate the DISTRIBUTIONS of the reference's own generators
(pydcop/commands/generators/graphcoloring.py:355-375 soft costs randint(0,9);
pydcop/commands/generators/ising.py:274-331,362-420) — the reference generators themselves build
Python objects and cannot produce 10^5..10^6-variable instances.  numpy PCG64, seed 0 by default.
"""
import numpy as np


def _distinct_scopes(rng, n_vars, n_factors, arity):
    """`n_factors` scopes of `arity` distinct variables each, uniform."""
    s = rng.integers(0, n_vars, size=(n_factors, arity), dtype=np.int64)
    for _ in range(64):
        srt = np.sort(s, axis=1)
        bad = (srt[:, 1:] == srt[:, :-1]).any(axis=1)
        if not bad.any():
            break
        s[bad] = rng.integers(0, n_vars, size=(int(bad.sum()), arity), dtype=np.int64)
    return s.astype(np.int32)


def random_factor_graph(n_vars, d, n_factors, arity=2, seed=0, noise=0.01, int_tables=True):
    """C2 / C5 / target family: uniform random scopes, tables integers(0,10), unary 0 + U(0,noise)
    (the reference's default `noise`, maxsum.py:218, drawn per (variable, value))."""
    rng = np.random.default_rng(seed)
    scopes = _distinct_scopes(rng, n_vars, n_factors, arity)
    if int_tables:
        tables = rng.integers(0, 10, size=n_factors * d ** arity).astype(np.float32)
    else:
        tables = rng.uniform(0, 10, size=n_factors * d ** arity).astype(np.float32)
    unary = rng.uniform(0, noise, size=n_vars * d) if noise else np.zeros(n_vars * d)
    return dict(dom_size=np.full(n_vars, d, np.int32),
                factor_ptr=np.arange(n_factors + 1, dtype=np.int64) * arity,
                edge_var=scopes.reshape(-1), tables=tables, unary=unary)


def mixed_shape_graph(n_vars, doms, shapes, seed=0, noise=0.01, int_tables=False):
    """Variables with domain sizes drawn from `doms`, factors of several arities: `shapes` is a list of
    (arity, n_factors).  Tables follow the scopes' domain sizes (mixed-domain classes, the SECP /
    meeting-scheduling kind of problem).  Factors are stored arity by arity."""
    rng = np.random.default_rng(seed)
    dom = rng.choice(np.asarray(doms, dtype=np.int32), size=n_vars).astype(np.int32)
    ev, ptr, tabs = [], [0], []
    for arity, n_f in shapes:
        sc = _distinct_scopes(rng, n_vars, n_f, arity) if arity > 1 else rng.integers(0, n_vars, (n_f, 1)).astype(np.int32)
        ev.append(sc.reshape(-1))
        ptr.extend((ptr[-1] + arity * np.arange(1, n_f + 1)).tolist())
        size = int(np.prod(dom[sc].astype(np.int64), axis=1).sum())
        tabs.append(rng.integers(0, 10, size).astype(np.float32) if int_tables else rng.uniform(0, 10, size).astype(np.float32))
    n_un = int(dom.sum())
    unary = rng.uniform(0, noise, n_un) if noise else np.zeros(n_un)
    return dict(dom_size=dom, factor_ptr=np.asarray(ptr, dtype=np.int64), edge_var=np.concatenate(ev).astype(np.int32),
                tables=np.concatenate(tabs), unary=unary)


def config_mixed(seed=0, n_vars=200_000):
    """side workload for the runtime-dimension kernels: domains {3, 5, 7, 12}, binary + ternary + arity-4 factors."""
    return mixed_shape_graph(n_vars, (3, 5, 7, 12), [(2, n_vars * 3 // 2), (3, n_vars // 4), (4, n_vars // 16)], seed,
                             int_tables=True)


def config_c2(seed=0, n_vars=100_000):
    """random binary DCOP 100k vars d=10 deg=4 (F = V*deg/2)."""
    return random_factor_graph(n_vars, 10, n_vars * 2, 2, seed)


def config_target(seed=0, n_vars=1_000_000):
    """north-star instance: 1M variables, d=10, binary, mean degree 4."""
    return random_factor_graph(n_vars, 10, n_vars * 2, 2, seed)


def config_c5(seed=0, n_factors=50_000):
    """arity-3 factors 50k, d=8, over 50k variables."""
    return random_factor_graph(n_factors, 8, n_factors, 3, seed)


def config_c4(seed=0, n_vars=1_000_000):
    """DSA: random 1M vars d=20 deg=6 (3M binary constraints), integer tables."""
    return random_factor_graph(n_vars, 20, n_vars * 3, 2, seed, noise=0.0)


def ising_grid(rows, cols, seed=0, noise=0.01):
    """C3: toroidal Ising grid (ising.py:285 periodic grid), d=2, binary table [[k,-k],[-k,k]]
    with k~U(-1.6,1.6) (:369), unary factor [u,-u], u~U(-0.05,0.05) (:417).  Variables in raster
    order; factor order: all 'down' + 'right' couplings in raster order, then the unary factors."""
    rng = np.random.default_rng(seed)
    n = rows * cols
    idx = np.arange(n, dtype=np.int64).reshape(rows, cols)
    down = np.roll(idx, -1, axis=0)
    right = np.roll(idx, -1, axis=1)
    pairs = np.stack([np.stack([idx, down], -1), np.stack([idx, right], -1)], 2).reshape(-1, 2)
    pairs = pairs[pairs[:, 0] != pairs[:, 1]]
    nb = len(pairs)
    k = rng.uniform(-1.6, 1.6, size=nb)
    tb = np.stack([k, -k, -k, k], 1).reshape(-1)
    u = rng.uniform(-0.05, 0.05, size=n)
    tu = np.stack([u, -u], 1).reshape(-1)
    factor_ptr = np.concatenate([np.arange(nb + 1, dtype=np.int64) * 2,
                                 2 * nb + np.arange(1, n + 1, dtype=np.int64)])
    edge_var = np.concatenate([pairs.reshape(-1), np.arange(n, dtype=np.int64)]).astype(np.int32)
    unary = rng.uniform(0, noise, size=n * 2) if noise else np.zeros(n * 2)
    return dict(dom_size=np.full(n, 2, np.int32), factor_ptr=factor_ptr, edge_var=edge_var,
                tables=np.concatenate([tb, tu]).astype(np.float32), unary=unary)


def config_c3(seed=0, side=1024):
    return ising_grid(side, side, seed)


def algorithmic_bytes_per_cycle(layout, value_bytes=4):
    """SURVEY.md §8(d): B = sum_f [4 d^a + a (12 d + 6)] + sum_v [4 d + k (12 d + 6) + 12]
    with value_bytes in place of 4 for the value arrays."""
    w = value_bytes
    b = 0
    for c in layout.classes:
        b += c.n_factors * (w * c.table_size + sum(3 * w * dj + 6 for dj in c.dom))
    deg = np.diff(layout.var_ptr).astype(np.int64)
    d = layout.dom_size.astype(np.int64)
    b += int((w * d + deg * (3 * w * d + 6) + 12).sum())
    return int(b)


def algorithmic_bytes_per_cycle_inst(inst, value_bytes=4):
    """Same figure as algorithmic_bytes_per_cycle, straight from the instance arrays (no layout):
    used by the multi-GPU bench where no rank builds the global layout."""
    w = value_bytes
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"], dtype=np.int64)
    ed = dom[ev]
    arity = np.diff(fp)
    efac = np.repeat(np.arange(len(arity)), arity)
    tsize = np.ones(len(arity), dtype=np.int64)
    np.multiply.at(tsize, efac, ed)
    b = int((w * tsize).sum() + (3 * w * ed + 6).sum())
    deg = np.bincount(ev, minlength=len(dom)).astype(np.int64)
    b += int((w * dom + deg * (3 * w * dom + 6) + 12).sum())
    return b


def bounded_separator_instance(n_vars, d, back, span=2, p_back=1.0, seed=0, float_costs=False):
    """DPOP workloads: a random tree (the parent of variable i is one of the `span` variables before it, so
    the tree is deep) plus, from each variable with probability `p_back`, one binary constraint to each of
    its ancestors 2..back+1 levels up.  Every constraint joins a variable to an ancestor, so pseudo-tree
    separators stay near `back` + 1 variables (tools/dpop_throughput.py reports the ones the DFS actually
    builds).  Tables are integers(0,10) (or uniform floats), no variable costs."""
    rng = np.random.default_rng(seed)
    parent = np.zeros(n_vars, dtype=np.int64)
    if n_vars > 1:
        i = np.arange(1, n_vars)
        parent[1:] = i - 1 - (rng.integers(0, span, size=n_vars - 1) % i)
    pairs = [np.stack([parent[1:], np.arange(1, n_vars)], 1)]
    anc = parent.copy()
    for _ in range(back):
        anc = np.where(anc > 0, parent[anc], -1) if n_vars else anc
        take = (anc >= 0) & (rng.uniform(size=n_vars) < p_back)
        take[0] = False
        pairs.append(np.stack([anc[take], np.nonzero(take)[0]], 1))
        anc = np.where(anc >= 0, anc, 0)
    scopes = np.concatenate(pairs).astype(np.int32) if n_vars > 1 else np.zeros((0, 2), np.int32)
    n_f = len(scopes)
    tables = (rng.uniform(-5, 5, size=n_f * d * d) if float_costs
              else rng.integers(0, 10, size=n_f * d * d).astype(np.float64))
    return dict(dom_size=np.full(n_vars, d, dtype=np.int32), factor_ptr=np.arange(0, 2 * n_f + 1, 2, dtype=np.int64),
                edge_var=scopes.reshape(-1), tables=tables, unary=np.zeros(n_vars * d))
