"""Hard constraints (+/-inf table cells) for the MaxSum tests: which factor->variable outputs have only
NaN candidates, which device kernel computes them, and a way to forbid assignments in a random instance.

An output (factor f, position j, value x) of factor_costs_for_var (maxsum.py:382-447) is the optimum
over the assignments a with a_j = x of T[a] + sum_{i != j} q_i[a_i], the sum over the q rows the factor
holds.  The reference starts from +/-inf and replaces it only on a strict < / >, so when every candidate
is NaN (a q row of a variable with every value forbidden is inf - inf = NaN) the output stays +/-inf.
A kernel that takes the optimum without that start value produces NaN there instead.
"""
import numpy as np

# compiled shapes of the device kernels (csrc/maxsum_fast.cuh FG_FAST_DOMS*, csrc/maxsum_warp.cuh dispatch_f2v_warp)
FAST_DOMS = (2, 3, 4, 5, 6, 8, 10, 16, 20)
FAST_DOMS_A3 = (2, 3, 4, 5, 8)
WARP_DOMS = (4, 6, 8, 10, 16, 20)


def factor_family(shape):
    """Kernel family that computes a factor of this shape (domain sizes in scope order) in the default
    configuration: "warp" (k_f2v_warp), "pipe" (k_f2v_pipe) or "tiled_rt" (k_f2v_tiled_rt)."""
    a, d = len(shape), int(shape[0])
    uniform = len(set(int(x) for x in shape)) == 1
    if a == 2 and uniform and d in WARP_DOMS:
        return "warp"
    if uniform and ((a <= 2 and d in FAST_DOMS) or (a == 3 and d in FAST_DOMS_A3)):
        return "pipe"
    return "tiled_rt"


def output_site(shape, j, x):
    """Code path of output (position j, value x) of a factor of this shape in the default configuration.
    Position 0 of the warp kernel: a lane owns D/2 table rows, in pairs ("warp pair"); when D/2 is odd the
    last two rows of the factor are the lanes' single rows ("warp single")."""
    fam = factor_family(shape)
    if fam == "warp" and j == 0:
        hd = int(shape[0]) // 2
        return "warp single" if hd % 2 == 1 and x >= 2 * (hd - 1) else "warp pair"
    if fam == "pipe" and j == 0:
        return f"pipe arity {len(shape)}"
    return f"{fam} position {j}" if fam != "tiled_rt" else "tiled_rt"


def all_nan_outputs(inst, q, q_valid):
    """(factor, position, value) of every output whose candidates are all NaN, for the q rows `q` (flat,
    canonical edge order) of which the edges with q_valid set have been received.  `inst` holds the
    flat instance arrays (dom_size, factor_ptr, edge_var, tables; table_off optional)."""
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"], dtype=np.int64)
    tables = np.asarray(inst["tables"], dtype=np.float64)
    ed = dom[ev]
    moff = np.concatenate([[0], np.cumsum(ed)])
    sizes = np.array([int(np.prod(ed[fp[f]:fp[f + 1]])) for f in range(len(fp) - 1)], dtype=np.int64)
    toff = (np.asarray(inst["table_off"], dtype=np.int64) if inst.get("table_off") is not None
            else np.concatenate([[0], np.cumsum(sizes)]))
    q = np.asarray(q, dtype=np.float64)
    q_valid = np.asarray(q_valid).astype(bool)
    groups = {}
    for f in range(len(fp) - 1):
        groups.setdefault(tuple(int(x) for x in ed[fp[f]:fp[f + 1]]), []).append(f)
    out = []
    for shape, fs in groups.items():
        fs = np.asarray(fs, dtype=np.int64)
        a = len(shape)
        t = tables[toff[fs][:, None] + np.arange(int(np.prod(shape)))[None, :]].reshape((len(fs),) + shape)
        rows = []
        for i in range(a):
            e = fp[fs] + i
            r = q[moff[e][:, None] + np.arange(shape[i])[None, :]]
            r[~q_valid[e]] = 0.0          # not received yet: not part of the sum (maxsum.py:430-436)
            bshape = [len(fs)] + [1] * a
            bshape[i + 1] = shape[i]
            rows.append(r.reshape(bshape))
        for j in range(a):
            tot = t.copy()
            with np.errstate(invalid="ignore"):   # inf - inf: the NaN candidates looked for
                for i in range(a):
                    if i != j:
                        tot = tot + rows[i]
            nan = np.isnan(tot)
            axes = tuple(1 + i for i in range(a) if i != j)
            alln = nan.all(axis=axes) if axes else nan
            for k, x in zip(*np.nonzero(alln)):
                out.append((int(fs[k]), j, int(x)))
    return out


def sites_reached(inst, q, q_valid):
    """Set of output_site() names over all_nan_outputs()."""
    dom = np.asarray(inst["dom_size"])
    fp, ev = np.asarray(inst["factor_ptr"]), np.asarray(inst["edge_var"])
    return {output_site(tuple(int(d) for d in dom[ev[fp[f]:fp[f + 1]]]), j, x)
            for f, j, x in all_nan_outputs(inst, q, q_valid)}


def forbid(inst, sign, seed, share=0.3, dead_share=0.03):
    """Copy of a random instance (flat arrays) with hard constraints: about `share` of the cells of every
    other table set to sign * inf, and a unary factor whose whole row is sign * inf on about `dead_share`
    of the variables (every value of those forbidden)."""
    rng = np.random.default_rng(seed)
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"])
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    tables = np.array(inst["tables"], copy=True)
    sizes = np.array([int(np.prod(dom[ev[fp[f]:fp[f + 1]]])) for f in range(len(fp) - 1)], dtype=np.int64)
    toff = np.concatenate([[0], np.cumsum(sizes)])
    cell_factor = np.repeat(np.arange(len(sizes)), sizes)
    tables[(cell_factor % 2 == 0) & (rng.random(len(tables)) < share)] = sign * np.inf
    assert len(tables) == toff[-1]
    n_dead = max(1, int(round(dead_share * len(dom))))
    dead = np.sort(rng.choice(len(dom), n_dead, replace=False)).astype(ev.dtype)
    out = dict(inst)
    out["edge_var"] = np.concatenate([ev, dead])
    out["factor_ptr"] = np.concatenate([fp, fp[-1] + np.arange(1, n_dead + 1)]).astype(np.asarray(inst["factor_ptr"]).dtype)
    out["tables"] = np.concatenate([tables, np.full(int(dom[dead].sum()), sign * np.inf, dtype=tables.dtype)])
    return out
