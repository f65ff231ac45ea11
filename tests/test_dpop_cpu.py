"""CPU: the restated pseudo-tree (pydcop_b200/pseudotree.py) and the DPOP oracle (tests/_dpop_oracle.py)
against the reference's own runs (tests/golden/dpop_*.npz, tools/make_golden_dpop.py), the schedule's
round bound, and the oracle's optimum against brute force."""
import math
import os

import numpy as np
import pytest

import oracle as orc
import ref_shim
from _dpop_oracle import DpopOracle, brute_force
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200 import pseudotree as pt

NAMES = golden_names("dpop_")


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


def lists(inst, key):
    p, i = inst[key + "_ptr"], inst[key + "_idx"]
    return [i[p[k]:p[k + 1]].tolist() for k in range(len(p) - 1)]


def tree_of(inst):
    return pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])


def check_tree(t, inst):
    assert np.array_equal(t.parent, inst["parent"])
    assert t.children == lists(inst, "children")
    assert t.pseudo_parents == lists(inst, "pseudo_parents")
    assert t.pseudo_children == lists(inst, "pseudo_children")
    assert np.array_equal(t.owner, inst["owner"])


def golden_util(inst, u):
    """The reference's UTIL of u: (dimension variables in its order, table)."""
    dims = inst["util_var"][inst["util_var_ptr"][u]:inst["util_var_ptr"][u + 1]].tolist()
    flat = inst["util"][inst["util_ptr"][u]:inst["util_ptr"][u + 1]]
    return dims, flat.reshape(tuple(int(inst["dom_size"][v]) for v in dims))


def as_order(table, dims, target):
    return table.transpose([dims.index(v) for v in target])


def same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def check_against_golden(inst, meta, t, util_of, value, cost, dt=np.float64):
    """Every UTIL message (as the separator-ordered table `util_of(u)`), value and cost, bit for bit."""
    for u in range(len(inst["dom_size"])):
        if inst["parent"][u] < 0:
            continue
        dims, g = golden_util(inst, u)
        assert sorted(dims) == sorted(t.sep[u]), u
        assert same(util_of(u), as_order(g, dims, t.sep[u]).astype(dt)), u
    if meta["error"] is None:
        assert np.array_equal(value, inst["value"])
        assert same(np.asarray(cost, dtype=dt), inst["cost"].astype(dt))


@pytest.mark.parametrize("name", NAMES)
def test_restated_tree_matches_reference(name):
    inst, _ = load(name)
    check_tree(tree_of(inst), inst)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_f64(name):
    inst, meta = load(name)
    t = tree_of(inst)
    o = DpopOracle(inst, t, np.float64, meta["mode"]).run()
    check_against_golden(inst, meta, t, lambda u: o.util[u], o.value, o.cost)
    if meta["error"] is None:
        assert o.unresolved == 0
    else:
        assert meta["error"] == "IndexError" and o.unresolved > 0


def _integer_without_sentinel(inst):
    finite = np.isfinite(inst["tables"]).all() and np.isfinite(inst["unary"]).all()
    return (finite and np.array_equal(inst["tables"], np.round(inst["tables"])) and np.abs(inst["tables"]).max() < 2 ** 20
            and np.array_equal(inst["unary"], np.round(inst["unary"])) and not (inst["util"] == 2147483647.0).any())


@pytest.mark.parametrize("name", [n for n in NAMES if _integer_without_sentinel(load(n)[0])])
def test_oracle_matches_reference_f32(name):
    inst, meta = load(name)
    t = tree_of(inst)
    o = DpopOracle(inst, t, np.float32, meta["mode"]).run()
    check_against_golden(inst, meta, t, lambda u: o.util[u], o.value, o.cost, np.float32)


def test_fixtures_cover_the_quirks():
    """>= 3 children, the 2147483647 sentinel, ties, several roots, max mode, costs above 2^31, arity 4,
    the unresolved case."""
    seen = dict(children3=False, sentinel=False, ties=False, roots=False, max=False, above31=False,
                arity4=False, error=False)
    for name in NAMES:
        inst, meta = load(name)
        seen["children3"] |= bool((np.diff(inst["children_ptr"]) >= 3).any())
        seen["sentinel"] |= bool((inst["util"] == 2147483647.0).any())
        seen["roots"] |= len(meta["roots"]) > 1
        seen["max"] |= meta["mode"] == "max"
        seen["above31"] |= bool((inst["tables"][np.isfinite(inst["tables"])] > 2 ** 31).any())
        seen["arity4"] |= bool((np.diff(inst["factor_ptr"]) == 4).any())
        seen["error"] |= meta["error"] == "IndexError"
        t = tree_of(inst)
        o = DpopOracle(inst, t, np.float64, meta["mode"]).util_phase()
        for u in range(len(inst["dom_size"])):
            j = o.joined(u)
            if j.ndim and j.shape[0] > 1:
                best = j.min(0) if meta["mode"] == "min" else j.max(0)
                seen["ties"] |= bool(((j == best).sum(0) > 1).any())
    assert all(seen.values()), seen


def test_reference_unit_answers():
    """The answers of the reference's tests/unit/test_algorithms_dpop.py (max mode)."""
    two = dict(dom_size=np.array([2, 2]), factor_ptr=np.array([0, 2]), edge_var=np.array([0, 1]),
               tables=np.array([1.0, 2.0, 4.0, 3.0]))
    t = pt.build_tree(two["dom_size"], two["factor_ptr"], two["edge_var"])
    t.parent[:] = [-1, 0]
    t.children, t.roots = [[1], []], [0]
    t = pt.complete(t, two["dom_size"], [[0, 1]])
    o = DpopOracle(two, t, np.float64, "max").run()
    assert o.util[1].tolist() == [2.0, 4.0] and o.value.tolist() == [1, 0]      # x0 = b, x1 = a
    three = dict(dom_size=np.array([2, 2, 2]), factor_ptr=np.array([0, 2, 4]), edge_var=np.array([0, 1, 0, 2]),
                 tables=np.array([1.0, 2.0, 2.0, 3.0, 5.0, 2.0, 3.0, 1.0]))
    t = pt.build_tree(three["dom_size"], three["factor_ptr"], three["edge_var"])
    assert t.roots == [0] and t.children[0] == [1, 2]
    o = DpopOracle(three, t, np.float64, "max").run()
    assert o.util[1].tolist() == [2.0, 3.0] and o.util[2].tolist() == [5.0, 3.0]
    assert o.value.tolist() == [0, 1, 0]                                        # x0 = a, x1 = b, x2 = a


def random_instance(rng, n, doms, n_cons, arities, floats=True):
    dom = np.array([doms[i % len(doms)] for i in range(n)], dtype=np.int32)
    fp, ev, tabs = [0], [], []
    for j in range(n_cons):
        a = min(int(arities[j % len(arities)]), n)
        s = rng.choice(n, size=a, replace=False)
        ev += s.tolist()
        fp.append(len(ev))
        size = int(np.prod(dom[s]))
        tabs.append(np.round(rng.uniform(-5, 5, size), 3) if floats else rng.integers(0, 4, size).astype(float))
    unary = np.round(rng.uniform(0, 1, int(dom.sum())), 2)
    return dict(dom_size=dom, factor_ptr=np.array(fp), edge_var=np.array(ev, dtype=np.int32),
                tables=np.concatenate(tabs) if tabs else np.zeros(0), unary=unary)


def test_oracle_cost_is_the_optimum():
    """300 random instances of <= 9 variables: the roots' costs add up to the brute-force optimum."""
    rng = np.random.default_rng(11)
    for k in range(300):
        n = int(rng.integers(1, 10))
        inst = random_instance(rng, n, [2, 3], int(rng.integers(0, 2 * n + 1)), [2, 3, 1, 2], floats=bool(k % 2))
        mode = "max" if k % 3 == 0 else "min"
        t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
        o = DpopOracle(inst, t, np.float64, mode).run()
        assert o.unresolved == 0
        total = sum(o.cost[r] for r in t.roots)
        assert math.isclose(total, brute_force(inst, mode), rel_tol=1e-9, abs_tol=1e-9), k


def test_schedule_rounds_on_a_long_chain():
    """A 10^5-node chain (rooted at its last inner node): two heavy paths, so two rounds each way, not
    10^5 launches."""
    n = 100000
    ev = np.stack([np.arange(n - 1), np.arange(1, n)], 1).reshape(-1)
    dom = np.full(n, 3, dtype=np.int32)
    t = pt.build_tree(dom, np.arange(0, 2 * n - 1, 2), ev)
    assert t.height == n - 1
    s = pt.schedule(t)
    assert s.rounds == 2 and s.n_launches == 4


def test_schedule_rounds_bound_on_random_trees():
    rng = np.random.default_rng(5)
    for n in (50, 2000, 20000):
        p = np.array([int(rng.integers(0, i)) for i in range(1, n)])
        ev = np.stack([p, np.arange(1, n)], 1).reshape(-1)
        dom = np.full(n, 2, dtype=np.int32)
        t = pt.build_tree(dom, np.arange(0, 2 * n - 1, 2), ev)
        s = pt.schedule(t)
        assert s.rounds <= int(math.log2(n)) + 1
        assert sorted(s.util_nodes.tolist()) == list(range(n)) and sorted(s.value_nodes.tolist()) == list(range(n))


@pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference")
def test_restated_tree_matches_live_reference_on_random_graphs():
    ref_shim.install()
    from pydcop.computations_graph import pseudotree
    from pydcop.dcop.objects import Domain, Variable
    from pydcop.dcop.relations import NAryMatrixRelation
    rng = np.random.default_rng(3)
    for k in range(200):
        n = int(rng.integers(1, 16))
        inst = random_instance(rng, n, [2, 3], int(rng.integers(0, 2 * n + 2)), [2, 2, 3, 1, 4], floats=False)
        dom = {d: Domain(f"d{d}", "", list(range(d))) for d in (2, 3)}
        vs = [Variable(f"x{i:02d}", dom[int(inst["dom_size"][i])]) for i in range(n)]
        fp, ev = inst["factor_ptr"], inst["edge_var"]
        cs = [NAryMatrixRelation([vs[v] for v in ev[fp[f]:fp[f + 1]]], name=f"c{f:02d}") for f in range(len(fp) - 1)]
        g = pseudotree.build_computation_graph(None, variables=vs, constraints=cs)
        t = pt.build_tree(inst["dom_size"], fp, ev)
        idx = {v.name: i for i, v in enumerate(vs)}
        cidx = {c.name: f for f, c in enumerate(cs)}
        links = {}
        for node in g.nodes:
            u = idx[node.name]
            par, pp, ch, pc = pseudotree.get_dfs_relations(node)
            assert t.parent[u] == (idx[par] if par is not None else -1), k
            assert t.children[u] == [idx[x] for x in ch], k
            assert t.pseudo_parents[u] == [idx[x] for x in pp], k
            assert t.pseudo_children[u] == [idx[x] for x in pc], k
            # DpopAlgo keeps the constraints that involve none of its children or pseudo-children (dpop.py:188-199)
            below = set(ch) | set(pc)
            for c in node.constraints:
                if not below & {v.name for v in c.dimensions}:
                    assert t.owner[cidx[c.name]] == u, k
            links[node.name] = [(l.type, l.target) for l in node.links if l.source == node.name]
        assert t.roots == [idx[r.variable.name] for r in g.roots], k
        assert_same_tree(pt.tree_from_links([v.name for v in vs], links, inst["dom_size"], fp, ev), t)


def assert_same_tree(a, b):
    assert np.array_equal(a.parent, b.parent) and a.roots == b.roots
    assert a.children == b.children and a.pseudo_parents == b.pseudo_parents
    assert a.pseudo_children == b.pseudo_children and np.array_equal(a.owner, b.owner)
    assert a.owned == b.owned and a.sep == b.sep and a.util_size == b.util_size


@pytest.mark.parametrize("name", NAMES)
def test_tree_from_links_matches_build_tree(name):
    """The plugin path (the tree from the orchestrator's links, in the reference's link order) and the
    direct path give the same tree arrays."""
    inst, meta = load(name)
    names = [str(n) for n in inst["var_names"]]
    links = {}
    for u, n in enumerate(names):
        lst = [("parent", names[inst["parent"][u]])] if inst["parent"][u] >= 0 else []
        lst += [("children", names[c]) for c in lists(inst, "children")[u]]
        lst += [("pseudo_children", names[c]) for c in lists(inst, "pseudo_children")[u]]
        lst += [("pseudo_parent", names[c]) for c in lists(inst, "pseudo_parents")[u]]
        links[n] = lst
    t = pt.tree_from_links(names, links, inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    assert_same_tree(t, tree_of(inst))
    assert t.roots == meta["roots"]
