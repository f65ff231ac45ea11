"""The factor order inside a class (layout.build_layout): factors of every untagged class follow the q row of their
position-0 edge, so that a tile of consecutive factors reads its position-0 rows from one short window of q; the
layout stays a pure re-ordering of the caller's graph, and tagged classes (the multi-GPU ghost stubs) keep the
caller's order."""
import numpy as np
import pytest

from pydcop_b200.generators import config_c2, random_factor_graph
from pydcop_b200.layout import build_layout


def _mixed(seed):
    """Binary factors over two domain sizes, ternary and unary factors, a hub: several classes of each side."""
    rng = np.random.default_rng(seed)
    n = 600
    dom = np.where(rng.random(n) < 0.7, 10, 6).astype(np.int32)
    scopes = []
    for a, m in ((2, 1500), (3, 200), (1, 150)):
        for _ in range(m):
            s = rng.choice(n, a, replace=False)
            if a == 2 and rng.random() < 0.05:
                s[0] = 5                                       # hub: degree far above the class limit
            scopes.append(s)
    rng.shuffle(scopes)
    # binary factors whose scopes mix the two domain sizes stay in classes of their own (not uniform)
    factor_ptr = np.concatenate([[0], np.cumsum([len(s) for s in scopes])]).astype(np.int64)
    edge_var = np.concatenate(scopes).astype(np.int32)
    tsize = [int(np.prod(dom[s])) for s in scopes]
    tables = rng.integers(0, 9, int(sum(tsize))).astype(np.float32)
    unary = rng.random(int(dom.sum()))
    return dict(dom_size=dom, factor_ptr=factor_ptr, edge_var=edge_var, tables=tables, unary=unary)


def _check_pure_reordering(inst, L):
    fp = np.asarray(inst["factor_ptr"], dtype=np.int64)
    ev = np.asarray(inst["edge_var"])
    tables = np.asarray(inst["tables"]).reshape(-1)
    toff = np.concatenate([[0], np.cumsum([int(np.prod(np.asarray(inst["dom_size"])[ev[fp[f]:fp[f + 1]]]))
                                           for f in range(len(fp) - 1)])]).astype(np.int64)
    F, E = len(fp) - 1, len(ev)
    assert np.array_equal(np.sort(L.factor_perm), np.arange(F))
    assert np.array_equal(np.sort(L.edge_perm), np.arange(E))
    order = np.empty(F, dtype=np.int64)
    order[L.factor_perm] = np.arange(F)
    for c in L.classes:
        for i in range(c.n_factors):
            f = int(order[c.first_factor + i])
            a = int(fp[f + 1] - fp[f])
            assert a == c.arity
            # edges of internal factor i are its canonical edges, in scope order
            assert np.array_equal(L.edge_perm[fp[f]:fp[f + 1]], c.first_edge + i * a + np.arange(a))
            got = L.tables[c.table_base + i * c.table_size:c.table_base + (i + 1) * c.table_size]
            assert np.array_equal(got, tables[toff[f]:toff[f + 1]])
    assert np.array_equal(L.edge_var, L.var_perm[ev[np.argsort(L.edge_perm)]])
    # both sides address the same rows: slot s reads the r row of its edge and owns the q row of its edge
    assert np.array_equal(L.slot_roff, L.edge_msg_off[L.slot_edge])
    assert np.array_equal(L.edge_var[L.slot_edge], L.slot_var)
    # each variable still lists its factors in `links` order
    assert np.array_equal(L.slot_canon_edge, np.argsort(L.edge_perm)[L.slot_edge])
    # and the canonical round trip of the messages covers every element once
    g = L.message_gather_index()
    assert len(np.unique(g)) == len(g) == L.n_msg_canonical


def _check_order(L):
    for c in L.classes:
        if c.tag != 0 or c.n_factors < 2:
            continue
        q0 = L.edge_qoff[c.first_edge:c.first_edge + c.n_factors * c.arity:c.arity]
        assert (np.diff(q0) > 0).all(), c


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mixed_classes_are_ordered_by_position0_q_row(seed):
    inst = _mixed(seed)
    L = build_layout(**inst)
    assert len(L.classes) >= 4
    _check_order(L)
    _check_pure_reordering(inst, L)


def test_given_links_order_is_kept():
    """var_ptr / var_edge in an order other than ascending edge id: the factor order follows it."""
    inst = random_factor_graph(300, 4, 700, 2, seed=5)
    L0 = build_layout(**inst)
    rng = np.random.default_rng(3)
    var_ptr, var_edge = L0.canon_var_ptr.copy(), L0.canon_var_edge.copy()
    for v in range(len(var_ptr) - 1):
        seg = var_edge[var_ptr[v]:var_ptr[v + 1]]
        var_edge[var_ptr[v]:var_ptr[v + 1]] = seg[rng.permutation(len(seg))]
    L = build_layout(**inst, var_ptr=var_ptr, var_edge=var_edge)
    _check_order(L)
    _check_pure_reordering(inst, L)
    for i in range(0, L.n_vars, 7):
        v = int(L.var_order[i])
        assert np.array_equal(L.slot_canon_edge[L.var_ptr[i]:L.var_ptr[i + 1]], var_edge[var_ptr[v]:var_ptr[v + 1]])


def test_c2_position0_windows():
    """On the bench instance almost every 16-factor tile has its position-0 q rows within 2 KB (f32)."""
    inst = config_c2(seed=0, n_vars=20_000)
    L = build_layout(**inst)
    assert len(L.classes) == 1
    _check_order(L)
    c = L.classes[0]
    q0 = L.edge_qoff[c.first_edge:c.first_edge + 2 * c.n_factors:2]
    nt = c.n_factors // 16
    w = q0[:nt * 16].reshape(nt, 16)
    span = (w.max(1) - w.min(1) + 10) * 4
    assert (span <= 2048).mean() > 0.99
    # the permutation of the tables is deferred (the engine applies it on the device) until `tables` is read; then
    # the rows come from a row gather (writable input) or numpy's take (read-only input): same rows
    assert L.table_rows is not None and L._tables is None
    order = np.empty(c.n_factors, dtype=np.int64)
    order[L.factor_perm] = np.arange(c.n_factors)
    want = np.asarray(inst["tables"]).reshape(-1, 100)[order]
    assert np.array_equal(L.tables[:c.n_factors * 100].reshape(-1, 100), want)
    ro = dict(inst, tables=np.asarray(inst["tables"]).copy())
    ro["tables"].flags.writeable = False
    assert np.array_equal(build_layout(**ro).tables, L.tables)


@pytest.mark.parametrize("world", [2, 3])
def test_shard_stub_classes_keep_the_caller_order(world):
    from pydcop_b200.multigpu import build_shard
    inst = random_factor_graph(500, 6, 1200, 2, seed=11)
    for r in range(world):
        L = build_shard(inst, r, world).layout
        tagged = [c for c in L.classes if c.tag != 0]
        assert tagged and any(c.tag == 0 for c in L.classes)
        order = np.empty(L.n_factors, dtype=np.int64)
        order[L.factor_perm] = np.arange(L.n_factors)
        for c in tagged:
            assert (np.diff(order[c.first_factor:c.first_factor + c.n_factors]) > 0).all()
        _check_order(L)
