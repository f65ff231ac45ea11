"""Host-side packing of a DCOP factor graph into the engine's class-major CSR layout.

Input ("array front door", canonical order = the order the caller lists factors in):
    dom_size[V]            domain size of each variable
    factor_ptr[F+1]        scope of factor f = edge_var[factor_ptr[f]:factor_ptr[f+1]]
    edge_var[E]            variable of each factor->variable edge; scope order == table axis order
                           (NAryMatrixRelation._m, pydcop/dcop/relations.py:716-733)
    tables, table_off[F+1] dense row-major cost tables, flattened
    unary[sum dom_size]    variable costs (Variable.cost_for_val, pydcop/dcop/objects.py:231)
    var_ptr, var_edge      optional: incident edges of each variable in the reference's `links`
                           order (pydcop/algorithms/maxsum.py:466); default = ascending edge id,
                           which is the order factor_graph.build_computation_graph produces
                           (pydcop/computations_graph/factor_graph.py:277-280)

Output: factors grouped into classes of identical shape so that tables and message rows are
affine in the factor index (include/pydcop_b200.h), plus the permutations needed to move between
canonical and internal order.  Everything is vectorised numpy: 10^6-variable graphs pack in
seconds (the reference's own graph build is O(|V|*|C|), pydcop/dcop/relations.py:1245-1247).
`FactorGraphLayout.tables` may be a VIEW of the caller's `tables` (one class, factors already adjacent): treat the
input as read-only while the layout is in use.
"""
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

MAX_ARITY = 8
MAX_DOM = 256
ALIGN = 32  # elements: class bases are 128-B aligned (f32) for bulk async copies
MAX_CLASS_DEGREE = 16  # variables of larger degree share one irregular (CSR-driven) class


@dataclass
class FactorClass:
    arity: int
    dom: tuple
    n_factors: int
    first_factor: int
    first_edge: int
    table_size: int
    table_base: int
    msg_base: int
    tag: int = 0

    @property
    def uniform(self):
        return all(d == self.dom[0] for d in self.dom)

    @property
    def row_off(self):
        """Offset of each scope position's message row inside the factor's row block.  Classes
        whose positions have different domain sizes start every row on a 4-element boundary so
        that a row of a D-valued variable is always aligned to gcd(16 bytes, D*sizeof(T))."""
        out, s = [], 0
        for d in self.dom:
            out.append(s)
            s += d if self.uniform else (d + 3) // 4 * 4
        return tuple(out)

    @property
    def row_total(self):
        if self.uniform:
            return int(sum(self.dom))
        return int(sum((d + 3) // 4 * 4 for d in self.dom))


@dataclass
class VarClass:
    """Variables of identical (domain size, degree): unary rows, q rows and slots are affine in
    the variable's rank inside the class.  degree == -1: irregular class (CSR via var_ptr)."""
    dom: int
    degree: int
    n_vars: int
    first_var: int
    first_slot: int
    unary_base: int
    q_base: int
    n_slots: int = 0
    tag: int = 0


@dataclass
class FactorGraphLayout:
    n_vars: int
    n_factors: int
    n_edges: int
    n_msg: int                 # internal r-array elements (class-major edge order, padded bases)
    n_msg_q: int               # internal q-array elements (slot order)
    n_msg_canonical: int
    classes: List[FactorClass]
    var_classes: List[VarClass]
    # NOTE: every per-variable / per-slot array below is in INTERNAL variable order (variables
    # sorted by class); var_perm / var_order translate from / to the caller's canonical order.
    dom_size: np.ndarray       # int32 [V]
    unary_off: np.ndarray      # int64 [V+1]
    unary: np.ndarray          # float64 [sum dom]
    tables: np.ndarray         # float64, internal (class-major) order, padded
    var_ptr: np.ndarray        # int32 [V+1]
    slot_edge: np.ndarray      # int32 [E]  internal edge id of slot s
    slot_var: np.ndarray       # int32 [E]
    slot_roff: np.ndarray      # int64 [E]  offset in r of the row of slot s's edge
    var_qbase: np.ndarray      # int64 [V+1] offset in q of the first slot of v
    edge_qoff: np.ndarray      # int64 [E]  internal edge order: offset in q of the edge's row
    uniform_dom: int           # D when all variables share one domain size, else 0
    max_degree: int
    edge_var: np.ndarray       # int32 [E]  internal edge order
    edge_class: np.ndarray     # int32 [E]  internal edge order
    edge_msg_off: np.ndarray   # int64 [E]  internal edge order -> internal message offset
    edge_perm: np.ndarray      # int32 [E]  canonical edge -> internal edge
    factor_perm: np.ndarray    # int32 [F]  canonical factor -> internal factor
    var_perm: np.ndarray       # int32 [V]  canonical variable -> internal variable
    var_order: np.ndarray      # int32 [V]  internal variable -> canonical variable
    canon_edge_var: np.ndarray  # int32 [E]  canonical edge -> canonical variable
    canon_msg_off: np.ndarray  # int64 [E+1]
    canon_var_ptr: np.ndarray  # int32 [V+1] canonical CSR (the reference's `links` order)
    canon_var_edge: np.ndarray  # int32 [E]
    canon_dom_size: np.ndarray  # int32 [V]
    slot_canon_edge: np.ndarray  # int32 [E] canonical edge id of INTERNAL slot s
    init_value: np.ndarray     # int32 [V] (-1 = none), internal order
    msg_gather: Optional[np.ndarray] = field(default=None, repr=False)
    msg_gather_q: Optional[np.ndarray] = field(default=None, repr=False)
    # deferred table permutation (one class only): internal tables = rows table_rows of table_src viewed as
    # (n_rows, table_size), then zeros up to table_total elements; `tables` is None until first read
    table_src: Optional[np.ndarray] = field(default=None, repr=False)
    table_rows: Optional[np.ndarray] = field(default=None, repr=False)
    table_total: int = 0

    # -- canonical <-> internal helpers (used by tests / readback, not by the hot path) ---------
    def message_gather_index(self):
        """Index array g with canonical_r = internal_r[g] (canonical = edge order of the input)."""
        if self.msg_gather is None:
            d = np.diff(self.canon_msg_off)
            start = self.edge_msg_off[self.edge_perm] - self.canon_msg_off[:-1]
            self.msg_gather = (np.repeat(start, d)
                               + np.arange(self.n_msg_canonical, dtype=np.int64))
        return self.msg_gather

    def message_gather_index_q(self):
        """Index array g with canonical_q = internal_q[g]."""
        if self.msg_gather_q is None:
            d = np.diff(self.canon_msg_off)
            start = self.edge_qoff[self.edge_perm] - self.canon_msg_off[:-1]
            self.msg_gather_q = (np.repeat(start, d)
                                 + np.arange(self.n_msg_canonical, dtype=np.int64))
        return self.msg_gather_q

    def edges_to_canonical(self, arr_internal):
        return np.asarray(arr_internal)[self.edge_perm]

    def slots_to_canonical_edges(self, arr_slot):
        out = np.zeros(self.n_edges, dtype=np.asarray(arr_slot).dtype)
        out[self.slot_canon_edge] = np.asarray(arr_slot)
        return out

    def vars_to_canonical(self, arr_internal):
        return np.asarray(arr_internal)[self.var_perm]

    def canonical_unary(self):
        """Unary costs back in canonical order, without class padding."""
        d = self.canon_dom_size.astype(np.int64)
        start = self.unary_off[:-1][self.var_perm]
        idx = np.repeat(start, d) + (np.arange(int(d.sum()), dtype=np.int64)
                                     - np.repeat(np.cumsum(d) - d, d))
        return self.unary[idx]


def _layout_tables(self):
    if self._tables is None and self.table_rows is not None:
        self._tables = _take_rows(self.table_src, self.table_rows, self.table_src.size // len(self.table_rows),
                                  self.table_total)
    return self._tables


def _set_layout_tables(self, value):
    self._tables = value


FactorGraphLayout.tables = property(_layout_tables, _set_layout_tables,
                                    doc="tables in internal (class-major) order; a deferred permutation is applied on "
                                        "first read")


def _as(a, dt):
    return np.ascontiguousarray(np.asarray(a), dtype=dt)


def _unique_rows(key):
    """np.unique(key, axis=0, return_inverse=True) — same rows, same (lexicographic) order, same
    inverse — for the factor class keys (8 domain sizes <= MAX_DOM, then the tag): the first seven
    columns are packed into one int64 (base MAX_DOM + 1, most significant first), the last two into
    another, and two 1-D integer sorts replace the row sort, which dominates the packing of 10^6 factors."""
    key = np.asarray(key)
    n, m = key.shape
    if n and (key == key[0]).all():     # one shape (the usual generated instance): nothing to sort
        return key[:1].copy(), np.zeros(n, dtype=np.int64)
    if n == 0 or m != MAX_ARITY + 1 or key.min() < 0 or key[:, :MAX_ARITY].max() > MAX_DOM:
        u, inv = np.unique(key, axis=0, return_inverse=True)
        return u, inv.reshape(-1)
    base = MAX_DOM + 1
    k = key.astype(np.int64)
    lo = np.zeros(n, dtype=np.int64)
    for i in range(7):
        lo = lo * base + k[:, i]
    tag_base = int(k[:, MAX_ARITY].max()) + 1
    hi = k[:, 7] * tag_base + k[:, MAX_ARITY]
    _, inv_lo = np.unique(lo, return_inverse=True)
    u_hi, inv_hi = np.unique(hi, return_inverse=True)
    code = inv_lo.astype(np.int64) * len(u_hi) + inv_hi
    _, first, inv = np.unique(code, return_index=True, return_inverse=True)
    return key[first], inv.reshape(-1)


def _gather_tables(tables, starts, size):
    """Tables of `size` elements starting at `starts`, concatenated.  Factors of one class usually sit
    next to each other in the caller's array: contiguous runs are taken as slices (one run = a view,
    no copy) instead of through an (n x size) index array, which at 10^6 factors costs more than
    everything else in the packing."""
    n = len(starts)
    if n == 0:
        return tables[:0]
    brk = np.nonzero(np.diff(starts) != size)[0] + 1
    if len(brk) == 0:
        return tables[starts[0]:starts[0] + n * size]
    if len(brk) <= max(1, n // 64):
        bounds = np.concatenate([[0], brk, [n]])
        return np.concatenate([tables[starts[a]:starts[a] + (b - a) * size]
                               for a, b in zip(bounds[:-1], bounds[1:])])
    if tables.flags.writeable and tables.size % size == 0 and not (starts % size).any():
        return _take_rows(tables, starts // size, size, n * size)      # one table shape tiles the array: a row gather
    idx = starts[:, None] + np.arange(size, dtype=np.int64)[None, :]
    return tables[idx.reshape(-1)]


def _take_rows(src, rows, size, total):
    """Rows `rows` of src viewed as (-1, size), flattened, then zeros up to `total` elements: a row gather on torch's CPU
    threads (4-5x faster than numpy's single-threaded take at 10^5 rows)."""
    out = np.zeros(total, dtype=src.dtype)
    if not src.flags.writeable:     # torch wants writable memory (e.g. not a read-only memory map): numpy's take
        out[:len(rows) * size] = src.reshape(-1, size)[rows].reshape(-1)
        return out
    import torch
    torch.index_select(torch.from_numpy(src.reshape(-1, size)), 0, torch.from_numpy(np.asarray(rows, dtype=np.int64)),
                       out=torch.from_numpy(out[:len(rows) * size].reshape(-1, size)))
    return out


def stable_group_order(keys, n_groups=None):
    """np.argsort(keys, kind="stable") for small non-negative integer keys, plus the group pointer array:
    a counting sort (scipy's COO -> CSR kernel, O(n)) instead of a comparison sort — the packing of a
    10^5-variable problem spent a third of its time in three such sorts.  Returns (order int32, ptr int32)."""
    keys = np.ascontiguousarray(keys)
    n = len(keys)
    if n_groups is None:
        n_groups = int(keys.max()) + 1 if n else 0
    if n and n < 2 ** 31 - 1 and n_groups < 2 ** 31 - 1:
        try:
            from scipy.sparse import _sparsetools
            k32 = keys.astype(np.int32, copy=False)
            ptr = np.empty(n_groups + 1, dtype=np.int32)
            order = np.empty(n, dtype=np.int32)
            junk = np.empty(n, dtype=np.int8)
            _sparsetools.coo_tocsr(n_groups, n, n, k32, np.arange(n, dtype=np.int32), np.zeros(n, dtype=np.int8),
                                   ptr, order, junk)
            return order, ptr
        except Exception:  # noqa: BLE001 — scipy missing or its private kernel moved: comparison sort below
            pass
    order = np.argsort(keys, kind="stable").astype(np.int32)
    ptr = np.zeros(n_groups + 1, dtype=np.int32)
    if n:
        np.cumsum(np.bincount(keys, minlength=n_groups), out=ptr[1:])
    return order, ptr


def default_var_csr(n_vars, edge_var):
    """Incident edges per variable in ascending (canonical) edge id == constraint order."""
    order, var_ptr = stable_group_order(_as(edge_var, np.int32), n_vars)
    return var_ptr, order


def build_layout(dom_size, factor_ptr, edge_var, tables, table_off=None, unary=None,
                 var_ptr=None, var_edge=None, init_value=None, factor_tag=None,
                 var_tag=None) -> FactorGraphLayout:
    """factor_tag / var_tag (optional small ints): factors / variables with different tags never
    share a class.  The multi-GPU shards tag their ghost stubs so the engine can skip them."""
    dom_size = _as(dom_size, np.int32)
    factor_ptr = _as(factor_ptr, np.int64)
    edge_var = _as(edge_var, np.int32)
    tables = np.ascontiguousarray(np.asarray(tables)).reshape(-1)
    if tables.dtype != np.float32:      # float32 tables are kept as they are (half the host memory)
        tables = tables.astype(np.float64, copy=False)
    V, F, E = len(dom_size), len(factor_ptr) - 1, len(edge_var)
    if F < 0 or factor_ptr[0] != 0 or factor_ptr[-1] != E:
        raise ValueError("factor_ptr must start at 0 and end at len(edge_var)")
    if E and (edge_var.min() < 0 or edge_var.max() >= V):
        raise ValueError("edge_var out of range")
    if V and (dom_size.min() < 1 or dom_size.max() > MAX_DOM):
        raise ValueError(f"domain sizes must be in 1..{MAX_DOM}")
    arity = np.diff(factor_ptr)
    if F and (arity.min() < 1 or arity.max() > MAX_ARITY):
        raise ValueError(f"factor arity must be in 1..{MAX_ARITY}")
    edge_dom = dom_size[edge_var] if E else np.zeros(0, np.int32)

    # shape key per factor: domain sizes padded with zeros
    key = np.zeros((F, MAX_ARITY + 1), dtype=np.int32)
    if E:
        efac = np.repeat(np.arange(F, dtype=np.int64), arity)
        epos = np.arange(E, dtype=np.int64) - factor_ptr[:-1][efac]
        key[efac, epos] = edge_dom
    # arity >= 1 everywhere (checked above): the table size is the product over each factor's run of edges
    tsize = np.multiply.reduceat(edge_dom.astype(np.int64), factor_ptr[:-1]) if F else np.zeros(0, np.int64)
    if factor_tag is not None and F:
        key[:, MAX_ARITY] = _as(factor_tag, np.int32)
    if table_off is None:
        table_off = np.zeros(F + 1, dtype=np.int64)
        np.cumsum(tsize, out=table_off[1:])
    table_off = _as(table_off, np.int64)
    if F and not np.array_equal(np.diff(table_off), tsize):
        raise ValueError("table sizes do not match the scopes' domain sizes")
    if tables.size != (table_off[-1] if F else 0):
        raise ValueError("tables has the wrong number of elements")

    if F:
        uniq, cls_of_factor = _unique_rows(key)
    else:
        uniq, cls_of_factor = np.zeros((0, MAX_ARITY + 1), np.int32), np.zeros(0, np.int64)
    counts = np.bincount(cls_of_factor, minlength=len(uniq)) if F else np.zeros(0, np.int64)

    canon_msg_off = np.zeros(E + 1, dtype=np.int64)
    np.cumsum(edge_dom, out=canon_msg_off[1:])

    # ---------------- variable side: classes of identical (domain size, degree) ----------------
    if var_ptr is None or var_edge is None:
        var_ptr, var_edge = default_var_csr(V, edge_var)
    c_var_ptr = _as(var_ptr, np.int32)
    c_var_edge = _as(var_edge, np.int32)
    if c_var_ptr[-1] != E or len(c_var_edge) != E:
        raise ValueError("var_ptr / var_edge must cover every edge exactly once")
    c_slot_var = np.repeat(np.arange(V, dtype=np.int32), np.diff(c_var_ptr)).astype(np.int32)
    if E and not np.array_equal(edge_var[c_var_edge], c_slot_var):
        raise ValueError("var_edge lists an edge under the wrong variable")
    c_deg = np.diff(c_var_ptr).astype(np.int64)
    c_unary_off = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(dom_size, out=c_unary_off[1:])
    c_unary = (np.zeros(int(c_unary_off[-1])) if unary is None
               else _as(unary, np.float64).reshape(-1))
    if c_unary.size != c_unary_off[-1]:
        raise ValueError("unary has the wrong number of elements")
    c_init = np.full(V, -1, np.int32) if init_value is None else _as(init_value, np.int32)

    # class key: (domain size, degree), degrees above MAX_CLASS_DEGREE share one irregular class
    kdeg = np.where(c_deg <= MAX_CLASS_DEGREE, c_deg, MAX_CLASS_DEGREE + 1)
    vkey = dom_size.astype(np.int64) * (MAX_CLASS_DEGREE + 2) + kdeg
    vtag = np.zeros(V, dtype=np.int64) if var_tag is None else _as(var_tag, np.int64)
    vkey = vkey + vtag * ((MAX_DOM + 1) * (MAX_CLASS_DEGREE + 2))
    _, vk_inv = np.unique(vkey, return_inverse=True)               # dense class index, same order as the keys
    var_order = stable_group_order(vk_inv.reshape(-1))[0]           # internal -> canonical
    var_perm = np.empty(V, dtype=np.int32)
    var_perm[var_order] = np.arange(V, dtype=np.int32)              # canonical -> internal
    i_dom = dom_size[var_order]
    i_deg = c_deg[var_order]
    i_var_ptr = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(i_deg, out=i_var_ptr[1:])
    slot_var = np.repeat(np.arange(V, dtype=np.int32), i_deg).astype(np.int32)
    # canonical slot feeding each internal slot (per-variable `links` order is preserved)
    src_slot = (c_var_ptr[:-1].astype(np.int64)[var_order][slot_var]
                + (np.arange(E, dtype=np.int64) - i_var_ptr[:-1].astype(np.int64)[slot_var])) \
        if E else np.zeros(0, np.int64)
    slot_canon_edge = c_var_edge[src_slot].astype(np.int32) if E else np.zeros(0, np.int32)
    var_classes: List[VarClass] = []
    i_unary_off = np.zeros(V + 1, dtype=np.int64)
    var_qbase = np.zeros(V + 1, dtype=np.int64)
    ukeys, ustart, ucount = (np.unique(vkey[var_order], return_index=True, return_counts=True)
                             if V else (np.zeros(0, np.int64),) * 3)
    unary_base = q_base = 0
    unary_parts = []
    for k, st, n in zip(ukeys, ustart, ucount):
        st, n = int(st), int(n)
        D = int(i_dom[st])
        K = int(k % (MAX_CLASS_DEGREE + 2))
        regular = K <= MAX_CLASS_DEGREE
        vc = VarClass(D, K if regular else -1, n, st, int(i_var_ptr[st]), unary_base, q_base,
                      int(i_deg[st:st + n].sum()), tag=int(k // ((MAX_DOM + 1) * (MAX_CLASS_DEGREE + 2))))
        var_classes.append(vc)
        i_unary_off[st:st + n] = unary_base + np.arange(n, dtype=np.int64) * D
        # the class's rows of own costs, gathered from the canonical array (rows of D contiguous elements)
        src0 = c_unary_off[:-1][var_order[st:st + n]]
        unary_parts.append((unary_base, c_unary[(src0[:, None] + np.arange(D, dtype=np.int64)[None, :]).reshape(-1)]))
        slots_before = (i_var_ptr[st:st + n].astype(np.int64) - int(i_var_ptr[st]))
        var_qbase[st:st + n] = q_base + slots_before * D
        unary_base += n * D
        unary_base += (-unary_base) % ALIGN
        q_base += int(i_deg[st:st + n].sum()) * D
        q_base += (-q_base) % ALIGN
    i_unary_off[V] = unary_base
    var_qbase[V] = q_base
    i_unary = np.zeros(int(unary_base))
    for base, part in unary_parts:
        i_unary[base:base + len(part)] = part
    slot_qoff = (var_qbase[:-1][slot_var]
                 + (np.arange(E, dtype=np.int64) - i_var_ptr[:-1].astype(np.int64)[slot_var])
                 * i_dom.astype(np.int64)[slot_var]) if E else np.zeros(0, np.int64)

    # ---------------- factor order ----------------
    # Inside a class with tag 0, factors follow the q row of their position-0 edge: the internal index of the
    # first variable, then the factor's place in that variable's `links`.  The position-0 rows a tile of factors
    # gathers then lie within a window of about a kilobyte, and so do the r rows a tile of variables reads at
    # its position-0 slots; the warp kernels load that window with one bulk copy (DESIGN.md §3).  Tagged classes
    # (the multi-GPU ghost stubs) keep the caller's order.  Two stable counting sorts: key, then class.
    slot_of_edge = np.empty(E, dtype=np.int64)
    slot_of_edge[slot_canon_edge] = np.arange(E, dtype=np.int64)
    tag0 = (uniq[:, MAX_ARITY] == 0)[cls_of_factor] if F else np.zeros(0, dtype=bool)
    fkey = np.where(tag0, slot_of_edge[factor_ptr[:-1]], np.arange(F, dtype=np.int64))
    by_key = stable_group_order(fkey, max(E, F))[0]
    order = by_key[stable_group_order(cls_of_factor[by_key], len(uniq))[0]].astype(np.int64)   # internal -> canonical
    factor_perm = np.empty(F, dtype=np.int32)
    factor_perm[order] = np.arange(F, dtype=np.int32)          # canonical -> internal

    classes: List[FactorClass] = []
    table_rows = None
    edge_perm = np.zeros(E, dtype=np.int32)
    edge_msg_off = np.zeros(E, dtype=np.int64)
    edge_class = np.zeros(E, dtype=np.int32)
    int_edge_var = np.zeros(E, dtype=np.int32)
    tab_parts = []
    first_factor = first_edge = table_base = msg_base = 0
    for ci in range(len(uniq)):
        dom = tuple(int(x) for x in uniq[ci][:MAX_ARITY] if x > 0)
        a, n = len(dom), int(counts[ci])
        S = int(np.prod(dom, dtype=np.int64))
        fc = FactorClass(a, dom, n, first_factor, first_edge, S, table_base, msg_base,
                         tag=int(uniq[ci][MAX_ARITY]))
        R = fc.row_total
        classes.append(fc)
        fs = order[first_factor:first_factor + n]               # canonical factor ids, in order
        # tables.  One class whose tables tile the caller's array in another order (C2 after the factor order of
        # DESIGN.md §3): the permutation is recorded, not applied: MaxSumEngine uploads the caller's array and permutes
        # the rows on the device, every other reader gets the host copy on first access of `tables`
        if len(uniq) == 1 and tables.size == n * S and n > 1 and (table_off[fs] != np.arange(n) * S).any():
            table_rows = np.ascontiguousarray(table_off[fs] // S)
            t = tables[:0]
            t_size = n * S
        else:
            t = _gather_tables(tables, table_off[fs], S)
            t_size = t.size
        pad = (-t_size) % ALIGN
        tab_parts.append(t)
        if pad:
            tab_parts.append(np.zeros(pad, dtype=tables.dtype))
        # edges
        ce = (factor_ptr[fs][:, None] + np.arange(a, dtype=np.int64)[None, :]).reshape(-1)
        ie = first_edge + np.arange(n * a, dtype=np.int64)
        edge_perm[ce] = ie
        int_edge_var[ie] = edge_var[ce]
        edge_class[ie] = ci
        row_off = np.array(fc.row_off, dtype=np.int64)
        edge_msg_off[ie] = (msg_base + (np.arange(n, dtype=np.int64) * R)[:, None]
                            + row_off[None, :]).reshape(-1)
        first_factor += n
        first_edge += n * a
        table_base += t_size + pad
        msg_base += n * R
        msg_base += (-msg_base) % ALIGN
    n_msg = msg_base
    tables_int = (tab_parts[0] if len(tab_parts) == 1 else np.concatenate(tab_parts)) if tab_parts \
        else np.zeros(0, dtype=tables.dtype)
    table_src = None
    if table_rows is not None:      # deferred: the rows of `tables` in internal order, then the class padding
        table_src, tables_int = tables, None

    slot_edge = edge_perm[slot_canon_edge].astype(np.int32)
    slot_roff = edge_msg_off[slot_edge]
    edge_qoff = np.zeros(E, dtype=np.int64)
    edge_qoff[slot_edge] = slot_qoff
    uniform_dom = int(dom_size[0]) if V and (dom_size == dom_size[0]).all() else 0
    int_edge_var = var_perm[int_edge_var] if E else int_edge_var

    return FactorGraphLayout(
        n_vars=V, n_factors=F, n_edges=E, n_msg=int(n_msg), n_msg_q=int(q_base),
        n_msg_canonical=int(canon_msg_off[-1]), classes=classes, var_classes=var_classes,
        dom_size=i_dom.astype(np.int32), unary_off=i_unary_off, unary=i_unary, tables=tables_int,
        var_ptr=i_var_ptr, slot_edge=slot_edge, slot_var=slot_var, slot_roff=slot_roff,
        var_qbase=var_qbase, edge_qoff=edge_qoff, uniform_dom=uniform_dom,
        max_degree=int(c_deg.max(initial=0)), edge_var=int_edge_var.astype(np.int32),
        edge_class=edge_class, edge_msg_off=edge_msg_off, edge_perm=edge_perm,
        factor_perm=factor_perm, var_perm=var_perm, var_order=var_order,
        canon_edge_var=edge_var, canon_msg_off=canon_msg_off, canon_var_ptr=c_var_ptr,
        canon_var_edge=c_var_edge, canon_dom_size=dom_size, slot_canon_edge=slot_canon_edge,
        init_value=c_init[var_order].astype(np.int32), table_src=table_src, table_rows=table_rows,
        table_total=int(table_base))


def layout_from_instance(inst) -> FactorGraphLayout:
    """From a dict/npz with the array front-door keys (tests/golden fixtures use these names)."""
    def get(k):
        return inst[k] if k in inst else None
    var_edge = get("var_edge")
    if var_edge is None and get("var_con") is not None:
        var_edge = var_con_to_edges(inst)
    return build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"],
                        get("table_off"), get("unary"), get("var_ptr"), var_edge,
                        get("init_value"))


def var_con_to_edges(inst):
    """DSA lists constraint ids per variable (node.constraints order); turn into edge ids."""
    factor_ptr = np.asarray(inst["factor_ptr"], dtype=np.int64)
    edge_var = np.asarray(inst["edge_var"], dtype=np.int64)
    var_ptr = np.asarray(inst["var_ptr"], dtype=np.int64)
    var_con = np.asarray(inst["var_con"], dtype=np.int64)
    V = len(var_ptr) - 1
    slot_var = np.repeat(np.arange(V, dtype=np.int64), np.diff(var_ptr))
    # position of slot_var inside the scope of var_con: compare against each scope position
    out = np.full(len(var_con), -1, dtype=np.int64)
    arity = np.diff(factor_ptr)
    for j in range(int(arity.max(initial=0))):
        ok = (arity[var_con] > j) & (out < 0)
        e = factor_ptr[var_con] + j
        hit = ok & (edge_var[np.where(ok, e, 0)] == slot_var)
        out[hit] = e[hit]
    if (out < 0).any():
        raise ValueError("var_con lists a constraint that does not contain the variable")
    return out.astype(np.int32)
