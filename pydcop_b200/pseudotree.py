"""DFS pseudo-tree of a DCOP and the static DPOP schedule over it.

`build_tree` restates pyDcop's `pseudotree.build_computation_graph` (pydcop/computations_graph/
pseudotree.py:218-539) from the canonical arrays (`dom_size`, `factor_ptr`, `edge_var`, file order),
iteratively and in O(V + sum deg^2) instead of the reference's recursive O(V*C):
- one DFS tree per connected component; the root is the remaining variable with the most distinct
  neighbours, the LAST one in variable order among ties (stable sort, then [-1], :353-354);
- a node lists its neighbours in constraint order, within one constraint in VARIABLE order (the loop
  over `nodes`, :314-321), dropping repeats;
- before it descends, a node stably sorts its neighbours by how many of THEIR neighbours lie on the
  root-to-node path, highest first (:269-280); unvisited neighbours become children in that order, an
  adjacent ancestor is a pseudo-parent (kept in neighbour order), an adjacent descendant that is not a
  child a pseudo-child (in the order the DFS reaches it);
- each constraint belongs to the deepest variable of its scope (dpop.py:188-199).

`tree_from_links` reads the same arrays from the orchestrator's PseudoTreeNode links (the plugin path).
`schedule` turns a tree into the device schedule (heavy/light path rounds, big nodes) and `terms` into
the per-node term descriptors of csrc/dpop_kernels.cuh.
"""
from dataclasses import dataclass
from typing import List

import numpy as np

#: a node with more UTIL entries than this is computed by the grid-wide kernel (one thread per UTIL entry)
#: instead of one warp
BIG_UTIL = 1 << 13
#: separator variables per node the kernels decode (csrc/dpop_kernels.cuh FG_DPOP_MAX_SEP)
MAX_SEP = 32


@dataclass
class PseudoTree:
    n_vars: int
    parent: np.ndarray            # int32 [V], -1 at a root
    children: List[List[int]]     # per node, in visiting order
    pseudo_parents: List[List[int]]
    pseudo_children: List[List[int]]
    roots: List[int]              # in the order the components were built
    owner: np.ndarray = None      # int32 [F] node that owns each constraint
    depth: np.ndarray = None      # int32 [V]
    sep: List[List[int]] = None   # per node, separator in depth order (root side first)
    util_size: List[int] = None   # per node, product of the separator's domain sizes (Python int)
    owned: List[List[int]] = None  # per node, the constraints it owns in summation order

    @property
    def height(self):
        return int(self.depth.max(initial=-1)) + 1

    def preorder(self):
        out = []
        for r in self.roots:
            stack = [r]
            while stack:
                u = stack.pop()
                out.append(u)
                stack.extend(reversed(self.children[u]))
        return out


def _scopes(factor_ptr, edge_var):
    fp = np.asarray(factor_ptr, dtype=np.int64).tolist()
    ev = np.asarray(edge_var, dtype=np.int64).tolist()
    return [ev[fp[f]:fp[f + 1]] for f in range(len(fp) - 1)]


def neighbours(n_vars, scopes):
    """Distinct neighbours of every variable in the reference's order (:303-322)."""
    var_facs = [[] for _ in range(n_vars)]
    for f, s in enumerate(scopes):
        for v in s:
            lst = var_facs[v]
            if not lst or lst[-1] != f:
                lst.append(f)
    sorted_scopes = [sorted(set(s)) for s in scopes]
    out = []
    for v in range(n_vars):
        seen, lst = {v}, []
        for f in var_facs[v]:
            for x in sorted_scopes[f]:
                if x not in seen:
                    seen.add(x)
                    lst.append(x)
        out.append(lst)
    return out


def build_tree(dom_size, factor_ptr, edge_var) -> PseudoTree:
    V = len(dom_size)
    scopes = _scopes(factor_ptr, edge_var)
    nbrs = neighbours(V, scopes)
    parent = [-1] * V
    children = [[] for _ in range(V)]
    pparents = [[] for _ in range(V)]
    pchildren = [[] for _ in range(V)]
    on_path = bytearray(V)
    in_tree = bytearray(V)
    roots = []

    def enter(u, p, stack):
        in_tree[u] = 1
        parent[u] = p
        pparents[u] = [x for x in nbrs[u] if on_path[x] and x != p]
        on_path[u] = 1
        cnt = {x: sum(on_path[y] for y in nbrs[x]) for x in nbrs[u]}
        stack.append([u, sorted(nbrs[u], key=lambda x: -cnt[x]), 0])

    # the root of each component: the remaining variable with most neighbours, last among ties
    for r in sorted(range(V), key=lambda v: (-len(nbrs[v]), -v)):
        if in_tree[r]:
            continue
        roots.append(r)
        stack = []
        enter(r, -1, stack)
        while stack:
            top = stack[-1]
            u, lst, i = top
            if i == len(lst):
                stack.pop()
                on_path[u] = 0
                continue
            top[2] = i + 1
            x = lst[i]
            if x == parent[u]:
                continue
            if on_path[x]:                 # pseudo-parent: the token tells it about its pseudo-child
                pchildren[x].append(u)
                continue
            if in_tree[x]:                 # a descendant that already reached u
                continue
            children[u].append(x)
            enter(x, u, stack)
    t = PseudoTree(V, np.array(parent, dtype=np.int32), children, pparents, pchildren, roots)
    return complete(t, dom_size, scopes)


def tree_from_links(var_names, links, dom_size, factor_ptr, edge_var, con_order=None) -> PseudoTree:
    """The tree the orchestrator built: `links[name]` lists (type, target) of that node's
    PseudoTreeLinks in their order (pseudotree.py:412-433).  `con_order[u]` (optional): the constraint
    indices of node u in its `node.constraints` order, the order DpopAlgo joins the ones it owns in
    (dpop.py:191-199, :381-382); default: constraint index order.  The roots come in the order
    build_computation_graph builds the components: most neighbours first, the later variable first among
    ties (:353-354)."""
    V = len(var_names)
    idx = {n: i for i, n in enumerate(var_names)}
    parent = np.full(V, -1, dtype=np.int32)
    children = [[] for _ in range(V)]
    pparents = [[] for _ in range(V)]
    pchildren = [[] for _ in range(V)]
    for n, lst in links.items():
        u = idx[n]
        for kind, target in lst:
            t = idx[target]
            if kind == "parent":
                parent[u] = t
            elif kind == "children":
                children[u].append(t)
            elif kind == "pseudo_parent":
                pparents[u].append(t)
            elif kind == "pseudo_children":
                pchildren[u].append(t)
    roots = sorted((u for u in range(V) if parent[u] < 0),
                   key=lambda u: (-(len(children[u]) + len(pchildren[u])), -u))
    t = PseudoTree(V, parent, children, pparents, pchildren, roots)
    return complete(t, dom_size, _scopes(factor_ptr, edge_var), con_order)


def complete(t: PseudoTree, dom_size, scopes, con_order=None) -> PseudoTree:
    """Depths, constraint owners (deepest scope variable) and the constraints each node owns (in
    con_order[u] order when given, else constraint order), separators and UTIL sizes."""
    V = t.n_vars
    order = t.preorder()
    if len(order) != V:
        raise ValueError("the pseudo-tree does not cover every variable exactly once")
    depth = [0] * V
    for u in order:
        for c in t.children[u]:
            depth[c] = depth[u] + 1
    owned = [[] for _ in range(V)]
    owner = np.zeros(len(scopes), dtype=np.int32)
    for f, s in enumerate(scopes):
        o = max(s, key=lambda v: depth[v])
        owner[f] = o
        owned[o].append(f)
    if con_order is not None:
        for u in range(V):
            rank = {f: i for i, f in enumerate(con_order[u])}
            owned[u].sort(key=lambda f: rank[f])
    dom = np.asarray(dom_size, dtype=np.int64).tolist()
    sep_sets = [None] * V
    for u in reversed(order):
        s = set()
        for c in t.children[u]:
            s |= sep_sets[c]
        for f in owned[u]:
            s.update(scopes[f])
        s.discard(u)
        sep_sets[u] = s
    sep, util = [], []
    for u in range(V):
        lst = sorted(sep_sets[u], key=lambda v: depth[v])
        sz = 1
        for v in lst:
            sz *= dom[v]
        sep.append(lst)
        util.append(sz)
    t.depth = np.array(depth, dtype=np.int32)
    t.owner = owner
    t.sep = sep
    t.util_size = util
    t.owned = owned
    return t


def heavy_paths(t: PseudoTree):
    """Heavy/light decomposition: the heavy child is the one with the largest subtree (first in
    children order among ties).  Returns (paths top-down, light depth of each path)."""
    V = t.n_vars
    order = t.preorder()
    size = [1] * V
    for u in reversed(order):
        for c in t.children[u]:
            size[u] += size[c]
    heavy = [-1] * V
    for u in range(V):
        best = -1
        for c in t.children[u]:
            if best < 0 or size[c] > size[best]:
                best = c
        heavy[u] = best
    paths, ldepth = [], []
    head_ld = [(r, 0) for r in reversed(t.roots)]
    while head_ld:
        h, ld = head_ld.pop()
        path = []
        u = h
        while u >= 0:
            path.append(u)
            for c in t.children[u]:
                if c != heavy[u]:
                    head_ld.append((c, ld + 1))
            u = heavy[u]
        paths.append(path)
        ldepth.append(ld)
    return paths, ldepth


@dataclass
class Schedule:
    util_nodes: np.ndarray        # int32: nodes of every UTIL segment, bottom-up
    util_seg_ptr: np.ndarray      # int32 [n_util_segs + 1]
    value_nodes: np.ndarray       # int32: nodes of every heavy path, top-down
    value_seg_ptr: np.ndarray     # int32 [n_paths + 1]
    util_launches: list           # (kind, first, count): kind 0 = warp walk over segments, 1 = big node
    value_launches: list          # (0, first path, count) per round
    rounds: int
    big_nodes: list

    @property
    def n_launches(self):
        return len(self.util_launches) + len(self.value_launches)


def schedule(t: PseudoTree) -> Schedule:
    """UTIL runs in rounds from the largest light depth to 0; in a round one warp walks each heavy-path
    segment from the bottom up.  A big node cuts its path: the segments below it, then the node on the
    whole grid, then the part above.  VALUE runs the same rounds top down, one warp per whole path."""
    paths, ldepth = heavy_paths(t)
    rounds = max(ldepth, default=-1) + 1
    by_round = [[] for _ in range(rounds)]
    for p, ld in zip(paths, ldepth):
        by_round[ld].append(p)
    util_nodes, util_ptr, util_launches, big = [], [0], [], []
    for ld in range(rounds - 1, -1, -1):
        pieces = []                      # per path: [seg, big, seg, big, ..., seg]
        for p in by_round[ld]:
            cur, pc = [], []
            for u in reversed(p):
                if t.util_size[u] > BIG_UTIL:
                    pc += [cur, u]
                    cur = []
                else:
                    cur.append(u)
            pc.append(cur)
            pieces.append(pc)
        for k in range(0, max(len(pc) for pc in pieces), 2):
            segs = [pc[k] for pc in pieces if k < len(pc) and pc[k]]
            if segs:
                util_launches.append((0, len(util_ptr) - 1, len(segs)))
                for s in segs:
                    util_nodes += s
                    util_ptr.append(len(util_nodes))
            for b in (pc[k + 1] for pc in pieces if k + 1 < len(pc)):
                util_launches.append((1, b, 1))
                big.append(b)
    value_nodes, value_ptr, value_launches = [], [0], []
    for ld in range(rounds):
        value_launches.append((0, len(value_ptr) - 1, len(by_round[ld])))
        for p in by_round[ld]:
            value_nodes += p
            value_ptr.append(len(value_nodes))
    i32 = lambda a: np.asarray(a, dtype=np.int32)  # noqa: E731
    return Schedule(i32(util_nodes), i32(util_ptr), i32(value_nodes), i32(value_ptr), util_launches,
                    value_launches, rounds, big)


def arena_layout(t: PseudoTree):
    """Start of every node's UTIL in the arena and the arena's size in entries (Python ints)."""
    off, n = [], 0
    for s in t.util_size:
        off.append(n)
        n += s
    return off, n


def largest_separator(t: PseudoTree):
    u = max(range(t.n_vars), key=lambda v: t.util_size[v]) if t.n_vars else -1
    return u, (t.sep[u] if u >= 0 else [])


def canonical_factor_ptr(layout):
    """factor_ptr of the caller's (canonical) constraint order, from the layout's classes."""
    arity_int = np.zeros(layout.n_factors, dtype=np.int64)
    for c in layout.classes:
        arity_int[c.first_factor:c.first_factor + c.n_factors] = c.arity
    fp = np.zeros(layout.n_factors + 1, dtype=np.int64)
    np.cumsum(arity_int[layout.factor_perm], out=fp[1:])
    return fp


def terms(t: PseudoTree, layout):
    """Per-node descriptors of csrc/dpop_kernels.cuh, canonical variable order.  The terms of node u
    are, in summation order after its own cost row: each child's UTIL in children order (kind 0, in the
    arena), then each constraint u owns in constraint order (kind 1, in the layout's class-major
    tables).  A term's offset is base + own value * own stride + sum over (separator position, stride)."""
    L = layout
    V = t.n_vars
    dom = L.canon_dom_size.astype(np.int64).tolist()
    fp = canonical_factor_ptr(L).tolist()
    ev = L.canon_edge_var.tolist()
    cls_of = {}
    for c in L.classes:
        cls_of.update({fi: c for fi in range(c.first_factor, c.first_factor + c.n_factors)})
    fperm = L.factor_perm.tolist()
    util_off, arena = arena_layout(t)
    owned = t.owned
    sep_ptr, sep_var = [0], []
    term_ptr, kind, base, own = [0], [], [], []
    tdim_ptr, tdim_pos, tdim_stride = [0], [], []

    def add(u, pos, b, k, scope):
        o = 0
        st = [1] * len(scope)
        for j in range(len(scope) - 2, -1, -1):
            st[j] = st[j + 1] * dom[scope[j + 1]]
        for w, s in zip(scope, st):
            if w == u:
                o += s
            else:
                tdim_pos.append(pos[w])
                tdim_stride.append(s)
        kind.append(k)
        base.append(b)
        own.append(o)
        tdim_ptr.append(len(tdim_pos))

    for u in range(V):
        pos = {w: i for i, w in enumerate(t.sep[u])}
        sep_var += t.sep[u]
        sep_ptr.append(len(sep_var))
        for c in t.children[u]:
            add(u, pos, util_off[c], 0, t.sep[c])
        for f in owned[u]:
            fi = fperm[f]
            c = cls_of[fi]
            add(u, pos, c.table_base + (fi - c.first_factor) * c.table_size, 1, ev[fp[f]:fp[f + 1]])
        term_ptr.append(len(kind))
    i32 = lambda a: np.asarray(a, dtype=np.int32)  # noqa: E731
    i64 = lambda a: np.asarray(a, dtype=np.int64)  # noqa: E731
    return dict(dom_size=i32(dom), unary_off=i64(L.unary_off[:-1][L.var_perm]) if V else i64([]),
                util_off=i64(util_off), util_size=i64(t.util_size), arena_size=arena,
                sep_ptr=i32(sep_ptr), sep_var=i32(sep_var), term_ptr=i32(term_ptr), term_kind=i32(kind),
                term_base=i64(base), term_own=i64(own), tdim_ptr=i32(tdim_ptr), tdim_pos=i32(tdim_pos),
                tdim_stride=i64(tdim_stride))
