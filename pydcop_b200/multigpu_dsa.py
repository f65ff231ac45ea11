"""Multi-GPU DSA: variables split over the GPUs of one box, one process per GPU, one exchange of
boundary VALUES per cycle (SURVEY.md §8e for the DSA half of the path).

DSA's only inter-variable traffic is the value message (dsa.py:297-299,339-357: every variable
posts its value to its neighbours each cycle).  Partition = the MaxSum one (`variable_owner`:
contiguous blocks).  Each rank builds a CLOSED local problem so the single-GPU engine runs
unchanged:
  * the variables it owns, with ALL their constraints (so costs, `p_mode=arity` counts and the
    variant-B violation test see exactly what the single-GPU run sees);
  * a GHOST variable for every remote variable in the scope of one of those constraints.  Ghosts
    are frozen (`DsaEngine(frozen=…)`: the local kernels never write them) and their value is
    supplied by the owner every cycle.
Random draws are keyed by the GLOBAL variable id (`DsaEngine(var_global_id=…)`), so the sharded
trajectory equals the single-GPU trajectory bit for bit, for any world size.

Per cycle: compute (writes the `next` value buffer) -> pack the boundary values (CUDA kernel
fg_halo_pack, rows of one 4-byte element) -> ONE all_to_all over NCCL/NVLink -> unpack into the
ghosts of `next` -> commit.  This replaces Messaging.post_msg for the value messages that cross
ranks (pydcop/infrastructure/communication.py:588-698).
"""
import ctypes as C
from dataclasses import dataclass
from typing import Dict, List

import numpy as np

from .layout import FactorGraphLayout, build_layout, default_var_csr, var_con_to_edges
from .multigpu import _ranges, resolve_owner


@dataclass
class DsaShard:
    rank: int
    world: int
    inst: Dict[str, np.ndarray]     # closed local instance (front-door arrays, local ids)
    layout: FactorGraphLayout
    own_vars: np.ndarray            # global ids of the owned variables (ascending) = local 0..n_own-1
    n_own_vars: int
    local_global_id: np.ndarray     # global id of every local variable (owned, then ghosts)
    frozen: np.ndarray              # bool per local variable: ghost
    send_var: np.ndarray            # local ids whose value goes out, grouped by peer, ascending global id
    recv_var: np.ndarray            # local ghost ids filled by the peers, grouped by peer
    send_split: List[int]
    recv_split: List[int]
    n_boundary: int                 # (variable, remote rank) pairs over the whole job


def boundary_pairs(edge_var, factor_ptr, owner_v):
    """All (variable u, rank r) with r != owner(u) such that a variable owned by r shares a
    constraint with u — u is a ghost on r.  Sorted by (r, u), unique."""
    F = len(factor_ptr) - 1
    arity = np.diff(factor_ptr)
    if not F or not len(edge_var):
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    efac = np.repeat(np.arange(F, dtype=np.int64), arity)
    e0 = factor_ptr[:-1][efac]
    ea = arity[efac]
    us, rs = [], []
    for j in range(int(arity.max())):
        m = ea > j
        u = edge_var[m]
        r = owner_v[edge_var[(e0 + j)[m]]].astype(np.int64)
        keep = r != owner_v[u]
        us.append(u[keep])
        rs.append(r[keep])
    u, r = np.concatenate(us), np.concatenate(rs)
    if not len(u):
        return u, r
    key = np.unique(r * (int(owner_v.shape[0]) + 1) + u)
    return key % (int(owner_v.shape[0]) + 1), key // (int(owner_v.shape[0]) + 1)


def build_dsa_shard(inst: Dict[str, np.ndarray], rank: int, world: int, partition="blocks") -> DsaShard:
    dom_size = np.asarray(inst["dom_size"], dtype=np.int32)
    factor_ptr = np.asarray(inst["factor_ptr"], dtype=np.int64)
    edge_var = np.asarray(inst["edge_var"], dtype=np.int64)
    tables = np.asarray(inst["tables"])
    V, F = len(dom_size), len(factor_ptr) - 1
    arity = np.diff(factor_ptr)
    efac = np.repeat(np.arange(F, dtype=np.int64), arity)
    tsize = np.ones(F, dtype=np.int64)
    np.multiply.at(tsize, efac, dom_size[edge_var].astype(np.int64))
    table_off = np.zeros(F + 1, dtype=np.int64)
    np.cumsum(tsize, out=table_off[1:])
    unary = (np.asarray(inst["unary"], dtype=np.float64) if inst.get("unary") is not None
             else np.zeros(int(dom_size.sum())))
    unary_off = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(dom_size, out=unary_off[1:])
    if inst.get("var_ptr") is not None and inst.get("var_edge") is not None:
        g_var_ptr = np.asarray(inst["var_ptr"], dtype=np.int64)
        g_var_edge = np.asarray(inst["var_edge"], dtype=np.int64)
    elif inst.get("var_ptr") is not None and inst.get("var_con") is not None:
        g_var_ptr = np.asarray(inst["var_ptr"], dtype=np.int64)
        g_var_edge = var_con_to_edges(inst).astype(np.int64)
    else:
        vp, ve = default_var_csr(V, edge_var)
        g_var_ptr, g_var_edge = vp.astype(np.int64), ve.astype(np.int64)

    owner_v = resolve_owner(inst, world, partition)
    own_v = np.nonzero(owner_v == rank)[0]
    n_own = len(own_v)
    # constraints with at least one owned variable, in global order
    touched = np.zeros(F, dtype=bool)
    touched[efac[owner_v[edge_var] == rank]] = True
    loc_f = np.nonzero(touched)[0]
    loc_edges = _ranges(factor_ptr[loc_f], arity[loc_f])
    scope_vars = edge_var[loc_edges] if len(loc_edges) else np.zeros(0, np.int64)
    ghosts = np.unique(scope_vars[owner_v[scope_vars] != rank]) if len(scope_vars) else np.zeros(0, np.int64)
    ghosts = ghosts[np.argsort(owner_v[ghosts], kind="stable")]     # one block of values per peer
    n_ghost = len(ghosts)
    local_global = np.concatenate([own_v, ghosts]).astype(np.int64)
    g2l_var = np.full(V, -1, dtype=np.int64)
    g2l_var[local_global] = np.arange(n_own + n_ghost)
    g2l_edge = np.full(len(edge_var), -1, dtype=np.int64)
    g2l_edge[loc_edges] = np.arange(len(loc_edges))

    l_factor_ptr = np.zeros(len(loc_f) + 1, dtype=np.int64)
    np.cumsum(arity[loc_f], out=l_factor_ptr[1:])
    l_edge_var = g2l_var[scope_vars].astype(np.int32)
    l_tables = tables[_ranges(table_off[loc_f], tsize[loc_f])] if len(loc_f) else tables[:0]
    l_table_off = np.zeros(len(loc_f) + 1, dtype=np.int64)
    np.cumsum(tsize[loc_f], out=l_table_off[1:])
    l_dom = dom_size[local_global].astype(np.int32)
    l_unary = unary[_ranges(unary_off[local_global], dom_size[local_global].astype(np.int64))] \
        if len(local_global) else unary[:0]
    # incident edges: owned variables keep their `node.constraints` order (dsa.py:255); a ghost
    # lists its local edges in ascending order (it is never evaluated)
    own_deg = (g_var_ptr[own_v + 1] - g_var_ptr[own_v]) if n_own else np.zeros(0, np.int64)
    own_inc = g2l_edge[g_var_edge[_ranges(g_var_ptr[own_v], own_deg)]] if n_own else np.zeros(0, np.int64)
    if len(own_inc) and (own_inc < 0).any():
        raise AssertionError("an owned variable's constraint is missing from the shard")
    l_edge_ids = np.arange(len(l_edge_var), dtype=np.int64)
    ghost_edge_mask = l_edge_var >= n_own
    g_edges = l_edge_ids[ghost_edge_mask]
    g_order = np.argsort(l_edge_var[ghost_edge_mask], kind="stable")
    ghost_inc = g_edges[g_order]
    ghost_deg = np.bincount(l_edge_var[ghost_edge_mask] - n_own, minlength=n_ghost) if n_ghost \
        else np.zeros(0, np.int64)
    l_var_ptr = np.zeros(n_own + n_ghost + 1, dtype=np.int32)
    np.cumsum(np.concatenate([own_deg, ghost_deg]), out=l_var_ptr[1:])
    l_var_edge = np.concatenate([own_inc, ghost_inc]).astype(np.int32)
    local = dict(dom_size=l_dom, factor_ptr=l_factor_ptr, edge_var=l_edge_var, tables=l_tables,
                 table_off=l_table_off, unary=l_unary, var_ptr=l_var_ptr, var_edge=l_var_edge)
    layout = build_layout(**local)

    u, r = boundary_pairs(edge_var, factor_ptr, owner_v)
    ou = owner_v[u] if len(u) else np.zeros(0, np.int32)
    send_var, recv_var, send_split, recv_split = [], [], [], []
    for p in range(world):
        s = u[(ou == rank) & (r == p)]        # my variables that rank p holds as ghosts
        g = u[(r == rank) & (ou == p)]        # my ghosts owned by rank p (same order on p's side)
        send_var.append(g2l_var[s])
        recv_var.append(g2l_var[g])
        send_split.append(len(s))
        recv_split.append(len(g))
    send_var = np.concatenate(send_var).astype(np.int64) if world else np.zeros(0, np.int64)
    recv_var = np.concatenate(recv_var).astype(np.int64) if world else np.zeros(0, np.int64)
    if (send_var < 0).any() or (recv_var < 0).any() or sorted(recv_var.tolist()) != list(range(n_own, n_own + n_ghost)):
        raise AssertionError("halo lists do not cover the ghosts")
    frozen = np.zeros(n_own + n_ghost, dtype=bool)
    frozen[n_own:] = True
    return DsaShard(rank=rank, world=world, inst=local, layout=layout, own_vars=own_v, n_own_vars=n_own,
                    local_global_id=local_global, frozen=frozen, send_var=send_var, recv_var=recv_var,
                    send_split=send_split, recv_split=recv_split, n_boundary=len(u))


class ValueHalo:
    """Boundary values: pack -> ONE all_to_all -> unpack.  `pack(src, packed, row_off, packed_off,
    row_len, n)` / `unpack(dst, packed, …)` are injected: the product passes the CUDA kernels behind
    fg_halo_pack / fg_halo_unpack (a value is a row of one 4-byte element, moved bit for bit); the
    CPU (gloo) tests pass index-based stand-ins."""

    def __init__(self, shard: DsaShard, layout: FactorGraphLayout, device, pack, unpack, group=None):
        import torch
        self.torch, self.shard, self.pack, self.unpack, self.group = torch, shard, pack, unpack, group

        def dv(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dt)

        perm = np.asarray(layout.var_perm, dtype=np.int64)     # canonical local id -> internal id
        ns, nr = len(shard.send_var), len(shard.recv_var)
        self.n_send, self.n_recv = ns, nr
        self.send = (dv(perm[shard.send_var], torch.int64), dv(np.arange(ns), torch.int64),
                     dv(np.ones(ns), torch.int32))
        self.recv = (dv(perm[shard.recv_var], torch.int64), dv(np.arange(nr), torch.int64),
                     dv(np.ones(nr), torch.int32))
        self.buf_send = torch.zeros(max(ns, 1), dtype=torch.int32, device=device)
        self.buf_recv = torch.zeros(max(nr, 1), dtype=torch.int32, device=device)
        self.send_split, self.recv_split = list(shard.send_split), list(shard.recv_split)
        self.launches = 0

    def pack_values(self, values):
        if self.n_send:
            self.pack(values, self.buf_send, *self.send, self.n_send)
            self.launches += 1

    def unpack_values(self, values):
        if self.n_recv:
            self.unpack(values, self.buf_recv, *self.recv, self.n_recv)
            self.launches += 1

    def exchange(self, values):
        import torch.distributed as dist
        self.pack_values(values)
        dist.all_to_all_single(self.buf_recv[:self.n_recv], self.buf_send[:self.n_send],
                               self.recv_split, self.send_split, group=self.group)
        self.unpack_values(values)


def value_push_tables(shard: DsaShard, base: np.ndarray, dst_idx):
    """Source indices (internal variable order) and absolute destination addresses of the value
    push.  base[rank] = addresses of that rank's two value buffers as mapped into this process;
    dst_idx = the consumers' internal ghost indices of my send list (my send order).  Issued in
    destination order inside each peer group, like multigpu.push_tables."""
    from .multigpu import destination_order
    perm = np.asarray(shard.layout.var_perm, dtype=np.int64)
    dst_idx = np.asarray(dst_idx, dtype=np.int64)
    peer_of = np.repeat(np.arange(shard.world), np.asarray(shard.send_split, dtype=np.int64))
    order = destination_order(dst_idx, shard.send_split)
    return dict(dst=[(base[peer_of, b] + dst_idx * 4)[order] for b in range(2)],
                src=perm[shard.send_var][order])


class ValuePeerPush:
    """Boundary values over NVLink peer memory, the DSA twin of multigpu.PeerPush: every rank maps
    the peers' two value buffers (CUDA IPC) and ONE push kernel (rows of one 4-byte element) stores
    each boundary value straight into the ghost entry of the consumer's `next` buffer; the cycle is
    closed by the device-side epoch barrier (pydcop_b200/peer.py).  Ghost entries are written ONLY by
    their owner's push (the local kernels skip them, has_nbr == 2), so a fast rank's push cannot be
    overwritten by a slow rank's own kernel.  Whole cycles are enqueued by fg_dsa_shard_step."""

    def __init__(self, sharded, group=None):
        import torch
        import torch.distributed as dist
        from . import _cabi
        from .peer import PeerMap, PeerSync
        self.torch, self.dist, self.group = torch, dist, group
        e, sh = sharded.engine, sharded.shard
        self.engine = e
        dev = e.device
        W, me = sh.world, sh.rank
        self.pmap = PeerMap(e.lib, dev, me, W, group)
        base = self.pmap.map([e.value[0], e.value[1]])
        # where my values land: the consumers' ghost indices (internal order), in my send order
        perm = np.asarray(sh.layout.var_perm, dtype=np.int64)
        out = torch.zeros(len(sh.send_var), dtype=torch.int64, device=dev)
        inp = torch.from_numpy(np.ascontiguousarray(perm[sh.recv_var])).to(dev)
        dist.all_to_all_single(out, inp, list(sh.send_split), list(sh.recv_split), group=group)
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)  # noqa: E731
        t = value_push_tables(sh, base, out.cpu().numpy())
        self.dst, self.src = [to(a) for a in t["dst"]], to(t["src"])
        self.n = len(sh.send_var)
        peers = [b for b in range(W) if b != me and (sh.send_split[b] or sh.recv_split[b])]
        self.sync = PeerSync(self.pmap, peers)
        plan = _cabi.FgHaloPlan()
        plan.elem_bytes, plan.dom, plan.n_r, plan.n_q = 4, 1, self.n, 0
        plan.dev_src_r_off = self.src.data_ptr()
        for b in range(2):
            plan.dev_dst_r[b] = self.dst[b].data_ptr()
        plan.dev_counter = self.sync.counter.data_ptr()
        plan.sync = self.sync.struct
        self._plan = plan
        rc = e.lib.fg_dsa_shard_attach(e._h, C.byref(plan))
        if rc != 0:
            raise RuntimeError(f"fg_dsa_shard_attach failed rc={rc}: {e._last_error()}")
        self.launches = 0      # counted inside the engine handle
        dist.barrier(group=group)

    def step(self, n_cycles):
        e, torch = self.engine, self.torch
        with torch.cuda.device(e.device):
            rc = e.lib.fg_dsa_shard_step(e._h, int(n_cycles),
                                         C.c_void_p(torch.cuda.current_stream(e.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"fg_dsa_shard_step failed rc={rc}: {e._last_error()}")


class ShardResults:
    """The whole problem's results from one rank of a sharded local search (ShardedDsa, ShardedMgm2): subclasses
    provide shard, engine, torch, device, global_n_vars, global_dom_size, group, local_values() and _value_tensor()
    (the current values, internal order, on the engine's device)."""

    def solution_cost(self, infinity=float("inf"), unary=None):
        """(cost, violations) of the whole problem's current assignment.  A DSA shard keeps ALL constraints of
        its variables, so a cut constraint lives on several ranks: a rank counts a constraint only if it
        owns the constraint's FIRST scope variable (the MaxSum ownership rule) and a variable cost only for
        the variables it owns; it reduces on its device and the ranks all-reduce the two sums
        (pydcop/dcop/dcop.py:319-367)."""
        import torch.distributed as dist
        sh, e, torch = self.shard, self.engine, self.torch
        L = sh.layout
        if not hasattr(self, "_cost_masks"):
            ghost_internal = np.zeros(L.n_vars, dtype=np.uint8)
            ghost_internal[L.var_perm[np.nonzero(sh.frozen)[0]]] = 1
            first_e = (np.concatenate([c.first_edge + np.arange(c.n_factors, dtype=np.int64) * c.arity
                                       for c in L.classes]) if L.n_factors else np.zeros(0, np.int64))
            fskip = ghost_internal[L.edge_var[first_e]] if L.n_factors else np.zeros(1, np.uint8)
            self._cost_masks = (torch.from_numpy(np.ascontiguousarray(fskip, dtype=np.uint8)).to(e.device),
                                torch.from_numpy(ghost_internal).to(e.device))
        local_unary = None
        if unary is not None:
            dom = np.asarray(self.global_dom_size, dtype=np.int64)
            uoff = np.concatenate([[0], np.cumsum(dom)])
            gid = sh.local_global_id
            local_unary = np.asarray(unary, dtype=np.float64)[_ranges(uoff[gid], dom[gid])]
        out = e._solution_cost(self._value_tensor(), infinity, local_unary, factor_skip=self._cost_masks[0],
                               var_skip=self._cost_masks[1])
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.group)
        o = out.cpu().numpy()
        return float(o[0]), int(round(o[1]))

    def values(self):
        """All-gathered assignment in global variable order (every rank gets the full vector)."""
        import torch.distributed as dist
        torch = self.torch
        ids, val = self.local_values()
        out = torch.zeros(self.global_n_vars, dtype=torch.int32, device=self.device)
        if len(ids):
            out[torch.from_numpy(np.asarray(ids)).to(self.device)] = \
                torch.from_numpy(val.astype(np.int32)).to(self.device)
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.group)
        return out.cpu().numpy()


class ShardedDsa(ShardResults):
    """One rank of the partitioned DSA: same driving API as DsaEngine (init / step / values).

    `engine_factory(layout, inst=local arrays, **kwargs)` and `pack` / `unpack` exist so the partition and exchange
    logic can run on CPU under gloo in the tests; the product path leaves them at None and gets
    DsaEngine + the CUDA halo kernels."""

    def __init__(self, inst, rank, world, device, precision="f32", group=None, engine_factory=None,
                 pack=None, unpack=None, partition="blocks", halo="nccl", **params):
        import torch
        self.torch = torch
        self.shard = sh = build_dsa_shard(inst, rank, world, partition)
        self.rank, self.world = rank, world
        self.global_n_vars = int(len(np.asarray(inst["dom_size"])))
        self.global_dom_size = np.asarray(inst["dom_size"], dtype=np.int32)
        iso = params.pop("isolated_value", None)
        if iso is not None:
            iso = np.asarray(iso, dtype=np.int32)[sh.local_global_id]
        kwargs = dict(precision=precision, var_global_id=sh.local_global_id.astype(np.int32),
                      frozen=sh.frozen, isolated_value=iso, **params)
        if engine_factory is not None:
            self.engine = engine_factory(sh.layout, inst=sh.inst, **kwargs)
            self.device = torch.device(device) if device is not None else torch.device("cpu")
        else:
            from . import _cabi
            from .engine import DsaEngine
            self.engine = DsaEngine(sh.layout, device=device, **kwargs)
            self.device = self.engine.device
            lib = self.engine.lib

            def stream():
                return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

            # the halo kernels run on the current device: make it the shard's (shards of one process may be on several)
            def mover(fn, name):
                def move(buf, packed, row_off, packed_off, row_len, n):
                    with torch.cuda.device(self.device):
                        rc = fn(_cabi.FG_F32, C.c_void_p(buf.data_ptr()), C.c_void_p(packed.data_ptr()),
                                C.c_void_p(row_off.data_ptr()), C.c_void_p(packed_off.data_ptr()),
                                C.c_void_p(row_len.data_ptr()), n, stream())
                    if rc != _cabi.FG_OK:
                        raise _cabi.EngineError(f"{name} failed rc={rc}")
                return move

            pack, unpack = mover(lib.fg_halo_pack, "fg_halo_pack"), mover(lib.fg_halo_unpack, "fg_halo_unpack")
        self.halo = ValueHalo(sh, sh.layout, self.device, pack, unpack, group)
        self.halo_mode = halo if engine_factory is None else "nccl"
        self.peer = None

    @property
    def layout(self):
        return self.shard.layout

    def init(self):
        e = self.engine
        e.init()
        self.halo.exchange(e.value[e.cur])       # ghosts learn their owners' initial values
        if self.halo_mode in ("p2p", "auto") and self.peer is None and self.world > 1:
            try:
                self.peer = ValuePeerPush(self, self.halo.group)
            except Exception as ex:  # noqa: BLE001 — no peer mapping: keep the NCCL exchange
                if self.halo_mode == "p2p":
                    raise
                self.peer_error = repr(ex)
        return self

    def step(self, n_cycles=1):
        e = self.engine
        if self.peer is not None:       # whole cycles enqueued by one C call, closed on the device
            self.peer.step(n_cycles)
            return self
        for _ in range(int(n_cycles)):
            before = e.cycle
            e.cycle_compute()
            self.halo.exchange(e.value[e.cur ^ 1])
            e.cycle_commit()
            if e.cycle == before:                 # stop_cycle reached: nothing moves any more
                break
        return self

    @property
    def cycle(self):
        return self.engine.cycle

    @property
    def launch_count(self):
        return self.engine.launch_count + self.halo.launches

    def check(self):
        """Raise if the device-side barrier timed out (synchronises the device)."""
        if self.peer is not None:
            self.peer.sync.check()

    def local_values(self):
        """(global variable ids, value indices) of the variables this rank owns."""
        val = self.engine.values()
        return self.shard.own_vars, np.asarray(val)[:self.shard.n_own_vars]

    def _value_tensor(self):
        e = self.engine
        return e.value[e.cur]

    @property
    def group(self):
        return self.halo.group
