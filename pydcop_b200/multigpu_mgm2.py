"""Multi-GPU MGM-2: variables split over the GPUs of one box, one process per GPU, five boundary exchanges per
cycle (DESIGN.md §6).

Each rank builds the closed local problem of multigpu_dsa.build_dsa_shard: the variables it owns with all their
constraints, in `node.constraints` order, plus a GHOST for every remote variable in their scopes.  The phase kernels
run on the owned variables only (csrc/mgm2_shard_kernels.cuh); draws are keyed by the GLOBAL variable id and ties are
broken on the GLOBAL name rank, so the sharded trajectory equals the single-GPU one bit for bit.  MGM-2 moves data
between neighbours at five points of a cycle (owner A, a rank B that holds the variable as a ghost):

  0 offers   A -> B after the value phase: offerer flag, partner (B's id of it when B owns it, else -1) and the
             first dom(u) x (max dom of u's neighbours owned by B) entries of the offer table: all B's receivers read
  1 answers  B -> A after the answer phase: the joint move B's receiver accepted for A's offerer (at most one rank
             holds the partner, so at most one answer per offerer), merged into A's flags
  2 gains    A -> B after the commit phase
  3 go       A -> B after the gain phase
  4 values   A -> B after the go phase (and after init)

Each exchange is pack -> transport -> unpack.  The transport is one NCCL all_to_all (halo='nccl'), or NVLink stores
into the peers' receive buffers closed by the device-side epoch barrier of pydcop_b200/peer.py (halo='p2p'; one C call
enqueues whole cycles, fg_mgm2_shard_step).
"""
from dataclasses import dataclass
from typing import Dict, List

import numpy as np

from .layout import FactorGraphLayout
from .multigpu import _ranges, resolve_owner
from .multigpu_dsa import DsaShard, ShardResults, build_dsa_shard

EXCHANGES = 5
OFFERS, ANSWERS, GAINS, GO, VALUES = range(EXCHANGES)


def canonical_neighbours(inst, variables):
    """Distinct neighbours of each of `variables` (global ids) in the WHOLE problem, in first-appearance order over
    the variable's constraints (var_ptr / var_edge order, then scope order): the order of
    engine.distinct_neighbours, in global ids.  Returns a list of arrays."""
    factor_ptr = np.asarray(inst["factor_ptr"], dtype=np.int64)
    edge_var = np.asarray(inst["edge_var"], dtype=np.int64)
    var_ptr = np.asarray(inst["var_ptr"], dtype=np.int64)
    var_edge = np.asarray(inst["var_edge"], dtype=np.int64)
    variables = np.asarray(variables, dtype=np.int64)
    arity = np.diff(factor_ptr)
    efac = np.repeat(np.arange(len(arity), dtype=np.int64), arity)
    deg = var_ptr[variables + 1] - var_ptr[variables]
    slots = _ranges(var_ptr[variables], deg)
    who = np.repeat(np.arange(len(variables), dtype=np.int64), deg)
    f = efac[var_edge[slots]] if len(slots) else np.zeros(0, np.int64)
    A = int(arity.max()) if len(arity) else 0
    vs, us, seqs = [], [], []
    for j in range(A):
        m = arity[f] > j
        u = edge_var[factor_ptr[f[m]] + j]
        keep = u != variables[who[m]]
        vs.append(who[m][keep])
        us.append(u[keep])
        seqs.append((slots[m] * A + j)[keep])
    out = [np.zeros(0, np.int64) for _ in variables]
    if not vs or not sum(len(v) for v in vs):
        return out
    v, u, seq = np.concatenate(vs), np.concatenate(us), np.concatenate(seqs)
    o = np.lexsort((seq, u, v))
    v, u, seq = v[o], u[o], seq[o]
    first = np.ones(len(v), dtype=bool)
    first[1:] = (v[1:] != v[:-1]) | (u[1:] != u[:-1])
    v, u, seq = v[first], u[first], seq[first]
    o = np.lexsort((seq, v))
    v, u = v[o], u[o]
    ptr = np.concatenate([[0], np.cumsum(np.bincount(v, minlength=len(variables)))])
    return [u[ptr[i]:ptr[i + 1]] for i in range(len(variables))]


@dataclass
class Mgm2Shard:
    rank: int
    world: int
    base: DsaShard                  # the closed local problem, ghosts and the (forward) boundary lists
    inst: Dict[str, np.ndarray]     # closed local instance (front-door arrays, local ids), with initial values
    layout: FactorGraphLayout
    own_vars: np.ndarray            # global ids of the owned variables = local 0..n_own-1
    n_own_vars: int
    local_global_id: np.ndarray     # global id of every local variable (canonical local order)
    frozen: np.ndarray              # bool per local variable (canonical): ghost
    var_rank: np.ndarray            # canonical local order: the GLOBAL name rank
    nbr_ptr: np.ndarray             # distinct-neighbour CSR of the local layout (internal ids)
    nbr_idx: np.ndarray
    ghost: np.ndarray               # uint8 per internal local id
    owner_rank: np.ndarray          # int32 per internal local id
    send_int: np.ndarray            # internal ids of the forward send list (grouped by peer)
    recv_int: np.ndarray            # internal ids of the forward receive list (ghosts, grouped by owner)
    send_split: List[int]           # entries per peer
    recv_split: List[int]
    send_peer: np.ndarray           # rank each forward send entry goes to
    send_plen: np.ndarray           # offer prefix (elements) of every forward send entry
    recv_plen: np.ndarray           # ... of every forward receive entry
    n_boundary: int

    def record_lengths(self, x):
        """(send, receive) record length per entry of exchange x, in elements of the run's precision."""
        ns, nr = len(self.send_int), len(self.recv_int)
        if x == OFFERS:
            return 1 + self.send_plen, 1 + self.recv_plen
        if x == ANSWERS:                 # the reverse direction: ghosts out, owned variables in
            return np.full(nr, 2, np.int64), np.full(ns, 2, np.int64)
        return np.ones(ns, np.int64), np.ones(nr, np.int64)

    def splits(self, x, lengths=True):
        """(send, receive) elements per peer of exchange x (entries per peer with lengths=False)."""
        ss, rs = (self.recv_split, self.send_split) if x == ANSWERS else (self.send_split, self.recv_split)
        if not lengths:
            return list(ss), list(rs)
        sl, rl = self.record_lengths(x)
        cut = lambda l, sp: [int(a.sum()) for a in np.split(l, np.cumsum(sp)[:-1])]  # noqa: E731
        return cut(sl, ss), cut(rl, rs)

    def plan_arrays(self, owner_local):
        """Host arrays of fg_mgm2_shard_plan_t (internal order).  owner_local: every local variable's internal id on
        its owner (ghost_owner_ids)."""
        xs = []
        for x in range(EXCHANGES):
            sv, rv = (self.recv_int, self.send_int) if x == ANSWERS else (self.send_int, self.recv_int)
            sl, rl = self.record_lengths(x)
            off = lambda l: np.concatenate([[0], np.cumsum(l)]).astype(np.int64)  # noqa: E731
            xs.append(dict(send_var=sv.astype(np.int32), send_off=off(sl), recv_var=rv.astype(np.int32),
                           recv_off=off(rl)))
        return dict(x=xs, ghost=self.ghost, send_peer=self.send_peer.astype(np.int32),
                    owner_rank=self.owner_rank.astype(np.int32), owner_local=np.asarray(owner_local, np.int32))

    def owner_local_ids(self, ghost_owner_ids):
        """Internal id of every local variable on its owner: its own for an owned variable; for the ghosts,
        `ghost_owner_ids` in forward receive order (what the owners send: their internal ids of their send lists)."""
        out = np.arange(self.layout.n_vars, dtype=np.int32)
        out[self.recv_int] = np.asarray(ghost_owner_ids, dtype=np.int32)
        return out


def build_mgm2_shard(inst: Dict[str, np.ndarray], rank: int, world: int, partition="blocks",
                     var_rank=None) -> Mgm2Shard:
    from .engine import mgm_host_arrays
    V = len(np.asarray(inst["dom_size"]))
    owner_v = resolve_owner(inst, world, partition)
    base = build_dsa_shard(inst, rank, world, owner_v)
    L = base.layout
    n_loc, n_own = L.n_vars, base.n_own_vars
    gid = base.local_global_id
    g_rank = np.arange(V, dtype=np.int32) if var_rank is None else np.asarray(var_rank, dtype=np.int32)
    loc_rank = g_rank[gid]
    h = mgm_host_arrays(L, var_rank=loc_rank)
    nbr_ptr, nbr_idx = h["nbr_ptr"], h["nbr_idx"]
    perm = np.asarray(L.var_perm, dtype=np.int64)
    order = np.asarray(L.var_order, dtype=np.int64)
    gid_int = gid[order]                                   # global id of every internal local id
    local_inst = dict(base.inst)
    if inst.get("init_value") is not None:   # MGM-2 starts from the initial values; the DSA shard has none
        local_inst["init_value"] = np.asarray(inst["init_value"], dtype=np.int32)[gid]
        L.init_value = local_inst["init_value"][order]
    # the partner pick nbr_idx[n0 + choice] must see the single-problem order
    full = dict(inst)
    if full.get("var_ptr") is None or full.get("var_edge") is None:
        from .layout import default_var_csr
        full["var_ptr"], full["var_edge"] = default_var_csr(V, np.asarray(inst["edge_var"]))
    want = canonical_neighbours(full, base.own_vars)
    for c, w in enumerate(want):
        i = perm[c]
        got = gid_int[nbr_idx[nbr_ptr[i]:nbr_ptr[i + 1]]]
        if not np.array_equal(got, w):
            raise AssertionError(f"variable {int(base.own_vars[c])}: shard neighbour order differs from the problem's")
    ghost = np.zeros(n_loc, dtype=np.uint8)
    ghost[perm[n_own:]] = 1
    owner_rank = owner_v[gid_int].astype(np.int32) if n_loc else np.zeros(0, np.int32)
    dom = L.dom_size.astype(np.int64)
    deg = np.diff(nbr_ptr).astype(np.int64)
    nb = nbr_idx[:int(nbr_ptr[-1])].astype(np.int64) if n_loc else np.zeros(0, np.int64)
    who = np.repeat(np.arange(n_loc, dtype=np.int64), deg)
    # slot capacity of every local variable (engine.mgm2_offer_offsets): dom x max dom of its local neighbours
    widest = np.zeros(n_loc, dtype=np.int64)
    np.maximum.at(widest, who, dom[nb])
    send_int, recv_int = perm[base.send_var], perm[base.recv_var]
    send_peer = np.repeat(np.arange(world), np.asarray(base.send_split, dtype=np.int64)).astype(np.int32)
    # offer prefix of (u, peer p): dom(u) x max dom of u's neighbours owned by p
    if len(send_int):
        key = who * world + owner_rank[nb]
        best = np.zeros(n_loc * world, dtype=np.int64)
        np.maximum.at(best, key, dom[nb])
        send_plen = dom[send_int] * best[send_int * world + send_peer]
    else:
        send_plen = np.zeros(0, np.int64)
    if len(recv_int):                                     # a ghost's neighbours owned here
        mine = ghost[nb] == 0
        best = np.zeros(n_loc, dtype=np.int64)
        np.maximum.at(best, who[mine], dom[nb[mine]])
        recv_plen = dom[recv_int] * best[recv_int]
    else:
        recv_plen = np.zeros(0, np.int64)
    if (send_plen > dom[send_int] * widest[send_int]).any() or (recv_plen > dom[recv_int] * widest[recv_int]).any():
        raise AssertionError("an offer prefix exceeds its offer slot")
    if (send_plen <= 0).any() or (recv_plen <= 0).any():
        raise AssertionError("a boundary variable has no neighbour on the rank that holds it")
    return Mgm2Shard(rank=rank, world=world, base=base, inst=local_inst, layout=L, own_vars=base.own_vars, n_own_vars=n_own,
                     local_global_id=gid, frozen=base.frozen, var_rank=loc_rank, nbr_ptr=nbr_ptr, nbr_idx=nbr_idx,
                     ghost=ghost, owner_rank=owner_rank, send_int=send_int, recv_int=recv_int,
                     send_split=list(base.send_split), recv_split=list(base.recv_split), send_peer=send_peer,
                     send_plen=send_plen, recv_plen=recv_plen, n_boundary=base.n_boundary)


class Mgm2PeerPush:
    """The five exchanges over NVLink peer memory: every rank maps the peers' receive buffers (CUDA IPC); per
    exchange one copy kernel stores each peer's block straight into the peer's buffer and its last block releases the
    next epoch; the rank then waits for the same epoch from every peer and unpacks (fg_mgm2_shard_step)."""

    def __init__(self, sharded, group=None):
        import torch
        import torch.distributed as dist
        from . import _cabi
        from .peer import PeerMap, PeerSync
        e, sh = sharded.engine, sharded.shard
        W, me = sh.world, sh.rank
        self.engine = e
        self.pmap = PeerMap(e.lib, e.device, me, W, group)
        base = self.pmap.map(e.recv_buf)                 # [world, exchange]
        # where each sender's block starts in my receive buffers
        recv_start = [np.concatenate([[0], np.cumsum(sh.splits(x)[1])])[:-1].astype(int).tolist()
                      for x in range(EXCHANGES)]
        starts = [None] * W
        dist.all_gather_object(starts, recv_start, group=group)
        esize = e.send_buf[0].element_size()
        peers = [b for b in range(W) if b != me and (sh.send_split[b] or sh.recv_split[b])]
        self.sync = PeerSync(self.pmap, peers)
        plan = _cabi.FgMgm2PeerPlan()
        for x in range(EXCHANGES):
            send = sh.splits(x)[0]
            src = np.concatenate([[0], np.cumsum(send)])
            k = 0
            for b in range(W):
                if b == me or not send[b]:
                    continue
                plan.src[x][k] = int(src[b])
                plan.n_elems[x][k] = int(send[b])
                plan.dst[x][k] = int(base[b, x]) + int(starts[b][x][me]) * esize
                k += 1
            plan.n_blocks[x] = k
        plan.dev_counter = self.sync.counter.data_ptr()
        plan.sync = self.sync.struct
        self._plan = plan
        e.shard_attach_peer(plan)
        torch.cuda.synchronize(e.device)
        dist.barrier(group=group)

    def step(self, n_cycles):
        self.engine.shard_step(n_cycles)


class ShardedMgm2(ShardResults):
    """One rank of the partitioned MGM-2: the driving API of ShardedDsa (init / step / values / local_values /
    solution_cost / check / launch_count).

    var_rank: the GLOBAL name ranks (canonical order), MGM-2's tie break.  halo: nccl | p2p | auto (p2p when the
    peers' memory can be mapped, else NCCL).  `engine_factory(layout, inst=local arrays, **kwargs)` exists so the
    partition and exchange logic can run on CPU under gloo in the tests (an engine with Mgm2Engine's shard_* surface);
    the product path leaves it at None and gets Mgm2Engine."""

    def __init__(self, inst, rank, world, device, precision="f32", group=None, engine_factory=None,
                 partition="blocks", halo="nccl", var_rank=None, **params):
        import torch
        self.torch, self.group_ = torch, group
        self.shard = sh = build_mgm2_shard(inst, rank, world, partition, var_rank)
        self.rank, self.world = rank, world
        self.global_n_vars = int(len(np.asarray(inst["dom_size"])))
        self.global_dom_size = np.asarray(inst["dom_size"], dtype=np.int32)
        kwargs = dict(precision=precision, var_global_id=sh.local_global_id.astype(np.int32), var_rank=sh.var_rank,
                      **params)
        if engine_factory is not None:
            self.engine = engine_factory(sh.layout, inst=sh.inst, **kwargs)
            self.device = torch.device(device) if device is not None else torch.device("cpu")
        else:
            from .engine import Mgm2Engine
            self.engine = Mgm2Engine(sh.layout, device=device, **kwargs)
            self.device = self.engine.device
        self.halo_mode = halo if engine_factory is None else "nccl"
        self.peer = None
        self.attached = False

    def attach(self, ghost_owner_ids=None):
        """Give the engine its shard plan.  ghost_owner_ids: the owners' internal ids of this rank's ghosts, in
        receive order; default: the owners send them over torch.distributed (with the offer prefix lengths they
        pack, which must equal what this rank unpacks).  init() attaches when this was not called."""
        sh = self.shard
        if ghost_owner_ids is None:
            send = np.stack([sh.send_int, sh.send_plen]).T.astype(np.int64)
            got = self._all_to_all(send, sh.send_split, sh.recv_split, 2)
            if not np.array_equal(got[:, 1], sh.recv_plen):
                raise AssertionError("offer prefix lengths differ between owner and holder")
            ghost_owner_ids = got[:, 0]
        self.engine.shard_attach(sh.plan_arrays(sh.owner_local_ids(ghost_owner_ids)))
        self.attached = True
        return self

    def _all_to_all(self, rows, send_split, recv_split, width):
        import torch.distributed as dist
        torch = self.torch
        out = torch.zeros((max(sum(recv_split), 0), width), dtype=torch.int64, device=self.device)
        inp = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.int64).reshape(-1, width)).to(self.device)
        dist.all_to_all_single(out, inp, list(recv_split), list(send_split), group=self.group)
        return out.cpu().numpy()

    @property
    def group(self):
        return self.group_

    @property
    def layout(self):
        return self.shard.layout

    def _exchange(self, x):
        """Transport exchange x over torch.distributed, then unpack it."""
        import torch.distributed as dist
        e = self.engine
        ss, rs = self.shard.splits(x)
        dist.all_to_all_single(e.recv_buf[x][:sum(rs)], e.send_buf[x][:sum(ss)], rs, ss, group=self.group)
        e.shard_unpack(x)

    def init(self):
        if not self.attached:
            self.attach()
        self.engine.shard_init()
        self._exchange(VALUES)                   # ghosts learn their owners' start values
        if self.halo_mode in ("p2p", "auto") and self.peer is None and self.world > 1:
            try:
                self.peer = Mgm2PeerPush(self, self.group)
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
            if e.finished:
                break
            for x in range(EXCHANGES):
                e.shard_phase(x)
                self._exchange(x)
        return self

    @property
    def cycle(self):
        return self.engine.cycle

    @property
    def finished(self):
        return self.engine.finished

    @property
    def launch_count(self):
        return self.engine.launch_count

    def check(self):
        """Raise if the device-side barrier timed out (synchronises the device)."""
        if self.peer is not None:
            self.peer.sync.check()

    def _value_tensor(self):
        return self.engine.value

    def local_values(self):
        """(global variable ids, value indices) of the variables this rank owns."""
        val = self.engine.values()[0]
        return self.shard.own_vars, np.asarray(val)[:self.shard.n_own_vars]

    def local_record(self):
        """(global ids, state of the last cycle) of the owned variables: value, cost, gain, committed, partner (a
        GLOBAL id, -1 for none) and go."""
        sh, e = self.shard, self.engine
        idx = np.asarray(sh.layout.var_perm, dtype=np.int64)[:sh.n_own_vars]
        host = lambda a: (a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a))[idx]  # noqa: E731
        partner = host(e.partner).astype(np.int64)
        gid_int = sh.local_global_id[np.asarray(sh.layout.var_order, dtype=np.int64)]
        out = dict(value=host(e.value), cost=host(e.cost), gain=host(e.gain), committed=host(e.committed),
                   partner=np.where(partner >= 0, gid_int[np.maximum(partner, 0)], -1), go=host(e.go))
        return sh.own_vars, out
