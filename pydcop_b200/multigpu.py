"""Multi-GPU MaxSum: the factor graph partitioned by VARIABLE CUT over the GPUs of one box, one
process per GPU, one halo exchange of boundary messages per cycle (SURVEY.md §8e).

Partition: variables are split into `world` contiguous blocks (row strips for a raster-ordered
grid); a factor lives with its first scope variable.  For a CUT edge (factor F on rank B, variable v
on rank A != B) the message r_{F->v} is produced on B and consumed on A, q_{v->F} the other way.

Each rank builds a CLOSED local graph so the single-GPU engine runs unchanged:
  * its own factors and its own variables;
  * a GHOST VARIABLE for every remote variable in the scope of an own factor — its slots are
    exactly the q rows that arrive from the owner;
  * a unary GHOST STUB FACTOR on the own variable for every remote factor touching it — its r row
    is exactly the row that arrives from the factor's owner, and it keeps the variable's true
    degree and `links` order (maxsum.py:466), so sums are bit-identical to the single-GPU run.
Ghost classes carry FG_CLASS_GHOST: their rows exist but are never computed, only filled by the
exchange.  Per cycle: compute (writes the `next` buffers) -> pack boundary rows (CUDA kernel,
fg_halo_pack) -> ONE all_to_all per direction over NCCL/NVLink -> unpack into `next` -> commit.
This replaces Messaging.post_msg for cut edges (pydcop/infrastructure/communication.py:588-698).
"""
import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np

from .layout import FactorGraphLayout, build_layout, default_var_csr


def variable_owner(n_vars: int, world: int) -> np.ndarray:
    """Contiguous blocks of ceil(V / world) variables."""
    per = -(-n_vars // world) if world > 0 else n_vars
    return (np.arange(n_vars, dtype=np.int64) // max(per, 1)).astype(np.int32)


@dataclass
class ShardPlan:
    """Everything rank `rank` needs: the closed local instance and the halo index lists."""
    rank: int
    world: int
    layout: FactorGraphLayout
    own_vars: np.ndarray            # global ids of the variables this rank owns (ascending)
    n_own_vars: int
    ghost_vars: np.ndarray          # global ids of the other ranks' variables in the scopes of this rank's factors
    # halo, one entry per cut edge touching this rank, grouped by peer in ascending global edge id
    send_r_off: np.ndarray          # int64 element offsets into r (rows this rank produces)
    send_q_off: np.ndarray          # int64 element offsets into q
    recv_r_off: np.ndarray          # where arriving r rows go (ghost stub rows)
    recv_q_off: np.ndarray          # where arriving q rows go (ghost variable slots)
    send_r_len: np.ndarray          # int32 row lengths
    send_q_len: np.ndarray
    recv_r_len: np.ndarray
    recv_q_len: np.ndarray
    send_r_edge: np.ndarray         # internal edge ids (for the validity flags exchanged at init)
    send_q_edge: np.ndarray
    recv_r_edge: np.ndarray
    recv_q_edge: np.ndarray
    send_r_split: List[int]         # elements per peer
    send_q_split: List[int]
    recv_r_split: List[int]
    recv_q_split: List[int]
    send_r_rows: List[int]          # rows per peer
    send_q_rows: List[int]
    recv_r_rows: List[int]
    recv_q_rows: List[int]
    n_cut_edges: int
    own_factor_edges: Optional[np.ndarray] = None   # global edge ids of the local real edges
    stub_edges: Optional[np.ndarray] = None         # global edge ids behind the local stub factors
    local_inst: Optional[Dict[str, np.ndarray]] = None   # the closed local graph as front-door arrays


def resolve_owner(inst, world: int, partition="blocks") -> np.ndarray:
    """Owner rank of every variable: an explicit int array, or the name of a method of
    pydcop_b200.partition.partition_variables ('blocks' | 'multilevel' | 'auto').  Every rank
    must pass the same value (the methods are deterministic)."""
    n_vars = len(np.asarray(inst["dom_size"]))
    if isinstance(partition, str):
        if partition == "blocks":
            return variable_owner(n_vars, world)
        from .partition import partition_variables
        return partition_variables(n_vars, inst["factor_ptr"], inst["edge_var"], world, method=partition)
    owner = np.asarray(partition, dtype=np.int32)
    if owner.shape != (n_vars,) or (len(owner) and (owner.min() < 0 or owner.max() >= world)):
        raise ValueError("owner array must give a rank in [0, world) for every variable")
    return owner


def broadcast_owner(inst, world: int, rank: int, device, method="auto", group=None):
    """Owner array for a multi-process run, computed ONCE on rank 0 and broadcast so that every
    rank builds its shard from the same array whatever the host libraries do.  Falls back to
    contiguous blocks when the partitioner fails.  Returns (owner array or 'blocks', error text
    or None); a collective — every rank must call it."""
    import torch
    import torch.distributed as dist
    if method == "blocks" or world <= 1:
        return "blocks", None
    n_vars = len(np.asarray(inst["dom_size"]))
    owner_t = torch.zeros(n_vars, dtype=torch.int32, device=device)
    ok = torch.zeros(1, dtype=torch.int32, device=device)
    err = None
    if rank == 0:
        try:
            owner_t.copy_(torch.from_numpy(np.ascontiguousarray(resolve_owner(inst, world, method), dtype=np.int32)))
            ok[0] = 1
        except Exception as ex:  # noqa: BLE001 — keep the run: contiguous blocks always work
            err = repr(ex)
    dist.broadcast(ok, 0, group=group)
    if int(ok.item()) != 1:
        return "blocks", err or "partition failed on rank 0"
    dist.broadcast(owner_t, 0, group=group)
    return owner_t.cpu().numpy(), None


def build_shard(inst: Dict[str, np.ndarray], rank: int, world: int, partition="blocks") -> ShardPlan:
    dom_size = np.asarray(inst["dom_size"], dtype=np.int32)
    factor_ptr = np.asarray(inst["factor_ptr"], dtype=np.int64)
    edge_var = np.asarray(inst["edge_var"], dtype=np.int64)
    tables = np.asarray(inst["tables"])
    V, F, E = len(dom_size), len(factor_ptr) - 1, len(edge_var)
    arity = np.diff(factor_ptr)
    tsize = np.ones(F, dtype=np.int64)
    efac = np.repeat(np.arange(F, dtype=np.int64), arity)
    np.multiply.at(tsize, efac, dom_size[edge_var].astype(np.int64))
    table_off = np.zeros(F + 1, dtype=np.int64)
    np.cumsum(tsize, out=table_off[1:])
    unary = np.asarray(inst["unary"], dtype=np.float64) if "unary" in inst and inst["unary"] is not None \
        else np.zeros(int(dom_size.sum()))
    unary_off = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(dom_size, out=unary_off[1:])
    if "var_ptr" in inst and inst.get("var_edge") is not None:
        g_var_ptr = np.asarray(inst["var_ptr"], dtype=np.int64)
        g_var_edge = np.asarray(inst["var_edge"], dtype=np.int64)
    else:
        vp, ve = default_var_csr(V, edge_var)
        g_var_ptr, g_var_edge = vp.astype(np.int64), ve.astype(np.int64)

    owner_v = resolve_owner(inst, world, partition)
    fac_owner = owner_v[edge_var[factor_ptr[:-1]]] if F else np.zeros(0, np.int32)
    e_fowner = fac_owner[efac]
    e_vowner = owner_v[edge_var]
    cut = e_fowner != e_vowner

    own_f = np.nonzero(fac_owner == rank)[0]
    own_v = np.nonzero(owner_v == rank)[0]
    # edges of own factors, in factor order
    own_f_edges = _ranges(factor_ptr[own_f], arity[own_f])
    ghost_vars = np.unique(edge_var[own_f_edges][e_vowner[own_f_edges] != rank]) if len(own_f_edges) \
        else np.zeros(0, np.int64)
    # grouped by owner (ascending id inside a group): one dense block of q rows per peer and class
    ghost_vars = ghost_vars[np.argsort(owner_v[ghost_vars], kind="stable")]
    # remote-factor edges of own variables (-> stub factors), grouped by the rank that produces
    # their row, ascending global edge id inside a group: the rows one peer sends land in ONE
    # contiguous block of this rank's r buffer, so its remote stores coalesce
    stub_edges = np.nonzero((e_vowner == rank) & (e_fowner != rank))[0]
    stub_edges = stub_edges[np.argsort(e_fowner[stub_edges], kind="stable")]

    # local variable ids: own (ascending global id) then ghosts
    n_own, n_ghost = len(own_v), len(ghost_vars)
    g2l_var = np.full(V, -1, dtype=np.int64)
    g2l_var[own_v] = np.arange(n_own)
    g2l_var[ghost_vars] = n_own + np.arange(n_ghost)
    l_dom = np.concatenate([dom_size[own_v], dom_size[ghost_vars]]).astype(np.int32)
    # variable tags (classes never mix tags): 0 = own, interior; 1 = own with at least one REMOTE factor — its q rows
    # towards those factors cross the cut, the engine computes these classes first so that their push overlaps the
    # interior variables' compute; 2 = ghost of another rank's variable (never computed here)
    own_tag = np.zeros(n_own, np.int32)
    if len(stub_edges):
        own_tag[g2l_var[edge_var[stub_edges]]] = 1
    l_var_tag = np.concatenate([own_tag, np.full(n_ghost, 2, np.int32)])

    # local factors: own factors then one unary stub per remote-factor edge
    n_real, n_stub = len(own_f), len(stub_edges)
    real_ar = arity[own_f]
    l_factor_ptr = np.zeros(n_real + n_stub + 1, dtype=np.int64)
    np.cumsum(np.concatenate([real_ar, np.ones(n_stub, np.int64)]), out=l_factor_ptr[1:])
    l_edge_var = np.concatenate([g2l_var[edge_var[own_f_edges]], g2l_var[edge_var[stub_edges]]])
    l_factor_tag = np.concatenate([np.zeros(n_real, np.int32), np.ones(n_stub, np.int32)])
    real_tab = _gather_blocks(tables, table_off, tsize, own_f) if n_real else np.zeros(0)
    l_tables = np.concatenate([real_tab, np.zeros(int(dom_size[edge_var[stub_edges]].sum()))])
    # global edge id -> local (canonical) edge id
    g2l_edge = np.full(E, -1, dtype=np.int64)
    g2l_edge[own_f_edges] = np.arange(len(own_f_edges))
    g2l_edge[stub_edges] = len(own_f_edges) + np.arange(n_stub)

    # variable CSR: own variables keep the global `links` order; ghosts list their local edges
    own_deg = (g_var_ptr[own_v + 1] - g_var_ptr[own_v]) if n_own else np.zeros(0, np.int64)
    own_slots_g = _ranges(g_var_ptr[own_v], own_deg) if n_own else np.zeros(0, np.int64)
    own_var_edge = g2l_edge[g_var_edge[own_slots_g]] if len(own_slots_g) else np.zeros(0, np.int64)
    assert (own_var_edge >= 0).all()
    ghost_edge_l = np.nonzero(l_edge_var[:len(own_f_edges)] >= n_own)[0]
    order = np.argsort(l_edge_var[ghost_edge_l], kind="stable")
    ghost_var_edge = ghost_edge_l[order]
    ghost_deg = np.bincount(l_edge_var[ghost_edge_l] - n_own, minlength=n_ghost) if n_ghost \
        else np.zeros(0, np.int64)
    l_var_ptr = np.zeros(n_own + n_ghost + 1, dtype=np.int64)
    np.cumsum(np.concatenate([own_deg, ghost_deg]), out=l_var_ptr[1:])
    l_var_edge = np.concatenate([own_var_edge, ghost_var_edge])
    l_unary = np.concatenate([unary[_ranges(unary_off[own_v], dom_size[own_v].astype(np.int64))]
                              if n_own else np.zeros(0),
                              np.zeros(int(dom_size[ghost_vars].sum()))])
    init = inst.get("init_value") if hasattr(inst, "get") else None
    l_init = None
    if init is not None:
        init = np.asarray(init, dtype=np.int32)
        l_init = np.concatenate([init[own_v], np.full(n_ghost, -1, np.int32)])

    L = build_layout(l_dom, l_factor_ptr, l_edge_var, l_tables, None, l_unary, l_var_ptr, l_var_edge,
                     l_init, factor_tag=l_factor_tag, var_tag=l_var_tag)

    # ---- halo lists: every cut edge touching this rank, grouped by peer, ascending global id ----
    def rows(global_edges):
        ie = L.edge_perm[g2l_edge[global_edges]]
        return (L.edge_msg_off[ie], L.edge_qoff[ie], dom_size[edge_var[global_edges]].astype(np.int32),
                ie.astype(np.int32))

    cut_e = np.nonzero(cut)[0]
    mine_f = cut_e[e_fowner[cut_e] == rank]     # I own the factor: I send r, receive q
    mine_v = cut_e[e_vowner[cut_e] == rank]     # I own the variable: I send q, receive r
    mine_f = mine_f[np.argsort(e_vowner[mine_f], kind="stable")]   # grouped by peer (variable owner)
    mine_v = mine_v[np.argsort(e_fowner[mine_v], kind="stable")]   # grouped by peer (factor owner)
    fr, fq, fl, fe = rows(mine_f)
    vr, vq, vl, ve = rows(mine_v)

    def per_peer(peers, lens):
        el = np.bincount(peers, weights=lens, minlength=world).astype(np.int64)
        rw = np.bincount(peers, minlength=world).astype(np.int64)
        return [int(x) for x in el], [int(x) for x in rw]

    sr_split, sr_rows = per_peer(e_vowner[mine_f], fl)
    rq_split, rq_rows = sr_split, sr_rows           # q rows come back along the same edges
    sq_split, sq_rows = per_peer(e_fowner[mine_v], vl)
    rr_split, rr_rows = sq_split, sq_rows
    return ShardPlan(
        rank=rank, world=world, layout=L, own_vars=own_v.astype(np.int64), n_own_vars=n_own,
        ghost_vars=np.asarray(ghost_vars, dtype=np.int64),
        send_r_off=fr, send_q_off=vq, recv_r_off=vr, recv_q_off=fq,
        send_r_len=fl, send_q_len=vl, recv_r_len=vl, recv_q_len=fl,
        send_r_edge=fe, send_q_edge=ve, recv_r_edge=ve, recv_q_edge=fe,
        send_r_split=sr_split, send_q_split=sq_split, recv_r_split=rr_split, recv_q_split=rq_split,
        send_r_rows=sr_rows, send_q_rows=sq_rows, recv_r_rows=rr_rows, recv_q_rows=rq_rows,
        n_cut_edges=int(cut.sum()), own_factor_edges=own_f_edges, stub_edges=stub_edges,
        local_inst=dict(dom_size=l_dom, factor_ptr=l_factor_ptr, edge_var=l_edge_var, tables=l_tables,
                        unary=l_unary, var_ptr=l_var_ptr, var_edge=l_var_edge, init_value=l_init))


def _ranges(starts, lengths):
    """Concatenation of arange(s, s + l) for every (s, l), vectorised."""
    starts = np.asarray(starts, dtype=np.int64)
    lengths = np.asarray(lengths, dtype=np.int64)
    total = int(lengths.sum())
    if total == 0:
        return np.zeros(0, dtype=np.int64)
    rep = np.repeat(starts - np.concatenate([[0], np.cumsum(lengths)[:-1]]), lengths)
    return rep + np.arange(total, dtype=np.int64)


def _gather_blocks(flat, off, size, which):
    """Concatenation of flat[off[i] : off[i] + size[i]] for i in `which`.  When every block has the same size and
    the blocks tile `flat` (the usual case: one table shape) this is a row gather of a 2-D view — a memcpy per row
    instead of one index per ELEMENT (20 M indices for the 200k tables a rank of C2 x 8 owns: 3 s of a solve)."""
    which = np.asarray(which, dtype=np.int64)
    n = len(size)
    if n and len(which):
        s0 = int(size[0])
        if s0 > 0 and len(flat) == n * s0 and (size == s0).all() and int(off[0]) == 0 and int(off[n - 1]) == (n - 1) * s0:
            return flat.reshape(n, s0)[which].reshape(-1)
    return flat[_ranges(off[which], size[which])]


class HaloExchange:
    """Packs boundary rows, exchanges them with one all_to_all per direction, unpacks them.

    `pack(src, packed, row_off, packed_off, row_len)` / `unpack(dst, packed, ...)` are injected:
    the product passes the CUDA kernels behind fg_halo_pack / fg_halo_unpack; the CPU (gloo) tests
    pass index-based stand-ins to exercise the plumbing without a GPU."""

    def __init__(self, plan: ShardPlan, torch_dtype, device, pack, unpack, group=None):
        import torch
        self.torch, self.plan, self.pack, self.unpack, self.group = torch, plan, pack, unpack, group
        dev = device

        def dv(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt)

        p = plan
        # ONE exchange per cycle: the block for peer b is [r rows for b | q rows for b]
        W = p.world
        sr_rows, sq_rows = np.asarray(p.send_r_rows), np.asarray(p.send_q_rows)
        rr_rows, rq_rows = np.asarray(p.recv_r_rows), np.asarray(p.recv_q_rows)
        sr_el, sq_el = np.asarray(p.send_r_split, np.int64), np.asarray(p.send_q_split, np.int64)
        rr_el, rq_el = np.asarray(p.recv_r_split, np.int64), np.asarray(p.recv_q_split, np.int64)
        self.send_split = [int(a + b) for a, b in zip(sr_el, sq_el)]
        self.recv_split = [int(a + b) for a, b in zip(rr_el, rq_el)]
        s_base = np.concatenate([[0], np.cumsum(sr_el + sq_el)])[:-1]
        r_base = np.concatenate([[0], np.cumsum(rr_el + rq_el)])[:-1]

        def packed_offsets(lens, rows_per_peer, base, shift):
            """offset of every row inside the combined buffer: rows are grouped by peer"""
            out = np.zeros(len(lens), dtype=np.int64)
            pos = 0
            for b in range(W):
                n = int(rows_per_peer[b])
                if n:
                    ln = np.asarray(lens[pos:pos + n], dtype=np.int64)
                    out[pos:pos + n] = base[b] + shift[b] + np.concatenate([[0], np.cumsum(ln)[:-1]])
                pos += n
            return out

        zero = np.zeros(W, dtype=np.int64)
        self.sr = (dv(p.send_r_off, torch.int64), dv(packed_offsets(p.send_r_len, sr_rows, s_base, zero), torch.int64),
                   dv(p.send_r_len, torch.int32))
        self.sq = (dv(p.send_q_off, torch.int64), dv(packed_offsets(p.send_q_len, sq_rows, s_base, sr_el), torch.int64),
                   dv(p.send_q_len, torch.int32))
        self.rr = (dv(p.recv_r_off, torch.int64), dv(packed_offsets(p.recv_r_len, rr_rows, r_base, zero), torch.int64),
                   dv(p.recv_r_len, torch.int32))
        self.rq = (dv(p.recv_q_off, torch.int64), dv(packed_offsets(p.recv_q_len, rq_rows, r_base, rr_el), torch.int64),
                   dv(p.recv_q_len, torch.int32))
        z = lambda n: torch.zeros(max(int(n), 1), dtype=torch_dtype, device=dev)  # noqa: E731
        self.buf_send, self.buf_recv = z(sum(self.send_split)), z(sum(self.recv_split))
        self.launches = 0
        # uniform-domain fast form: one launch moves the r and the q rows (fg_halo_rows_uniform)
        self.fused = None
        self.uniform_dom = int(p.layout.uniform_dom)
        c64 = lambda a: (C.c_int64 * len(a))(*[int(x) for x in a])  # noqa: E731
        cs = lambda a: np.concatenate([[0], np.cumsum(a)])  # noqa: E731
        self.peers_send = (c64(cs(sr_rows)), c64(cs(sq_rows)), c64(s_base))
        self.peers_recv = (c64(cs(rr_rows)), c64(cs(rq_rows)), c64(r_base))

    def pack_rows(self, q, r):
        p = self.plan
        n_sr, n_sq = len(p.send_r_len), len(p.send_q_len)
        if self.fused is not None and self.uniform_dom and (n_sr + n_sq):
            self.fused(1, r, q, self.buf_send, self.sr[0], self.sq[0], n_sr, n_sq, self.uniform_dom,
                       p.world, *self.peers_send)
            self.launches += 1
            return
        if n_sr:
            self.pack(r, self.buf_send, *self.sr, n_sr)
        if n_sq:
            self.pack(q, self.buf_send, *self.sq, n_sq)
        self.launches += int(n_sr > 0) + int(n_sq > 0)

    def unpack_rows(self, q, r):
        p = self.plan
        n_rr, n_rq = len(p.recv_r_len), len(p.recv_q_len)
        if self.fused is not None and self.uniform_dom and (n_rr + n_rq):
            self.fused(0, r, q, self.buf_recv, self.rr[0], self.rq[0], n_rr, n_rq, self.uniform_dom,
                       p.world, *self.peers_recv)
            self.launches += 1
            return
        if n_rr:
            self.unpack(r, self.buf_recv, *self.rr, n_rr)
        if n_rq:
            self.unpack(q, self.buf_recv, *self.rq, n_rq)
        self.launches += int(n_rr > 0) + int(n_rq > 0)

    def exchange(self, q, r):
        """Boundary rows of the given q / r buffers -> the peers' ghost rows: pack, ONE
        all_to_all (NCCL grouped send/recv over NVLink), unpack."""
        import torch.distributed as dist
        self.pack_rows(q, r)
        ts, tr = sum(self.send_split), sum(self.recv_split)
        dist.all_to_all_single(self.buf_recv[:tr], self.buf_send[:ts], self.recv_split, self.send_split,
                               group=self.group)
        self.unpack_rows(q, r)

    def exchange_flags(self, q_valid, r_valid):
        """Validity bytes of the cycle-0 (on_start) messages along the cut edges."""
        import torch.distributed as dist
        torch, p = self.torch, self.plan
        dev = q_valid.device

        def idx(a):
            return torch.from_numpy(np.ascontiguousarray(a).astype(np.int64)).to(dev)

        for flags, send_e, recv_e, s_rows, r_rows in (
                (r_valid, p.send_r_edge, p.recv_r_edge, p.send_r_rows, p.recv_r_rows),
                (q_valid, p.send_q_edge, p.recv_q_edge, p.send_q_rows, p.recv_q_rows)):
            out = flags[idx(send_e)].contiguous() if len(send_e) else flags[:0].clone()
            inn = torch.zeros(int(sum(r_rows)), dtype=flags.dtype, device=dev)
            dist.all_to_all_single(inn, out, list(r_rows), list(s_rows), group=self.group)
            if len(recv_e):
                flags[idx(recv_e)] = inn


def destination_order(dst_off, rows_per_peer) -> np.ndarray:
    """Permutation of the send rows (which are grouped by peer) that sorts every peer's group by
    destination offset and leaves the grouping intact."""
    dst_off = np.asarray(dst_off, dtype=np.int64)
    peer = np.repeat(np.arange(len(rows_per_peer)), np.asarray(rows_per_peer, dtype=np.int64))
    assert len(peer) == len(dst_off)
    return np.lexsort((dst_off, peer)).astype(np.int64)


def push_tables(plan: ShardPlan, base: np.ndarray, dst_r_off, dst_q_off, elem: int):
    """Source offsets and absolute destination addresses of the peer push.
    base[rank] = addresses of that rank's (q[0], q[1], r[0], r[1]) as mapped into this process;
    dst_*_off = the consumers' element offsets of my send rows (my send order).
    Rows are independent: they are issued in DESTINATION order inside each peer group, so that
    consecutive threads of the push kernel store to consecutive remote addresses (the local reads
    become gathers instead, which HBM absorbs)."""
    W = plan.world
    peer_of_r = np.repeat(np.arange(W), np.asarray(plan.send_r_rows, dtype=np.int64))
    peer_of_q = np.repeat(np.arange(W), np.asarray(plan.send_q_rows, dtype=np.int64))
    dst_r_off = np.asarray(dst_r_off, dtype=np.int64)
    dst_q_off = np.asarray(dst_q_off, dtype=np.int64)
    perm_r = destination_order(dst_r_off, plan.send_r_rows)
    perm_q = destination_order(dst_q_off, plan.send_q_rows)
    return dict(
        dst_r=[(base[peer_of_r, 2 + b] + dst_r_off * elem)[perm_r] for b in range(2)],
        dst_q=[(base[peer_of_q, 0 + b] + dst_q_off * elem)[perm_q] for b in range(2)],
        src_r_off=np.asarray(plan.send_r_off, dtype=np.int64)[perm_r],
        src_q_off=np.asarray(plan.send_q_off, dtype=np.int64)[perm_q])


def fused_destinations(plan: ShardPlan, base: np.ndarray, dst_r_off, dst_q_off, elem: int):
    """Per-edge / per-slot destination addresses of the FUSED halo (fg_halo_plan_t::dev_edge_dst_r / dev_slot_dst_q):
    for buffer index b, edge_dst[b][e] = address in the consumer's r[b] of the row edge e's factor produces (internal,
    class-major edge ids), slot_dst[b][s] = address in the consumer's q[b] of slot s's row; 0 = the row stays here.
    Same inputs as push_tables.  Pure function (tested on CPU)."""
    L, W = plan.layout, plan.world
    peer_of_r = np.repeat(np.arange(W), np.asarray(plan.send_r_rows, dtype=np.int64))
    peer_of_q = np.repeat(np.arange(W), np.asarray(plan.send_q_rows, dtype=np.int64))
    dst_r_off = np.asarray(dst_r_off, dtype=np.int64)
    dst_q_off = np.asarray(dst_q_off, dtype=np.int64)
    slot_of_edge = np.empty(L.n_edges, dtype=np.int64)
    slot_of_edge[np.asarray(L.slot_edge, dtype=np.int64)] = np.arange(L.n_edges)
    edge_dst, slot_dst = [], []
    for b in range(2):
        er = np.zeros(max(L.n_edges, 1), dtype=np.int64)
        er[np.asarray(plan.send_r_edge, dtype=np.int64)] = base[peer_of_r, 2 + b] + dst_r_off * elem
        sq = np.zeros(max(L.n_edges, 1), dtype=np.int64)
        sq[slot_of_edge[np.asarray(plan.send_q_edge, dtype=np.int64)]] = base[peer_of_q, 0 + b] + dst_q_off * elem
        edge_dst.append(er)
        slot_dst.append(sq)
    return edge_dst, slot_dst


def push_runs(dst_addr, row_bytes: int):
    """Cut a push list (absolute destination address per row, in push order) into RUNS of rows whose
    destinations are consecutive addresses.  Returns (int64 [n_runs, 4], total_units): per run the first
    destination address, the index of its first row, its length in bytes, and the index of its first
    16-byte aligned destination unit (the run-based push kernel maps one thread to one unit, fg_halo_plan_t)."""
    dst = np.asarray(dst_addr, dtype=np.int64)
    if not len(dst):
        return np.zeros((0, 4), dtype=np.int64), 0
    brk = np.ones(len(dst), dtype=bool)
    brk[1:] = dst[1:] != dst[:-1] + row_bytes
    first = np.nonzero(brk)[0]
    n_rows = np.diff(np.concatenate([first, [len(dst)]]))
    a0 = dst[first]
    nbytes = n_rows * row_bytes
    units = (a0 + nbytes + 15) // 16 - a0 // 16
    first_unit = np.concatenate([[0], np.cumsum(units)[:-1]])
    return np.ascontiguousarray(np.stack([a0, first, nbytes, first_unit], axis=1), dtype=np.int64), int(units.sum())


class PeerPush:
    """Halo over NVLink peer memory: every rank maps the peers' message buffers (CUDA IPC) and its
    push kernel stores each boundary row straight into the consumer's `next` buffer.  The cycle is
    closed on the DEVICE: the last block of the push kernel releases the new epoch into the peers'
    flag arrays and a one-warp kernel acquires the peers' epochs (pydcop_b200/peer.py,
    csrc/peer_sync.cuh) — no NCCL call, no host round trip per cycle.  The whole cycle
    (compute -> push + release -> wait -> commit) is enqueued by ONE C call, fg_maxsum_shard_step."""

    def __init__(self, sharded, group=None):
        import torch
        import torch.distributed as dist
        from . import _cabi
        from .peer import PeerMap, PeerSync
        self.torch, self.dist, self.group = torch, dist, group
        e, p = sharded.engine, sharded.plan
        self.engine, self.plan, self.sharded = e, p, sharded
        dev = e.device
        W, me = p.world, p.rank
        if not p.layout.uniform_dom:
            raise RuntimeError("peer push needs a uniform domain size")
        # 1. map everybody's four message buffers with MY device as the accessor
        self.pmap = PeerMap(e.lib, dev, me, W, group)
        base = self.pmap.map([e.q[0], e.q[1], e.r[0], e.r[1]])
        # 2. where do my rows land?  the consumer's recv offsets, in my send order
        def peer_offsets(recv_off, recv_rows, send_rows):
            out = torch.zeros(int(sum(send_rows)), dtype=torch.int64, device=dev)
            inp = torch.from_numpy(np.ascontiguousarray(recv_off, dtype=np.int64)).to(dev)
            dist.all_to_all_single(out, inp, list(send_rows), list(recv_rows), group=group)
            return out.cpu().numpy()

        dst_r_off = peer_offsets(p.recv_r_off, p.recv_r_rows, p.send_r_rows)   # offsets in the peer's r
        dst_q_off = peer_offsets(p.recv_q_off, p.recv_q_rows, p.send_q_rows)
        elem = e.q[0].element_size()
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)  # noqa: E731
        t = push_tables(p, base, dst_r_off, dst_q_off, elem)
        self.dst_r, self.dst_q = [to(a) for a in t["dst_r"]], [to(a) for a in t["dst_q"]]
        self.src_r_off, self.src_q_off = to(t["src_r_off"]), to(t["src_q_off"])
        self.n_r, self.n_q = len(p.send_r_len), len(p.send_q_len)
        self.dom = int(p.layout.uniform_dom)
        # 3. device-side barrier with the ranks I share cut edges with
        peers = [b for b in range(W) if b != me and (p.send_r_rows[b] or p.send_q_rows[b]
                                                    or p.recv_r_rows[b] or p.recv_q_rows[b])]
        self.sync = PeerSync(self.pmap, peers)
        plan = _cabi.FgHaloPlan()
        plan.elem_bytes, plan.dom, plan.n_r, plan.n_q = elem, self.dom, self.n_r, self.n_q
        plan.dev_src_r_off, plan.dev_src_q_off = self.src_r_off.data_ptr(), self.src_q_off.data_ptr()
        for b in range(2):
            plan.dev_dst_r[b], plan.dev_dst_q[b] = self.dst_r[b].data_ptr(), self.dst_q[b].data_ptr()
        plan.dev_counter = self.sync.counter.data_ptr()
        plan.sync = self.sync.struct
        # destination runs: whole 16-byte stores over NVLink whatever the row size (PYDCOP_B200_PUSH_RUNS=0: per row)
        self.runs = []
        import os
        if (self.dom * elem) % 8 == 0 and os.environ.get("PYDCOP_B200_PUSH_RUNS", "1") != "0":
            for b in range(2):
                for name, dst in (("r", t["dst_r"][b]), ("q", t["dst_q"][b])):
                    runs, units = push_runs(dst, self.dom * elem)
                    rt = to(runs.reshape(-1)) if len(runs) else None
                    self.runs.append(rt)
                    if rt is not None:
                        getattr(plan, "dev_runs_" + name)[b] = rt.data_ptr()
                        getattr(plan, "n_runs_" + name)[b] = len(runs)
                        getattr(plan, "units_" + name)[b] = units
        self.n_runs = [int(plan.n_runs_r[0]), int(plan.n_runs_q[0])]
        # fused halo: the warp kernels store each boundary row from the lane that produced it (the engine decides at
        # attach time whether every class of this shard runs on them; PYDCOP_B200_PUSH_FUSED=0 keeps the push kernels)
        ed, sd = fused_destinations(p, base, dst_r_off, dst_q_off, elem)
        self.edge_dst, self.slot_dst = [to(a) for a in ed], [to(a) for a in sd]
        for b in range(2):
            plan.dev_edge_dst_r[b], plan.dev_slot_dst_q[b] = self.edge_dst[b].data_ptr(), self.slot_dst[b].data_ptr()
        self._plan = plan
        rc = e.lib.fg_maxsum_shard_attach(e._h, C.byref(plan))
        if rc != 0:
            raise RuntimeError(f"fg_maxsum_shard_attach failed rc={rc}: {e._last_error()}")
        self.launches = 0      # counted inside the engine handle now
        self.fused = bool(e.lib.fg_maxsum_shard_fused(e._h))
        dist.barrier(group=group)

    def step(self, n_cycles):
        e, torch = self.engine, self.torch
        with torch.cuda.device(e.device):
            rc = e.lib.fg_maxsum_shard_step(e._h, int(n_cycles),
                                            C.c_void_p(torch.cuda.current_stream(e.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"fg_maxsum_shard_step failed rc={rc}: {e._last_error()}")

    def phase(self, ph):
        e, torch = self.engine, self.torch
        with torch.cuda.device(e.device):
            rc = e.lib.fg_maxsum_shard_phase(e._h, int(ph),
                                             C.c_void_p(torch.cuda.current_stream(e.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"fg_maxsum_shard_phase({ph}) failed rc={rc}: {e._last_error()}")


class ShardedMaxSum:
    """One rank of the partitioned MaxSum: same driving API as MaxSumEngine (init / step / values)."""

    def __init__(self, inst, rank, world, device, precision="f32", group=None, halo="nccl",
                 partition="blocks", engine_factory=None, pack=None, unpack=None, **params):
        """`engine_factory(layout, precision=…, **params)`, `pack` and `unpack` exist so that the
        partition, the exchange and this class's own cycle logic can run on a box without a GPU
        (tests: the kernel source through the host shim, gloo); the product path leaves them at
        None and gets MaxSumEngine + the CUDA halo kernels."""
        import torch
        from . import _cabi
        from .engine import MaxSumEngine, PRECISIONS
        self.torch = torch
        self.plan = build_shard(inst, rank, world, partition)
        self.rank, self.world = rank, world
        prec, tdt, _ = PRECISIONS[precision]
        self.global_n_edges = int(len(np.asarray(inst["edge_var"])))
        self.global_n_vars = int(len(np.asarray(inst["dom_size"])))
        self.global_dom_size = np.asarray(inst["dom_size"], dtype=np.int32)
        self.peer = None
        if engine_factory is not None:
            self.engine = engine_factory(self.plan.layout, precision=precision, **params)
            self.device = torch.device(device) if device is not None else torch.device("cpu")
            self.halo = HaloExchange(self.plan, tdt, self.device, pack, unpack, group)
            self.halo_mode = "nccl"
            return
        self.engine = MaxSumEngine(self.plan.layout, device=device, precision=precision, **params)
        self.device = self.engine.device
        lib = self.engine.lib

        def stream():
            return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

        # the halo kernels run on the current device: make it the shard's (shards of one process may be on several)
        def pack(src, packed, row_off, packed_off, row_len, n):
            with torch.cuda.device(self.device):
                rc = lib.fg_halo_pack(prec, C.c_void_p(src.data_ptr()), C.c_void_p(packed.data_ptr()),
                                      C.c_void_p(row_off.data_ptr()), C.c_void_p(packed_off.data_ptr()),
                                      C.c_void_p(row_len.data_ptr()), n, stream())
            if rc != _cabi.FG_OK:
                raise _cabi.EngineError(f"fg_halo_pack failed rc={rc}")

        def unpack(dst, packed, row_off, packed_off, row_len, n):
            with torch.cuda.device(self.device):
                rc = lib.fg_halo_unpack(prec, C.c_void_p(dst.data_ptr()), C.c_void_p(packed.data_ptr()),
                                        C.c_void_p(row_off.data_ptr()), C.c_void_p(packed_off.data_ptr()),
                                        C.c_void_p(row_len.data_ptr()), n, stream())
            if rc != _cabi.FG_OK:
                raise _cabi.EngineError(f"fg_halo_unpack failed rc={rc}")

        self.halo = HaloExchange(self.plan, tdt, self.device, pack, unpack, group)

        def fused(is_pack, r, q, packed, off_r, off_q, n_r, n_q, dom, n_peers, pr, pq, pb):
            with torch.cuda.device(self.device):
                rc = lib.fg_halo_rows_uniform(prec, is_pack, C.c_void_p(r.data_ptr()), C.c_void_p(q.data_ptr()),
                                              C.c_void_p(packed.data_ptr()), C.c_void_p(off_r.data_ptr()),
                                              C.c_void_p(off_q.data_ptr()), n_r, n_q, dom, n_peers,
                                              C.cast(pr, C.c_void_p), C.cast(pq, C.c_void_p),
                                              C.cast(pb, C.c_void_p), stream())
            if rc != _cabi.FG_OK:
                raise _cabi.EngineError(f"fg_halo_rows_uniform failed rc={rc}")

        if self.plan.layout.uniform_dom:
            self.halo.fused = fused
        self.halo_mode = halo

    @property
    def layout(self):
        return self.plan.layout

    def init(self):
        e = self.engine
        e.init()
        self.halo.exchange(e.q[0], e.r[0])
        self.halo.exchange_flags(e.q_valid, e.r_valid)
        if self.halo_mode in ("p2p", "auto") and self.peer is None and self.world > 1:
            try:
                self.peer = PeerPush(self, self.halo.group)
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
            e.cycle_compute()
            nxt = e.cur ^ 1
            self.halo.exchange(e.q[nxt], e.r[nxt])
            e.cycle_commit()
        return self

    def check(self):
        """Raise if the device-side barrier timed out (synchronises the device)."""
        if self.peer is not None:
            self.peer.sync.check()

    def timed_breakdown(self, n_cycles=50):
        """Device time (ms per cycle) of the phases of a cycle on this rank: peer push path ->
        compute / push (+ release) / wait; NCCL path -> compute / pack / all_to_all / unpack."""
        import torch.distributed as dist
        torch, e, h = self.torch, self.engine, self.halo
        ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
        if self.peer is not None:   # timing events recorded inside the C cycle: no host time between the kernels
            out = (C.c_double * 7)()
            with torch.cuda.device(self.device):
                rc = e.lib.fg_maxsum_shard_profile(e._h, int(n_cycles), e._stream(), out)
            if rc != 0:
                raise RuntimeError(f"fg_maxsum_shard_profile failed rc={rc}: {e._last_error()}")
            keys = ("factor_side", "push_r", "variable_side", "push_q", "push_release", "wait", "cycle")
            return {k: out[i] * 1e-3 for i, k in enumerate(keys)}
        acc = np.zeros(4)
        for _ in range(n_cycles):
            t = [ev() for _ in range(5)]
            t[0].record()
            e.cycle_compute()
            t[1].record()
            nxt = e.cur ^ 1
            h.pack_rows(e.q[nxt], e.r[nxt])
            t[2].record()
            ts, tr = sum(h.send_split), sum(h.recv_split)
            dist.all_to_all_single(h.buf_recv[:tr], h.buf_send[:ts], h.recv_split, h.send_split, group=h.group)
            t[3].record()
            h.unpack_rows(e.q[nxt], e.r[nxt])
            t[4].record()
            e.cycle_commit()
            torch.cuda.synchronize(self.device)
            acc += [t[i].elapsed_time(t[i + 1]) for i in range(4)]
        return dict(zip(("compute", "pack", "all_to_all", "unpack"), (acc / n_cycles).tolist()))

    @property
    def launch_count(self):
        return self.engine.launch_count + self.halo.launches

    def local_values(self):
        """(global variable ids, value indices) of the variables this rank owns."""
        val, _ = self.engine.values()
        return self.plan.own_vars, val[:self.plan.n_own_vars]

    def solution_cost(self, infinity=float("inf"), unary=None):
        """(cost, violations) of the current assignment of the WHOLE problem: every rank reduces its own
        factors and variables on its device (fg_solution_cost skips the ghost classes), one NCCL
        all-reduce of the two sums (pydcop/dcop/dcop.py:319-367, orchestrator.py:1229-1231).
        `unary`: the variables' own costs of the whole problem, global canonical order, without noise."""
        import torch.distributed as dist
        p, e = self.plan, self.engine
        local_unary = None
        if unary is not None:
            dom = np.asarray(self.global_dom_size, dtype=np.int64)
            uoff = np.concatenate([[0], np.cumsum(dom)])
            own = p.own_vars
            n_ghost_el = int(np.asarray(p.local_inst["dom_size"], dtype=np.int64)[p.n_own_vars:].sum())
            local_unary = np.concatenate([np.asarray(unary, dtype=np.float64)[_ranges(uoff[own], dom[own])],
                                          np.zeros(n_ghost_el)])
        n_own_internal = sum(c.n_vars for c in p.layout.var_classes if c.tag != 2)
        # a cut factor's entry needs the value of a variable another rank owns, and ghost variables are never
        # evaluated here: take them from the all-gathered assignment (local canonical order = own, then ghosts)
        full = self.values()
        L = p.layout
        local = np.concatenate([full[p.own_vars], full[p.ghost_vars]]).astype(np.int32)
        val = self.torch.from_numpy(np.ascontiguousarray(local[L.var_order])).to(e.value.device)
        out = e._solution_cost(val, infinity, local_unary, n_vars=n_own_internal)
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.halo.group)
        o = out.cpu().numpy()
        return float(o[0]), int(round(o[1]))

    def values(self):
        """All-gathered assignment (every rank gets the full vector)."""
        import torch.distributed as dist
        torch = self.torch
        ids, val = self.local_values()
        out = torch.zeros(self.global_n_vars, dtype=torch.int32, device=self.device)
        out[torch.from_numpy(ids).to(self.device)] = torch.from_numpy(val.astype(np.int32)).to(self.device)
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.halo.group)
        return out.cpu().numpy()
