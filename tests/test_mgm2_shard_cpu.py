"""Sharded MGM-2 on CPU: the shard builder, and the whole init / five-exchange cycle over torch.distributed (gloo,
world 2 and 3) with the sharded kernel SOURCE on the CPU (tests/hostshim/mgm2_shard_host.cpp runs
the fg_mgm2_shard_* launch sequences of pydcop_b200/csrc/mgm2_shard_kernels.cuh) in the engine seam of ShardedMgm2.  Every cycle must equal the
single-process run of the kernel source (tests/hostshim/mgm2_host.cpp) and Mgm2Oracle bit for bit."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _hostshim as hs
import oracle as orc
from _mgm2_oracle import Mgm2Oracle
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array, distinct_neighbours, fill_desc, fill_header, host_state, mgm2_plan
from pydcop_b200.layout import layout_from_instance
from pydcop_b200.multigpu import resolve_owner
from pydcop_b200.multigpu_mgm2 import EXCHANGES, build_mgm2_shard
from test_mgm2_hostshim import HostMgm2

KEYS = ("value", "cost", "gain", "committed", "partner", "go")


@pytest.fixture(scope="module")
def shims():
    """Both shims built before the gloo workers start (they load the cached libraries)."""
    return hs.build("mgm2_shard_host"), hs.build("mgm2_host")


class HostShardMgm2:
    """Mgm2Engine's plan and shard_* surface over the host-shimmed sharded kernels (host arrays; the exchange
    buffers are torch CPU tensors for gloo)."""

    def __init__(self, layout, inst=None, precision="f64", mode="min", threshold=0.5, favor="unilateral",
                 stop_cycle=0, seed=0, var_rank=None, var_global_id=None):
        self.lib = hs.build("mgm2_shard_host")
        self.layout, self.precision = layout, precision
        inputs, state, scalars = mgm2_plan(layout, precision, mode, threshold, favor, stop_cycle, seed, var_rank,
                                           var_global_id=var_global_id)
        self.k = dict(inputs, **host_state(state))
        self.classes = _class_array(layout)
        self.d = fill_desc(fill_header(_cabi.FgMgm2Desc(), precision, layout, self.classes), self.k, scalars)
        self.stop_cycle, self.cycle, self.launch_count = scalars["stop_cycle"], 0, 0
        for key in ("value", "cost", "gain", "committed", "partner", "go", "has_cost"):
            setattr(self, key, self.k[key])

    @property
    def finished(self):
        return bool(self.stop_cycle and self.cycle + 1 >= self.stop_cycle)

    def shard_attach(self, arrays):
        tdt = torch.float64 if self.precision == "f64" else torch.float32
        self._keep = arrays
        self.send_buf = [torch.zeros(max(int(x["send_off"][-1]), 1), dtype=tdt) for x in arrays["x"]]
        self.recv_buf = [torch.zeros(max(int(x["recv_off"][-1]), 1), dtype=tdt) for x in arrays["x"]]
        plan = _cabi.FgMgm2ShardPlan()
        addr = lambda a: a.ctypes.data if len(a) else None  # noqa: E731
        for i, x in enumerate(arrays["x"]):
            p = plan.x[i]
            p.n_send, p.n_recv = len(x["send_var"]), len(x["recv_var"])
            p.dev_send_var, p.dev_recv_var = addr(x["send_var"]), addr(x["recv_var"])
            p.dev_send_off, p.dev_recv_off = addr(x["send_off"]), addr(x["recv_off"])
            p.dev_send_buf, p.dev_recv_buf = self.send_buf[i].data_ptr(), self.recv_buf[i].data_ptr()
        for key in ("ghost", "send_peer", "owner_rank", "owner_local"):
            setattr(plan, "dev_" + key, addr(arrays[key]))
        self.plan = plan

    def shard_init(self):
        self.lib.mgm2_shard_host_init(C.byref(self.d), C.byref(self.plan))
        self.cycle = 0

    def shard_phase(self, x):
        self.lib.mgm2_shard_host_phase(C.byref(self.d), C.byref(self.plan), C.c_int32(x), C.c_int64(self.cycle))
        if x == EXCHANGES - 1:
            self.cycle += 1

    def shard_unpack(self, x):
        self.lib.mgm2_shard_host_unpack(C.byref(self.d), C.byref(self.plan), C.c_int32(x))

    def values(self):
        L = self.layout
        return L.vars_to_canonical(self.k["value"][:L.n_vars].copy()), None


class HostMgm2Single(HostMgm2):
    """The single-process run (tests/hostshim/mgm2_host.cpp): every variable's state per cycle."""

    def state(self):
        L, n = self.L, self.L.n_vars
        out = {k: L.vars_to_canonical(self.k[k][:n].copy()) for k in KEYS}
        p = out["partner"].astype(np.int64)
        out["partner"] = np.where(p >= 0, np.asarray(L.var_order)[np.maximum(p, 0)], -1)
        return out


def random_instance(n, d, seed, levels=0, isolated=0):
    """Mixed arities 1-3 (unary-only variables), float costs or few integer levels (ties), random name ranks and
    initial values; `isolated` extra variables without any constraint."""
    from test_mgm2_hostshim import random_mgm2_instance
    from pydcop_b200.layout import default_var_csr
    inst = random_mgm2_instance(n, d, [2, 3, 1], seed=seed, n_factors=n // 2, levels=levels)
    if isolated:
        m = n + isolated
        inst["dom_size"] = np.concatenate([inst["dom_size"], np.full(isolated, d, np.int32)])
        inst["unary"] = np.concatenate([inst["unary"], np.zeros(isolated * d)])
        rng = np.random.default_rng(seed)
        inst["var_rank"] = rng.permutation(m).astype(np.int32)
        inst["init_value"] = np.concatenate([inst["init_value"], np.full(isolated, -1, np.int32)])
        inst["var_ptr"], inst["var_edge"] = default_var_csr(m, inst["edge_var"])
    return inst


def imbalanced_owner(V, world, seed=0):
    rng = np.random.default_rng(seed)
    w = np.arange(1, world + 1, dtype=np.float64) ** 2
    return rng.choice(world, size=V, p=w / w.sum()).astype(np.int32)


# ---- the shard builder ----

@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("partition", ["blocks", "multilevel", "imbalanced"])
def test_shard_builder(world, partition):
    inst = random_instance(240, 4, seed=3, isolated=5)
    inst["dom_size"] = np.where(np.arange(len(inst["dom_size"])) % 3 == 0, 2, 4).astype(np.int32)
    sizes = [int(np.prod(inst["dom_size"][inst["edge_var"][inst["factor_ptr"][f]:inst["factor_ptr"][f + 1]]]))
             for f in range(len(inst["factor_ptr"]) - 1)]
    inst["tables"] = np.random.default_rng(1).random(int(np.sum(sizes)))
    inst["unary"] = np.zeros(int(inst["dom_size"].sum()))
    V = len(inst["dom_size"])
    part = imbalanced_owner(V, world) if partition == "imbalanced" else partition
    owner = resolve_owner(inst, world, part)
    shards = [build_mgm2_shard(inst, r, world, owner, var_rank=inst["var_rank"]) for r in range(world)]
    G = layout_from_instance(inst)
    gp, gi = distinct_neighbours(G)
    for a, s in enumerate(shards):
        L = s.layout
        order = np.asarray(L.var_order, dtype=np.int64)
        gid_int = s.local_global_id[order]
        # neighbour lists of the owned variables equal the single problem's (global ids, same order)
        for c in range(s.n_own_vars):
            i = L.var_perm[c]
            v = int(s.own_vars[c])
            gv = G.var_perm[v]
            want = np.asarray(G.var_order)[gi[gp[gv]:gp[gv + 1]]]
            assert np.array_equal(gid_int[s.nbr_idx[s.nbr_ptr[i]:s.nbr_ptr[i + 1]]], want), (a, v)
        # the receive lists cover every ghost exactly once; ghosts are never owned here
        assert sorted(s.recv_int.tolist()) == sorted(np.nonzero(s.ghost)[0].tolist())
        assert (owner[gid_int[s.recv_int]] != a).all() and (owner[gid_int[s.send_int]] == a).all()
        assert np.array_equal(s.var_rank, np.asarray(inst["var_rank"])[s.local_global_id])
        # the owners' ids of my ghosts, as ShardedMgm2 learns them, name the same global variables
        ids = np.concatenate([shards[b].send_int[sum(shards[b].send_split[:a]):sum(shards[b].send_split[:a + 1])]
                              for b in range(world)]) if len(s.recv_int) else np.zeros(0, np.int64)
        ol = s.owner_local_ids(ids)
        for i in range(L.n_vars):
            b = s.owner_rank[i]
            assert shards[b].local_global_id[shards[b].layout.var_order[ol[i]]] == gid_int[i]
        # offer prefixes: what a sends to b is what b unpacks, fits both slots, and covers every b-owned partner
        pos = 0
        dom = np.asarray(inst["dom_size"], dtype=np.int64)
        for b in range(world):
            n = s.send_split[b]
            assert n == shards[b].recv_split[a]
            off = sum(shards[b].recv_split[:a])
            assert np.array_equal(s.send_plen[pos:pos + n], shards[b].recv_plen[off:off + n])
            for k in range(pos, pos + n):
                u = int(gid_int[s.send_int[k]])
                nb = np.asarray(G.var_order)[gi[gp[G.var_perm[u]]:gp[G.var_perm[u] + 1]]]
                on_b = nb[owner[nb] == b]
                assert len(on_b) and s.send_plen[k] == dom[u] * dom[on_b].max()
            pos += n
        # partner translation: an offerer's partner reaches rank b as b's id when b owns it, else as -1
        xl_rank, xl_local = s.owner_rank, ol
        for k in range(len(s.send_int)):
            u = s.send_int[k]
            b = s.send_peer[k]
            for p in s.nbr_idx[s.nbr_ptr[u]:s.nbr_ptr[u + 1]]:
                tp = xl_local[p] if xl_rank[p] == b else -1
                if owner[gid_int[p]] == b:
                    sb = shards[b]
                    assert tp >= 0 and sb.local_global_id[sb.layout.var_order[tp]] == gid_int[p]
                    assert not sb.ghost[tp]
                else:
                    assert tp == -1


# ---- the sharded run over gloo ----

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _case(case):
    """(instance, parameters, precision, cycles, partition) of a named case."""
    kind = case[0]
    if kind == "fixture":
        inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, case[1] + ".npz"))
        return inst, dict(mode=meta["mode"], seed=meta["seed"], **meta["params"]), "f64", meta["n_cycles"], "blocks"
    _, precision, params, levels, partition = case
    inst = random_instance(300, 4 if not levels else 3, seed=11, levels=levels, isolated=4)
    return inst, params, precision, 10, partition


def _worker(rank, world, port, cases, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from pydcop_b200.multigpu_mgm2 import ShardedMgm2
        out = []
        for case in cases:
            inst, params, precision, cycles, partition = _case(case)
            if partition == "imbalanced":
                partition = imbalanced_owner(len(inst["dom_size"]), world, seed=4)
            sm = ShardedMgm2(inst, rank, world, torch.device("cpu"), precision=precision,
                             engine_factory=HostShardMgm2, partition=partition, var_rank=inst.get("var_rank"),
                             **params).init()
            traj = [(sm.local_record(), sm.values())]
            for _ in range(cycles):
                sm.step()
                traj.append((sm.local_record(), sm.values()))
            out.append((traj, sm.cycle))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL " + repr(e) + traceback.format_exc(), None))


def _run(world, cases):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in res:
        assert status == "ok", (rank, status)
    return [r[2] for r in sorted(res, key=lambda r: r[0])]


def _check(shims, world, cases):
    per_rank = _run(world, cases)
    for ci, case in enumerate(cases):
        inst, params, precision, cycles, _ = _case(case)
        dt = np.float64 if precision == "f64" else np.float32
        L = layout_from_instance(inst)
        kw = dict(params, var_rank=inst.get("var_rank"))
        single = HostMgm2Single(L, precision, **kw).init()
        o = Mgm2Oracle(inst, dt, **params).init()
        V = L.n_vars
        moved = 0
        for k in range(cycles + 1):
            if k:
                single.step()
                o.step()
            want = single.state()
            assert np.array_equal(want["value"], o.values()[0]), (case, k)
            got = {key: np.full(V, -7, dtype=np.float64) for key in KEYS}
            for rank in range(world):
                traj, cyc = per_rank[rank][ci]
                (ids, rec), allval = traj[k]
                assert np.array_equal(allval, o.values()[0]), (case, k, rank)
                for key in KEYS:
                    got[key][ids] = rec[key]
            for key in KEYS:
                if key in ("cost", "gain"):
                    conn = np.diff(distinct_neighbours(L)[0])[L.var_perm] > 0 if key == "gain" else np.ones(V, bool)
                    assert np.array_equal(got[key].astype(dt)[conn], want[key].astype(dt)[conn]), (case, k, key)
                else:
                    assert np.array_equal(got[key].astype(np.int64), want[key].astype(np.int64)), (case, k, key)
            if k:
                moved += int((want["value"] != prev).sum())
            prev = want["value"]
        assert all(per_rank[rank][ci][1] == single.cycle for rank in range(world)), case
        if case[0] != "fixture":
            assert moved > 0, case


def test_sharded_mgm2_reproduces_every_fixture_over_gloo(shims):
    _check(shims, 2, [("fixture", name) for name in golden_names("mgm2_")])


RANDOM = [
    ("random", "f64", dict(mode="min", favor="unilateral", threshold=0.5, seed=5), 0, "blocks"),
    ("random", "f32", dict(mode="min", favor="no", threshold=0.4, seed=6), 0, "multilevel"),
    ("random", "f32", dict(mode="max", favor="coordinated", threshold=0.7, seed=7), 0, "imbalanced"),
    ("random", "f64", dict(mode="min", favor="no", threshold=0.5, seed=8), 2, "blocks"),
    ("random", "f32", dict(mode="max", favor="coordinated", threshold=1.0, seed=9), 3, "imbalanced"),
    ("random", "f64", dict(mode="min", favor="unilateral", threshold=0.0, seed=10), 2, "blocks"),
    ("random", "f64", dict(mode="min", favor="no", threshold=0.5, seed=12, stop_cycle=6), 2, "blocks"),
]


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_mgm2_equals_single_process_over_gloo(shims, world):
    """Float and tie-rich integer costs, f64 and f32, threshold 0 / 1, all three favor modes, max mode, isolated and
    unary-only variables, stop_cycle, blocks / multilevel / imbalanced partitions."""
    _check(shims, world, RANDOM)


def _solve_worker(rank, world, port, params, kw, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from pydcop_b200 import solve as S
        from test_solve_distributed_gloo import SPLIT
        res = S.solve(SPLIT, "mgm2", params, precision="f64", sharded_kwargs=dict(engine_factory=HostShardMgm2), **kw)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", res))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL " + repr(e) + traceback.format_exc(), None))


@pytest.mark.parametrize("params,kw", [({"stop_cycle": 12, "favor": "no"}, dict(seed=3, partition="blocks")),
                                       ({"stop_cycle": 9, "threshold": 0.8}, dict(partition="multilevel"))])
def test_distributed_solve_mgm2_equals_single_process(shims, params, kw):
    from pydcop_b200 import solve as S
    from test_solve_distributed_gloo import SPLIT
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_solve_worker, args=(r, world, port, params, kw, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in res:
        assert status == "ok", (rank, status)
    a, b = res[0][2], res[1][2]
    assert a["assignment"] == b["assignment"] and a["n_gpus"] == 2

    def single_engine(kind, layout, inst, p):
        e = HostMgm2Single(layout, "f64", mode=p["mode"], threshold=p["threshold"], favor=p["favor"],
                           stop_cycle=p["stop_cycle"], seed=p["seed"], var_rank=inst["var_rank"])

        class Run:
            cycle = property(lambda s: e.cycle)

            def init(s):
                e.init()

            def step(s, n):
                for _ in range(n):
                    e.step()

            def values(s):
                return e.state()["value"], None
        return Run()

    single = S.solve(SPLIT, "mgm2", params, precision="f64", engine_factory=single_engine,
                     **dict({k: v for k, v in kw.items() if k != "partition"}, seed=kw.get("seed", 0)))
    assert a["assignment"] == single["assignment"] and a["cost"] == pytest.approx(single["cost"], rel=1e-12)
    assert a["cycle"] == single["cycle"] and a["status"] == single["status"] == "FINISHED"
