"""GPU: the sharded MGM-2 path emulated on ONE device: `world` shard engines live in one process on cuda:0 and move
their five exchanges per cycle through an in-process copy that follows exactly the per-peer blocks of the NCCL
all_to_all (the phase, pack and unpack kernels are the real ones).  Every cycle must equal the single-GPU
Mgm2Engine: value, cost, gain, committed, partner (as a global id) and GO of every variable."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KEYS = ("value", "cost", "gain", "committed", "partner", "go")


def _fabric(shards, x, phase=True):
    """Exchange x: every shard's phase kernel and pack (unless phase=False), the per-peer blocks copied as the
    all_to_all moves them, every shard's unpack."""
    import torch
    if phase:
        for s in shards:
            s.engine.shard_phase(x)
    torch.cuda.synchronize()
    for a, sa in enumerate(shards):
        so = np.concatenate([[0], np.cumsum(sa.shard.splits(x)[0])]).astype(int)
        for b, sb in enumerate(shards):
            ro = np.concatenate([[0], np.cumsum(sb.shard.splits(x)[1])]).astype(int)
            n = so[b + 1] - so[b]
            assert n == ro[a + 1] - ro[a]
            if n:
                sb.engine.recv_buf[x][ro[a]:ro[a + 1]] = sa.engine.send_buf[x][so[b]:so[b + 1]]
    for s in shards:
        s.engine.shard_unpack(x)


def _attach(shards):
    world = len(shards)
    for a, s in enumerate(shards):
        ids = [shards[b].shard.send_int[sum(shards[b].shard.send_split[:a]):sum(shards[b].shard.send_split[:a + 1])]
               for b in range(world)]
        s.attach(np.concatenate(ids) if ids else np.zeros(0, np.int64))


def _single_state(e):
    L, n = e.layout, e.layout.n_vars
    out = {k: L.vars_to_canonical(getattr(e, k)[:n].cpu().numpy()) for k in KEYS}
    p = out["partner"].astype(np.int64)
    out["partner"] = np.where(p >= 0, np.asarray(L.var_order)[np.maximum(p, 0)], -1)
    return out


def _sharded_state(shards, V):
    got = {k: np.full(V, -7, dtype=np.float64) for k in KEYS}
    seen = np.zeros(V, dtype=int)
    for s in shards:
        ids, rec = s.local_record()
        seen[ids] += 1
        for k in KEYS:
            got[k][ids] = rec[k]
    assert (seen == 1).all()
    return got


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("levels,precision,params", [
    (0, "f32", dict(mode="min", favor="unilateral", threshold=0.5, seed=3)),
    (0, "f64", dict(mode="max", favor="coordinated", threshold=0.6, seed=4)),
    (3, "f32", dict(mode="min", favor="no", threshold=0.5, seed=5)),        # tie-rich integer costs
    (2, "f64", dict(mode="max", favor="no", threshold=0.4, seed=6)),
])
def test_sharded_mgm2_equals_single_gpu(levels, precision, params, world):
    import torch
    from pydcop_b200.engine import Mgm2Engine, distinct_neighbours
    from pydcop_b200.layout import layout_from_instance
    from pydcop_b200.multigpu_mgm2 import EXCHANGES, VALUES, ShardedMgm2
    from test_mgm2_hostshim import random_mgm2_instance
    inst = random_mgm2_instance(20000, 4 if not levels else 3, [2, 3, 1], seed=17, levels=levels)
    V = len(inst["dom_size"])
    dt = np.float64 if precision == "f64" else np.float32
    L = layout_from_instance(inst)
    single = Mgm2Engine(L, precision=precision, var_rank=inst["var_rank"], **params).init()
    conn = np.diff(distinct_neighbours(L)[0])[L.var_perm] > 0
    shards = [ShardedMgm2(inst, r, world, "cuda:0", precision=precision, var_rank=inst["var_rank"], **params)
              for r in range(world)]
    _attach(shards)
    for s in shards:
        s.engine.shard_init()           # init kernel, then the pack of the values
    _fabric(shards, VALUES, phase=False)
    torch.cuda.synchronize()
    assert np.array_equal(_sharded_state(shards, V)["value"], _single_state(single)["value"])
    moved = pairs = 0
    for k in range(8):
        prev = _single_state(single)["value"]
        single.step()
        for x in range(EXCHANGES):
            _fabric(shards, x)
        torch.cuda.synchronize()
        want, got = _single_state(single), _sharded_state(shards, V)
        for key in KEYS:
            if key in ("cost", "gain"):
                m = conn if key == "gain" else np.ones(V, bool)
                assert np.array_equal(got[key].astype(dt)[m], want[key].astype(dt)[m]), (k, key)
            else:
                assert np.array_equal(got[key].astype(np.int64), want[key].astype(np.int64)), (k, key)
        moved += int((want["value"] != prev).sum())
        pairs += int(want["go"].sum())
    assert moved > 0 and pairs > 0
    assert all(s.cycle == single.cycle for s in shards) and shards[0].shard.n_boundary > 0


def _peer_plans(shards, timeout_s=10.0):
    """The NVLink transport of Mgm2PeerPush for shards that share one device and one process: the peers' receive
    buffers and epoch flags are plain device addresses, so no CUDA IPC is needed."""
    import torch
    from pydcop_b200 import _cabi
    world = len(shards)
    flags = [torch.zeros(world, dtype=torch.int64, device="cuda:0") for _ in shards]
    keep = []
    for a, s in enumerate(shards):
        sh = s.shard
        peers = [b for b in range(world) if b != a and (sh.send_split[b] or sh.recv_split[b])]
        err = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        counter = torch.zeros(1, dtype=torch.int32, device="cuda:0")
        sync = _cabi.FgPeerSync()
        sync.n_peers, sync.my_rank, sync.dev_flags = len(peers), a, flags[a].data_ptr()
        for i, b in enumerate(peers):
            sync.peer_rank[i] = b
            sync.peer_slot[i] = flags[b].data_ptr() + 8 * a
        sync.dev_error, sync.timeout_ns = err.data_ptr(), int(timeout_s * 1e9)
        plan = _cabi.FgMgm2PeerPlan()
        esize = s.engine.send_buf[0].element_size()
        for x in range(len(s.engine.send_buf)):
            send = sh.splits(x)[0]
            src = np.concatenate([[0], np.cumsum(send)])
            k = 0
            for b in range(world):
                if b == a or not send[b]:
                    continue
                start = int(np.concatenate([[0], np.cumsum(shards[b].shard.splits(x)[1])])[a])
                plan.src[x][k], plan.n_elems[x][k] = int(src[b]), int(send[b])
                plan.dst[x][k] = shards[b].engine.recv_buf[x].data_ptr() + start * esize
                k += 1
            plan.n_blocks[x] = k
        plan.dev_counter, plan.sync = counter.data_ptr(), sync
        s.engine.shard_attach_peer(plan)
        keep.append((err, counter))
    return flags, keep


@pytest.mark.parametrize("world,precision,stop_cycle,steps", [(2, "f32", 0, [3, 4]), (4, "f64", 6, [4, 4])])
def test_sharded_mgm2_device_step_equals_single_gpu(world, precision, stop_cycle, steps):
    """fg_mgm2_shard_step (phase -> pack -> copy into the peers' receive buffers + release -> wait -> unpack, five
    epochs per cycle) with every shard on its own stream of one device, against the single-GPU engine."""
    import torch
    from pydcop_b200.engine import Mgm2Engine
    from pydcop_b200.layout import layout_from_instance
    from pydcop_b200.multigpu_mgm2 import VALUES, ShardedMgm2
    from test_mgm2_hostshim import random_mgm2_instance
    inst = random_mgm2_instance(20000, 3, [2, 3, 1], seed=29, levels=3)
    params = dict(mode="min", favor="no", threshold=0.5, seed=8, stop_cycle=stop_cycle)
    single = Mgm2Engine(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **params).init()
    shards = [ShardedMgm2(inst, r, world, "cuda:0", precision=precision, var_rank=inst["var_rank"], **params)
              for r in range(world)]
    _attach(shards)
    for s in shards:
        s.engine.shard_init()
    _fabric(shards, VALUES, phase=False)
    _, keep = _peer_plans(shards)
    streams = [torch.cuda.Stream(device="cuda:0") for _ in shards]
    torch.cuda.synchronize()
    V = len(inst["dom_size"])
    for n in steps:
        for s, st in zip(shards, streams):
            with torch.cuda.stream(st):
                s.engine.shard_step(n)
        torch.cuda.synchronize()
        single.step(n)
        assert all(int(err.item()) == 0 for err, _ in keep)
        got = _sharded_state(shards, V)["value"]
        assert np.array_equal(got, _single_state(single)["value"])
        assert all(s.cycle == single.cycle for s in shards)
    assert single.cycle == (min(sum(steps), stop_cycle - 1) if stop_cycle else sum(steps))
