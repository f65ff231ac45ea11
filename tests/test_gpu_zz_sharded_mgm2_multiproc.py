"""GPU (>= 2 devices): sharded MGM-2 in real processes, one per GPU, NCCL for the plumbing, in both halo modes: five
all_to_all per cycle, and the NVLink stores into the peers' receive buffers closed by the device-side epoch barrier
(fg_mgm2_shard_step).  The all-gathered assignment and the sharded solution cost must equal the single-GPU
Mgm2Engine's, and no barrier may time out.  Cases: several step() calls and a re-init (the epoch only grows),
stop_cycle, and an imbalanced partition (a fast rank's push must not be overwritten by a slow rank's kernels)."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, case, q):
    try:
        import torch
        import torch.distributed as dist
        from pydcop_b200.engine import Mgm2Engine
        from pydcop_b200.layout import layout_from_instance
        from pydcop_b200.multigpu_mgm2 import ShardedMgm2
        from test_mgm2_hostshim import random_mgm2_instance
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        n = case.get("n_vars", 20000)
        inst = random_mgm2_instance(n, 3, [2, 3, 1], seed=23, levels=3)
        part = case.get("partition", "blocks")
        if part == "imbalanced":             # rank 0 owns 85 % of the ids
            own = np.zeros(n, dtype=np.int32)
            tail = n - int(n * 0.85)
            own[n - tail:] = 1 + (np.arange(tail) % (world - 1))
            part = own
        kw = dict(precision=case.get("precision", "f32"), favor="no", threshold=0.5, seed=9,
                  stop_cycle=case.get("stop_cycle", 0), var_rank=inst["var_rank"])
        sh = ShardedMgm2(inst, rank, world, dev, halo=case["mode"], partition=part, **kw).init()
        cur = 0
        for steps in case.get("steps", [10]):
            if steps == "init":
                sh.init()
                cur = 0
                continue
            sh.step(steps)
            cur += steps
        sh.check()
        got = sh.values()
        cost = sh.solution_cost(2.0)         # table entries equal to 2 count as violations
        used = "p2p" if sh.peer is not None else "nccl"
        ok = True
        if rank == 0:
            ref = Mgm2Engine(layout_from_instance(inst), device=dev, **kw).init().step(cur)
            ok = bool(np.array_equal(got, ref.values()[0])) and sh.cycle == ref.cycle
            want = ref.solution_cost(2.0)
            ok = ok and cost[1] == want[1] and cost[1] > 0 and abs(cost[0] - want[0]) <= 1e-6 * max(1.0, abs(want[0]))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok" if ok else "MISMATCH", used))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL " + repr(e) + traceback.format_exc(), "?"))


CASES = {
    "nccl": dict(mode="nccl", partition="multilevel"),
    "p2p": dict(mode="p2p", partition="multilevel", precision="f64"),
    "p2p-steps-reinit": dict(mode="p2p", steps=[1, 3, "init", 2, 5, 4]),
    "p2p-stop-cycle": dict(mode="p2p", stop_cycle=6, steps=[4, 4, 2]),
    "nccl-stop-cycle": dict(mode="nccl", stop_cycle=6, steps=[4, 4, 2]),
    "p2p-imbalanced": dict(mode="p2p", partition="imbalanced", n_vars=100000, steps=[12]),
}


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("name", sorted(CASES))
def test_sharded_mgm2_processes_match_single_gpu(name, world):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    case = CASES[name]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = [q.get(timeout=300) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=20)
            if p.is_alive():
                p.kill()
    assert all(r[1] == "ok" for r in results), results
    assert all(r[2] == case["mode"] for r in results), results
