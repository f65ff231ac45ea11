#!/usr/bin/env python
"""Sharded MGM-2 throughput on the C4-shaped instance (generators.config_c4: d = 20, degree 6, binary constraints
with integer costs), one process per GPU under torchrun:

    torchrun --nproc_per_node N tools/mgm2_sharded_throughput.py [--scaling strong|weak] [--vars N]
             [--halo nccl,p2p] [--precision f32|f64] [--steps K] [--warmup W] [--repeats R] [--partition blocks]

strong: one instance of --vars variables split over the N ranks; weak: --vars x N variables.  For every halo mode
each rank times `--repeats` windows of `--steps` cycles with CUDA events after `--warmup` cycles and prints one JSON
line: milliseconds per cycle of every window and their median, the boundary bytes it sends per cycle (all five
exchanges; the offer prefixes go out whether or not the variable offered), its variables and ghosts, the card's name
and its power limit.  Exits non-zero without a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def power_limit_w(device_index):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(device_index)], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main(argv=None):
    ap = argparse.ArgumentParser(prog="mgm2_sharded_throughput")
    ap.add_argument("--scaling", default="strong", choices=["strong", "weak"])
    ap.add_argument("--vars", type=int, default=1_000_000)
    ap.add_argument("--halo", default="nccl,p2p")
    ap.add_argument("--precision", default="f32", choices=["f32", "f64"])
    ap.add_argument("--partition", default="blocks")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        print("mgm2_sharded_throughput: no CUDA device (the MGM-2 engine runs on the GPU only)", file=sys.stderr)
        return 2
    import torch.distributed as dist
    from pydcop_b200.generators import config_c4
    from pydcop_b200.multigpu_mgm2 import EXCHANGES, ShardedMgm2

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    n = args.vars * (world if args.scaling == "weak" else 1)
    inst = config_c4(args.seed, n_vars=n)
    esize = 8 if args.precision == "f64" else 4
    for mode in [m for m in args.halo.split(",") if m]:
        sm = ShardedMgm2(inst, rank, world, dev, precision=args.precision, halo=mode, partition=args.partition,
                         seed=args.seed + 1).init()
        used = "p2p" if sm.peer is not None else "nccl"
        sm.step(args.warmup)
        torch.cuda.synchronize()
        dist.barrier()
        ms = []
        for _ in range(args.repeats):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            sm.step(args.steps)
            t1.record()
            t1.synchronize()
            ms.append(t0.elapsed_time(t1) / args.steps)
        sm.check()
        sent = sum(sum(sm.shard.splits(x)[0]) for x in range(EXCHANGES)) * esize
        print(json.dumps({
            "workload": "mgm2_c4_sharded", "scaling": args.scaling, "n_vars": n, "world": world, "rank": rank,
            "halo": mode, "halo_used": used, "precision": args.precision, "partition": args.partition,
            "steps": args.steps, "warmup": args.warmup, "ms_per_cycle": [round(x, 3) for x in ms],
            "ms_per_cycle_median": round(float(np.median(ms)), 3), "own_vars": sm.shard.n_own_vars,
            "ghosts": int(sm.shard.layout.n_vars - sm.shard.n_own_vars), "boundary_bytes_per_cycle": int(sent),
            "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(local)}), flush=True)
        del sm
        torch.cuda.empty_cache()
        dist.barrier()
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
