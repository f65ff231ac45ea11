"""bench.py's contract on CPU: the reference arm prints ONE JSON line with the required keys; the
GPU arm refuses to run without a device (no CPU fallback); under a multi-rank launch only rank 0
of the reference arm prints.  (The GPU arm's own line is checked where it runs, on the H100.)"""
import json
import os
import subprocess
import sys

from conftest import ROOT

BENCH = os.path.join(ROOT, "bench.py")


def _run(args, env=None, timeout=600):
    e = dict(os.environ, **(env or {}))
    return subprocess.run([sys.executable, BENCH, *args], capture_output=True, text=True, timeout=timeout, env=e)


def test_reference_arm_prints_one_contract_line():
    r = _run(["--impl", "reference", "--steps", "2", "--warmup", "1", "--vars-per-gpu", "2000"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["steps"] == 2 and d["warmup"] == 1 and d["value"] > 0
    assert d["metric"] == "maxsum_edge_message_updates_per_s" and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and d["config"]["n_vars"] == 2000


def test_reference_arm_other_ranks_exit_quietly():
    r = _run(["--impl", "reference", "--steps", "1", "--warmup", "1", "--vars-per-gpu", "500", "--gpus", "2"],
             env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert r.returncode == 0 and not [ln for ln in r.stdout.splitlines() if ln.startswith("{")]


def test_gpu_arm_refuses_to_run_without_a_device():
    import torch
    if torch.cuda.is_available():
        return
    r = _run(["--steps", "1", "--warmup", "1"])
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_reference_arm_sets_its_threads_explicitly_and_shares_the_gpu_arms_config():
    """torchrun exports OMP_NUM_THREADS=1: the CPU arm must not inherit it silently (VERDICT r1: it printed
    "128 threads" while running one), and its `config` is the dict the GPU arm prints at the same N."""
    import bench
    r = _run(["--impl", "reference", "--steps", "2", "--warmup", "1", "--vars-per-gpu", "1000", "--gpus", "2"],
             env={"RANK": "0", "WORLD_SIZE": "2", "LOCAL_RANK": "0", "OMP_NUM_THREADS": "1",
                  "PYDCOP_B200_CPU_THREADS": "3"})
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][0])
    assert d["cpu_baseline"]["cores"] == 3 and "OpenMP 3 threads" in d["cpu_baseline"]["sample"]
    assert "median of" in d["cpu_baseline"]["sample"]
    os.environ.pop("PYDCOP_B200_PARTITION", None)
    assert d["config"] == bench.workload_config(2000, 2)
    assert d["n_gpus"] == 2 and d["config"]["n_vars"] == 2000
