"""solve_batch with one seed per problem on the device: every run of a batch gets what solve() gives that problem with
that seed alone, the repeats of one problem follow different streams, and create refuses a key array in host memory."""
import ctypes as C

import numpy as np
import pytest
import torch

from pydcop_b200 import _cabi, batch
from pydcop_b200.engine import make_engine
from pydcop_b200.solve import name_rank, solve_batch
from test_batch_cpu import batch_problems
from test_gpu_zz_batch import _against_solve

pytestmark = pytest.mark.gpu

FAMILIES = [("dsa", {}), ("dsa", {"variant": "C", "p_mode": "arity"}), ("adsa", {}), ("mgm", {}),
            ("mgm2", {"favor": "no"}), ("gdba", {"violation": "NM", "increase_mode": "T"}), ("mixeddsa", {})]
SEEDS = [0, 1, 29, -3, 2 ** 63 + 5]


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind,params", FAMILIES, ids=lambda x: x if isinstance(x, str) else "-".join(map(str, x.values())))
def test_every_seed_of_every_problem_equals_solve(kind, params, precision):
    dcops = [d for d in batch_problems(12, seed=70 + len(kind), hard=kind in ("mixeddsa", "gdba"), n_range=(20, 150))
             if len(d.arrays["tables"])][:6]
    assert len(dcops) == 6
    probs = [d for d in dcops for _ in SEEDS]
    seeds = SEEDS * len(dcops)
    p = dict(params, stop_cycle=25)
    res = solve_batch(probs, kind, p, precision=precision, seed=seeds)
    for d, s, r in zip(probs, seeds, res):
        _against_solve(kind, d, r, p, precision=precision, seed=s)
    for k in range(len(dcops)):
        runs = {tuple(sorted(r["assignment"].items())) for r in res[k * len(SEEDS):(k + 1) * len(SEEDS)]}
        assert len(runs) >= 2, (kind, k)


@pytest.mark.parametrize("kind", ["dsa", "mgm", "mgm2", "gdba", "mixeddsa"])
def test_mixed_objectives_with_seeds_cut_into_several_engines(kind):
    dcops = batch_problems(12, seed=80, modes=("min", "max", "max"), hard=kind == "mixeddsa", n_range=(20, 150))
    probs = [d for d in dcops for _ in range(3)]
    seeds = [7 * i + 2 for i in range(len(probs))]
    assert len(batch.groups(probs, max_vars=500)) >= 4
    p = {"stop_cycle": 20}
    res = solve_batch(probs, kind, p, precision="f32", seed=seeds, max_vars=500)
    for d, s, r in zip(probs, seeds, res):
        _against_solve(kind, d, r, p, precision="f32", seed=s)


@pytest.mark.parametrize("kind", ["dsa", "mgm", "mgm2", "gdba", "mixeddsa"])
def test_create_refuses_keys_in_host_memory(kind):
    dcops = batch_problems(4, seed=90, hard=kind == "mixeddsa", n_range=(20, 60))
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d), None), 0.0, [1, 2, 3, 4])
    L = batch.union_layout(u, dcops)
    eng = make_engine(kind, L, {"stop_cycle": 5}, precision="f32", seed=1, var_rank=u.var_rank,
                      var_global_id=u.var_global_id, var_seed=u.var_seed)
    assert eng._desc.dev_var_seed
    d = type(eng._desc).from_buffer_copy(eng._desc)
    host = np.full(L.n_vars, 7, dtype=np.uint64)
    d.dev_var_seed = host.ctypes.data
    fn = lambda name: getattr(eng.lib, f"fg_{kind}_{name}")  # noqa: E731
    h = C.c_void_p()
    torch.cuda.synchronize()
    rc = fn("create")(C.byref(d), C.byref(h))
    msg = (fn("last_error")(h) or b"").decode()
    fn("destroy")(h)
    assert rc == _cabi.FG_ERR_ARG, (rc, msg)
    assert msg == f"dev_var_seed is pageable host memory, not device memory of the handle's device {eng.device.index}"
    eng.init().step(3)
    torch.cuda.synchronize()
    eng.close()
