"""solve_batch with one parameter dict per problem on the device: every problem of a batch gets what solve() gives it
with its own parameters and seed, whether its parameters run inside one union (DSA, A-DSA, MGM-2, GDBA, MixedDSA
through parameter sets; MGM's break_mode; MaxSum's noise) or split the batch into groups (MaxSum's damping)."""
import ctypes as C

import numpy as np
import pytest
import torch

from pydcop_b200 import _cabi, batch, ingest
from pydcop_b200.engine import make_engine
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.solve import check_params, name_rank, solve, solve_batch
from test_batch_cpu import batch_problems
from test_gpu_zz_batch import _against_solve

pytestmark = pytest.mark.gpu

SETS = {"dsa": [dict(variant=v, probability=p) for v, p in (("A", 0.3), ("B", 0.9), ("C", 0.6))]
        + [dict(variant="B", p_mode="arity"), dict(variant="C", p_mode="arity")],
        "adsa": [dict(variant=v, probability=p, period=t) for v, p, t in (("A", 0.4, 0.5), ("B", 0.8, 1.0),
                                                                            ("C", 0.6, 0.5), ("B", 0.2, 2.0))],
        "mgm": [dict(break_mode="lexic"), dict(break_mode="random")] * 2,
        "mgm2": [dict(favor=f, threshold=t) for f, t in (("unilateral", 0.5), ("no", 0.2), ("coordinated", 0.8),
                                                        ("no", 0.9), ("coordinated", 0.1))],
        "gdba": [dict(modifier=m, violation=v, increase_mode="T") for m, v in (("A", "NZ"), ("M", "NM"), ("A", "MX"),
                                                                                ("M", "NZ"), ("M", "MX"), ("A", "NM"))],
        "mixeddsa": [dict(variant=v, proba_hard=h, proba_soft=s) for v, h, s in (("A", 0.7, 0.5), ("B", 0.9, 0.2),
                                                                                  ("C", 0.3, 0.8), ("B", 0.5, 0.5))],
        "maxsum": [dict(noise=z) for z in (0.0, 0.01, 0.05, 0.1)]}


def _engines(monkeypatch):
    """The engines solve_batch builds, in order, with their parameter-set inputs."""
    import pydcop_b200.engine as E
    made, real = [], E.make_engine

    def spy(kind, layout, params, **kw):
        made.append((kind, kw.get("var_pset"), kw.get("psets")))
        return real(kind, layout, params, **kw)

    monkeypatch.setattr(E, "make_engine", spy)
    return made


def _run(kind, dcops, precision, monkeypatch, stop_cycle=25, trace=False):
    sets = SETS[kind]
    probs = [d for d in dcops for _ in sets]
    params = [dict(s, stop_cycle=stop_cycle) for _ in dcops for s in sets]
    seeds = [5 * i - 3 for i in range(len(probs))]
    made = _engines(monkeypatch)
    res = solve_batch(probs, kind, params, precision=precision, seed=seeds, trace=trace)
    assert len(made) == 1
    if kind in ("dsa", "adsa", "mgm2", "gdba", "mixeddsa"):
        assert made[0][1] is not None and len(made[0][2]) == len({batch.pset_key(check_params(kind, p))
                                                                   for p in params})
    return probs, params, seeds, res


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind", sorted(SETS))
def test_every_parameter_set_equals_solve(kind, precision, monkeypatch):
    dcops = [d for d in batch_problems(12, seed=110 + len(kind), hard=kind in ("mixeddsa", "gdba"), n_range=(20, 150))
             if len(d.arrays["tables"])][:6]
    assert len(dcops) == 6
    probs, params, seeds, res = _run(kind, dcops, precision, monkeypatch)
    for d, p, s, r in zip(probs, params, seeds, res):
        _against_solve(kind, d, r, p, precision=precision, seed=s)


def _uniform(n, dom, seed):
    return [ingest.from_arrays(random_factor_graph(60 + 10 * i, dom, 90 + 15 * i, 2, seed=seed + i, noise=0),
                               name=f"u{i}") for i in range(n)]


@pytest.mark.parametrize("cache", ["1", "0"])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind", ["dsa", "adsa"])
def test_mixed_variants_on_the_oriented_table_kernels(kind, precision, cache, monkeypatch):
    """All-binary unions over one domain size: the active-row kernel (cache 1) and the oriented-table kernel (cache 0)
    run with every variable reading its own variant."""
    monkeypatch.setenv("PYDCOP_B200_DSA_CACHE", cache)
    dcops = _uniform(6, 4, 300)
    probs, params, seeds, res = _run(kind, dcops, precision, monkeypatch)
    for d, p, s, r in zip(probs, params, seeds, res):
        _against_solve(kind, d, r, p, precision=precision, seed=s)


def test_maxsum_damping_sweep_splits_into_groups(monkeypatch):
    dcops = [d for d in batch_problems(8, seed=130, n_range=(20, 120)) if len(d.arrays["tables"])][:5]
    damp = (0.0, 0.5, 0.9)
    probs = [d for d in dcops for _ in damp]
    params = [dict(damping=x, stop_cycle=20) for _ in dcops for x in damp]
    made = _engines(monkeypatch)
    res = solve_batch(probs, "maxsum", params, precision="f32", seed=3)   # the seed of MaxSum's noise draws
    assert len(made) == len(damp) and all(vp is None for _, vp, _ in made)
    for d, p, r in zip(probs, params, res):
        _against_solve("maxsum", d, r, p, precision="f32", seed=3)


@pytest.mark.parametrize("kind", ["dsa", "mgm2", "gdba", "mixeddsa"])
def test_traces_equal_every_solve_trace(kind, monkeypatch):
    dcops = [d for d in batch_problems(8, seed=140, hard=kind in ("mixeddsa", "gdba"), n_range=(20, 100))
             if len(d.arrays["tables"])][:4]
    probs, params, seeds, res = _run(kind, dcops, "f64", monkeypatch, stop_cycle=15, trace=True)
    for d, p, s, r in zip(probs, params, seeds, res):
        t = solve(d, kind, p, precision="f64", seed=s, trace=True)["trace"]
        assert r["trace"]["cycle"] == t["cycle"] and r["trace"]["violation"] == t["violation"]
        assert r["trace"]["cost"] == pytest.approx(t["cost"], rel=1e-12, abs=1e-9)


@pytest.mark.parametrize("kind", ["dsa", "mgm2", "gdba", "mixeddsa"])
def test_create_refuses_a_set_index_in_host_memory_and_frees_its_table(kind):
    dcops = batch_problems(4, seed=150, hard=kind == "mixeddsa", n_range=(20, 60))
    checked = [check_params(kind, dict(SETS[kind][i], stop_cycle=5)) for i in range(4)]
    u = batch.build_union(dcops, list(range(4)), lambda d: (name_rank(d), None), 0.0, 1, checked)
    L = batch.union_layout(u, dcops)
    eng = make_engine(kind, L, checked[0], precision="f32", seed=1, var_rank=u.var_rank, var_global_id=u.var_global_id,
                      var_pset=u.var_pset, psets=u.psets)
    assert eng._desc.dev_var_pset and eng._desc.n_psets == 4
    d = type(eng._desc).from_buffer_copy(eng._desc)
    host = np.zeros(L.n_vars, dtype=np.uint16)
    d.dev_var_pset = host.ctypes.data
    fn = lambda name: getattr(eng.lib, f"fg_{kind}_{name}")  # noqa: E731
    h = C.c_void_p()
    torch.cuda.synchronize()
    rc = fn("create")(C.byref(d), C.byref(h))
    msg = (fn("last_error")(h) or b"").decode()
    fn("destroy")(h)
    assert rc == _cabi.FG_ERR_ARG, (rc, msg)
    assert msg == f"dev_var_pset is pageable host memory, not device memory of the handle's device {eng.device.index}"
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(50):    # every handle's device copy of the table is freed with it
        d = type(eng._desc).from_buffer_copy(eng._desc)
        assert fn("create")(C.byref(d), C.byref(h)) == _cabi.FG_OK
        fn("destroy")(h)
    assert torch.cuda.mem_get_info()[0] >= free0 - (2 << 20)
    eng.init().step(3)
    torch.cuda.synchronize()
    eng.close()
