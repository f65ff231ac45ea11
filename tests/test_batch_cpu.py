"""Batches (pydcop_b200.batch, solve.solve_batch) without a GPU.

1. The kernel SOURCE of every batched family, run on the CPU through the host shims (tests/hostshim/*_host.cpp) on
   one union layout with per-problem var_global_id / var_rank: every problem's slice of the state equals its own run
   at every cycle, bit for bit, in f32 and f64.
2. solve_batch's host logic through the engine seam: grouping, cutting, order, refusals, the CLI."""
import ctypes as C
import functools
import json
import os
import subprocess
from unittest import mock

import numpy as np
import pytest

import test_gdba_hostshim as tg
import test_mgm2_hostshim as tm2
import test_mgm_hostshim as tm
import test_mixeddsa_hostshim as tmx
from conftest import ROOT
from pydcop_b200 import batch, engine as eng_mod, ingest
from pydcop_b200.generators import mixed_shape_graph
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import main, name_rank, solve, solve_batch
from test_dsa_generic_hostshim import HostDsa
from test_maxsum_generic_hostshim import CUDA_INC, HostMaxSum

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA toolkit headers not present")


# ------------------------------------------------------------------------------------------------------------------
# problems
# ------------------------------------------------------------------------------------------------------------------
def batch_problem(seed, mode="min", hard=False, n_range=(6, 40)):
    """One small problem, its shape drawn from `seed`: one domain size or mixed ones, binary factors plus ternary and
    unary-scope ones on some, integer or float tables and variable costs, three variables without constraints, initial
    values on about a third of the variables; every seventh problem has no constraints at all.  `hard`: +inf (min) or
    -inf (max) on the equal-value entries of half the binary and ternary constraints."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(*n_range))
    ints = seed % 2 == 0
    if seed % 7 == 3:
        dom = rng.integers(1, 6, n).astype(np.int32)
        inst = dict(dom_size=dom, factor_ptr=np.zeros(1, np.int64), edge_var=np.zeros(0, np.int32),
                    tables=np.zeros(0, np.float32))
    else:
        doms = [int(rng.integers(2, 6))] if seed % 3 else [2, 3, 5]
        shapes = [(2, int(n * 1.3))] + ([(3, n // 5)] if seed % 4 == 0 else []) + ([(1, n // 6)] if seed % 5 == 1 else [])
        inst = mixed_shape_graph(n - 3, doms, shapes, seed=seed, noise=0, int_tables=ints)
        inst["dom_size"] = np.concatenate([inst["dom_size"], rng.integers(1, 5, 3)]).astype(np.int32)
    dom = inst["dom_size"]
    n_un = int(dom.sum())
    inst["unary"] = rng.integers(0, 4, n_un).astype(np.float64) if ints else rng.uniform(0, 2, n_un)
    inst["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, 1 << 30, n) % dom, -1).astype(np.int32)
    if hard:
        fp, ev = inst["factor_ptr"], inst["edge_var"]
        t = np.asarray(inst["tables"], dtype=np.float64).copy()
        off = 0
        for f in range(len(fp) - 1):
            sc = ev[fp[f]:fp[f + 1]]
            shape = tuple(int(dom[u]) for u in sc)
            size = int(np.prod(shape, dtype=np.int64))
            if len(sc) > 1 and rng.uniform() < 0.5:
                idx = np.indices(shape).reshape(len(sc), -1)
                t[off:off + size][(idx == idx[0]).all(0)] = np.inf if mode == "min" else -np.inf
            off += size
        inst["tables"] = t
    return ingest.from_arrays(inst, name=f"p{seed}", objective=mode)


def batch_problems(n, seed=0, modes=("min",), hard=False, n_range=(6, 40)):
    return [batch_problem(seed * 1000 + i, modes[i % len(modes)], hard, n_range) for i in range(n)]


# ------------------------------------------------------------------------------------------------------------------
# 1. kernel source: the union against every problem's own run
# ------------------------------------------------------------------------------------------------------------------
def _shim(name):
    """tests/hostshim/<name>_host.cpp built for this file (the kernel headers are its dependencies)."""
    src = os.path.join(ROOT, "tests", "hostshim", f"{name}_host.cpp")
    so = os.path.join(ROOT, "tests", "hostshim", "_build", f"batch_{name}_host.so")
    csrc = os.path.join(ROOT, "pydcop_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "pydcop_b200.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-w", "-I", CUDA_INC, "-shared", "-fPIC",
                        "-o", so, src], check=True, capture_output=True)
    lib = C.CDLL(so)
    for fn in ("gdba_host_cycle", "mixeddsa_host_cycle"):
        if hasattr(lib, fn):
            getattr(lib, fn).argtypes = [C.c_void_p, C.c_int64]
    return lib


_PLANS = {"mgm": (tm, "mgm_plan"), "mgm2": (tm2, "mgm2_plan"), "gdba": (tg, "gdba_plan"),
          "mixeddsa": (tmx, "mixeddsa_plan")}
_HOSTS = {"mgm": (tm.HostMgm, "mgm"), "mgm2": (tm2.HostMgm2, "mgm2"), "gdba": (tg.HostGdba, "gdba"),
          "mixeddsa": (tmx.HostMixedDsa, "mixeddsa")}


@functools.lru_cache(maxsize=None)
def shim(name):
    return _shim(name)


def host_engine(kind, layout, inst, precision, mode, params, seed, var_rank=None, var_global_id=None):
    """The host-shimmed engine of `kind` over `layout`: the engine's own plan (with var_global_id) stepped by the
    kernel source."""
    if kind in ("dsa", "adsa"):
        return HostDsa(inst, precision=precision, mode=mode, seed=seed, var_global_id=var_global_id,
                       var_costs=kind == "adsa", **params)
    if kind == "maxsum":
        return HostMaxSum(layout, precision=precision, mode=mode, **params)
    module, plan = _PLANS[kind]
    cls, lib = _HOSTS[kind]
    with mock.patch.object(module, plan, functools.partial(getattr(eng_mod, plan), var_global_id=var_global_id)):
        return cls(shim(lib), layout, precision=precision, mode=mode, seed=seed, var_rank=var_rank, **params)


def _values(e):
    out = e.values()
    return out if isinstance(out, tuple) else (out,)


def check_union(kind, dcops, precision, params, n_cycles=12, seed=5, noise=0.0):
    mode = dcops[0].objective
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d), None), noise, seed)
    L = batch.union_layout(u, dcops)
    whole = host_engine(kind, L, u.inst, precision, mode, params, seed, u.var_rank, u.var_global_id).init()
    alone = []
    for d in dcops:
        inst = d.instance()
        inst["unary"] = ingest.add_noise(inst["unary"], noise, seed)
        alone.append(host_engine(kind, build_layout(**inst), inst, precision, mode, params, seed, name_rank(d)).init())
    moved = 0
    for k in range(n_cycles + 1):
        if k:
            whole.step()
            for e in alone:
                e.step()
        got = _values(whole)
        for i, e in enumerate(alone):
            a, b = u.var_start[i], u.var_start[i + 1]
            for x, y in zip(got, _values(e)):
                assert np.array_equal(x[a:b], y, equal_nan=True), (kind, i, k)
        moved += k > 0 and int((got[0] != prev).sum())
        prev = got[0].copy()
    assert moved > 0


FAMILY_CASES = [("dsa", dict(variant="B", stop_cycle=0)), ("dsa", dict(variant="A", p_mode="arity")),
                ("adsa", dict(variant="C")), ("mgm", {}),
                ("mgm2", dict(favor="unilateral")), ("mgm2", dict(favor="no", threshold=0.8)),
                ("mgm2", dict(favor="coordinated")),
                ("gdba", dict(modifier="A", violation="NZ", increase_mode="E")),
                ("gdba", dict(modifier="M", violation="NM", increase_mode="R")),
                ("gdba", dict(modifier="A", violation="MX", increase_mode="C")),
                ("gdba", dict(modifier="M", violation="NZ", increase_mode="T")),
                ("maxsum", dict(damping=0.5))]


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("kind,params", FAMILY_CASES, ids=lambda x: x if isinstance(x, str) else "-".join(map(str, x.values())))
@pytest.mark.parametrize("mode", ["min", "max"])
def test_union_kernel_source_equals_every_problem_alone(kind, params, precision, mode):
    check_union(kind, batch_problems(9, seed=len(kind) + len(params), modes=(mode,)), precision, params)


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("mode", ["min", "max"])
def test_union_kernel_source_mixeddsa_hard_constraints(precision, mode):
    check_union("mixeddsa", batch_problems(9, seed=3, modes=(mode,), hard=True), precision, dict(variant="B"))
    check_union("mixeddsa", batch_problems(7, seed=4, modes=(mode,), hard=True), precision,
                dict(variant="A", proba_hard=0.9, proba_soft=0.3))


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_union_kernel_source_maxsum_with_noise(precision):
    """MaxSum's noise is drawn per problem before the union, as solve() draws it for the problem alone."""
    check_union("maxsum", batch_problems(8, seed=7), precision, dict(damping=0.5, start_messages="all"), noise=0.01)


def test_union_arrays():
    dcops = batch_problems(5, seed=11)
    u = batch.build_union(dcops, [0, 2, 4], lambda d: (name_rank(d), None))
    assert list(u.var_start) == list(np.cumsum([0] + [dcops[i].n_vars for i in (0, 2, 4)]))
    assert np.array_equal(u.var_global_id, np.concatenate([np.arange(dcops[i].n_vars) for i in (0, 2, 4)]))
    assert len(u.seg_factor) == len(u.inst["factor_ptr"]) - 1 and len(u.seg_var) == u.var_start[-1]
    L = batch.union_layout(u, dcops)
    for k, i in enumerate((0, 2, 4)):           # problem i's factors, cut back out of the union, are its own
        a = dcops[i].arrays
        f = np.nonzero(u.seg_factor == k)[0]
        fp, to = u.inst["factor_ptr"], u.inst["table_off"]
        assert np.array_equal(np.concatenate([u.inst["edge_var"][fp[g]:fp[g + 1]] for g in f] or [[]]) - u.var_start[k],
                              a["edge_var"])
        assert np.array_equal(np.concatenate([u.inst["tables"][to[g]:to[g + 1]] for g in f] or [[]]),
                              np.asarray(a["tables"], dtype=u.inst["tables"].dtype))
    assert L.n_vars == u.var_start[-1]


# ------------------------------------------------------------------------------------------------------------------
# 2. solve_batch through the engine seam
# ------------------------------------------------------------------------------------------------------------------
def factory(kind, layout, inst, params):
    p = {k: v for k, v in params.items() if k not in ("mode", "seed", "noise")}
    return host_engine(kind, layout, inst, "f64", params["mode"], p, params["seed"], inst.get("var_rank"),
                       inst.get("var_global_id"))


def _same(r, s):
    assert r["assignment"] == s["assignment"]
    assert (r["status"], r["cycle"], r["violation"]) == (s["status"], s["cycle"], s["violation"])
    assert r["cost"] == pytest.approx(s["cost"], rel=1e-12, abs=1e-12)
    assert set(r) == set(s)


@pytest.mark.parametrize("kind,params", [("dsa", {}), ("mgm", {}), ("mgm2", {}), ("gdba", {"increase_mode": "T"}),
                                         ("mixeddsa", {}), ("adsa", {}), ("maxsum", {})])
def test_solve_batch_equals_solve_with_mixed_objectives_and_cuts(kind, params):
    dcops = batch_problems(11, seed=21, modes=("min", "max", "min"), hard=kind == "mixeddsa")
    p = dict(params, stop_cycle=9)
    one = solve_batch(dcops, kind, p, seed=4, engine_factory=factory)
    cut = solve_batch(dcops, kind, p, seed=4, engine_factory=factory, max_vars=45)
    for d, r, c in zip(dcops, one, cut):
        s = solve(d, kind, p, seed=4, engine_factory=factory)
        _same(r, s)
        _same(c, s)
        assert r["n_gpus"] == 1 and r["time"] == one[0]["time"] and list(r["assignment"]) == list(d.var_names)


def test_groups_by_objective_and_size():
    dcops = batch_problems(7, seed=2, modes=("max", "min", "min"))
    n = [d.n_vars for d in dcops]
    assert batch.groups(dcops) == [[0, 3, 6], [1, 2, 4, 5]]
    cut = batch.groups(dcops, max_vars=max(n))
    assert sorted(i for g in cut for i in g) == list(range(7))
    for g in cut:
        assert len({dcops[i].objective for i in g}) == 1 and g == sorted(g)
        assert len(g) == 1 or sum(n[i] for i in g) <= max(n)
    assert batch.groups(dcops, max_vars=1) == [[0], [3], [6], [1], [2], [4], [5]]


def test_solve_batch_timeout():
    """The timeout bounds the whole batch: the group running when it expires stops at the cycle it reached, the
    groups after it report TIMEOUT at cycle 0."""
    import time
    dcops = batch_problems(4, seed=5)

    def slow(kind, layout, inst, params):
        e = factory(kind, layout, inst, params)
        step = e.step
        e.step = lambda n=1: (time.sleep(0.3), step(n))[1]
        return e
    res = solve_batch(dcops, "dsa", {"stop_cycle": 0}, timeout=0.2, engine_factory=slow, chunk=3,
                      max_vars=dcops[0].n_vars + dcops[1].n_vars)
    assert [(r["status"], r["cycle"]) for r in res] == [("TIMEOUT", 3)] * 2 + [("TIMEOUT", 0)] * 2
    res = solve_batch(dcops, "dsa", {"stop_cycle": 7}, timeout=600.0, engine_factory=factory, chunk=3)
    assert [(r["status"], r["cycle"]) for r in res] == [("FINISHED", 7)] * 4


@pytest.mark.parametrize("algo", ["dba", "dpop", "syncbb", "dba_gpu"])
def test_refuses_self_stopping_and_search_families(algo):
    with pytest.raises(ValueError, match=r"^(dba|dpop|syncbb) is not batched: "):
        solve_batch(batch_problems(2), algo, engine_factory=factory)


def test_refusals():
    with pytest.raises(ValueError, match="at least one problem"):
        solve_batch([], "dsa", {"stop_cycle": 3}, engine_factory=factory)
    with pytest.raises(ValueError, match="does not stop by itself"):
        solve_batch(batch_problems(2), "dsa", engine_factory=factory)
    with pytest.raises(ValueError, match="Unknown parameter"):
        solve_batch(batch_problems(2), "dsa", {"stop_cycle": 3, "nope": 1}, engine_factory=factory)
    good = batch_problems(3)
    bad = dict(good[1].arrays)
    bad["edge_var"] = np.asarray(bad["edge_var"]).copy()
    bad["edge_var"][0] = len(bad["dom_size"])      # points at the next problem's first variable in a union
    with pytest.raises(ValueError) as alone:
        solve(bad, "dsa", {"stop_cycle": 3}, engine_factory=factory)
    with pytest.raises(ValueError) as batched:
        solve_batch([good[0], bad, good[2]], "dsa", {"stop_cycle": 3}, engine_factory=factory)
    assert str(batched.value) == f"problem 1: {alone.value}"
    big = dict(good[2].arrays, dom_size=np.asarray(good[2].arrays["dom_size"]).copy())
    big["dom_size"][-1] = 300                     # a variable without constraints: only the domain check sees it
    big["unary"] = np.zeros(int(big["dom_size"].sum()))
    with pytest.raises(ValueError) as alone:
        solve(big, "dsa", {"stop_cycle": 3}, engine_factory=factory)
    with pytest.raises(ValueError) as batched:
        solve_batch([good[0], good[1], big], "dsa", {"stop_cycle": 3}, engine_factory=factory)
    assert str(batched.value) == f"problem 2: {alone.value}"
    with pytest.raises(ValueError, match="^problem 1: cannot load"):
        solve_batch([good[0], 42], "dsa", {"stop_cycle": 3}, engine_factory=factory)


def test_refused_under_torchrun():
    with mock.patch("pydcop_b200.solve._under_torchrun", return_value=True):
        with pytest.raises(ValueError, match="without torchrun"):
            solve_batch(batch_problems(2), "dsa", {"stop_cycle": 3}, engine_factory=factory)


def test_cli_batch(tmp_path, capsys):
    dcops = batch_problems(3, seed=9, modes=("min", "max"))
    paths = []
    for i, d in enumerate(dcops):
        paths.append(str(tmp_path / f"p{i}.fgb"))
        ingest.save_instance(paths[-1], d)
    with mock.patch("pydcop_b200.solve.solve_batch",
                    side_effect=functools.partial(solve_batch, engine_factory=factory)):
        assert main(["--batch", "-a", "mgm", "-p", "stop_cycle:6", "--seed", "2", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert [r["problem"] for r in out] == paths
        for path, r in zip(paths, out):
            s = solve(path, "mgm", {"stop_cycle": 6}, seed=2, engine_factory=factory)
            assert r["assignment"] == {k: v for k, v in s["assignment"].items()} and r["cycle"] == 6
        assert main(["--batch", "--no-assignment", "-a", "dsa", "-p", "stop_cycle:3", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert len(out) == 3 and all("assignment" not in r for r in out)
    for extra in (["--run_metrics", str(tmp_path / "m.csv")], ["--save", str(tmp_path / "s.fgb")]):
        with pytest.raises(SystemExit):
            main(["--batch", "-a", "dsa", "-p", "stop_cycle:3", *extra, *paths])
        assert "--batch" in capsys.readouterr().err
    with mock.patch.dict(os.environ, {"WORLD_SIZE": "2"}), pytest.raises(SystemExit):
        main(["--batch", "-a", "dsa", "-p", "stop_cycle:3", *paths])
