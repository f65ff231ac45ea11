"""The best cycle of a run (fg_trace_set_best, engine start_trace(best=True) / best(), solve(best=True), --best)
without a GPU.

1. The rule (csrc/cost.cuh's best_better), run on the CPU by tests/hostshim/best_host.cpp, against a Python statement
   of it on crafted rows: violation precedence, equal violations, exact ties, NaN and +-inf costs, min and max mode,
   costs rounded from f32 and from f64.  solve.best_better, the engine seam's copy of it, agrees too.
2. The C-ABI entry point: bound by ctypes, and a NULL trace refused before any device work.
3. solve / solve_batch / the CLI through the engine seam, whose engines keep their best on the host."""
import ctypes as C
import functools
import json
import math
import os
import struct
from unittest import mock

import numpy as np
import pytest

import test_batch_cpu as tb
from _hostshim import build as build_shim
from pydcop_b200 import _cabi, ingest
from pydcop_b200.solve import best_better, main, solve, solve_batch
from test_batch_params_cpu import pset_factory
from test_batch_seeds_cpu import seeded_factory
from test_maxsum_generic_hostshim import CUDA_INC
from test_trace_cpu import ITERATIVE, dba_factory

needs_cuda_headers = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                        reason="CUDA toolkit headers not present")


def rule(cost, viol, best_cost, best_viol, mode):
    """The issue's statement of the rule, written independently of the code under test."""
    if viol < best_viol:
        return True
    if viol > best_viol:
        return False
    if math.isnan(cost):
        return False
    if math.isnan(best_cost):
        return True
    return cost < best_cost if mode == "min" else cost > best_cost


def first_best(costs, viols, mode):
    """0-based index of the best row of one trace column under `rule` (the first of equal rows), -1 for none."""
    k = -1
    for i, (c, v) in enumerate(zip(costs, viols)):
        if k < 0 or rule(float(c), float(v), float(costs[k]), float(viols[k]), mode):
            k = i
    return k


def bits(x):
    return struct.pack("<d", float(x))


# costs an f32 table sums to (rounded through float32) and costs only f64 represents
COSTS = [0.0, -0.0, 1.0, 2.0, -3.5, float(np.float32(0.1)), 0.1, float(np.float32(0.1)) + 1e-12, 1e300, -1e300,
         float("inf"), float("-inf"), float("nan"), float(np.float32(1 / 3)), 1 / 3]
VIOLS = [0.0, 1.0, 2.0, 7.0]


@pytest.fixture(scope="module")
def shim():
    lib = build_shim("best_host")
    lib.best_host_better.argtypes = [C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32]
    lib.best_host_better.restype = C.c_int64
    lib.best_host_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.best_host_rows.restype = C.c_int64
    return lib


# ------------------------------------------------------------------------------------------------------------------
# 1. the rule
# ------------------------------------------------------------------------------------------------------------------
@needs_cuda_headers
@pytest.mark.parametrize("mode", ["min", "max"])
def test_rule_on_every_pair_of_rows(shim, mode):
    seen = set()
    for c in COSTS:
        for v in VIOLS:
            for bc in COSTS:
                for bv in VIOLS:
                    want = rule(c, v, bc, bv, mode)
                    assert bool(shim.best_host_better(c, v, bc, bv, int(mode == "max"))) == want, (c, v, bc, bv)
                    assert best_better(c, v, bc, bv, mode == "max") == want, (c, v, bc, bv)
                    seen.add((v < bv, v == bv and c == bc, math.isnan(c), math.isnan(bc), want))
    # the cases the rule separates all occur: fewer violations, exact ties, NaN row, NaN best, better and not
    assert {s[0] for s in seen} == {True, False} and any(s[1] for s in seen)
    assert any(s[2] for s in seen) and any(s[3] and not s[2] and s[4] for s in seen)
    assert bool(shim.best_host_better(-0.0, 0, 0.0, 0, 0)) is False   # -0 == 0: a tie
    assert bool(shim.best_host_better(5.0, 0, float("nan"), 0, 1)) is True
    assert bool(shim.best_host_better(float("nan"), 0, 5.0, 1, 0)) is True   # fewer violations first
    assert bool(shim.best_host_better(float("-inf"), 3, 0.0, 2, 0)) is False


@needs_cuda_headers
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("seed", range(4))
def test_best_rows_equal_the_first_best_of_every_column(shim, precision, mode, seed):
    rng = np.random.default_rng(seed)
    n_rows, n_seg = 60, 9
    pool = np.array(COSTS[:12] + [float("nan")] * 2 + list(rng.normal(0, 4, 20).round(1)))
    if precision == "f32":
        with np.errstate(over="ignore"):   # +-1e300 round to +-inf in f32
            pool = pool.astype(np.float32).astype(np.float64)
    rows = np.zeros((n_rows, n_seg, 2))
    rows[:, :, 0] = rng.choice(pool, (n_rows, n_seg))
    rows[:, :, 1] = rng.choice([0.0, 1.0, 2.0], (n_rows, n_seg), p=[0.2, 0.4, 0.4])
    rows[:, 0] = rows[0, 0]                 # one column of exact ties: the first row stays
    rows[:, 1, 0] = float("nan")            # one all-NaN column
    best, cyc = np.zeros(2 * n_seg), np.zeros(n_seg, dtype=np.int64)
    shim.best_host_rows(np.ascontiguousarray(rows).ctypes.data, n_rows, n_seg, int(mode == "max"), best.ctypes.data,
                        cyc.ctypes.data)
    for s in range(n_seg):
        k = first_best(rows[:, s, 0], rows[:, s, 1], mode)
        assert cyc[s] == k + 1, s
        assert bits(best[2 * s]) == bits(rows[k, s, 0]) and best[2 * s + 1] == rows[k, s, 1], s
    assert cyc[0] == 1 and cyc[1] == first_best(rows[:, 1, 0], rows[:, 1, 1], mode) + 1
    assert len(set(cyc.tolist())) > 2, "the draws put every best in the same row"


# ------------------------------------------------------------------------------------------------------------------
# 2. the C-ABI entry point
# ------------------------------------------------------------------------------------------------------------------
def test_set_best_binding_and_null_trace():
    lib = _cabi.load()
    res, args = _cabi.SYMBOLS["fg_trace_set_best"]
    assert res is C.c_int and args == [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert lib.fg_trace_set_best(None, 0, None, None, None, None) == _cabi.FG_ERR_ARG
    assert lib.fg_trace_set_best(None, 0, 8, 8, 8, None) == _cabi.FG_ERR_ARG


# ------------------------------------------------------------------------------------------------------------------
# 3. solve, solve_batch and the CLI through the engine seam
# ------------------------------------------------------------------------------------------------------------------
def _check_best(res, dcop, after):
    """res["best"] is the first best row of res["trace"] and its assignment the one after that many cycles
    (after[c]: the value indices after cycle c)."""
    tr, b = res["trace"], res["best"]
    k = first_best(tr["cost"], tr["violation"], dcop.objective)
    assert b is not None and b["cycle"] == k + 1
    assert (bits(b["cost"]), b["violation"]) == (bits(tr["cost"][k]), tr["violation"][k])
    assert b["assignment"] == dcop.assignment(after[b["cycle"]])


def _after_every_cycle(d, kind, p, seed, factory):
    after = {}
    solve(d, kind, p, seed=seed, engine_factory=factory, chunk=1,
          on_cycle=lambda c, idx: after.__setitem__(c, np.array(idx)))
    return after


@pytest.mark.parametrize("kind,params,mode", [(k, p, m) for k, p in ITERATIVE for m in ("min", "max")
                                               if (k, m) != ("dba", "max")])   # DBA is min only
def test_solve_best_is_the_first_best_row_of_the_trace(kind, params, mode):
    d = tb.batch_problem(30, mode, hard=kind in ("mixeddsa", "dba"), n_range=(30, 40))
    p = dict(params, stop_cycle=14)
    res = solve(d, kind, p, seed=3, engine_factory=dba_factory, trace=True, best=True)
    _check_best(res, d, _after_every_cycle(d, kind, p, 3, dba_factory))
    only = solve(d, kind, p, seed=3, engine_factory=dba_factory, best=True)
    plain = solve(d, kind, p, seed=3, engine_factory=dba_factory)
    assert "trace" not in only and only["best"] == res["best"]
    skip = ("trace", "best", "time", "ingest_time")
    assert {k: v for k, v in only.items() if k not in skip} == {k: v for k, v in plain.items() if k not in skip}


def test_solve_best_differs_from_the_final_result():
    """A run whose last cycle is not its best: DSA with probability 0.9 keeps moving away from good assignments."""
    gains = 0
    for seed in range(6):
        d = tb.batch_problem(40 + seed, n_range=(30, 40))
        res = solve(d, "dsa", {"stop_cycle": 20, "probability": 0.9}, seed=seed, engine_factory=tb.factory,
                    trace=True, best=True)
        b = res["best"]
        assert (b["violation"], b["cost"]) <= (res["violation"], res["cost"])
        gains += (b["violation"], b["cost"]) < (res["violation"], res["cost"])
    assert gains > 0


@pytest.mark.parametrize("kind,params", [k for k in ITERATIVE if k[0] != "dba"])
def test_solve_batch_best_equals_solve_best(kind, params):
    dcops = tb.batch_problems(7, seed=33, modes=("min", "max", "min"), hard=kind == "mixeddsa")
    p = dict(params, stop_cycle=8)
    res = solve_batch(dcops, kind, p, seed=4, engine_factory=tb.factory, max_vars=50, trace=True, best=True)
    assert len({r["best"]["cycle"] for r in res}) > 1 or kind == "mgm"
    for d, r in zip(dcops, res):
        s = solve(d, kind, p, seed=4, engine_factory=tb.factory, trace=True, best=True)
        tb._same(r, s)
        assert r["best"] == s["best"]
        _check_best(r, d, _after_every_cycle(d, kind, p, 4, tb.factory))
    only = solve_batch(dcops, kind, p, seed=4, engine_factory=tb.factory, max_vars=50, best=True)
    assert [r["best"] for r in only] == [r["best"] for r in res] and all("trace" not in r for r in only)


def test_solve_batch_best_is_none_for_a_group_that_never_started():
    import time
    dcops = tb.batch_problems(4, seed=35)

    def slow(kind, layout, inst, params):
        e = tb.factory(kind, layout, inst, params)
        step = e.step
        e.step = lambda n=1: (time.sleep(0.1), step(n))[1]
        return e
    res = solve_batch(dcops, "dsa", {"stop_cycle": 0}, timeout=0.25, engine_factory=slow, chunk=2,
                      max_vars=dcops[0].n_vars + dcops[1].n_vars, best=True)
    assert [r["status"] for r in res] == ["TIMEOUT"] * 4
    assert res[0]["cycle"] > 0 and all(1 <= r["best"]["cycle"] <= r["cycle"] for r in res[:2])
    assert [r["best"] for r in res[2:]] == [None, None]


def test_best_refusals():
    d = tb.batch_problem(32)
    for algo in ("dpop", "syncbb", "dpop_gpu"):
        with pytest.raises(ValueError, match="best: .* has no cycles to trace"):
            solve(d, algo, engine_factory=tb.factory, best=True)
    with pytest.raises(ValueError, match="best: .*without torchrun"):
        solve(d, "dsa", {"stop_cycle": 3}, engine_factory=tb.factory, distributed=True, best=True)
    for algo in ("dba", "dpop", "syncbb"):
        with pytest.raises(ValueError, match="is not batched"):
            solve_batch([d, d], algo, {"stop_cycle": 3}, engine_factory=tb.factory, best=True)
    with mock.patch("pydcop_b200.solve._under_torchrun", return_value=True), \
            pytest.raises(ValueError, match="without torchrun"):
        solve_batch([d, d], "dsa", {"stop_cycle": 3}, engine_factory=tb.factory, best=True)


def test_cli_best(tmp_path, capsys):
    dcops = tb.batch_problems(2, seed=64, modes=("min", "max"))
    paths = []
    for i, d in enumerate(dcops):
        paths.append(str(tmp_path / f"p{i}.fgb"))
        ingest.save_instance(paths[-1], d)
    with mock.patch("pydcop_b200.solve.solve", side_effect=functools.partial(solve, engine_factory=tb.factory)):
        assert main(["-a", "dsa", "-p", "stop_cycle:9", "--seed", "2", "--best", paths[0]]) == 0
        res = json.loads(capsys.readouterr().out)
        assert res["best"] == solve(paths[0], "dsa", {"stop_cycle": 9}, seed=2, engine_factory=tb.factory,
                                    best=True)["best"]
        assert main(["-a", "dsa", "-p", "stop_cycle:9", "--best", "--no-assignment", paths[0]]) == 0
        res = json.loads(capsys.readouterr().out)
        assert "assignment" not in res and set(res["best"]) == {"cycle", "cost", "violation"}
        assert main(["-a", "dsa", "-p", "stop_cycle:9", paths[0]]) == 0
        assert "best" not in json.loads(capsys.readouterr().out)
    with mock.patch("pydcop_b200.solve.solve_batch",
                    side_effect=functools.partial(solve_batch, engine_factory=seeded_factory)):
        assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:7", "--best", "--iterations", "2", "--seed", "5",
                     *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert len(out) == 4
        for e in out:
            want = solve(e["problem"], "dsa", {"stop_cycle": 7}, seed=e["seed"], engine_factory=tb.factory, best=True)
            assert e["best"] == want["best"]
    with mock.patch("pydcop_b200.solve.solve_batch",
                    side_effect=functools.partial(solve_batch, engine_factory=pset_factory)):
        assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:7", "--best", "--no-assignment", "--sweep",
                     "probability:0.9,0.3", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert len(out) == 4
        for e in out:
            assert "assignment" not in e and set(e["best"]) == {"cycle", "cost", "violation"}
            want = solve(e["problem"], "dsa", e["algo_params"], engine_factory=tb.factory, best=True)["best"]
            assert e["best"] == {k: v for k, v in want.items() if k != "assignment"}
        assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:7", *paths]) == 0
        assert all("best" not in e for e in json.loads(capsys.readouterr().out))
