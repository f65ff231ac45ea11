"""The best cycle of a run kept on the device (fg_trace_set_best, engine start_trace(best=True) / best(),
solve(best=True), solve_batch(best=True)).

The best each record keeps is the first best row of the trace under the rule (test_best_cpu.rule), bit for bit, and its
values are those of a twin engine stepped that many cycles; keeping it changes neither the families' launch counts nor
what a run computes."""
import ctypes as C

import numpy as np
import pytest
import torch

from pydcop_b200 import _cabi
from pydcop_b200.engine import EngineError, make_engine
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import DEFAULTS, _var_inputs, solve, solve_batch
from test_batch_cpu import batch_problem, batch_problems
from test_best_cpu import bits, first_best
from test_gpu_zz_trace import _problem

pytestmark = pytest.mark.gpu

KINDS = ["maxsum", "dsa", "adsa", "mgm", "mgm2", "gdba", "dba", "mixeddsa"]
N_CYCLES = 30
INF = float("inf")


def _engine(kind, d, precision, mode="min", seed=3, **kw):
    L = build_layout(**d.instance())
    var_rank, iso = _var_inputs(kind, d, mode)
    return make_engine(kind, L, dict(DEFAULTS[kind], **kw), mode=mode, precision=precision, seed=seed,
                       var_rank=var_rank, isolated_value=iso).init()


def _values(e):
    v = e.values()
    return np.asarray(v[0] if isinstance(v, tuple) else v)


def _check_engine_best(kind, d, precision, mode, e, n_rows=None):
    """e's best (one segment) against the first best row of its trace and a twin engine stepped best.cycle cycles;
    returns the best cycle."""
    tr, b = e.trace(), e.best()
    n = len(tr["time"]) if n_rows is None else n_rows
    k = first_best(tr["cost"][:n, 0], tr["violation"][:n, 0], mode)
    assert k >= 0 and b["cycle"].tolist() == [k + 1]
    assert bits(b["cost"][0]) == bits(tr["cost"][k, 0]) and b["violation"][0] == tr["violation"][k, 0]
    twin = _engine(kind, d, precision, mode)
    twin.step(k + 1)
    assert np.array_equal(b["value"], _values(twin))
    return k + 1


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("chunk", [1, 7, N_CYCLES])
def test_best_is_the_first_best_row_and_its_values(kind, precision, chunk):
    mode = "max" if chunk == 7 and kind != "dba" else "min"
    cycles = set()
    for seed in range(2):
        d = _problem(kind, seed)
        e = _engine(kind, d, precision, mode)
        e.start_trace(N_CYCLES, INF, d.arrays["unary"], best=True)
        done = 0
        while done < N_CYCLES:
            e.step(min(chunk, N_CYCLES - done))
            done += min(chunk, N_CYCLES - done)
        cycles.add(_check_engine_best(kind, d, precision, mode, e, e.cycle if kind == "dba" else None))
    assert cycles


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind", ["maxsum", "dsa", "adsa", "mgm", "mgm2", "gdba", "mixeddsa"])
def test_batch_best_per_problem(kind, precision):
    dcops = batch_problems(36, seed=len(kind) + 7, modes=("min", "max"), hard=True, n_range=(20, 120))
    dcops = [d for d in dcops if len(d.arrays["tables"]) or kind not in ("mgm2", "gdba")]
    assert len(dcops) >= 30
    p = {"stop_cycle": 16}
    res = solve_batch(dcops, kind, p, precision=precision, seed=3, trace=True, best=True, max_vars=1200)
    plain = solve_batch(dcops, kind, p, precision=precision, seed=3, max_vars=1200)
    assert any(r["trace"]["violation"][0] for r in res), "no violated hard constraint"
    for d, r, q in zip(dcops, res, plain):
        assert (r["assignment"], r["status"], r["cycle"], r["violation"]) == \
            (q["assignment"], q["status"], q["cycle"], q["violation"])
        tr, b = r["trace"], r["best"]
        k = first_best(tr["cost"], tr["violation"], d.objective)
        assert b["cycle"] == k + 1
        assert (bits(b["cost"]), b["violation"]) == (bits(tr["cost"][k]), tr["violation"][k])
        after = {}
        solve(d, kind, p, precision=precision, seed=3, chunk=1,
              on_cycle=lambda c, idx: after.__setitem__(c, np.array(idx)))
        assert b["assignment"] == d.assignment(after[b["cycle"]])
    assert len({r["best"]["cycle"] for r in res}) > 1


@pytest.mark.parametrize("kind", ["maxsum", "dsa", "mgm", "mgm2", "gdba", "dba", "mixeddsa"])
def test_rotation_and_best_only(kind):
    d = _problem(kind, 1)
    for precision in ("f32", "f64"):
        kept, only = _engine(kind, d, precision), _engine(kind, d, precision)
        kept.start_trace(5, INF, d.arrays["unary"], best=True)
        only.start_trace(5, INF, d.arrays["unary"], best=True, rows=False)
        for _ in range(8):
            for e in (kept, only):
                e.step(5)
        a, b = kept.best(), only.best()
        assert all(np.array_equal(a[k], b[k]) for k in ("cycle", "cost", "violation", "value"))
        assert len(kept.trace()["time"]) == 40 or kind == "dba"
        _check_engine_best(kind, d, precision, "min", kept, kept.cycle if kind == "dba" else None)
        with pytest.raises(EngineError, match="keeps no rows"):
            only.trace()
    dcops = [x for x in batch_problems(12, seed=71, modes=("min", "max"), hard=True, n_range=(20, 80))
             if len(x.arrays["tables"])]
    if kind != "dba":
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr("pydcop_b200.solve.TRACE_BYTES", 16 * len(dcops) * 5)   # 5 rows per block
            both = solve_batch(dcops, kind, {"stop_cycle": 40}, seed=2, trace=True, best=True)
            alone = solve_batch(dcops, kind, {"stop_cycle": 40}, seed=2, best=True)
        assert [r["best"] for r in both] == [r["best"] for r in alone]


def test_dba_best_ignores_the_rounds_after_the_finish():
    d = _problem("dba", 0)
    e = _engine("dba", d, "f32")
    e.start_trace(200, INF, d.arrays["unary"], best=True)
    while not e.finished:
        e.step(50)
    rows = len(e.trace()["time"])
    assert e.cycle < rows, "DBA finished at the end of a step: no round after the finish was recorded"
    b = _check_engine_best("dba", d, "f32", "min", e, e.cycle)
    assert b <= e.cycle
    res = solve(d, "dba", {"stop_cycle": 0}, timeout=60, precision="f32", seed=3, best=True)
    assert res["status"] == "FINISHED" and res["best"]["cycle"] == b


@pytest.mark.parametrize("kind", KINDS)
def test_launch_count_unchanged(kind):
    d = _problem(kind, 0)
    plain, kept = _engine(kind, d, "f32"), _engine(kind, d, "f32")
    kept.start_trace(4, INF, d.arrays["unary"], best=True, rows=False)
    for e in (plain, kept):
        e.step(9)
    assert kept.launch_count == plain.launch_count
    assert np.array_equal(_values(plain), _values(kept))


def test_best_beats_the_final_assignment():
    """DSA at probability 0.9 keeps moving away from good assignments: some problems end worse than they were."""
    dcops = [d for d in batch_problems(40, seed=90, n_range=(40, 120)) if len(d.arrays["tables"])]
    res = solve_batch(dcops, "dsa", {"probability": 0.9, "stop_cycle": 30}, precision="f64", seed=5, best=True)
    assert any((r["best"]["violation"], r["best"]["cost"]) < (r["violation"], r["cost"]) for r in res)


def test_set_best_refusals():
    d = batch_problem(4)
    e = _engine("dsa", d, "f32")
    e.start_trace(4, INF, d.arrays["unary"])
    lib, h = _cabi.load(), e._trace["h"]
    dev = [torch.zeros(8, dtype=t, device="cuda") for t in (torch.float64, torch.int64, torch.int32)]
    ptr = [C.c_void_p(t.data_ptr()) for t in dev]
    err = lambda: lib.fg_trace_last_error(h).decode()  # noqa: E731
    assert lib.fg_trace_set_best(h, 2, *ptr, None) == _cabi.FG_ERR_ARG and "mode_max" in err()
    assert lib.fg_trace_set_best(h, 0, ptr[0], None, ptr[2], None) == _cabi.FG_ERR_ARG and "together" in err()
    host = np.zeros(8, dtype=np.int32)
    assert lib.fg_trace_set_best(h, 0, ptr[0], ptr[1], C.c_void_p(host.ctypes.data), None) == _cabi.FG_ERR_ARG
    assert "dev_best_value is pageable host memory" in err()
    assert lib.fg_trace_set_best(h, 1, *ptr, None) == _cabi.FG_OK
    assert lib.fg_trace_set_best(h, 0, None, None, None, None) == _cabi.FG_OK   # detach
    e.step(3)
    torch.cuda.synchronize()
    assert all(int(t.abs().sum()) == 0 for t in dev)
