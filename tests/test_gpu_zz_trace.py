"""The cost trace on the device (fg_trace_*, engine start_trace / trace, solve(trace=True)).

Every row the record kernel writes inside the step loop equals solution_cost() of the same engine stepped one cycle
at a time, exactly on integer costs (the f64 sums of integers are order-free), to rel 1e-12 on non-dyadic f64 costs;
the trace neither adds to the family's launch count nor changes what the run computes."""
import numpy as np
import pytest
import torch

from pydcop_b200.engine import make_engine
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import DEFAULTS, _var_inputs, solve, solve_batch
from test_batch_cpu import batch_problem, batch_problems

pytestmark = pytest.mark.gpu

KINDS = ["maxsum", "dsa", "adsa", "mgm", "mgm2", "gdba", "mixeddsa", "dba"]
N_CYCLES = 30


def _problem(kind, seed, ints=True):
    """batch_problem with integer (even seed) or float costs, hard entries for the families built for them"""
    s = 2 * seed + (0 if ints else 1)
    if s % 7 == 3:       # batch_problem's constraint-free shape
        s += 14
    return batch_problem(s, hard=kind in ("mixeddsa", "dba", "gdba") or seed % 2 == 1, n_range=(60, 200))


def _engine(kind, d, precision, seed=3, **kw):
    inst = d.instance()
    L = build_layout(**inst)
    var_rank, iso = _var_inputs(kind, d, "min")
    params = dict(DEFAULTS[kind], **kw)
    return make_engine(kind, L, params, mode="min", precision=precision, seed=seed, var_rank=var_rank,
                       isolated_value=iso).init()


def _stepped_costs(kind, d, precision, n):
    e = _engine(kind, d, precision)
    out, last = [], e.cycle
    for _ in range(n):
        e.step(1)
        if kind == "dba" and e.cycle == last:   # DBA has finished: no more rounds change the state
            break
        last = e.cycle
        out.append(e.solution_cost(float("inf"), d.arrays["unary"]))
    return out


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("chunk", [1, 7, N_CYCLES])
def test_rows_equal_solution_cost_after_every_cycle(kind, precision, chunk):
    for seed in range(2):
        d = _problem(kind, seed)
        want = _stepped_costs(kind, d, precision, N_CYCLES)
        e = _engine(kind, d, precision)
        e.start_trace(N_CYCLES, float("inf"), d.arrays["unary"])
        done = 0
        while done < N_CYCLES:
            k = min(chunk, N_CYCLES - done)
            e.step(k)
            done += k
        tr = e.trace()
        n = len(want) if kind == "dba" else len(tr["time"])
        assert n == len(want) and len(tr["time"]) >= n
        assert [(float(c), int(v)) for c, v in zip(tr["cost"][:n, 0], tr["violation"][:n, 0])] == want
        assert np.all(np.diff(tr["time"]) >= 0) and tr["time"][0] > 0
        if kind in ("mixeddsa", "dba", "gdba"):
            assert any(v for _, v in want), "no violated hard constraint in the run"


@pytest.mark.parametrize("kind", KINDS)
def test_float_costs_in_f64(kind):
    d = _problem(kind, 2, ints=False)
    assert not np.all(np.asarray(d.arrays["unary"]) == np.round(d.arrays["unary"]))
    want = _stepped_costs(kind, d, "f64", 12)
    e = _engine(kind, d, "f64")
    e.start_trace(5, float("inf"), d.arrays["unary"])   # three blocks
    e.step(12)
    tr = e.trace()
    n = len(want)
    assert [int(v) for v in tr["violation"][:n, 0]] == [v for _, v in want]
    np.testing.assert_allclose(tr["cost"][:n, 0], [c for c, _ in want], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("kind", KINDS)
def test_launch_count_unchanged_and_detach(kind):
    d = _problem(kind, 0)
    plain, traced = _engine(kind, d, "f32"), _engine(kind, d, "f32")
    traced.start_trace(4, float("inf"), d.arrays["unary"])
    for e in (plain, traced):
        e.step(9)
    assert traced.launch_count == plain.launch_count
    rows = len(traced.trace()["time"])
    traced.stop_trace()
    for e in (plain, traced):
        e.step(3)
    assert traced.launch_count == plain.launch_count
    assert len(traced.trace()["time"]) == rows
    assert np.array_equal(np.asarray(plain.values()[0] if isinstance(plain.values(), tuple) else plain.values()),
                          np.asarray(traced.values()[0] if isinstance(traced.values(), tuple) else traced.values()))


def test_timeout_only_run_spans_several_blocks():
    d = _problem("dsa", 0)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr("pydcop_b200.solve.TRACE_BYTES", 16 * 64)   # 64 rows per block
        res = solve(d, "dsa", {"stop_cycle": 0}, timeout=1.0, chunk=50, precision="f32", seed=3, trace=True)
    tr = res["trace"]
    assert res["status"] == "TIMEOUT" and res["cycle"] > 3 * 64
    assert tr["cycle"] == list(range(1, res["cycle"] + 1))
    assert np.all(np.diff(tr["time"]) >= 0)
    assert (tr["cost"][-1], tr["violation"][-1]) == (res["cost"], res["violation"])
    e = _engine("dsa", d, "f32")
    e.step(res["cycle"])
    assert e.solution_cost(float("inf"), d.arrays["unary"]) == (res["cost"], res["violation"])


@pytest.mark.parametrize("kind", KINDS)
def test_solve_trace_ends_at_the_result(kind):
    d = _problem(kind, 1)
    res = solve(d, kind, {"stop_cycle": 20}, precision="f64", seed=5, trace=True)
    plain = solve(d, kind, {"stop_cycle": 20}, precision="f64", seed=5)
    assert (res["assignment"], res["cost"], res["violation"], res["cycle"]) == \
        (plain["assignment"], plain["cost"], plain["violation"], plain["cycle"])
    tr = res["trace"]
    assert len(tr["cycle"]) == (res["cycle"] if kind in ("dba", "maxsum", "dsa", "adsa", "mixeddsa") else 19)
    assert (tr["cost"][-1], tr["violation"][-1]) == (res["cost"], res["violation"])


BATCHED = [("maxsum", {}), ("dsa", {}), ("adsa", {}), ("mgm", {}), ("mgm2", {"favor": "coordinated"}),
           ("gdba", {"violation": "NM", "increase_mode": "T"}), ("mixeddsa", {})]


def _int_problem(d):
    t, u = np.asarray(d.arrays["tables"], np.float64), np.asarray(d.arrays["unary"], np.float64)
    return bool(np.all(t[np.isfinite(t)] == np.round(t[np.isfinite(t)])) and np.all(u == np.round(u)))


def _same_trace(d, r, s):
    assert (r["status"], r["cycle"], r["assignment"]) == (s["status"], s["cycle"], s["assignment"])
    a, b = r["trace"], s["trace"]
    assert a["cycle"] == b["cycle"] and a["violation"] == b["violation"]
    if _int_problem(d):
        assert a["cost"] == b["cost"]
    else:
        np.testing.assert_allclose(a["cost"], b["cost"], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("kind,params", BATCHED, ids=[k for k, _ in BATCHED])
def test_batch_trace_equals_solve_trace(kind, params):
    dcops = batch_problems(36, seed=len(kind), modes=("min", "max"), hard=kind in ("mixeddsa", "gdba"),
                           n_range=(20, 150))
    dcops = [d for d in dcops if len(d.arrays["tables"]) or kind not in ("mgm2", "gdba")]
    p = dict(params, stop_cycle=15)
    res = solve_batch(dcops, kind, p, precision="f64", seed=3, trace=True, max_vars=1500)
    plain = solve_batch(dcops, kind, p, precision="f64", seed=3, max_vars=1500)
    for d, r, q in zip(dcops, res, plain):
        # the trace uploads its own segment arrays (h2d_bytes); float costs are f64 atomic sums in no fixed order
        skip = ("trace", "time", "ingest_time", "h2d_bytes") + (() if _int_problem(d) else ("cost",))
        assert {k: v for k, v in r.items() if k not in skip} == {k: v for k, v in q.items() if k not in skip}
        assert r["cost"] == pytest.approx(q["cost"], rel=1e-12, abs=1e-12)
        _same_trace(d, r, solve(d, kind, p, precision="f64", seed=3, trace=True))


def test_batch_trace_seed_sweep():
    dcops = [d for d in batch_problems(7, seed=50, n_range=(40, 120)) if len(d.arrays["tables"])]
    probs = [d for d in dcops for _ in range(5)]
    seeds = [7 * i + 2 for i in range(len(probs))]
    for kind in ("dsa", "mgm2"):
        res = solve_batch(probs, kind, {"stop_cycle": 12}, precision="f32", seed=seeds, trace=True)
        for d, s, r in zip(probs, seeds, res):
            _same_trace(d, r, solve(d, kind, {"stop_cycle": 12}, precision="f32", seed=s, trace=True))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_traced_engine_on_a_second_device():
    d = _problem("mgm", 0)
    want = _stepped_costs("mgm", d, "f32", 6)
    torch.cuda.set_device(0)
    inst = d.instance()
    e = make_engine("mgm", build_layout(**inst), {}, precision="f32", device="cuda:1", seed=3,
                    var_rank=_var_inputs("mgm", d, "min")[0], isolated_value=_var_inputs("mgm", d, "min")[1]).init()
    e.start_trace(8, float("inf"), d.arrays["unary"])
    e.step(6)
    assert torch.cuda.current_device() == 0
    tr = e.trace()
    assert [(float(c), int(v)) for c, v in zip(tr["cost"][:, 0], tr["violation"][:, 0])] == want
