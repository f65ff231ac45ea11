"""The cost trace (fg_trace_*, engine start_trace / trace, solve(trace=True), --collect_on cycle_change) without a GPU.

1. The C-ABI: the ctypes mirror of fg_trace_desc_t lays out as the C compiler does, and fg_trace_create refuses a
   bad descriptor with FG_ERR_ARG and a message before it looks for a device.
2. The cost terms the record kernel shares with fg_solution_cost (csrc/cost.cuh), run on the CPU by
   tests/hostshim/cost_host.cpp, against solve.solution_cost, in f32 and f64, with `infinity` entries.
3. solve / solve_batch / the CLI through the engine seam, whose engines get their trace on the host."""
import csv
import ctypes as C
import functools
import json
import os
import subprocess
import tempfile
from unittest import mock

import numpy as np
import pytest

import test_batch_cpu as tb
from _hostshim import build as build_shim
from conftest import ROOT
from pydcop_b200 import _cabi, ingest
from pydcop_b200.engine import _class_array
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import main, solution_cost, solve, solve_batch
from test_batch_seeds_cpu import seeded_factory
from test_maxsum_generic_hostshim import CUDA_INC

_FIELDS = [name for name, _ in _cabi.FgTraceDesc._fields_]


def test_struct_size_and_offsets_match_header():
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"pydcop_b200.h\"\nint main(void){printf(\"%zu\", " \
           "sizeof(fg_trace_desc_t));" + "".join(f'printf(" %zu", offsetof(fg_trace_desc_t, {f}));' for f in _FIELDS) \
           + "return 0;}\n"
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "s.c"), os.path.join(td, "s")
        open(src, "w").write(prog)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I",
                        os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [C.sizeof(_cabi.FgTraceDesc)] + [getattr(_cabi.FgTraceDesc, f).offset for f in _FIELDS]


def _good_desc(cls):
    d = _cabi.FgTraceDesc()
    d.abi_version, d.precision, d.n_vars, d.n_classes = _cabi.FG_ABI_VERSION, _cabi.FG_F64, 2, 1
    d.classes = C.cast(cls, C.POINTER(_cabi.FgClass))
    d.dev_tables = d.dev_edge_var = d.dev_rows = d.dev_stamp = 8
    d.n_seg, d.capacity, d.infinity = 1, 4, float("inf")
    return d


def test_create_refuses_bad_descriptors_before_the_device():
    import torch
    lib = _cabi.load()
    h = C.c_void_p()
    assert lib.fg_trace_create(None, C.byref(h)) == _cabi.FG_ERR_ARG
    cls = (_cabi.FgClass * 1)()
    cls[0].arity, cls[0].n_factors, cls[0].table_size, cls[0].row_total = 2, 1, 4, 4
    cls[0].dom[0] = cls[0].dom[1] = 2
    cls[0].row_off[1] = 2
    for change, msg in [(dict(abi_version=_cabi.FG_ABI_VERSION + 1), None), (dict(precision=5), None),
                        (dict(capacity=0), "capacity"), (dict(n_seg=0), "n_seg must be"),
                        (dict(n_seg=3), "n_seg > 1 needs the segment arrays"),
                        (dict(dev_factor_seg=8), "both segment arrays or neither"),
                        (dict(dev_rows=None), "missing dev_rows"), (dict(n_vars=-1), "negative n_vars"),
                        (dict(dev_unary=8), "dev_unary needs dev_unary_off"),
                        (dict(dev_tables=None), "missing dev_tables"),
                        (dict(capacity=2 ** 62), "overflow")]:
        d = _good_desc(cls)
        for k, v in change.items():
            setattr(d, k, v)
        rc = lib.fg_trace_create(C.byref(d), C.byref(h))
        assert rc == _cabi.FG_ERR_ARG, change
        if msg is None:
            assert not h.value
        else:
            assert msg in lib.fg_trace_last_error(h).decode(), change
        lib.fg_trace_destroy(h)
    cls[0].table_size = 5
    assert lib.fg_trace_create(C.byref(_good_desc(cls)), C.byref(h)) == _cabi.FG_ERR_ARG
    assert b"class size mismatch" in lib.fg_trace_last_error(h)
    lib.fg_trace_destroy(h)
    if not torch.cuda.is_available():
        cls[0].table_size = 4
        assert lib.fg_trace_create(C.byref(_good_desc(cls)), C.byref(h)) == _cabi.FG_ERR_CUDA
        assert b"no CUDA device visible" in lib.fg_trace_last_error(h)
        lib.fg_trace_destroy(h)
    for fam in ("maxsum", "dsa", "mgm", "mgm2", "gdba", "dba", "mixeddsa"):
        assert getattr(lib, f"fg_{fam}_set_trace")(None, None) == _cabi.FG_ERR_ARG
    n = C.c_int64()
    assert lib.fg_trace_start(None, None) == _cabi.FG_ERR_ARG and lib.fg_trace_rows(None, C.byref(n)) == _cabi.FG_ERR_ARG


# ------------------------------------------------------------------------------------------------------------------
# 2. the shared cost terms on the CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")), reason="CUDA toolkit headers not present")
@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("seed", range(6))
def test_cost_terms_equal_solution_cost(precision, seed):
    rng = np.random.default_rng(seed)
    infinity = float("inf") if seed % 2 else 3.0
    dt = np.float64 if precision == "f64" else np.float32
    dcops = []
    for d in tb.batch_problems(4, seed=40 + seed, hard=True):
        a = dict(d.arrays)
        if infinity != float("inf"):   # a finite `infinity`: some table entries and variable costs equal it
            a["tables"] = np.where(rng.random(len(a["tables"])) < 0.2, infinity, a["tables"])
            a["unary"] = np.where(rng.random(len(a["unary"])) < 0.2, infinity, a["unary"])
        a["tables"], a["unary"] = np.asarray(a["tables"]).astype(dt), np.asarray(a["unary"]).astype(dt)
        dcops.append(ingest.from_arrays(a))
    u = tb.batch.build_union(dcops, list(range(len(dcops))), lambda d: (None, None))
    L = build_layout(**u.inst)
    canon = (rng.integers(0, 1 << 30, L.n_vars) % u.inst["dom_size"]).astype(np.int32)
    value, v_seg = np.zeros(L.n_vars, np.int32), np.zeros(L.n_vars, np.int32)
    value[L.var_perm], v_seg[L.var_perm] = canon, u.seg_var
    f_seg = np.zeros(max(L.n_factors, 1), np.int32)
    f_seg[L.factor_perm] = u.seg_factor
    tables, unary = np.ascontiguousarray(L.tables, dt), np.ascontiguousarray(L.unary, dt)
    ev, uoff = np.ascontiguousarray(L.edge_var, np.int32), np.ascontiguousarray(L.unary_off, np.int64)
    lib = build_shim("cost_host")
    lib.cost_host.argtypes = [C.c_int32, C.c_void_p, C.c_int32] + [C.c_void_p] * 5 + [
        C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    out = np.zeros(2 * len(dcops))
    lib.cost_host(_cabi.FG_F64 if precision == "f64" else _cabi.FG_F32, C.cast(_class_array(L), C.c_void_p),
                  len(L.classes), tables.ctypes.data, ev.ctypes.data, value.ctypes.data, unary.ctypes.data,
                  uoff.ctypes.data, L.n_vars, infinity, f_seg.ctypes.data, v_seg.ctypes.data, len(dcops),
                  out.ctypes.data)
    assert out[1::2].sum() > 0, "no violation drawn"
    for k, d in enumerate(dcops):
        viol, cost = solution_cost(d, canon[u.var_start[k]:u.var_start[k + 1]], float(dt(infinity)))
        assert out[2 * k + 1] == viol, k
        assert out[2 * k] == pytest.approx(cost, rel=1e-12, abs=1e-9), k


# ------------------------------------------------------------------------------------------------------------------
# 3. solve, solve_batch and the CLI through the engine seam
# ------------------------------------------------------------------------------------------------------------------
ITERATIVE = [("maxsum", {}), ("dsa", {}), ("adsa", {}), ("mgm", {}), ("mgm2", {}), ("gdba", {"increase_mode": "T"}),
             ("mixeddsa", {}), ("dba", {})]


def dba_factory(kind, layout, inst, params):
    if kind != "dba":
        return tb.factory(kind, layout, inst, params)
    from test_dba_hostshim import HostDba
    return HostDba(layout, precision="f64", stop_cycle=params.get("stop_cycle", 0), seed=params["seed"],
                   var_rank=inst.get("var_rank"))


def _check_trace(res, cycles):
    tr = res["trace"]
    assert tr["cycle"] == list(range(1, cycles + 1))
    assert len(tr["time"]) == len(tr["cost"]) == len(tr["violation"]) == cycles
    assert all(b >= a for a, b in zip(tr["time"], tr["time"][1:]))
    if cycles:
        assert tr["violation"][-1] == res["violation"]
        assert tr["cost"][-1] == pytest.approx(res["cost"], rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("kind,params", ITERATIVE)
def test_solve_trace_has_a_row_per_cycle_ending_at_the_result(kind, params):
    d = tb.batch_problem(30, hard=kind in ("mixeddsa", "dba"), n_range=(30, 40))
    p = dict(params, stop_cycle=11)
    res = solve(d, kind, p, seed=3, engine_factory=dba_factory, trace=True)
    plain = solve(d, kind, p, seed=3, engine_factory=dba_factory)
    assert {k: v for k, v in res.items() if k not in ("trace", "time", "ingest_time")} == \
        {k: v for k, v in plain.items() if k not in ("time", "ingest_time")}
    # MGM, MGM-2, GDBA and DBA run stop_cycle - 1 rounds (cycle + 1 >= stop_cycle), DBA fewer once it has finished
    ran = res["cycle"] if kind == "dba" else 11 if kind in ("maxsum", "dsa", "adsa", "mixeddsa") else 10
    _check_trace(res, ran)
    assert len(set(res["trace"]["cost"])) > 1 or kind == "dba"


def test_solve_trace_refusals():
    d = tb.batch_problem(32)
    for algo in ("dpop", "syncbb", "dpop_gpu"):
        with pytest.raises(ValueError, match="has no cycles to trace"):
            solve(d, algo, engine_factory=tb.factory, trace=True)
    with pytest.raises(ValueError, match="without torchrun"):
        solve(d, "dsa", {"stop_cycle": 3}, engine_factory=tb.factory, distributed=True, trace=True)


def _same_trace(r, s):
    assert r["trace"]["cycle"] == s["trace"]["cycle"] and r["trace"]["violation"] == s["trace"]["violation"]
    assert r["trace"]["cost"] == pytest.approx(s["trace"]["cost"], rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("kind,params", [k for k in ITERATIVE if k[0] != "dba"])
def test_solve_batch_trace_equals_solve_trace(kind, params):
    dcops = tb.batch_problems(7, seed=33, modes=("min", "max", "min"), hard=kind == "mixeddsa")
    p = dict(params, stop_cycle=8)
    res = solve_batch(dcops, kind, p, seed=4, engine_factory=tb.factory, max_vars=50, trace=True)
    for d, r in zip(dcops, res):
        s = solve(d, kind, p, seed=4, engine_factory=tb.factory, trace=True)
        tb._same(r, s)
        _same_trace(r, s)


@pytest.mark.parametrize("kind", ["dsa", "mgm2", "maxsum"])
def test_solve_batch_trace_with_seed_lists(kind):
    dcops = tb.batch_problems(3, seed=34, modes=("min", "max"))
    probs = [d for d in dcops for _ in range(3)]
    seeds = [5 * i + 1 for i in range(len(probs))]
    res = solve_batch(probs, kind, {"stop_cycle": 7}, seed=seeds, engine_factory=seeded_factory, trace=True)
    for d, s, r in zip(probs, seeds, res):
        want = solve(d, kind, {"stop_cycle": 7}, seed=s, engine_factory=tb.factory, trace=True)
        tb._same(r, want)
        _same_trace(r, want)


def test_solve_batch_trace_on_timeout():
    import time
    dcops = tb.batch_problems(4, seed=35)

    def slow(kind, layout, inst, params):
        e = tb.factory(kind, layout, inst, params)
        step = e.step
        e.step = lambda n=1: (time.sleep(0.1), step(n))[1]
        return e
    res = solve_batch(dcops, "dsa", {"stop_cycle": 0}, timeout=0.25, engine_factory=slow, chunk=2,
                      max_vars=dcops[0].n_vars + dcops[1].n_vars, trace=True)
    assert [r["status"] for r in res] == ["TIMEOUT"] * 4
    for r in res:
        _check_trace(r, r["cycle"])
    assert res[0]["cycle"] > 0 and [r["trace"]["cycle"] for r in res[2:]] == [[], []]


def test_cli_collect_on_cycle_change(tmp_path, capsys):
    d = tb.batch_problem(36)
    path = str(tmp_path / "p.fgb")
    ingest.save_instance(path, d)
    metrics = str(tmp_path / "m.csv")
    with mock.patch("pydcop_b200.solve.solve", side_effect=functools.partial(solve, engine_factory=tb.factory)):
        assert main(["-a", "dsa", "-p", "stop_cycle:9", "--seed", "2", "--collect_on", "cycle_change",
                     "--run_metrics", metrics, path]) == 0
    res = json.loads(capsys.readouterr().out)
    assert "trace" not in res
    rows = list(csv.reader(open(metrics)))
    assert rows[0] == ["cycle", "time", "cost", "violation", "msg_count", "msg_size", "status"]
    assert [int(r[0]) for r in rows[1:]] == list(range(1, 10)) + [9]
    assert [r[6] for r in rows[1:]] == ["RUNNING"] * 9 + ["FINISHED"]
    want = solve(d, "dsa", {"stop_cycle": 9}, seed=2, engine_factory=tb.factory, trace=True)["trace"]
    assert [float(r[2]) for r in rows[1:-1]] == pytest.approx(want["cost"])
    assert [int(r[3]) for r in rows[1:-1]] == want["violation"]
    assert float(rows[-1][2]) == pytest.approx(res["cost"])

    paths = [path, str(tmp_path / "q.fgb")]
    ingest.save_instance(paths[1], tb.batch_problem(37, "max"))
    with mock.patch("pydcop_b200.solve.solve_batch",
                    side_effect=functools.partial(solve_batch, engine_factory=tb.factory)):
        assert main(["--batch", "-a", "mgm", "-p", "stop_cycle:6", "--collect_on", "cycle_change", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        for p, r in zip(paths, out):
            _same_trace(r, solve(p, "mgm", {"stop_cycle": 6}, engine_factory=tb.factory, trace=True))
        assert main(["--batch", "-a", "mgm", "-p", "stop_cycle:6", *paths]) == 0
        assert all("trace" not in r for r in json.loads(capsys.readouterr().out))
    with pytest.raises(SystemExit):
        main(["-a", "dsa", "-p", "stop_cycle:3", "--collect_on", "value_change", path])
    assert "--collect_on" in capsys.readouterr().err
