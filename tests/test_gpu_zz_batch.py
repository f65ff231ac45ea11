"""solve_batch on the device: every problem of a batch gets what solve() gives it alone, and the per-problem device
reduction (fg_solution_cost_segmented) equals the unsegmented one restricted to each problem.

The batches mix one-domain problems (DSA's and MGM's fast and active-row paths, MaxSum's warp kernels) with
mixed-domain ones, and integer tables (8-bit copies on the MaxSum warp path) with float ones, so the union runs other
kernels than many of its problems do alone."""
import numpy as np
import pytest
import torch

from pydcop_b200 import batch
from pydcop_b200.engine import DsaEngine, EngineError, MaxSumEngine
from pydcop_b200.solve import name_rank, solve, solve_batch
from test_batch_cpu import batch_problems

pytestmark = pytest.mark.gpu

FAMILIES = [("maxsum", {}), ("dsa", {}), ("adsa", {}), ("mgm", {}), ("mgm2", {"favor": "coordinated"}),
            ("gdba", {"violation": "NM", "increase_mode": "T"}), ("mixeddsa", {})]


def _int_costs(d):
    a = d.arrays
    t = np.asarray(a["tables"], dtype=np.float64)
    u = np.asarray(a["unary"], dtype=np.float64)
    return bool(np.all(t[np.isfinite(t)] == np.round(t[np.isfinite(t)])) and np.all(u == np.round(u)))


def _same(d, r, s):
    assert r["assignment"] == s["assignment"]
    assert (r["status"], r["cycle"], r["violation"]) == (s["status"], s["cycle"], s["violation"])
    if _int_costs(d):
        assert r["cost"] == s["cost"]
    else:
        assert r["cost"] == pytest.approx(s["cost"], rel=1e-9, abs=1e-12)
    assert r["n_gpus"] == 1 and set(r) == set(s)


def _against_solve(kind, d, r, p, **kw):
    if kind in ("mgm2", "gdba") and not len(d.arrays["tables"]):
        # alone, these engines refuse a problem without any constraint table (no table array to bind); in a union it
        # runs, and tests/test_batch_cpu.py pins its trajectory on the kernel source
        with pytest.raises(EngineError, match="missing device array"):
            solve(d, kind, p, **kw)
        assert (r["status"], r["cycle"], r["violation"]) == ("FINISHED", p["stop_cycle"], 0)
        return
    _same(d, r, solve(d, kind, p, **kw))


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind,params", FAMILIES, ids=[k for k, _ in FAMILIES])
def test_batch_equals_solve_of_every_problem(kind, params, precision):
    dcops = batch_problems(36, seed=len(kind), hard=kind in ("mixeddsa", "gdba"), n_range=(20, 150))
    p = dict(params, stop_cycle=25)
    res = solve_batch(dcops, kind, p, precision=precision, seed=3)
    assert len(res) == len(dcops)
    for d, r in zip(dcops, res):
        _against_solve(kind, d, r, p, precision=precision, seed=3)


@pytest.mark.parametrize("kind", ["dsa", "mgm", "maxsum"])
def test_mixed_objectives_cut_into_several_engines(kind):
    dcops = batch_problems(30, seed=40, modes=("min", "max", "max"), n_range=(20, 150))
    assert len(batch.groups(dcops, max_vars=400)) >= 4
    res = solve_batch(dcops, kind, {"stop_cycle": 20}, precision="f32", seed=0, max_vars=400)
    for d, r in zip(dcops, res):
        _against_solve(kind, d, r, {"stop_cycle": 20}, precision="f32", seed=0)


def test_timeout_reports_the_cycle_reached():
    dcops = batch_problems(20, seed=50, n_range=(20, 150))
    res = solve_batch(dcops, "dsa", {"stop_cycle": 0}, timeout=0.0, seed=0)
    for d, r in zip(dcops, res):
        assert (r["status"], r["cycle"]) == ("TIMEOUT", 0)
        _same(d, r, solve(d, "dsa", {"stop_cycle": 0}, timeout=0.0, seed=0))


def _masked_costs(eng, u, n_seg, seg_f, seg_v, infinity):
    """fg_solution_cost over each segment's factors and variables alone: every other one skipped by the masks."""
    L = eng.layout
    out = []
    for k in range(n_seg):
        fs = np.ones(max(L.n_factors, 1), dtype=np.uint8)
        fs[L.factor_perm] = (seg_f != k)
        vs = (seg_v != k)[L.var_order].astype(np.uint8)
        with torch.cuda.device(eng.device):
            c = eng._solution_cost(eng._assignment(), infinity, u.unary, factor_skip=eng._dev(fs, torch.uint8),
                                   var_skip=eng._dev(vs, torch.uint8)).cpu().numpy()
        out.append((float(c[0]), int(c[1])))
    return out


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("engine", ["dsa", "maxsum"])
def test_segmented_cost_equals_the_masked_cost_of_every_problem(engine, precision):
    """Problems of 6 to 70 variables, so segments start and end inside warps, hard entries counted, and an arbitrary
    (not run-ordered) assignment of segments, with ids outside 0..n_seg-1 not counted."""
    dcops = batch_problems(48, seed=60, hard=True, n_range=(6, 70))
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d), None))
    L = batch.union_layout(u, dcops)
    if engine == "dsa":
        eng = DsaEngine(L, precision=precision, seed=2, var_global_id=u.var_global_id).init().step(4)
    else:
        eng = MaxSumEngine(L, precision=precision).init().step(4)
    inf = float("inf")
    exact = [_int_costs(d) for d in dcops]
    for seg_f, seg_v, n_seg in [(u.seg_factor, u.seg_var, len(dcops)),
                                (np.random.default_rng(1).integers(-1, 9, len(u.seg_factor)),
                                 np.random.default_rng(2).integers(-1, 9, len(u.seg_var)), 7)]:
        cost, viol = eng.solution_costs_segmented(seg_f, seg_v, n_seg, inf, u.unary)
        want = _masked_costs(eng, u, n_seg, seg_f, seg_v, inf)
        assert [int(v) for v in viol] == [w[1] for w in want]
        for k in range(n_seg):
            if n_seg == len(dcops) and exact[k]:
                assert cost[k] == want[k][0], k
            else:
                assert cost[k] == pytest.approx(want[k][0], rel=1e-12, abs=1e-12), k
        if n_seg == len(dcops):
            total = eng.solution_cost(inf, u.unary)
            assert viol.sum() == total[1] > 0 and float(cost.sum()) == pytest.approx(total[0], rel=1e-12)
