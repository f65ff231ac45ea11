"""Per-problem algorithm parameters in a batch (parameter sets: dev_var_pset / psets) without a GPU.

1. The kernel SOURCE, run on the CPU by the existing host shims through tests/_hostshim.HostRun: one union whose
   problems have different parameter sets, against every problem run alone with its parameters as the scalar fields,
   at every cycle, bit for bit, in f32 and f64, with and without per-problem seeds.
2. create refuses a malformed set with FG_ERR_ARG before it looks for a device.
3. solve_batch with one parameter dict per problem through the engine seam: results, groups per key, refusals, and
   the CLI's --sweep."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import test_batch_cpu as tb
import test_batch_seeds_cpu as ts
from _hostshim import HostRun
from pydcop_b200 import _cabi, batch
from pydcop_b200.engine import dsa_plan, gdba_plan, mgm2_plan, mixeddsa_plan
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import check_params, main, name_rank, solve, solve_batch
from test_maxsum_generic_hostshim import CUDA_INC

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA toolkit headers not present")

FAMILY = {"dsa": "dsa", "adsa": "dsa", "mgm2": "mgm2", "gdba": "gdba", "mixeddsa": "mixeddsa"}


def plan_for(kind, L, precision, mode, seed, p, var_rank=None, var_global_id=None, var_seed=None, var_pset=None,
             psets=None):
    """The engine's plan of `kind` with the checked parameters `p` as its scalars."""
    ids = dict(var_global_id=var_global_id, var_seed=var_seed, var_pset=var_pset, psets=psets)
    if kind in ("dsa", "adsa"):
        return dsa_plan(L, precision, mode, p["probability"], p.get("p_mode", "fixed"), p["variant"], 0, seed,
                        var_costs=kind == "adsa", **ids)
    if kind == "mgm2":
        return mgm2_plan(L, precision, mode, p["threshold"], p["favor"], 0, seed, var_rank, **ids)
    if kind == "gdba":
        return gdba_plan(L, precision, mode, p["modifier"], p["violation"], p["increase_mode"], 0, seed, var_rank,
                         **ids)
    return mixeddsa_plan(L, precision, mode, p["proba_hard"], p["proba_soft"], p["variant"], 0, seed, **ids)


class HostEngine(HostRun):
    """A plan run by the family's shim, with the values (and costs) in canonical order."""

    def values(self):
        L, k = self.L, self.k
        out = L.vars_to_canonical(self.value[:L.n_vars].copy())
        if "cost" not in k:
            return out
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return out, L.vars_to_canonical(cost)


def _tuple(x):
    return x if isinstance(x, tuple) else (x,)


def check_union_params(kind, dcops, params, precision, seeds=None, n_cycles=12, seed=5):
    """params: one parameter dict per problem.  The union's run with its parameter sets against every problem alone."""
    mode = dcops[0].objective
    checked = [check_params(kind, p) for p in params]
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d), None),
                          seed=seed if seeds is None else seeds, params=checked)
    assert u.var_pset is not None and len(u.psets) == len({batch.pset_key(p) for p in checked})
    L = batch.union_layout(u, dcops)
    whole = HostEngine(FAMILY[kind], L, plan_for(kind, L, precision, mode, seed, u.psets[0], u.var_rank,
                                                 u.var_global_id, u.var_seed, u.var_pset, u.psets), precision).init()
    assert whole.d.n_psets == len(u.psets) and whole.d.dev_var_pset
    alone = []
    for i, d in enumerate(dcops):
        inst = d.instance()
        La = build_layout(**inst)
        s = seed if seeds is None else seeds[i]
        alone.append(HostEngine(FAMILY[kind], La, plan_for(kind, La, precision, mode, s, checked[i], name_rank(d)),
                                precision).init())
        assert not alone[-1].d.dev_var_pset
    moved = 0
    for k in range(n_cycles + 1):
        if k:
            whole.step()
            for e in alone:
                e.step()
        got = _tuple(whole.values())
        for i, e in enumerate(alone):
            a, b = u.var_start[i], u.var_start[i + 1]
            for x, y in zip(got, _tuple(e.values())):
                assert np.array_equal(x[a:b], y, equal_nan=True), (kind, i, k, checked[i])
        moved += k > 0 and int((got[0] != prev).sum())
        prev = got[0].copy()
    assert moved > 0


def _cycle(sets, n):
    return [sets[i % len(sets)] for i in range(n)]


DSA_SETS = [dict(variant=v, probability=p) for v in "ABC" for p in (0.3, 0.9)] + [dict(variant="B", p_mode="arity"),
                                                                                  dict(variant="C", p_mode="arity")]
CASES = [("dsa", DSA_SETS),
         ("adsa", [dict(variant=v, probability=p, period=t) for v, p, t in (("A", 0.5, 0.5), ("B", 0.9, 1.0),
                                                                             ("C", 0.2, 0.5), ("B", 0.6, 2.0))]),
         ("mgm2", [dict(favor=f, threshold=t) for f in ("unilateral", "no", "coordinated") for t in (0.2, 0.8)]),
         ("gdba", [dict(modifier=m, violation=v, increase_mode="E") for m in "AM" for v in ("NZ", "NM", "MX")]),
         ("gdba", [dict(modifier=m, violation=v, increase_mode="T") for m in "MA" for v in ("MX", "NZ")]),
         ("mixeddsa", [dict(variant=v, proba_hard=h, proba_soft=s) for v, h, s in
                       (("A", 0.7, 0.5), ("B", 0.9, 0.2), ("C", 0.3, 0.8), ("B", 0.5, 0.5), ("A", 1.0, 0.0))])]


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("kind,sets", CASES, ids=lambda x: x if isinstance(x, str) else str(len(x)))
@pytest.mark.parametrize("mode", ["min", "max"])
def test_union_with_parameter_sets_equals_every_problem_alone(kind, sets, precision, mode):
    dcops = tb.batch_problems(10, seed=31 + len(sets), modes=(mode,), hard=kind == "mixeddsa")
    check_union_params(kind, dcops, _cycle(sets, len(dcops)), precision)


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("kind,sets", [CASES[0], CASES[2], CASES[3], CASES[5]], ids=lambda x: x if isinstance(x, str)
                         else str(len(x)))
def test_parameter_sets_with_per_problem_seeds(kind, sets, precision):
    """One problem repeated: every (parameter set, seed) pair is its own run."""
    d = tb.batch_problems(1, seed=41, hard=kind == "mixeddsa", n_range=(30, 40))[0]
    n = 2 * len(sets)
    check_union_params(kind, [d] * n, _cycle(sets, n), precision, seeds=[3 * i - 5 for i in range(n)])


def test_dsa_plan_prob_per_set_and_unchanged_without_sets():
    dcops = tb.batch_problems(6, seed=7)
    checked = [check_params("dsa", p) for p in _cycle(DSA_SETS, 6)]
    u = batch.build_union(dcops, list(range(6)), lambda d: (None, None), params=checked)
    L = batch.union_layout(u, dcops)
    inputs, _, scalars = dsa_plan(L, "f64", var_pset=u.var_pset, psets=u.psets)
    prob = L.vars_to_canonical(inputs["prob"][:L.n_vars])
    for k, d in enumerate(dcops):   # every problem's slice is the prob its own plan computes
        La = build_layout(**d.instance())
        own = dsa_plan(La, "f64", probability=checked[k]["probability"], p_mode=checked[k]["p_mode"])[0]["prob"]
        assert np.array_equal(prob[u.var_start[k]:u.var_start[k + 1]], La.vars_to_canonical(own[:La.n_vars]))
    assert scalars["n_psets"] == len(u.psets) and inputs["var_pset"].dtype == np.uint16
    # without sets: no var_pset input, no psets scalars, the arrays of the scalar plan
    a = dsa_plan(L, "f32", probability=0.4, variant="C")
    b = dsa_plan(L, "f32", probability=0.4, variant="C", var_pset=None, psets=None)
    assert "var_pset" not in a[0] and "psets" not in a[2] and a[2] == b[2] and a[1] == b[1]
    for k in a[0]:
        x, y = a[0][k], b[0][k]
        assert (x is None and y is None) or all(np.array_equal(p, q) for p, q in zip(_tuple_list(x), _tuple_list(y)))
    with pytest.raises(ValueError, match="go together"):
        dsa_plan(L, "f32", var_pset=u.var_pset)
    with pytest.raises(ValueError, match="one index"):
        dsa_plan(L, "f32", var_pset=np.full(L.n_vars, len(u.psets)), psets=u.psets)


def _tuple_list(x):
    return x if isinstance(x, list) else [x]


# ------------------------------------------------------------------------------------------------------------------
# 2. create's checks of the parameter sets
# ------------------------------------------------------------------------------------------------------------------
BAD_SETS = {"dsa": (_cabi.FgDsaDesc, _cabi.FgDsaPset, [dict(variant=3), dict(variant=-1)]),
            "mgm2": (_cabi.FgMgm2Desc, _cabi.FgMgm2Pset,
                     [dict(threshold=1.5, favor=0), dict(threshold=float("nan"), favor=0),
                      dict(threshold=-0.1, favor=0), dict(threshold=float("inf"), favor=0),
                      dict(threshold=0.5, favor=3)]),
            "gdba": (_cabi.FgGdbaDesc, _cabi.FgGdbaPset, [dict(modifier=2, violation=0), dict(modifier=0, violation=3),
                                                          dict(modifier=0, violation=1)]),
            "mixeddsa": (_cabi.FgMixedDsaDesc, _cabi.FgMixedDsaPset,
                         [dict(proba_hard=0.5, proba_soft=0.5, variant=4), dict(proba_hard=1.01, proba_soft=0.5),
                          dict(proba_hard=0.5, proba_soft=float("nan")), dict(proba_hard=0.5, proba_soft=-2.0)])}
GOOD = {"dsa": dict(variant=1), "mgm2": dict(threshold=0.5, favor=1), "gdba": dict(modifier=1, violation=0),
        "mixeddsa": dict(proba_hard=0.7, proba_soft=0.5, variant=2)}


@pytest.mark.parametrize("family", sorted(BAD_SETS))
def test_create_refuses_malformed_sets_before_the_device(family):
    import torch
    lib = _cabi.load()
    desc_t, pset_t, bad = BAD_SETS[family]
    create = getattr(lib, f"fg_{family}_create")
    last = getattr(lib, f"fg_{family}_last_error")
    last.restype = C.c_char_p
    fake = C.c_void_p(0x1000)   # never read: the sets are checked first

    def desc(rows, var_pset=fake, n=None):
        d = desc_t()
        d.abi_version, d.precision, d.mode_max = _cabi.FG_ABI_VERSION, _cabi.FG_F32, 0
        if family == "mgm2":
            d.threshold = 0.5
        if family == "mixeddsa":
            d.proba_hard = d.proba_soft = 0.5
            d.variant = 1
        if family == "gdba":
            d.n_edges = 1   # so that NM needs dev_viol_ref
            d.dev_edge_var = d.dev_edge_class = d.dev_slot_edge = d.dev_violated = d.dev_mod = d.dev_mod_off = fake
        table = (pset_t * max(len(rows), 1))(*[pset_t(**dict(GOOD[family], **r)) for r in rows])
        d.dev_var_pset, d.psets, d.n_psets = var_pset, table if rows else None, len(rows) if n is None else n
        return d

    h = C.c_void_p()
    for row in bad:
        rc = create(C.byref(desc([GOOD[family], row])), C.byref(h))
        assert rc == _cabi.FG_ERR_ARG, row
        assert b"parameter set 1:" in last(h), (row, last(h))
        getattr(lib, f"fg_{family}_destroy")(h)
    for d, what in ((desc([GOOD[family]], var_pset=None), "go together"), (desc([]), "go together"),
                    (desc([GOOD[family]], n=0), "go together"), (desc([GOOD[family]], n=70000), "go together")):
        assert create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_ARG
        assert what.encode() in last(h)
        getattr(lib, f"fg_{family}_destroy")(h)
    if not torch.cuda.is_available():   # good sets pass the checks and reach the device lookup
        assert create(C.byref(desc([GOOD[family]] * 3)), C.byref(h)) == _cabi.FG_ERR_CUDA
        getattr(lib, f"fg_{family}_destroy")(h)


def test_descriptor_layout_matches_the_header():
    import subprocess
    import tempfile
    from conftest import ROOT
    names = ["fg_dsa_desc_t", "fg_mgm2_desc_t", "fg_gdba_desc_t", "fg_mixeddsa_desc_t", "fg_dsa_pset_t",
             "fg_mgm2_pset_t", "fg_gdba_pset_t", "fg_mixeddsa_pset_t"]
    mirrors = [_cabi.FgDsaDesc, _cabi.FgMgm2Desc, _cabi.FgGdbaDesc, _cabi.FgMixedDsaDesc, _cabi.FgDsaPset,
               _cabi.FgMgm2Pset, _cabi.FgGdbaPset, _cabi.FgMixedDsaPset]
    fields = [(n, f) for n in names[:4] for f in ("dev_var_pset", "psets", "n_psets")]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"pydcop_b200.h\"\nint main(void){" + "".join(
        f'printf("%zu\\n", sizeof({n}));' for n in names) + "".join(
        f'printf("%zu\\n", offsetof({n}, {f}));' for n, f in fields) + "return 0;}"
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "s.c"), os.path.join(td, "s")
        open(src, "w").write(prog)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    offs = [getattr(m, f).offset for m in mirrors[:4] for f in ("dev_var_pset", "psets", "n_psets")]
    assert out == [C.sizeof(m) for m in mirrors] + offs
    assert _cabi.FG_ABI_VERSION == 3


# ------------------------------------------------------------------------------------------------------------------
# 3. solve_batch through the engine seam
# ------------------------------------------------------------------------------------------------------------------
def pset_factory(kind, layout, inst, params, made=None):
    """The engine seam: host-shimmed engines with the union's parameter sets (inst["var_pset"], params["psets"])."""
    if made is not None:
        made.append((kind, inst.get("var_pset"), params.get("psets")))
    if kind not in FAMILY:
        return ts.seeded_factory(kind, layout, inst, params)
    p = {k: v for k, v in params.items() if k not in ("mode", "seed", "psets")}
    var_pset = inst.get("var_pset")
    plan = plan_for(kind, layout, "f64", params["mode"], params["seed"], p, inst.get("var_rank"),
                    inst.get("var_global_id"), inst.get("var_seed"), var_pset,
                    params["psets"] if var_pset is not None else None)
    plan[2]["stop_cycle"] = int(p["stop_cycle"])
    return HostEngine(FAMILY[kind], layout, plan, "f64")


SWEEPS = {"dsa": [dict(variant=v, probability=p) for v in "AC" for p in (0.2, 0.8)],
          "adsa": [dict(period=t, variant=v) for t in (0.5, 1.5) for v in "AB"],
          "mgm": [dict(break_mode=b) for b in ("lexic", "random")],
          "mgm2": [dict(favor=f, threshold=0.6) for f in ("no", "coordinated")] + [dict(threshold=0.1)],
          "gdba": [dict(modifier=m, violation=v) for m in "AM" for v in ("NM", "MX")],
          "mixeddsa": [dict(proba_hard=h, variant=v) for h in (0.4, 0.9) for v in "AB"],
          "maxsum": [dict(noise=z) for z in (0.0, 0.01, 0.05)]}


@pytest.mark.parametrize("kind", sorted(SWEEPS))
def test_solve_batch_per_problem_params_equals_solve(kind):
    dcops = tb.batch_problems(4, seed=53, modes=("min", "max"), hard=kind == "mixeddsa")
    sets = SWEEPS[kind]
    probs = [d for d in dcops for _ in sets]
    params = [dict(s, stop_cycle=8) for _ in dcops for s in sets]
    seeds = [7 * i + 1 for i in range(len(probs))]
    made = []
    res = solve_batch(probs, kind, params, seed=seeds,
                      engine_factory=lambda *a: pset_factory(*a, made=made))
    assert len(made) == 2   # one engine per objective: every parameter here varies inside one union
    if kind in FAMILY:
        assert all(vp is not None and len(ps) == len(sets) for _, vp, ps in made)
    else:
        assert all(vp is None and ps is None for _, vp, ps in made)
    for d, p, s, r in zip(probs, params, seeds, res):
        tb._same(r, solve(d, kind, p, seed=s, engine_factory=tb.factory))


def test_group_keys_split_and_single_dict_unchanged():
    dcops = tb.batch_problems(6, seed=61)
    made = []
    fac = lambda *a: pset_factory(*a, made=made)  # noqa: E731
    # stop_cycle is one scalar per engine: two groups, in order of first appearance
    params = [dict(stop_cycle=c, variant=v) for c, v in ((5, "A"), (7, "A"), (5, "C"), (7, "B"), (5, "A"), (7, "A"))]
    res = solve_batch(dcops, "dsa", params, engine_factory=fac)
    assert [vp is not None for _, vp, _ in made] == [True, True] and [len(ps) for *_, ps in made] == [2, 2]
    assert [r["cycle"] for r in res] == [5, 7, 5, 7, 5, 7]
    for d, p, r in zip(dcops, params, res):
        tb._same(r, solve(d, "dsa", p, engine_factory=tb.factory))
    made.clear()
    solve_batch(dcops, "gdba", [dict(stop_cycle=4, increase_mode=m) for m in "ETETRE"], engine_factory=fac)
    assert [len(ps) if ps else 1 for *_, ps in made] == [1, 1, 1] and all(vp is None for _, vp, _ in made)
    made.clear()
    solve_batch(dcops, "maxsum", [dict(stop_cycle=4, damping=x) for x in (0.5, 0.7) * 3], engine_factory=fac)
    assert len(made) == 2
    # one dict, or a list of equal dicts: the groups and engine inputs of today, no sets
    made.clear()
    solve_batch(dcops, "dsa", {"stop_cycle": 4}, engine_factory=fac)
    solve_batch(dcops, "dsa", [{"stop_cycle": 4}] * 6, engine_factory=fac)
    assert [(vp, ps) for _, vp, ps in made] == [(None, None)] * 2
    assert batch.groups(dcops) == batch.groups(dcops, keys=[1] * 6, sets=[2] * 6)


def test_groups_cut_at_the_set_limit(monkeypatch):
    dcops = tb.batch_problems(7, seed=62)
    monkeypatch.setattr(batch, "MAX_PSETS", 3)
    assert batch.groups(dcops, sets=[0, 1, 0, 2, 3, 1, 4]) == [[0, 1, 2, 3], [4, 5, 6]]


def test_per_problem_params_refusals():
    dcops = tb.batch_problems(3, seed=63)
    with pytest.raises(ValueError, match="2 parameter dicts for 3 problems"):
        solve_batch(dcops, "dsa", [{"stop_cycle": 3}] * 2, engine_factory=pset_factory)
    with pytest.raises(ValueError, match="problem 1: Unknown parameter"):
        solve_batch(dcops, "dsa", [{"stop_cycle": 3}, {"stop_cycle": 3, "nope": 1}, None],
                    engine_factory=pset_factory)
    with pytest.raises(ValueError, match="problem 2: Invalid value for parameter variant"):
        solve_batch(dcops, "dsa", [{"stop_cycle": 3}] * 2 + [{"stop_cycle": 3, "variant": "D"}],
                    engine_factory=pset_factory)
    with pytest.raises(ValueError, match="problem 2: dsa does not stop by itself"):
        solve_batch(dcops, "dsa", [{"stop_cycle": 3}] * 2 + [None], engine_factory=pset_factory)
    for algo in ("dba", "dpop", "syncbb"):   # refused first, as before
        with pytest.raises(ValueError, match=f"{algo} is not batched"):
            solve_batch(dcops, algo, [{"nope": 1}] * 5)
    from pydcop_b200.engine import make_engine
    L = build_layout(**dcops[0].instance())
    for kind in ("maxsum", "mgm", "dba", "dpop", "syncbb"):
        with pytest.raises(ValueError, match="parameter sets"):
            make_engine(kind, L, {}, var_pset=np.zeros(L.n_vars), psets=[{}])


def test_cli_sweep(tmp_path, capsys, monkeypatch):
    dcops = tb.batch_problems(2, seed=64)
    from pydcop_b200 import ingest
    paths = []
    for i, d in enumerate(dcops):
        paths.append(str(tmp_path / f"p{i}.bin"))
        ingest.save_instance(paths[-1], d)
    seen = []
    import pydcop_b200.solve as S
    real = S.solve_batch
    monkeypatch.setattr(S, "solve_batch", lambda *a, **k: seen.append((a, k)) or real(*a, **k,
                                                                                       engine_factory=pset_factory))
    assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:6", "--sweep", "variant:C,A", "--sweep",
                 "probability:0.9,0.25,1", "--iterations", "2", "--seed", "3", *paths]) == 0
    out = json.loads(capsys.readouterr().out)
    combos = [(p, v) for p in ("0.25", "0.9", "1") for v in ("A", "C")]   # names sorted, values sorted as strings
    assert len(out) == 2 * len(combos) * 2
    k = 0
    for f in range(2):
        for p, v in combos:
            for r in range(2):
                e = out[k]
                assert e["problem"] == paths[f] and (e["iteration"], e["seed"]) == (r, 3 + r)
                assert e["algo_params"] == check_params("dsa", dict(stop_cycle=6, probability=p, variant=v))
                want = solve(dcops[f], "dsa", e["algo_params"], seed=3 + r, engine_factory=tb.factory)
                assert e["assignment"] == want["assignment"] and e["cycle"] == 6
                k += 1
    assert len(seen) == 1
    for bad in (["--sweep", "variant:A,B", "-p", "variant:C", "--batch"], ["--sweep", "variant:A"],
                ["--batch", "--sweep", "variant"], ["--batch", "--sweep", "variant:"],
                ["--batch", "--sweep", "variant:A", "--sweep", "variant:B"]):
        with pytest.raises(SystemExit):
            main(["-a", "dsa", "-p", "stop_cycle:3", *bad, *paths])
    capsys.readouterr()
    # without --sweep: the output of before
    assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:4", *paths]) == 0
    assert all("algo_params" not in e for e in json.loads(capsys.readouterr().out))
