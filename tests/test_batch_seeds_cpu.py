"""Per-problem seeds in a batch (a per-variable Philox key, solve_batch(seed=[...]), --iterations) without a GPU.

1. The kernel source of every Philox family, run on the CPU through the host shims: a union of one problem repeated
   with several seeds, and a union of distinct problems with distinct seeds, equals every member run alone with its
   own scalar seed, at every cycle, bit for bit; the repeats do not all follow one trajectory.
2. A key array holding one value is the scalar seed; a plan without keys is the plan the engines always built.
3. solve_batch and the CLI through the engine seam."""
import ctypes as C
import functools
import json
from unittest import mock

import numpy as np
import pytest

import test_batch_cpu as tb
from pydcop_b200 import batch, engine as eng_mod, ingest
from pydcop_b200.layout import build_layout
from pydcop_b200.solve import main, name_rank, solve, solve_batch
from test_dsa_generic_hostshim import HostDsa
from test_mgm_hostshim import HostMgm

pytestmark = tb.pytestmark

SEEDS = [0, 1, 7, -5, 2 ** 40 + 3, 2 ** 64 - 1]   # -5 and 2**64 - 1 are keyed as solve() masks them


def _p(a):
    return C.c_void_p(a.ctypes.data if a is not None else 0)


class SeededDsa(HostDsa):
    """HostDsa with DsaSide::var_seed (tests/hostshim/dsa_seeded_host.cpp)."""

    def __init__(self, inst, var_seed=None, **kw):
        super().__init__(inst, **kw)
        self.lib = tb.shim("dsa_seeded")
        self.var_seed = None if var_seed is None else eng_mod._var_seeds(self.L, var_seed)

    def init(self):
        self.lib.dsa_host_init_seeded(C.byref(self.h), _p(self.var_seed))
        self.cur, self.cycle = 0, 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.stop_cycle and self.cycle >= self.stop_cycle:
                break
            self.lib.dsa_host_step_seeded(C.byref(self.h), self.cur, C.c_uint32(self.cycle), _p(self.var_seed))
            self.cur ^= 1
            self.cycle += 1
        return self


class SeededMgm(HostMgm):
    """HostMgm with MgmSide::var_seed (tests/hostshim/mgm_seeded_host.cpp); the shim's array struct has no field for
    it, so the keys are passed next to it."""

    def __init__(self, lib, layout, var_global_id=None, var_seed=None, **kw):
        keep = {}

        def plan(*a, **k):
            inputs, state, scalars = eng_mod.mgm_plan(*a, **k, var_global_id=var_global_id, var_seed=var_seed)
            keep["var_seed"] = inputs.pop("var_seed", None)
            return inputs, state, scalars
        with mock.patch("test_mgm_hostshim.mgm_plan", plan):
            super().__init__(lib, layout, **kw)
        self.var_seed = keep["var_seed"]

    def init(self):
        self.lib.mgm_host_init_seeded(C.byref(self.a), _p(self.var_seed))
        self.cycle = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.lib.mgm_host_cycle_seeded(C.byref(self.a), C.c_uint32(self.cycle + 1), _p(self.var_seed))
            self.cycle += 1
        return self


def seeded_engine(kind, layout, inst, precision, mode, params, seed, var_rank=None, var_global_id=None, var_seed=None):
    """tb.host_engine with the per-variable keys, stepped by tests/hostshim/<family>_seeded_host.cpp: the engine's own
    plan (mgm2, gdba, mixeddsa: dev_var_seed of the descriptor) or the keys next to the shim's arrays (dsa, adsa,
    mgm)."""
    if kind in ("dsa", "adsa"):
        return SeededDsa(inst, precision=precision, mode=mode, seed=seed, var_global_id=var_global_id,
                         var_costs=kind == "adsa", var_seed=var_seed, **params)
    if kind == "mgm":
        return SeededMgm(tb.shim("mgm_seeded"), layout, precision=precision, mode=mode, seed=seed, var_rank=var_rank,
                         var_global_id=var_global_id, var_seed=var_seed, **params)
    module, plan = tb._PLANS[kind]
    cls, lib = tb._HOSTS[kind]
    with mock.patch.object(module, plan, functools.partial(getattr(eng_mod, plan), var_global_id=var_global_id,
                                                           var_seed=var_seed)):
        return cls(tb.shim(lib + "_seeded"), layout, precision=precision, mode=mode, seed=seed, var_rank=var_rank,
                   **params)


def _trajectory(e, n_cycles):
    out = [tuple(x.copy() for x in tb._values(e))]
    for _ in range(n_cycles):
        e.step()
        out.append(tuple(x.copy() for x in tb._values(e)))
    return out


def check_seeds(kind, dcops, seeds, precision, params, n_cycles=12):
    """The union of `dcops` with `seeds` (one per problem) against every problem alone with its own scalar seed.
    Returns the union's per-problem trajectories of values."""
    mode = dcops[0].objective
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (name_rank(d), None), 0.0, seeds)
    assert u.var_seed is not None and u.var_seed.dtype == np.uint64
    L = batch.union_layout(u, dcops)
    # the scalar seed of the union is none of the members': every draw must take its variable's key
    whole = _trajectory(seeded_engine(kind, L, u.inst, precision, mode, params, 12345, u.var_rank, u.var_global_id,
                                      u.var_seed).init(), n_cycles)
    per_problem = []
    for i, (d, s) in enumerate(zip(dcops, seeds)):
        inst = d.instance()
        alone = _trajectory(tb.host_engine(kind, build_layout(**inst), inst, precision, mode, params, s,
                                           name_rank(d)).init(), n_cycles)
        a, b = u.var_start[i], u.var_start[i + 1]
        for k, (w, y) in enumerate(zip(whole, alone)):
            for x, z in zip(w, y):
                assert np.array_equal(x[a:b], z, equal_nan=True), (kind, i, k)
        per_problem.append([w[0][a:b] for w in whole])
    return per_problem


def _busy_problem(mode, hard=False):
    """A problem with constraints and variables without an initial value, so the seeds show."""
    for k in range(50):
        d = tb.batch_problem(700 + k, mode, hard, n_range=(25, 40))
        if len(d.arrays["tables"]) and (d.arrays["init_value"] < 0).sum() > 10:
            return d
    raise AssertionError("no busy problem")


SEED_CASES = [("dsa", dict(variant="A")), ("dsa", dict(variant="B")), ("dsa", dict(variant="C")),
              ("dsa", dict(variant="B", p_mode="arity")), ("adsa", dict(variant="B")),
              ("mgm", dict(break_mode="lexic")), ("mgm", dict(break_mode="random")),
              ("mgm2", dict(favor="unilateral")), ("mgm2", dict(favor="no", threshold=0.8)),
              ("mgm2", dict(favor="coordinated")),
              ("gdba", dict(modifier="A", violation="NZ", increase_mode="E")),
              ("gdba", dict(modifier="M", violation="NM", increase_mode="R")),
              ("gdba", dict(modifier="A", violation="MX", increase_mode="C")),
              ("gdba", dict(modifier="M", violation="NZ", increase_mode="T")),
              ("mixeddsa", dict(variant="B")), ("mixeddsa", dict(variant="A", proba_hard=0.9, proba_soft=0.3))]


def _host_params(kind, params):
    return {k: v for k, v in params.items() if not (kind == "mgm" and k == "break_mode")}


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("kind,params", SEED_CASES, ids=lambda x: x if isinstance(x, str) else "-".join(map(str, x.values())))
def test_repeated_problem_with_seeds_equals_every_seed_alone(kind, params, precision):
    mode = "max" if len(params) % 2 else "min"
    hard = kind == "mixeddsa"
    p = _host_params(kind, params)
    runs = check_seeds(kind, [_busy_problem(mode, hard)] * len(SEEDS), SEEDS, precision, p)
    distinct = {tuple(np.concatenate(r)) for r in runs}
    assert len(distinct) >= 2, "every seed followed the same trajectory"
    dcops = tb.batch_problems(7, seed=31 + len(params), modes=(mode,), hard=hard)
    check_seeds(kind, dcops, [3 * i + 1 for i in range(len(dcops))], precision, p)


@pytest.mark.parametrize("kind,params", [c for c in SEED_CASES if c[0] in ("dsa", "mgm", "mgm2", "gdba", "mixeddsa")][::2])
def test_one_key_everywhere_is_the_scalar_seed(kind, params):
    d = _busy_problem("min", kind == "mixeddsa")
    inst = d.instance()
    L = build_layout(**inst)
    p = _host_params(kind, params)
    keyed = _trajectory(seeded_engine(kind, L, inst, "f64", "min", p, 0, name_rank(d),
                                      var_seed=np.full(d.n_vars, 2 ** 33 + 9)).init(), 10)
    scalar = _trajectory(tb.host_engine(kind, L, inst, "f64", "min", p, 2 ** 33 + 9, name_rank(d)).init(), 10)
    for w, s in zip(keyed, scalar):
        for x, y in zip(w, s):
            assert np.array_equal(x, y, equal_nan=True)


PLANS = {"mgm": lambda L, **k: eng_mod.mgm_plan(L, "f32", "max", 5, 3, **k),
         "mgm2": lambda L, **k: eng_mod.mgm2_plan(L, "f64", "min", 0.5, "no", 5, 3, **k),
         "gdba": lambda L, **k: eng_mod.gdba_plan(L, "f32", "min", "M", "NM", "T", 5, 3, **k),
         "mixeddsa": lambda L, **k: eng_mod.mixeddsa_plan(L, "f64", "min", 0.7, 0.5, "B", 5, 3, **k)}


@pytest.mark.parametrize("kind", sorted(PLANS))
def test_plans_without_keys_are_unchanged(kind):
    d = _busy_problem("min")
    L = build_layout(**d.instance())
    gid = np.arange(d.n_vars, dtype=np.int32)[::-1].copy()
    pi, ps, pc = PLANS[kind](L, var_global_id=gid)
    ni, ns, nc = PLANS[kind](L, var_global_id=gid, var_seed=None)
    ki, ks, kc = PLANS[kind](L, var_global_id=gid, var_seed=[-1] * d.n_vars)
    assert "var_seed" not in pi and list(ni) == list(pi) and list(ki) == list(pi) + ["var_seed"]
    for name, a in pi.items():
        for other in (ni, ki):
            b = other[name]
            for x, y in (zip(a, b) if isinstance(a, list) else [(a, b)]):
                assert (x is None and y is None) or (x.dtype == y.dtype and np.array_equal(x, y)), name
    assert ps == ns == ks and pc == nc == kc
    key = ki["var_seed"]
    assert key.dtype == np.uint64 and key.flags.c_contiguous and (key == np.uint64(2 ** 64 - 1)).all()
    # internal order: variable v of the layout reads the key of canonical variable L.var_order[v]
    keys = PLANS[kind](L, var_seed=np.arange(d.n_vars) * 3)[0]["var_seed"]
    assert np.array_equal(keys, (L.var_order * 3).astype(np.uint64))


def test_make_engine_refuses_keys_where_nothing_draws_them():
    L = build_layout(**_busy_problem("min").instance())
    for kind in ("maxsum", "dba", "dpop", "syncbb"):
        with pytest.raises(ValueError, match=f"^{kind} takes no per-variable seeds"):
            eng_mod.make_engine(kind, L, {}, var_seed=np.zeros(L.n_vars, np.uint64))


# ------------------------------------------------------------------------------------------------------------------
# solve_batch and the CLI through the engine seam
# ------------------------------------------------------------------------------------------------------------------
def seeded_factory(kind, layout, inst, params, seen=None):
    if seen is not None:
        seen.append(inst.get("var_seed"))
    p = {k: v for k, v in params.items() if k not in ("mode", "seed", "noise")}
    if kind == "maxsum":
        return tb.factory(kind, layout, inst, params)
    return seeded_engine(kind, layout, inst, "f64", params["mode"], _host_params(kind, p), params["seed"],
                         inst.get("var_rank"), inst.get("var_global_id"), inst.get("var_seed"))


@pytest.mark.parametrize("kind,params", [("dsa", {}), ("adsa", {}), ("mgm", {}), ("mgm2", {}),
                                         ("gdba", {"increase_mode": "T"}), ("mixeddsa", {}), ("maxsum", {})])
def test_solve_batch_seed_list_equals_solve_of_every_seed(kind, params):
    dcops = tb.batch_problems(5, seed=23, modes=("min", "max"), hard=kind == "mixeddsa")
    probs = [d for d in dcops for _ in range(3)]
    seeds = [11 * i - 7 for i in range(len(probs))]
    p = dict(params, stop_cycle=9)
    one = solve_batch(probs, kind, p, seed=seeds, engine_factory=seeded_factory)
    cut = solve_batch(probs, kind, p, seed=tuple(seeds), engine_factory=seeded_factory, max_vars=60)
    assert len(batch.groups(probs, 60)) > 2
    for d, s, r, c in zip(probs, seeds, one, cut):
        want = solve(d, kind, p, seed=s, engine_factory=tb.factory)
        tb._same(r, want)
        tb._same(c, want)
    if kind != "maxsum":
        assert len({json.dumps(r["assignment"], sort_keys=True) for r in one}) > len(dcops)


def test_one_seed_for_all_runs_as_before():
    dcops = tb.batch_problems(6, seed=24, modes=("min", "max"))
    seen = []
    same = solve_batch(dcops, "mgm2", {"stop_cycle": 8}, seed=[4] * 6,
                       engine_factory=functools.partial(seeded_factory, seen=seen))
    assert seen == [None, None]       # one objective per engine, one seed: no key array
    for r, s in zip(same, solve_batch(dcops, "mgm2", {"stop_cycle": 8}, seed=4, engine_factory=tb.factory)):
        tb._same(r, s)
    seen.clear()
    solve_batch(dcops, "dsa", {"stop_cycle": 3}, seed=None, engine_factory=functools.partial(seeded_factory, seen=seen))
    assert seen == [None, None]


def test_seed_list_refusals():
    dcops = tb.batch_problems(3)
    for bad, msg in [([1, 2], "2 seeds for 3 problems"), ([1, 2, 3, 4], "4 seeds for 3 problems"),
                     ([1, 2.5, 3], "seed 1: expected an int"), ([1, "2", 3], "seed 1: expected an int"),
                     ([None, 1, 2], "seed 0: expected an int"), ([1, 2, True], "seed 2: expected an int"),
                     (2.5, "seed must be an int or a sequence of ints")]:
        with pytest.raises(ValueError, match=msg):
            solve_batch(dcops, "dsa", {"stop_cycle": 3}, seed=bad, engine_factory=seeded_factory)
    assert len(solve_batch(dcops, "dsa", {"stop_cycle": 3}, seed=np.array([1, 2, 3]), engine_factory=seeded_factory)) == 3


def test_maxsum_noise_is_drawn_per_problem_with_its_seed():
    dcops = tb.batch_problems(4, seed=25)
    seeds = [3, 9, 3, 40]
    u = batch.build_union(dcops, [0, 1, 2, 3], lambda d: (name_rank(d), None), 0.05, seeds)
    want = np.concatenate([ingest.add_noise(d.arrays["unary"], 0.05, s) for d, s in zip(dcops, seeds)])
    assert np.array_equal(u.inst["unary"], want)
    res = solve_batch(dcops, "maxsum", {"stop_cycle": 7, "noise": 0.05}, seed=seeds, engine_factory=seeded_factory)
    for d, s, r in zip(dcops, seeds, res):
        tb._same(r, solve(d, "maxsum", {"stop_cycle": 7, "noise": 0.05}, seed=s, engine_factory=tb.factory))


def test_cli_iterations(tmp_path, capsys):
    dcops = tb.batch_problems(3, seed=26, modes=("min", "max"))
    paths = []
    for i, d in enumerate(dcops):
        paths.append(str(tmp_path / f"p{i}.fgb"))
        ingest.save_instance(paths[-1], d)
    loads = []
    real_load = ingest.load_instance
    with mock.patch("pydcop_b200.solve.solve_batch",
                    side_effect=functools.partial(solve_batch, engine_factory=seeded_factory)), \
            mock.patch("pydcop_b200.ingest.load_instance", side_effect=lambda p: loads.append(p) or real_load(p)):
        assert main(["--batch", "--iterations", "3", "--seed", "5", "-a", "dsa", "-p", "stop_cycle:6", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert loads == paths               # every file read once
        assert [(r["problem"], r["iteration"], r["seed"]) for r in out] == [(p, r, 5 + r) for p in paths for r in range(3)]
        for r in out:
            s = solve(r["problem"], "dsa", {"stop_cycle": 6}, seed=r["seed"], engine_factory=tb.factory)
            assert r["assignment"] == s["assignment"] and r["cycle"] == 6
            assert set(r) == set(s) | {"problem", "iteration", "seed"}
        assert len({json.dumps(r["assignment"], sort_keys=True) for r in out}) > len(paths)
        assert main(["--batch", "--iterations", "2", "--no-assignment", "-a", "mgm", "-p", "stop_cycle:3", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert [r["seed"] for r in out] == [0, 1] * 3 and all("assignment" not in r for r in out)
        assert main(["--batch", "-a", "dsa", "-p", "stop_cycle:3", "--seed", "5", *paths]) == 0
        out = json.loads(capsys.readouterr().out)
        assert [r["problem"] for r in out] == paths and all("iteration" not in r and "seed" not in r for r in out)
    for argv in (["--iterations", "2", "-a", "dsa", "-p", "stop_cycle:3", paths[0]],
                 ["--batch", "--iterations", "0", "-a", "dsa", "-p", "stop_cycle:3", paths[0]]):
        with pytest.raises(SystemExit):
            main(argv)
        assert "--iterations" in capsys.readouterr().err
