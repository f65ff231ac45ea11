"""The DBA CUDA kernel SOURCE executed on the CPU (tests/hostshim/dba_host.cpp compiles pydcop_b200/csrc/dba_kernels.cuh
with g++ and loops over the threads) with exactly the arrays DbaEngine uploads (dba_plan): the violation bit rows
against numpy, and the trajectories against the reference's (tests/golden/dba_*.npz) and the oracle's.  The device
run is tests/test_gpu_zz_dba.py's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _dba_oracle import LIVE, ROW_KEYS, DbaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array, canonical_slot, dba_plan, fill_desc, fill_header, host_state
from pydcop_b200.layout import layout_from_instance
from test_dba_cpu import check_trajectory
from test_mgm2_hostshim import random_mgm2_instance

SHIM_SRC = os.path.join(ROOT, "tests", "hostshim", "dba_host.cpp")
SHIM_SO = os.path.join(ROOT, "tests", "hostshim", "_build", "dba_host.so")
P = C.c_void_p


@pytest.fixture(scope="module")
def shim():
    deps = [SHIM_SRC, os.path.join(ROOT, "include", "pydcop_b200.h")] + [
        os.path.join(ROOT, "pydcop_b200", "csrc", f) for f in ("dba_kernels.cuh", "mgm_kernels.cuh", "philox.cuh")]
    if not os.path.exists(SHIM_SO) or any(os.path.getmtime(d) > os.path.getmtime(SHIM_SO) for d in deps):
        os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SHIM_SO,
                        SHIM_SRC], check=True, capture_output=True)
    lib = C.CDLL(SHIM_SO)
    lib.dba_host_cycle.argtypes = [P, C.c_int64]
    return lib


class HostDba:
    """DbaEngine's plan (dba_plan) and driving API over the host-shimmed kernels."""

    def __init__(self, lib, layout, precision="f64", infinity=10000, max_distance=50, stop_cycle=0, seed=0,
                 var_rank=None, **_):
        self.lib, self.L = lib, layout
        inputs, state, scalars = dba_plan(layout, precision, infinity, max_distance, stop_cycle, seed, var_rank)
        self.has_nbr = np.diff(inputs["nbr_ptr"]) > 0
        self.k = dict(inputs, **host_state(state))
        self.value = self.k["value"]
        self.classes = _class_array(layout)
        self.d = fill_desc(fill_header(_cabi.FgDbaDesc(), precision, layout, self.classes), self.k, scalars)
        self.stop_cycle, self.rounds = scalars["stop_cycle"], 0

    @property
    def end_round(self):
        return int(self.k["status"][1])

    @property
    def finished(self):
        return self.end_round != LIVE or bool(self.stop_cycle and self.rounds + 1 >= self.stop_cycle)

    @property
    def cycle(self):
        return min(self.rounds, self.end_round)

    def init(self):
        self.lib.dba_host_init(C.byref(self.d))
        self.rounds = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.lib.dba_host_cycle(C.byref(self.d), self.rounds)
            self.rounds += 1
        return self

    def values(self):
        L, k = self.L, self.k
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return L.vars_to_canonical(self.value[self.cycle % 2][:L.n_vars].copy()), L.vars_to_canonical(cost)

    def record(self):
        L, k, n, E = self.L, self.k, self.L.n_vars, self.L.n_edges
        out = {key: L.vars_to_canonical(k[key][:n].copy()) for key in
               ("eval", "improve", "new_value", "can_move", "qlm", "consistent", "counter", "finish_phase")}
        cs = canonical_slot(L)
        for key in ("violated", "weight"):
            a = np.zeros(E, dtype=k[key].dtype)
            a[cs] = k[key][:E]
            out[key] = a
        return out


def compare_with_oracle(eng, o, n_cycles):
    """Every array of every round identical to the oracle in the same precision, and the same cycle."""
    assert np.array_equal(eng.values()[0], o.values()[0])
    for k in range(1, n_cycles + 1):
        o.step()
        eng.step()
        got, want = eng.record(), o.record()
        for key in ROW_KEYS:
            assert np.array_equal(got[key], want[key]), (k, key)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1], o.values()[1], equal_nan=True), k
        assert eng.cycle == o.cycle and eng.finished == o.finished, k
    assert int(eng.k["unresolved"][0]) == o.unresolved


def expected_bits(layout, infinity, dt):
    """The bit rows from numpy `tables >= infinity`, slot by slot in the layout's internal order."""
    L = layout
    words = []
    for s in range(L.n_edges):
        e = int(L.slot_edge[s])
        c = L.classes[int(L.edge_class[e])]
        le = e - c.first_edge
        f, j = le // c.arity, le % c.arity
        t = np.asarray(L.tables[c.table_base + f * c.table_size:c.table_base + (f + 1) * c.table_size], dtype=dt)
        bad = np.moveaxis((t >= dt(infinity)).reshape(tuple(c.dom[:c.arity])), j, -1).reshape(-1, c.dom[j])
        d = c.dom[j]
        W = (d + 31) // 32
        pad = np.zeros((bad.shape[0], W * 32), dtype=np.uint64)
        pad[:, :d] = bad
        w = (pad.reshape(-1, W, 32) << np.arange(32, dtype=np.uint64)).sum(axis=2)
        words.append(w.reshape(-1).astype(np.uint32))
    return np.concatenate(words) if words else np.zeros(0, np.uint32)


def check_bits(eng, precision, infinity):
    dt = np.float64 if precision == "f64" else np.float32
    got = eng.k["bits"][:eng.d.n_words].view(np.uint32)
    assert np.array_equal(got, expected_bits(eng.L, infinity, dt))


@pytest.mark.parametrize("name", golden_names("dba_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_fixture(shim, name, precision):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    eng = HostDba(shim, layout_from_instance(inst), precision=precision, seed=meta["seed"], var_rank=inst["var_rank"],
                  **meta["params"]).init()
    check_bits(eng, precision, meta["params"]["infinity"])
    check_trajectory(eng, inst, meta, name)


def random_dba_instance(n, d, seed, infinity=10000, frac=0.3):
    """Mixed-arity random graph (binary, ternary, unary constraints) with random name ranks; a fraction `frac` of
    the entries raised to infinity, exactly or above it, the others soft costs just below it or far below."""
    inst = random_mgm2_instance(n, d, [2, 3, 1], seed=seed, n_factors=n // 2, levels=4)
    rng = np.random.default_rng(seed + 7)
    t = np.asarray(inst["tables"], dtype=np.float64)
    r = rng.random(len(t))
    t = np.where(r < frac / 2, float(infinity), t)
    t = np.where((r >= frac / 2) & (r < frac), np.inf, t)
    t = np.where((r >= frac) & (r < frac + 0.05), infinity - 0.5, t)
    inst["tables"] = t
    return inst


@pytest.mark.parametrize("precision,max_distance,infinity", [("f64", 3, 10000), ("f32", 2, 100), ("f64", 0, 10000)])
def test_kernel_source_matches_oracle_on_random_graphs(shim, precision, max_distance, infinity):
    inst = random_dba_instance(500, 3, seed=13, infinity=infinity)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(infinity=infinity, max_distance=max_distance, seed=5)
    o = DbaOracle(inst, dt, **kw).init()
    eng = HostDba(shim, layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    check_bits(eng, precision, infinity)
    compare_with_oracle(eng, o, 12)
    assert o.stats["weight_raises"] > 0 and o.stats["moves"] > 0


def test_kernel_source_flood_on_a_solvable_colouring(shim):
    """A sparse 3-colouring: variables stop, the End flood reaches every variable with neighbours, and rounds after
    the end change nothing."""
    rng = np.random.default_rng(4)
    n, d = 300, 3
    pairs = set()
    while len(pairs) < 330:
        a, b = sorted(int(x) for x in rng.choice(n, 2, replace=False))
        pairs.add((a, b))
    pairs = sorted(pairs)
    inst = dict(dom_size=np.full(n, d, np.int32), factor_ptr=np.arange(0, 2 * len(pairs) + 1, 2, dtype=np.int64),
                edge_var=np.array(pairs, np.int32).reshape(-1),
                tables=np.tile(np.where(np.eye(d, dtype=bool), np.inf, 0.0).reshape(-1), len(pairs)))
    from pydcop_b200.layout import default_var_csr
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    kw = dict(max_distance=4, seed=9)
    o = DbaOracle(inst, **kw).init()
    eng = HostDba(shim, layout_from_instance(inst), **kw).init()
    compare_with_oracle(eng, o, 80)
    assert o.ended and o.stats["stops"] > 0 and o.stats["floods"] > 0
    c, before = eng.cycle, eng.record()
    for r in range(eng.rounds, eng.rounds + 2):              # rounds enqueued after the end change nothing
        eng.lib.dba_host_cycle(C.byref(eng.d), r)
    after = eng.record()
    assert all(np.array_equal(before[k], after[k]) for k in ROW_KEYS) and eng.cycle == c


@pytest.mark.parametrize("case", list(LM.LOCAL))
def test_kernel_source_at_the_limits(shim, case):
    """Domain sizes 1 and 256 (8 words per row) and the mix {1, 2, 256} (tests/_limits.py), some entries raised
    to infinity."""
    inst = LM.LOCAL[case]()
    rng = np.random.default_rng(5)
    t = np.asarray(inst["tables"], dtype=np.float64)
    inst["tables"] = np.where(rng.random(len(t)) < 0.4, 10000.0, t)
    kw = dict(max_distance=3, seed=23)
    o = DbaOracle(inst, np.float64, **kw).init()
    eng = HostDba(shim, layout_from_instance(inst), precision="f64", var_rank=inst["var_rank"], **kw).init()
    check_bits(eng, "f64", 10000)
    compare_with_oracle(eng, o, 6)


def test_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu",'
                   ' sizeof(fg_dba_desc_t), offsetof(fg_dba_desc_t, n_words), offsetof(fg_dba_desc_t, seed));'
                   'return 0;}\n' % os.path.join(ROOT, "include", "pydcop_b200.h"))
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = _cabi.FgDbaDesc
    assert out == [C.sizeof(D), D.n_words.offset, D.seed.offset]


def test_descriptor_validation():
    """fg_dba_create accepts the plan's descriptor (without a device the one refusal left is FG_ERR_CUDA) and
    refuses a bad one with FG_ERR_ARG and a message."""
    import torch
    lib = _cabi.load()
    inst = random_dba_instance(60, 3, seed=1)
    d = HostDba(None, layout_from_instance(inst)).d

    def create():
        h = P()
        rc = lib.fg_dba_create(C.byref(d), C.byref(h))
        msg = (lib.fg_dba_last_error(h) or b"").decode()
        lib.fg_dba_destroy(h)
        return rc, msg

    rc, msg = create()
    if torch.cuda.is_available():
        assert rc == _cabi.FG_OK, msg
    else:
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device visible" in msg, (rc, msg)
    for field, bad, word in (("max_distance", -1, "max_distance"), ("stop_cycle", -1, "stop_cycle"),
                             ("n_words", d.n_edges - 1, "bit-row size"), ("n_live", d.n_vars + 1, "n_live")):
        good = getattr(d, field)
        setattr(d, field, bad)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and word in msg, (field, msg)
        setattr(d, field, good)
    for field in ("dev_bits", "dev_bit_off", "dev_finish_phase", "dev_status", "dev_weight"):
        good = getattr(d, field)
        setattr(d, field, None)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and "missing" in msg, field
        setattr(d, field, good)


def test_bit_row_bytes():
    """One word per row up to 32 values, ceil(d / 32) above: d = 256 rows are 8 words."""
    from pydcop_b200.engine import dba_bit_offsets
    inst = LM.LOCAL["d256"]()
    L = layout_from_instance(inst)
    off = dba_bit_offsets(L)
    d = L.dom_size[L.slot_var].astype(np.int64)
    ts = np.array([c.table_size for c in L.classes])[L.edge_class[L.slot_edge]]
    assert np.array_equal(np.diff(off), ts // d * ((d + 31) // 32))
    assert (np.diff(off)[d == 256] % 8 == 0).all()


def unresolved_instance():
    """A chain of three binary variables whose constraints are violated at every assignment: with the weights
    raised past `infinity` every value's eval is above it, so improve > 0 with no value to draw (the reference
    raises on random.choice([]))."""
    from test_mgm2_cpu import unit_instance
    inf = lambda a, b: float("inf")  # noqa: E731
    return unit_instance([[0, 1], [0, 1], [0, 1]], [([0, 1], inf), ([1, 2], inf)])


def test_kernel_source_unresolved_keeps_the_value(shim):
    """Weights grown past infinity: the kernel keeps the current value, draws nothing, clears can_move and counts
    every such variable in every round, as the oracle does."""
    inst = unresolved_instance()
    kw = dict(infinity=3, max_distance=0, seed=2)
    o = DbaOracle(inst, **kw).init()
    eng = HostDba(shim, layout_from_instance(inst), **kw).init()
    o.weight = [[5] * len(c) for c in o.cons]
    eng.k["weight"][:] = 5
    start = o.values()[0].copy()
    compare_with_oracle(eng, o, 3)
    rec = eng.record()
    assert o.unresolved == 3 * 3 and int(eng.k["unresolved"][0]) == 9
    assert (rec["improve"] > 0).all() and (rec["can_move"] == 0).all() and (rec["new_value"] == -1).all()
    assert np.array_equal(eng.values()[0], start)
