"""The MixedDSA CUDA kernel SOURCE executed on the CPU (tests/hostshim/mixeddsa_host.cpp compiles
pydcop_b200/csrc/mixeddsa_kernels.cuh with g++ and loops over the threads) with exactly the arrays MixedDsaEngine
uploads (engine.mixeddsa_plan), against the reference trajectories (tests/golden/mixeddsa_*.npz) and the oracle, in
f64 and f32.  The device run is tests/test_gpu_zz_mixeddsa.py's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _mixeddsa_oracle import MixedDsaOracle
from conftest import GOLDEN_DIR, ROOT, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import (_class_array, fill_desc, fill_header, host_state, mixeddsa_hard_factors,
                                mixeddsa_plan, mixeddsa_slots)
from pydcop_b200.layout import layout_from_instance
from test_mixeddsa_cpu import EXACT_F32, check_trajectory

SHIM_SRC = os.path.join(ROOT, "tests", "hostshim", "mixeddsa_host.cpp")
SHIM_SO = os.path.join(ROOT, "tests", "hostshim", "_build", "mixeddsa_host.so")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
P = C.c_void_p


@pytest.fixture(scope="module")
def shim():
    deps = [SHIM_SRC, os.path.join(ROOT, "include", "pydcop_b200.h")] + [
        os.path.join(ROOT, "pydcop_b200", "csrc", f)
        for f in ("mixeddsa_kernels.cuh", "dsa_generic.cuh", "mgm_kernels.cuh", "philox.cuh")]
    if not os.path.exists(SHIM_SO) or any(os.path.getmtime(d) > os.path.getmtime(SHIM_SO) for d in deps):
        os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-w", "-I", CUDA_INC, "-shared", "-fPIC", "-o",
                        SHIM_SO, SHIM_SRC], check=True, capture_output=True)
    lib = C.CDLL(SHIM_SO)
    lib.mixeddsa_host_cycle.argtypes = [P, C.c_int64]
    return lib


class HostMixedDsa:
    """MixedDsaEngine's plan (mixeddsa_plan) and driving API over the host-shimmed kernels."""

    def __init__(self, lib, layout, precision="f64", mode="min", proba_hard=0.7, proba_soft=0.5, variant="B",
                 stop_cycle=0, seed=0, **_):
        self.lib, self.L = lib, layout
        inputs, state, scalars = mixeddsa_plan(layout, precision, mode, proba_hard, proba_soft, variant, stop_cycle,
                                               seed)
        self.k = dict(inputs, **host_state(state))
        self.value = self.k["value"]
        self.classes = _class_array(layout)
        self.d = fill_desc(fill_header(_cabi.FgMixedDsaDesc(), precision, layout, self.classes), self.k, scalars)
        self.stop_cycle, self.cycle = scalars["stop_cycle"], 0

    @property
    def finished(self):
        return bool(self.stop_cycle and self.cycle >= self.stop_cycle)

    def init(self):
        self.lib.mixeddsa_host_init(C.byref(self.d))
        self.cycle = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self.lib.mixeddsa_host_cycle(C.byref(self.d), self.cycle)
            self.cycle += 1
        return self

    def values(self):
        L, k = self.L, self.k
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return L.vars_to_canonical(self.value[self.cycle % 2][:L.n_vars].copy()), L.vars_to_canonical(cost)

    def record(self):
        L, k, n = self.L, self.k, self.L.n_vars
        return dict(h_best=L.vars_to_canonical(k["h_best"][:n].copy()), branch=L.vars_to_canonical(k["branch"][:n].copy()))


def compare_with_oracle(eng, o, dt, n_cycles):
    """Values, costs, best H and branch of every round bit-identical to the oracle in the same precision."""
    assert np.array_equal(eng.values()[0], o.values()[0])
    for k in range(1, n_cycles + 1):
        o.step()
        eng.step()
        got, want = eng.record(), o.record()
        for key in want:
            assert np.array_equal(got[key], want[key]), (k, key)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k


@pytest.mark.parametrize("name", golden_names("mixeddsa_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_fixture(shim, name, precision):
    """f64 against the reference's trajectory; f32 against it on the exact-cost fixtures, else against the f32
    oracle."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostMixedDsa(shim, layout_from_instance(inst), precision=precision, mode=meta["mode"], seed=meta["seed"],
                       **meta["params"]).init()
    if precision == "f64" or name in EXACT_F32:
        check_trajectory(eng, inst, meta, dt, name)
    else:
        o = MixedDsaOracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
        compare_with_oracle(eng, o, dt, meta["n_cycles"])


def harden(inst, share, seed, neg=False):
    """A share of the constraints of arity >= 2 made hard: +inf (or -inf) on every entry whose scope variables take
    equal value indices (hard `!=` colouring); the others stay soft."""
    rng = np.random.default_rng(seed)
    out = dict(inst)
    dom = np.asarray(inst["dom_size"], dtype=np.int64)
    fp, ev = np.asarray(inst["factor_ptr"], dtype=np.int64), np.asarray(inst["edge_var"], dtype=np.int64)
    t = np.asarray(inst["tables"], dtype=np.float64).copy()
    off = 0
    for f in range(len(fp) - 1):
        sc = ev[fp[f]:fp[f + 1]]
        shape = tuple(int(dom[u]) for u in sc)
        size = int(np.prod(shape, dtype=np.int64))
        if len(sc) > 1 and rng.uniform() < share:
            idx = np.indices(shape).reshape(len(sc), -1)
            eq = (idx == idx[0]).all(0)
            t[off:off + size][eq] = -np.inf if neg else np.inf
        off += size
    out["tables"] = t
    return out


def random_mixed(n, seed, levels=4, neg=False):
    """Mixed arities 1-4, hard and soft constraints, dyadic variable costs, some initial values."""
    inst = LM.random_graph(n, [2, 3, 4], [(2, n), (3, n // 5), (4, n // 20), (1, n // 8)], seed=seed, levels=levels)
    inst = harden(inst, 0.5, seed, neg)
    rng = np.random.default_rng(seed + 7)
    inst["unary"] = np.floor(rng.uniform(0, 8, len(inst["unary"]))) / 8.0
    return LM.with_local_search_arrays(inst, seed)


RANDOM_RUNS = [("f64", "min", "B", 0, False), ("f64", "max", "A", 4, False), ("f32", "min", "C", 4, True),
               ("f32", "max", "B", 0, False)]


@pytest.mark.parametrize("precision,mode,variant,levels,neg", RANDOM_RUNS)
def test_kernel_source_matches_oracle_on_random_graphs(shim, precision, mode, variant, levels, neg):
    inst = random_mixed(300, seed=17 + levels, levels=levels, neg=neg)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, variant=variant, proba_hard=0.8, proba_soft=0.6, seed=9)
    o = MixedDsaOracle(inst, dt, **kw).init()
    eng = HostMixedDsa(shim, layout_from_instance(inst), precision=precision, **kw).init()
    compare_with_oracle(eng, o, dt, 6)


LIMITS = {
    **{k: LM.LOCAL[k] for k in ("d1", "d256", "doms_1_2_256")},
    "arity8_d3": lambda: LM.with_local_search_arrays(LM.MAXSUM["arity8_d3"](), 4),
    "hub2400": lambda: LM.with_local_search_arrays(LM.MAXSUM["hub2400"](), 5),
    "unary_only": lambda: LM.with_local_search_arrays(LM.MAXSUM["unary_only"](), 6),
    "no_factors": lambda: LM.with_local_search_arrays(LM.MAXSUM["no_factors"](), 7),
}


def limits_instance(case):
    """The shape-limit instance `case` with half its constraints of arity >= 2 made hard."""
    return harden(LIMITS[case](), 0.5, 3)


@pytest.mark.parametrize("case", list(LIMITS))
def test_kernel_source_at_the_limits(shim, case):
    """Domain sizes 1 and 256, arity 8, a degree-2400 hub, unary-only and factor-free graphs."""
    inst = limits_instance(case)
    kw = dict(mode="min", variant="B", proba_hard=0.9, proba_soft=0.9, seed=23)
    for precision, dt in (("f64", np.float64), ("f32", np.float32)):
        o = MixedDsaOracle(inst, dt, **kw).init()
        eng = HostMixedDsa(shim, layout_from_instance(inst), precision=precision, **kw).init()
        compare_with_oracle(eng, o, dt, 3 if case == "hub2400" else 4)


def test_hard_classification_in_the_run_precision():
    """An f64 entry above the f32 range is a hard constraint in f32 only; each variable's soft slots come first."""
    inst = random_mixed(60, seed=3)
    inst["tables"] = np.where(np.isinf(inst["tables"]), 1e300, inst["tables"])
    L = layout_from_instance(inst)
    h64 = mixeddsa_hard_factors(L, np.asarray(L.tables, np.float64))
    with np.errstate(over="ignore"):
        h32 = mixeddsa_hard_factors(L, np.asarray(L.tables, np.float32))
    assert not h64.any() and h32.any()
    slot_edge, soft_end = mixeddsa_slots(L, h32)
    assert sorted(slot_edge.tolist()) == sorted(L.slot_edge.tolist())
    assert ((L.var_ptr[:-1] <= soft_end) & (soft_end <= L.var_ptr[1:])).all()


def test_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu",'
                   ' sizeof(fg_mixeddsa_desc_t), offsetof(fg_mixeddsa_desc_t, proba_hard), offsetof(fg_mixeddsa_desc_t,'
                   ' seed));return 0;}\n' % os.path.join(ROOT, "include", "pydcop_b200.h"))
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = _cabi.FgMixedDsaDesc
    assert out == [C.sizeof(D), D.proba_hard.offset, D.seed.offset]


def test_descriptor_validation():
    """fg_mixeddsa_create refuses a bad descriptor with FG_ERR_ARG and a message; the plan's own descriptor passes
    every check, and without a device create reports FG_ERR_CUDA — never a CPU path."""
    import torch
    lib = _cabi.load()
    d = HostMixedDsa(None, layout_from_instance(random_mixed(60, seed=1))).d

    def create():
        h = P()
        rc = lib.fg_mixeddsa_create(C.byref(d), C.byref(h))
        msg = (lib.fg_mixeddsa_last_error(h) or b"").decode()
        lib.fg_mixeddsa_destroy(h)
        return rc, msg

    for field, bad, word in (("variant", 3, "variant"), ("variant", -1, "variant"), ("mode_max", 2, "mode_max"),
                             ("stop_cycle", -1, "stop_cycle")):
        good = getattr(d, field)
        setattr(d, field, bad)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and word in msg, (field, msg)
        setattr(d, field, good)
    for field in ("dev_soft_end", "dev_con_opt", "dev_h_best", "dev_slot_edge"):
        good = getattr(d, field)
        setattr(d, field, None)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and "missing" in msg, field
        setattr(d, field, good)
    if not torch.cuda.is_available():
        rc, msg = create()
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device" in msg
