"""The SyncBB CUDA kernel SOURCE's step logic executed on the CPU (tests/hostshim/syncbb_host.cpp compiles
pydcop_b200/csrc/syncbb_kernels.cuh with g++) with exactly the arrays SyncbbEngine uploads (syncbb_plan): every
fixture step by step against the reference's trace and the oracle, in 1-step launches and in one launch.  The device
run is tests/test_gpu_zz_syncbb.py's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle as orc
from _syncbb_oracle import SyncbbOracle
from conftest import GOLDEN_DIR, ROOT
from pydcop_b200 import _cabi
from pydcop_b200.engine import fill_desc, host_state, syncbb_plan
from pydcop_b200.layout import layout_from_instance
from test_syncbb_cpu import INTEGER, RUNNABLE

SHIM_SRC = os.path.join(ROOT, "tests", "hostshim", "syncbb_host.cpp")
SHIM_SO = os.path.join(ROOT, "tests", "hostshim", "_build", "syncbb_host.so")
P = C.c_void_p


@pytest.fixture(scope="module")
def shim():
    deps = [SHIM_SRC, os.path.join(ROOT, "include", "pydcop_b200.h"),
            os.path.join(ROOT, "pydcop_b200", "csrc", "syncbb_kernels.cuh")]
    if not os.path.exists(SHIM_SO) or any(os.path.getmtime(d) > os.path.getmtime(SHIM_SO) for d in deps):
        os.makedirs(os.path.dirname(SHIM_SO), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SHIM_SO,
                        SHIM_SRC], check=True, capture_output=True)
    lib = C.CDLL(SHIM_SO)
    lib.syncbb_host_step.argtypes = [P, C.c_int64]
    lib.syncbb_host_init.argtypes = [P]
    return lib


class HostSyncbb:
    """SyncbbEngine's plan (syncbb_plan) and readers over the host-shimmed step logic."""

    def __init__(self, lib, inst, precision="f64", mode="min"):
        self.lib = lib
        L = layout_from_instance(inst)
        rank = inst.get("var_rank")
        inputs, state, scalars = syncbb_plan(L, precision, mode, rank)
        self.k = dict(inputs, **host_state(state))
        d = _cabi.FgSyncbbDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        self.d = fill_desc(d, self.k, scalars)
        self.chain = np.argsort(np.arange(L.n_vars) if rank is None else np.asarray(rank), kind="stable")
        self.n = L.n_vars

    def init(self):
        self.lib.syncbb_host_init(C.byref(self.d))
        return self

    def step(self, n=1):
        self.lib.syncbb_host_step(C.byref(self.d), int(n))
        return self

    def canonical(self, a):
        out = np.empty_like(a)
        out[self.chain] = a
        return out

    def values(self):
        return self.canonical(self.k["sel"][:self.n].copy())

    def bounds(self):
        return self.canonical(self.k["ub"][:self.n].copy())

    def message(self):
        m = self.k["msg"]
        return int(m[0]), int(self.chain[m[1]]), int(m[2]), self.k["msg_ub"][0]

    def cycle_counts(self):
        return self.canonical(self.k["cycles"][:self.n].copy())

    @property
    def finished(self):
        return bool(self.k["msg"][3])

    @property
    def steps(self):
        return int(self.k["count"][0])

    @property
    def messages(self):
        return int(self.k["count"][1])


def same_message(a, b):
    return a[:3] == b[:3] and ((np.isnan(a[3]) and np.isnan(b[3])) or a[3] == b[3])


def check_against_oracle(eng, o, split):
    """Step by step (split 1) or at the end of launches of `split` messages: message in flight, bounds, selections
    and counts identical to the oracle's in the same precision."""
    while not o.finished:
        for _ in range(split):
            if not o.step():
                break
        eng.step(split)
        assert same_message(eng.message(), o.message()), (o.steps, eng.message(), o.message())
        assert np.array_equal(eng.bounds(), o.bounds()) and np.array_equal(eng.values(), o.values()), o.steps
        assert (eng.steps, eng.messages, eng.finished) == (o.steps, o.messages, o.finished)
        assert np.array_equal(eng.cycle_counts(), o.cycle_counts())
    eng.step(3)                                            # nothing after the end
    assert (eng.steps, eng.messages) == (o.steps, o.messages)


def load(name):
    return orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))


@pytest.mark.parametrize("name", RUNNABLE)
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_oracle_and_fixture(shim, name, precision):
    inst, meta = load(name)
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostSyncbb(shim, inst, precision, meta["mode"]).init()
    o = SyncbbOracle(inst, dt, meta["mode"], inst["var_rank"]).init()
    if name in INTEGER or precision == "f64":              # the reference's own trace, message by message
        for k in range(int(inst["n_steps"])):
            kind, recv, plen, _ = eng.message()
            assert (kind, recv, plen) == (inst["step_type"][k], inst["step_recv"][k], inst["step_plen"][k]), k
            eng.step(1)
            assert np.array_equal(eng.bounds(), inst["ub"][k].astype(dt)), k
            assert np.array_equal(eng.values(), inst["sel"][k]), k
        assert eng.finished and eng.messages == int(inst["msg_count"])
        assert np.array_equal(eng.cycle_counts(), inst["cycle_count"])
        eng = HostSyncbb(shim, inst, precision, meta["mode"]).init()
    check_against_oracle(eng, o, 1)


@pytest.mark.parametrize("name", RUNNABLE)
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_in_one_launch(shim, name, precision):
    inst, meta = load(name)
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostSyncbb(shim, inst, precision, meta["mode"]).init().step(10 ** 9)
    o = SyncbbOracle(inst, dt, meta["mode"], inst["var_rank"]).init().run()
    assert eng.finished and (eng.steps, eng.messages) == (o.steps, o.messages)
    assert np.array_equal(eng.values(), o.values()) and np.array_equal(eng.bounds(), o.bounds())


def random_instance(n, d, n_edges, seed, levels=None, mode_inf=0.0):
    """Random binary constraints over shuffled names (var_rank a permutation), with duplicate pairs in both scope
    orders; entries from `levels` or uniform floats, a fraction `mode_inf` set to inf."""
    rng = np.random.default_rng(seed)
    pairs = [tuple(int(x) for x in rng.choice(n, 2, replace=False)) for _ in range(n_edges)]
    dom = rng.integers(1, d + 1, size=n).astype(np.int32)
    tabs = []
    for a, b in pairs:
        t = rng.choice(levels, size=dom[a] * dom[b]) if levels is not None else rng.random(dom[a] * dom[b]) * 10
        t = np.where(rng.random(t.size) < mode_inf, np.inf, t)
        tabs.append(t)
    return dict(dom_size=dom, factor_ptr=np.arange(0, 2 * len(pairs) + 1, 2, dtype=np.int64),
                edge_var=np.array(pairs, dtype=np.int32).reshape(-1), tables=np.concatenate(tabs),
                var_rank=rng.permutation(n).astype(np.int32))


@pytest.mark.parametrize("mode,precision,split", [("min", "f64", 1), ("min", "f32", 7), ("max", "f64", 5),
                                                  ("min", "f64", 1000)])
def test_kernel_source_on_random_instances(shim, mode, precision, split):
    dt = np.float64 if precision == "f64" else np.float32
    n = 7 if mode == "max" else 12
    inst = random_instance(n, 3, 20, seed=split + (100 if mode == "max" else 0) + (7 if precision == "f32" else 0), mode_inf=0.05)
    eng = HostSyncbb(shim, inst, precision, mode).init()
    o = SyncbbOracle(inst, dt, mode, inst["var_rank"]).init()
    check_against_oracle(eng, o, split)


def test_struct_size_matches_header(tmp_path):
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu",'
                   ' sizeof(fg_syncbb_desc_t), offsetof(fg_syncbb_desc_t, dev_count), offsetof(fg_syncbb_desc_t, '
                   'n_pair));return 0;}\n' % os.path.join(ROOT, "include", "pydcop_b200.h"))
    exe = tmp_path / "s"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    D = _cabi.FgSyncbbDesc
    assert out == [C.sizeof(D), D.dev_count.offset, D.n_pair.offset]


def test_descriptor_validation():
    """fg_syncbb_create accepts the plan's descriptor (without a device the one refusal left is FG_ERR_CUDA) and
    refuses a bad one with FG_ERR_ARG and a message."""
    import torch
    lib = _cabi.load()
    inst, _ = load("syncbb_tuto")
    d = HostSyncbb(None, inst).d

    def create():
        h = P()
        rc = lib.fg_syncbb_create(C.byref(d), C.byref(h))
        msg = (lib.fg_syncbb_last_error(h) or b"").decode()
        lib.fg_syncbb_destroy(h)
        return rc, msg

    rc, msg = create()
    if torch.cuda.is_available():
        assert rc == _cabi.FG_ERR_ARG and "host memory" in msg, (rc, msg)   # host arrays
    else:
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device visible" in msg, (rc, msg)
    for field, bad, word in (("n_vars", 1, "at least two"), ("mode_max", 2, "mode_max"), ("n_pair", 0, "n_elts")):
        good = getattr(d, field)
        setattr(d, field, bad)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and word in msg, (field, msg)
        setattr(d, field, good)
    for field in ("dev_ub", "dev_msg", "dev_pair", "dev_count", "dev_cycles"):
        good = getattr(d, field)
        setattr(d, field, None)
        rc, msg = create()
        assert rc == _cabi.FG_ERR_ARG and "missing" in msg, field
        setattr(d, field, good)


def test_plan_refuses_arity3_and_one_variable():
    inst, _ = load("syncbb_arity3")
    with pytest.raises(ValueError, match="constraint abc has arity 3"):
        syncbb_plan(layout_from_instance(inst), "f64", "min", inst["var_rank"], [str(x) for x in inst["factor_names"]])
    inst, _ = load("syncbb_one_var")
    with pytest.raises(ValueError, match="at least two variables"):
        syncbb_plan(layout_from_instance(inst), "f64", "min", inst["var_rank"])


def test_pair_tables_combine_in_constraint_order():
    """Two constraints between the same pair, in both scope orders: one [val_u][x] table, their sum from 0."""
    inst = dict(dom_size=np.array([2, 3], np.int32), factor_ptr=np.array([0, 2, 4]),
                edge_var=np.array([0, 1, 1, 0], np.int32), tables=np.concatenate([np.arange(6.0), 10 * np.arange(6.0)]))
    inputs, _, scalars = syncbb_plan(layout_from_instance(inst), "f64", "min")
    assert scalars["n_elts"] == 1 and list(inputs["elt_ptr"]) == [0, 0, 1]
    want = np.arange(6.0).reshape(2, 3) + (10 * np.arange(6.0)).reshape(3, 2).T
    assert np.array_equal(inputs["pair"].reshape(2, 3), want)
