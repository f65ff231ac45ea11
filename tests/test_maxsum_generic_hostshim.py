"""The generic MaxSum CUDA kernel SOURCE (pydcop_b200/csrc/maxsum_generic.cuh, unmodified) run on
the CPU through tests/hostshim/maxsum_generic_host.cpp with the arrays MaxSumEngine uploads, against
the oracle and the reference trajectories — including shapes the GPU tests do not reach (arity up
to 6, domain sizes up to 40, hub variables).  Needs the CUDA toolkit headers (not a GPU)."""
import ctypes as C
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import _hostshim as hs
from _hostshim import CUDA_INC
import _limits as LM
import oracle as orc
from bench import oracle_instance
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array, _varclass_array
from pydcop_b200.layout import build_layout, layout_from_instance

P = C.c_void_p

pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="CUDA toolkit headers not present")


class _Host(C.Structure):
    _fields_ = [("classes", P), ("varclasses", P), ("n_classes", C.c_int32), ("n_varclasses", C.c_int32),
                ("n_vars", C.c_int32), ("n_edges", C.c_int32), ("precision", C.c_int32),
                ("n_msg_r", C.c_int64), ("n_msg_q", C.c_int64), ("tables", P), ("unary", P),
                ("dom_size", P), ("var_ptr", P), ("slot_edge", P), ("slot_var", P), ("init_value", P),
                ("unary_off", P), ("var_qbase", P), ("slot_roff", P), ("edge_qoff", P),
                ("q", P * 2), ("r", P * 2), ("q_valid", P), ("r_valid", P), ("q_cnt", P), ("r_cnt", P),
                ("q_sent", P), ("r_sent", P), ("value", P), ("value_cost", P),
                ("mode_max", C.c_int32), ("damp_vars", C.c_int32), ("damp_factors", C.c_int32),
                ("start_messages", C.c_int32), ("damping", C.c_double), ("stability", C.c_double)]


def _lib():
    return hs.build("maxsum_generic_host")


class HostMaxSum:
    """MaxSumEngine's buffers and driving API over the host-shimmed generic kernels."""

    def __init__(self, layout, precision="f64", mode="min", damping=0.5, damping_nodes="both",
                 stability=0.1, start_messages="leafs", **_):
        self.lib, self.L = _lib(), layout
        L = layout
        dt = np.float64 if precision == "f64" else np.float32
        c = np.ascontiguousarray
        z = lambda n, d: np.zeros(max(int(n), 1), dtype=d)  # noqa: E731
        self.keep = dict(
            classes=_class_array(L), varclasses=_varclass_array(L), tables=c(L.tables, dt), unary=c(L.unary, dt),
            dom_size=c(L.dom_size, np.int32), var_ptr=c(L.var_ptr, np.int32), slot_edge=c(L.slot_edge, np.int32),
            slot_var=c(L.slot_var, np.int32), init_value=c(L.init_value, np.int32),
            unary_off=c(L.unary_off, np.int64), var_qbase=c(L.var_qbase, np.int64),
            slot_roff=c(L.slot_roff, np.int64), edge_qoff=c(L.edge_qoff, np.int64),
            q0=z(L.n_msg_q, dt), q1=z(L.n_msg_q, dt), r0=z(L.n_msg, dt), r1=z(L.n_msg, dt),
            q_valid=z(L.n_edges, np.uint8), r_valid=z(L.n_edges, np.uint8), q_cnt=z(L.n_edges, np.uint8),
            r_cnt=z(L.n_edges, np.uint8), q_sent=z(L.n_edges, np.uint8), r_sent=z(L.n_edges, np.uint8),
            value=z(L.n_vars, np.int32), value_cost=z(L.n_vars, dt))
        h = _Host()
        k = self.keep
        for name in ("tables", "unary", "dom_size", "var_ptr", "slot_edge", "slot_var", "init_value", "unary_off",
                     "var_qbase", "slot_roff", "edge_qoff", "q_valid", "r_valid", "q_cnt", "r_cnt", "q_sent",
                     "r_sent", "value", "value_cost"):
            setattr(h, name, P(k[name].ctypes.data))
        h.classes, h.varclasses = C.cast(k["classes"], P), C.cast(k["varclasses"], P)
        h.q[0], h.q[1], h.r[0], h.r[1] = (k["q0"].ctypes.data, k["q1"].ctypes.data, k["r0"].ctypes.data,
                                          k["r1"].ctypes.data)
        h.n_classes, h.n_varclasses, h.n_vars, h.n_edges = len(L.classes), len(L.var_classes), L.n_vars, L.n_edges
        h.n_msg_r, h.n_msg_q = L.n_msg, L.n_msg_q
        h.precision = _cabi.FG_F64 if precision == "f64" else _cabi.FG_F32
        h.mode_max = int(mode == "max")
        h.damp_vars = int(damping_nodes in ("vars", "both"))
        h.damp_factors = int(damping_nodes in ("factors", "both"))
        h.start_messages = _cabi.START_MESSAGES[start_messages]
        h.damping, h.stability = float(damping), float(stability)
        self.h, self.cur, self.cycle = h, 0, 0

    def init(self):
        self.lib.ms_host_init(C.byref(self.h))
        self.cur, self.cycle = 0, 0
        return self

    def step(self, n=1):
        for _ in range(n):
            self.lib.ms_host_cycle(C.byref(self.h), self.cur, int(self.cycle == 0))
            self.cur ^= 1
            self.cycle += 1
        return self

    def messages(self):
        L, k = self.L, self.keep
        q = k["q%d" % self.cur][L.message_gather_index_q()].astype(np.float64)
        r = k["r%d" % self.cur][L.message_gather_index()].astype(np.float64)
        return q, r

    def values(self):
        L, k = self.L, self.keep
        return L.vars_to_canonical(k["value"][:L.n_vars]), L.vars_to_canonical(k["value_cost"][:L.n_vars])

    def sent(self):
        L, k = self.L, self.keep
        return (L.slots_to_canonical_edges(k["q_sent"][:L.n_edges]), L.edges_to_canonical(k["r_sent"][:L.n_edges]))


def _compare(eng, o, k, dt):
    q, r = eng.messages()
    assert np.array_equal(q.astype(dt), o.q), ("q", k)
    assert np.array_equal(r.astype(dt), o.r), ("r", k)
    assert np.array_equal(eng.values()[0], o.value), ("value", k)
    qs, rs = eng.sent()
    assert np.array_equal(qs, o.q_sent) and np.array_equal(rs, o.r_sent), ("sent", k)


@pytest.mark.parametrize("name", golden_names("ms_"))
def test_generic_kernel_source_matches_reference_trajectory(name):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    params = {k: v for k, v in meta["params"].items() if k != "noise"}
    eng = HostMaxSum(layout_from_instance(inst), "f64", mode=meta["mode"], **params).init()
    o = orc.MaxSumOracle(inst, np.float64, mode=meta["mode"], **params).init()
    for k in range(min(meta["n_cycles"], 12) + 1):
        if k:
            eng.step()
            o.step()
        q, r = eng.messages()
        assert np.array_equal(q, inst["q_state"][k]) and np.array_equal(r, inst["r_state"][k]), (name, k)
        _compare(eng, o, k, np.float64)


def _mixed_instance(rng, n_vars, doms, shapes):
    """shapes: list of (arity, count); scopes of distinct variables; float tables and unary costs."""
    dom_size = rng.choice(doms, size=n_vars).astype(np.int32)
    fp, ev, tabs = [0], [], []
    for arity, count in shapes:
        for _ in range(count):
            scope = rng.choice(n_vars, size=arity, replace=False)
            ev.extend(scope.tolist())
            fp.append(len(ev))
            tabs.append(rng.uniform(-3, 3, size=int(np.prod(dom_size[scope]))).astype(np.float32))
    return dict(dom_size=dom_size, factor_ptr=np.array(fp, np.int64), edge_var=np.array(ev, np.int32),
                tables=np.concatenate(tabs) if tabs else np.zeros(0, np.float32),
                unary=rng.uniform(0, 0.5, size=int(dom_size.sum())))


@pytest.mark.parametrize("case", ["high_arity", "big_domains", "hub", "unary_only", "max_arity", "max_domain", "no_factors"]
                         + ["limits_" + c for c in LM.MAXSUM])
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_generic_kernel_source_on_shapes_beyond_the_gpu_tests(case, precision):
    """Small shapes of every kind, and the C-ABI limit instances of tests/_limits.py that
    tests/test_gpu_limits.py runs on the device kernels."""
    rng = np.random.default_rng(hash(case) % 1000)
    if case.startswith("limits_"):
        inst = LM.MAXSUM[case[len("limits_"):]]()
    elif case == "high_arity":        # arity 5 and 6 (FG_MAX_ARITY = 8), small domains
        inst = _mixed_instance(rng, 24, [2, 3], [(5, 6), (6, 3), (2, 10), (1, 3)])
    elif case == "big_domains":       # domains up to 40
        inst = _mixed_instance(rng, 14, [17, 33, 40], [(2, 12), (1, 2)])
    elif case == "hub":               # one variable in 40 factors (degree > the class limit of 16)
        inst = _mixed_instance(rng, 30, [3, 4], [(2, 25), (3, 5)])
        hub = np.zeros(0, np.int32)
        fp, ev, tabs = list(inst["factor_ptr"]), list(inst["edge_var"]), [inst["tables"]]
        for other in range(1, 30):
            ev.extend([0, other])
            fp.append(len(ev))
            tabs.append(rng.uniform(-3, 3, size=int(inst["dom_size"][0] * inst["dom_size"][other])).astype(np.float32))
        inst.update(factor_ptr=np.array(fp, np.int64), edge_var=np.array(ev, np.int32), tables=np.concatenate(tabs))
    elif case == "max_arity":         # FG_MAX_ARITY = 8 over binary variables (256-entry tables)
        inst = _mixed_instance(rng, 12, [2], [(8, 3), (2, 6)])
    elif case == "max_domain":        # FG_MAX_DOM = 256
        inst = _mixed_instance(rng, 5, [256, 3], [(2, 4), (1, 2)])
    elif case == "no_factors":        # variables only: every cycle is a no-op that must not crash
        inst = _mixed_instance(rng, 6, [2, 4], [])
    else:                              # unary factors only + isolated variables
        inst = _mixed_instance(rng, 12, [3, 5], [(1, 7)])
    L = build_layout(**inst)
    dt = np.float64 if precision == "f64" else np.float32
    for params in (dict(), dict(mode="max", damping_nodes="vars", start_messages="all"),
                   dict(damping_nodes="none", start_messages="leafs_vars", stability=0.01)):
        eng = HostMaxSum(L, precision, **params).init()
        o = orc.MaxSumOracle(oracle_instance(inst, L), dt, **params).init()
        for k in range(9):
            if k:
                eng.step()
                o.step()
            _compare(eng, o, (case, k), dt)


@settings(max_examples=25, deadline=None)
@given(st.integers(0, 10_000), st.integers(4, 20), st.sampled_from(["both", "vars", "factors", "none"]),
       st.sampled_from(["leafs", "leafs_vars", "all"]), st.sampled_from(["min", "max"]))
def test_generic_kernel_source_fuzz(seed, n_vars, damping_nodes, start, mode):
    rng = np.random.default_rng(seed)
    shapes = [(int(a), int(rng.integers(1, 8))) for a in rng.choice([1, 2, 3, 4], size=3) if a <= n_vars]
    inst = _mixed_instance(rng, n_vars, [2, 3, 5, 7], shapes)
    L = build_layout(**inst)
    params = dict(mode=mode, damping_nodes=damping_nodes, start_messages=start, damping=float(rng.uniform(0, 0.9)))
    eng = HostMaxSum(L, "f64", **params).init()
    o = orc.MaxSumOracle(oracle_instance(inst, L), np.float64, **params).init()
    for k in range(7):
        if k:
            eng.step()
            o.step()
        _compare(eng, o, k, np.float64)


@pytest.mark.parametrize("name", golden_names("msx_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_generic_kernel_source_with_infinite_costs(name, precision):
    """+/-inf table entries: inf and NaN messages.  f64 against the reference trajectory, f32 against
    the f32 oracle; NaN positions, send decisions and values included."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    params = {k: v for k, v in meta["params"].items() if k != "noise"}
    dt = np.float64 if precision == "f64" else np.float32
    eng = HostMaxSum(layout_from_instance(inst), precision, mode=meta["mode"], **params).init()
    o = orc.MaxSumOracle(inst, dt, mode=meta["mode"], **params).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            eng.step()
            o.step()
        q, r = eng.messages()
        assert np.array_equal(q.astype(dt), o.q, equal_nan=True) and np.array_equal(r.astype(dt), o.r, equal_nan=True), k
        if precision == "f64":
            assert np.array_equal(q, inst["q_state"][k], equal_nan=True), k
            assert np.array_equal(r, inst["r_state"][k], equal_nan=True), k
        assert np.array_equal(eng.values()[0], o.value), k
        qs, rs = eng.sent()
        assert np.array_equal(qs, o.q_sent) and np.array_equal(rs, o.r_sent), k
