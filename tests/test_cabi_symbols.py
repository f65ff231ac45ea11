"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/pydcop_b200.h declares; without a GPU the product path fails loudly (no CPU fallback)."""
import os
import re

import pytest

from conftest import ROOT


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "pydcop_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fg_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_all_exported_and_bound():
    from pydcop_b200 import _cabi, build
    build.build()
    lib = _cabi.load()
    declared = _declared_symbols()
    assert declared, "no declarations parsed"
    assert sorted(_cabi.SYMBOLS) == declared
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.fg_abi_version() == _cabi.FG_ABI_VERSION


def test_struct_sizes_match_header():
    """sizeof of the ctypes mirrors == what the C compiler lays out for include/pydcop_b200.h."""
    import ctypes as C
    import subprocess
    import tempfile
    from pydcop_b200 import _cabi
    prog = r'''
#include <stdio.h>
#include "pydcop_b200.h"
int main(void){printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(fg_class_t), sizeof(fg_maxsum_desc_t), sizeof(fg_dsa_desc_t), sizeof(fg_mgm_desc_t), sizeof(fg_varclass_t), sizeof(fg_peer_sync_t), sizeof(fg_halo_plan_t));return 0;}
'''
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "s.c"), os.path.join(td, "s")
        open(src, "w").write(prog)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I",
                        os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in out] == [C.sizeof(_cabi.FgClass), C.sizeof(_cabi.FgMaxSumDesc),
                                     C.sizeof(_cabi.FgDsaDesc), C.sizeof(_cabi.FgMgmDesc),
                                     C.sizeof(_cabi.FgVarClass), C.sizeof(_cabi.FgPeerSync),
                                     C.sizeof(_cabi.FgHaloPlan)]


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import numpy as np
    from pydcop_b200 import build_layout
    from pydcop_b200.engine import EngineError, MaxSumEngine, DsaEngine, MgmEngine
    L = build_layout([2, 2], [0, 2], [0, 1], np.zeros(4))
    with pytest.raises(EngineError):
        MaxSumEngine(L)
    with pytest.raises(EngineError):
        DsaEngine(L)
    with pytest.raises(EngineError):
        MgmEngine(L)


def test_create_validates_its_descriptor_before_touching_the_device():
    """fg_maxsum_create / fg_dsa_create reject malformed descriptors with FG_ERR_ARG and a
    message, and report FG_ERR_CUDA (never a silent CPU path) when no device is visible."""
    import ctypes as C
    import torch
    from pydcop_b200 import _cabi
    lib = _cabi.load()
    h = C.c_void_p()
    assert lib.fg_maxsum_create(None, C.byref(h)) == _cabi.FG_ERR_ARG
    assert lib.fg_dsa_create(None, C.byref(h)) == _cabi.FG_ERR_ARG
    assert lib.fg_mgm_create(None, C.byref(h)) == _cabi.FG_ERR_ARG
    m = _cabi.FgMgmDesc()
    m.abi_version, m.precision = _cabi.FG_ABI_VERSION, 9
    assert lib.fg_mgm_create(C.byref(m), C.byref(h)) == _cabi.FG_ERR_ARG and not h.value
    m.precision, m.n_vars = _cabi.FG_F64, 3  # device arrays missing
    assert lib.fg_mgm_create(C.byref(m), C.byref(h)) == _cabi.FG_ERR_ARG
    assert b"missing device array" in lib.fg_mgm_last_error(h)
    lib.fg_mgm_destroy(h)

    d = _cabi.FgMaxSumDesc()
    d.abi_version, d.precision = _cabi.FG_ABI_VERSION + 1, _cabi.FG_F32
    assert lib.fg_maxsum_create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_ARG and not h.value
    d.abi_version, d.precision = _cabi.FG_ABI_VERSION, 7
    assert lib.fg_maxsum_create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_ARG and not h.value

    # one binary class whose table_size disagrees with its domain sizes
    cls = (_cabi.FgClass * 1)()
    cls[0].arity, cls[0].n_factors, cls[0].table_size, cls[0].row_total = 2, 1, 5, 4
    cls[0].dom[0], cls[0].dom[1] = 2, 2
    cls[0].row_off[0], cls[0].row_off[1] = 0, 2
    d.precision, d.n_classes, d.n_edges, d.n_factors, d.n_vars = _cabi.FG_F32, 1, 2, 1, 2
    d.classes = C.cast(cls, C.POINTER(_cabi.FgClass))
    assert lib.fg_maxsum_create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_ARG
    assert b"class size mismatch" in lib.fg_maxsum_last_error(h)
    lib.fg_maxsum_destroy(h)

    # consistent class, but the variable classes do not cover the edges
    cls[0].table_size = 4
    assert lib.fg_maxsum_create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_ARG
    assert b"variable classes cover 0 slots, expected 2" in lib.fg_maxsum_last_error(h)
    lib.fg_maxsum_destroy(h)

    if not torch.cuda.is_available():
        vcs = (_cabi.FgVarClass * 1)()
        vcs[0].dom, vcs[0].degree, vcs[0].n_vars, vcs[0].n_slots = 2, 1, 2, 2
        d.n_varclasses, d.varclasses = 1, C.cast(vcs, C.POINTER(_cabi.FgVarClass))
        assert lib.fg_maxsum_create(C.byref(d), C.byref(h)) == _cabi.FG_ERR_CUDA
        assert b"no CPU fallback" in lib.fg_maxsum_last_error(h)
        lib.fg_maxsum_destroy(h)
        assert lib.fg_device_count() <= 0


@pytest.mark.parametrize("family", ["mgm", "mgm2", "gdba", "dpop"])
def test_plan_passes_every_create_check(family):
    """The descriptor a family's host-array plan fills (host arrays here) passes every argument check of
    fg_<family>_create: without a device the one refusal left is FG_ERR_CUDA."""
    import ctypes as C
    import torch
    from pydcop_b200 import _cabi, build_layout, engine as E, pseudotree as pt
    from pydcop_b200.generators import bounded_separator_instance
    inst = bounded_separator_instance(14, 4, back=3, span=1, seed=6, float_costs=True)
    L = build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"], unary=inst["unary"])
    if family == "dpop":
        tree = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
        inputs, state, scalars = E.dpop_plan(L, tree, pt.schedule(tree), "f64")
        d = _cabi.FgDpopDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, _cabi.FG_F64
    else:
        plan, desc, kw = {"mgm": (E.mgm_plan, _cabi.FgMgmDesc, {}), "mgm2": (E.mgm2_plan, _cabi.FgMgm2Desc, {}),
                          "gdba": (E.gdba_plan, _cabi.FgGdbaDesc, dict(violation="NM"))}[family]
        inputs, state, scalars = plan(L, "f64", **kw)
        classes = E._class_array(L)
        d = E.fill_header(desc(), "f64", L, classes)
    arrays = dict(inputs, **E.host_state(state))
    E.fill_desc(d, arrays, scalars)
    lib = _cabi.load()
    h = C.c_void_p()
    rc = getattr(lib, f"fg_{family}_create")(C.byref(d), C.byref(h))
    msg = (getattr(lib, f"fg_{family}_last_error")(h) or b"").decode()
    getattr(lib, f"fg_{family}_destroy")(h)
    if torch.cuda.is_available():
        assert rc == _cabi.FG_OK, msg
    else:
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device visible" in msg, (rc, msg)
