"""CPU: the hard-constraint fixtures (tests/golden/msx_*.npz, oracle/make_golden_extra.py) really reach
the corner they were built for: a factor->variable output whose candidates are all NaN, on the factor-kernel
site of the fixture, and the reference sends +/-inf there."""
import os

import numpy as np
import pytest

import oracle as orc
from _hard_constraints import all_nan_outputs, factor_family, output_site
from conftest import GOLDEN_DIR, golden_names

# fixture -> sites (tests/_hard_constraints.py::output_site) it must reach
EXPECTED_SITES = {
    "msx_hard_inf_min": {"pipe arity 2", "tiled_rt"},
    "msx_hard_inf_max": {"pipe arity 2", "tiled_rt"},
    "msx_warp_d4_min": {"warp pair"},
    "msx_warp_d4_max": {"warp pair"},
    "msx_warp_d10": {"warp pair", "warp single"},
    "msx_pipe_bin_d2_d5": {"pipe arity 2"},
    "msx_pipe_tern_min": {"pipe arity 3"},
    "msx_pipe_tern_max": {"pipe arity 3"},
    "msx_tiled_rt_mixed": {"tiled_rt"},
    "msx_p_nodamp": {"warp pair"},
    "msx_p_stab_tiny": {"warp pair"},
    "msx_p_start_all": {"warp pair"},
}


def _shape(inst, f):
    fp, ev, dom = inst["factor_ptr"], inst["edge_var"], inst["dom_size"]
    return tuple(int(d) for d in dom[ev[fp[f]:fp[f + 1]]])


def test_every_fixture_has_expected_sites():
    assert set(golden_names("msx_")) == set(EXPECTED_SITES)


@pytest.mark.parametrize("name", golden_names("msx_"))
def test_fixture_reaches_all_nan_marginals(name):
    """For every expected site, some cycle has an output there whose candidates (from the table and the
    q rows of the previous cycle) are all NaN, and for which the reference sends +/-inf."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    moff = np.concatenate([[0], np.cumsum(inst["dom_size"][inst["edge_var"]])])
    sign = np.inf if meta["mode"] == "min" else -np.inf
    seen = set()
    for k in range(1, meta["n_cycles"] + 1):
        for f, j, x in all_nan_outputs(inst, inst["q_state"][k - 1], inst["q_valid"][k - 1]):
            e = inst["factor_ptr"][f] + j
            # counted where the NaN a kernel without the +/-inf start would compute is not hidden by damping
            # with a non-finite previous message
            if inst["r_sent"][k][e] and inst["r_state"][k][moff[e] + x] == sign:
                seen.add(output_site(_shape(inst, f), j, x))
    assert EXPECTED_SITES[name] <= seen, (name, seen)


def test_fixtures_cover_the_shapes_of_every_kernel_site():
    """Across the fixture set: arity 7 and 8 over D = 2 and a binary factor wider than a warp on the
    runtime-shape kernel; unary factors whose whole row is infinite; variables of degree 1..8, 9..16 and
    > 16 next to binary D = 4 factors; min and max mode on the warp and the arity-3 sites."""
    shapes, degrees_d4, modes = set(), set(), {}
    unary_all_inf = False
    for name in golden_names("msx_"):
        inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
        fp, toff = inst["factor_ptr"], inst["table_off"]
        for f in range(len(fp) - 1):
            sh = _shape(inst, f)
            shapes.add(sh)
            t = inst["tables"][toff[f]:toff[f + 1]]
            unary_all_inf |= len(sh) == 1 and bool(np.isinf(t).all())
        if set(inst["dom_size"].tolist()) == {4}:
            degrees_d4.update(np.diff(inst["var_ptr"]).tolist())
        for site in EXPECTED_SITES[name]:
            modes.setdefault(site, set()).add(meta["mode"])
    assert (2,) * 7 in shapes and (2,) * 8 in shapes
    assert any(len(s) == 2 and max(s) > 32 and factor_family(s) == "tiled_rt" for s in shapes)
    assert any(len(set(s)) > 1 for s in shapes)
    assert unary_all_inf
    assert any(1 <= d <= 8 for d in degrees_d4) and any(9 <= d <= 16 for d in degrees_d4)
    assert max(degrees_d4) > 16
    assert modes["warp pair"] == {"min", "max"} and modes["pipe arity 3"] == {"min", "max"}
