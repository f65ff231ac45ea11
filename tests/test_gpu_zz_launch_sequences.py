"""The device entry points and the host shims run one launch sequence (the kernel headers' shared templates): after
init and k cycles, every engine's launch_count equals the launches the host shim ran for the same plan.  MGM's
active-row value phase replaces the shared gain launch one for one, so its count matches too."""
import numpy as np
import pytest

from pydcop_b200.engine import DbaEngine, GdbaEngine, MgmEngine, Mgm2Engine, MixedDsaEngine
from pydcop_b200.layout import layout_from_instance
from test_dba_hostshim import HostDba, random_dba_instance
from test_gdba_hostshim import HostGdba, random_gdba_instance
from test_mgm2_hostshim import HostMgm2, random_mgm2_instance
from test_mgm_hostshim import HostMgm
from test_mixeddsa_hostshim import HostMixedDsa, random_mixed

pytestmark = pytest.mark.gpu

CASES = [
    ("mgm", MgmEngine, HostMgm, lambda: random_mgm2_instance(60, 4, [2, 3], seed=1), {}),
    ("mgm2", Mgm2Engine, HostMgm2, lambda: random_mgm2_instance(60, 4, [2, 3], seed=2), dict(favor="coordinated")),
    ("gdba", GdbaEngine, HostGdba, lambda: random_gdba_instance(60, 4, seed=3), dict(increase_mode="T")),
    ("mixeddsa", MixedDsaEngine, HostMixedDsa, lambda: random_mixed(60, seed=4), {}),
    ("dba", DbaEngine, HostDba, lambda: random_dba_instance(60, 3, seed=5), {}),
]


@pytest.mark.parametrize("kind,engine,host,make,params", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_device_and_host_launch_the_same_sequence(kind, engine, host, make, params, precision):
    inst = make()
    L = layout_from_instance(inst)
    kw = dict(precision=precision, seed=7, **params)
    dev = engine(L, device="cuda:0", **kw).init()
    cpu = host(L, **kw).init()
    assert dev.launch_count == cpu.launches > 0
    for k in range(1, 6):
        dev.step()
        cpu.step()
        assert dev.launch_count == cpu.launches, (kind, k)
    assert np.array_equal(dev.values()[0], cpu.values()[0])
