"""solve(..., "syncbb") on the CPU: the algorithm names, parameters, refusals and the result dict's conventions,
with the oracle behind the engine seam.  The device runs are tests/test_gpu_zz_syncbb.py's."""
import os

import numpy as np
import pytest

import oracle as orc
from _syncbb_oracle import SyncbbOracle
from conftest import GOLDEN_DIR
from pydcop_b200 import solve as S


class OracleEngine:
    """The engine seam of solve(): SyncbbEngine's interface over the oracle."""

    def __init__(self, kind, layout, inst, params):
        assert kind == "syncbb"
        self.o = SyncbbOracle(inst, np.float64, params["mode"], inst["var_rank"])

    def init(self):
        self.o.init()
        return self

    def step(self, n):
        self.o.run(n)

    @property
    def finished(self):
        return self.o.finished

    @property
    def messages(self):
        return self.o.messages

    @property
    def cycle(self):
        return int(self.o.cycle_counts().max())

    def values(self):
        return self.o.values()


def fixture_dict(name):
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    keys = ("dom_size", "factor_ptr", "edge_var", "tables", "unary")
    d = {k: inst[k] for k in keys}
    d["var_names"] = [str(x) for x in inst["var_names"]]
    d["objective"] = meta["mode"]
    return d, inst


@pytest.mark.parametrize("algo", ["syncbb", "syncbb_gpu"])
def test_solve_reports_the_reference_run(algo):
    """graph_coloring_tuto.yaml through the seam: cost 12, 23 SyncBB messages, FINISHED, and cycle 9, the largest
    new_cycle count (v3's), which the reference's orchestrated run reports."""
    d, inst = fixture_dict("syncbb_tuto")
    res = S.solve(d, algo, engine_factory=OracleEngine)
    assert res["status"] == "FINISHED" and res["cost"] == 12 and res["violation"] == 0
    assert res["msg_count"] == 23 and res["cycle"] == 9 == int(inst["cycle_count"].max())
    assert list(res["assignment"].values()) == [1, 1, 1, 1]      # G G G G


def test_solve_infeasible_leaves_the_assignment_incomplete():
    d, inst = fixture_dict("syncbb_infeasible")
    res = S.solve(d, "syncbb", engine_factory=OracleEngine)
    assert res["status"] == "FINISHED" and res["assignment"] == {}
    assert res["cost"] is None and res["violation"] is None


def test_solve_timeout_keeps_the_state():
    d, inst = fixture_dict("syncbb_name_order")
    res = S.solve(d, "syncbb", timeout=0.0, engine_factory=OracleEngine)
    assert res["status"] == "TIMEOUT" and res["msg_count"] == 1


def test_solve_refuses_parameters_arity3_and_sharding():
    d, _ = fixture_dict("syncbb_tuto")
    with pytest.raises(ValueError, match="takes no parameters"):
        S.solve(d, "syncbb", {"stop_cycle": 3}, engine_factory=OracleEngine)
    d3, _ = fixture_dict("syncbb_arity3")
    d3["con_names"] = ["ab", "abc"]
    with pytest.raises(ValueError, match="has arity 3"):
        S.solve(d3, "syncbb", engine_factory=OracleEngine)
    with pytest.raises(ValueError, match="syncbb is not sharded"):
        S.solve(d, "syncbb", distributed=True)
