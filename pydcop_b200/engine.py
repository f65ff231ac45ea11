"""Python host of the GPU engine: device memory (torch), streams, and the C-ABI calls.

`MaxSumEngine` / `DsaEngine` are what the pyDcop plugin modules (pydcop_b200/algorithms/) and
bench.py drive.  All arithmetic on messages happens in libpydcop_b200.so (hand-written sm_90a
kernels); torch only owns the buffers.  There is no CPU path: constructing an engine without a
CUDA device raises EngineError.
"""
import ctypes as C
import functools
import os
from typing import Optional

import numpy as np
import torch

from . import _cabi
from ._cabi import EngineError, FgClass, FgDsaDesc, FgMaxSumDesc, FgMgmDesc, FgVarClass
from .layout import FactorGraphLayout

PRECISIONS = {"f32": (_cabi.FG_F32, torch.float32, np.float32),
              "f64": (_cabi.FG_F64, torch.float64, np.float64)}


def _require_cuda(device):
    if not torch.cuda.is_available():
        raise EngineError("no CUDA device: pydcop_b200 runs the MaxSum/DSA hot path on the GPU "
                          "only (no CPU fallback)")
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise EngineError(f"device must be a CUDA device, got {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _class_array(layout: FactorGraphLayout):
    arr = (FgClass * max(1, len(layout.classes)))()
    for i, c in enumerate(layout.classes):
        fc = arr[i]
        fc.arity = c.arity
        for j in range(c.arity):
            fc.dom[j] = c.dom[j]
            fc.row_off[j] = c.row_off[j]
        fc.row_total = c.row_total
        fc.n_factors, fc.first_factor, fc.first_edge = c.n_factors, c.first_factor, c.first_edge
        fc.flags = 1 if c.tag else 0
        fc.table_size, fc.table_base, fc.msg_base = c.table_size, c.table_base, c.msg_base
    return arr


def _varclass_array(layout: FactorGraphLayout):
    arr = (FgVarClass * max(1, len(layout.var_classes)))()
    for i, c in enumerate(layout.var_classes):
        vc = arr[i]
        vc.dom, vc.degree, vc.n_vars = c.dom, c.degree, c.n_vars
        vc.first_var, vc.first_slot, vc.n_slots = c.first_var, c.first_slot, c.n_slots
        vc.unary_base, vc.q_base = c.unary_base, c.q_base
        vc.flags = (1 if c.tag == 2 else 0) | (2 if c.tag == 1 else 0)   # FG_CLASS_GHOST | FG_CLASS_BOUNDARY (multigpu.build_shard)
    return arr


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr() if t is not None and t.numel() else 0) if t is not None \
        else C.c_void_p(0)


def _addr(a):
    """Address of a torch tensor (device) or numpy array (host); NULL for None or an empty one."""
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data if a.size else 0)
    return _ptr(a)


def fill_desc(d, arrays, scalars=(), prefix="dev_"):
    """d.<prefix><name> = the address of every array of `arrays` (name -> tensor, numpy array or None; a list of two
    fills a double-buffer field), then d.<name> = value for every scalar field.  An unknown field raises."""
    for name in [prefix + k for k in arrays] + list(dict(scalars)):
        if not hasattr(type(d), name):
            raise AttributeError(f"{type(d).__name__} has no field {name}")
    for name, a in arrays.items():
        if isinstance(a, list):
            for b, x in enumerate(a):
                getattr(d, prefix + name)[b] = _addr(x)
        else:
            setattr(d, prefix + name, _addr(a))
    for name, v in dict(scalars).items():
        setattr(d, name, v)
    return d


def fill_header(d, precision, layout, classes):
    """The fields every descriptor with a class table starts with; `classes` from _class_array(layout)."""
    L = layout
    d.abi_version, d.precision = _cabi.FG_ABI_VERSION, PRECISIONS[precision][0]
    d.n_vars, d.n_factors, d.n_edges, d.n_classes = L.n_vars, L.n_factors, L.n_edges, len(L.classes)
    d.classes = C.cast(classes, C.POINTER(FgClass))
    return d


def host_state(state):
    """The state of a host-array plan as numpy arrays (what the engines allocate on the device)."""
    return {k: np.full(max(n, 1), 0 if fill is None else fill, dtype=dt) for k, (n, dt, fill) in state.items()}


_TORCH_DTYPES = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64,
                 np.dtype(np.int32): torch.int32, np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8,
                 np.dtype(np.uint64): torch.uint64, np.dtype(np.uint16): torch.uint16}


class _EngineBase:
    """Lifecycle of an engine's handle: FAMILY names its fg_<FAMILY>_* functions.  Subclasses build the descriptor,
    call _create and supply _assignment (the current value of every variable, internal order, on the device)."""
    FAMILY = None

    def _open(self, layout, device, precision):
        self.lib = _cabi.load()
        self.device = _require_cuda(device)
        self.layout = layout
        self.precision = precision
        prec, tdt, self.np_dtype = PRECISIONS[precision]
        return tdt

    def _fn(self, name):
        return getattr(self.lib, f"fg_{self.FAMILY}_{name}")

    def _create(self, d):
        """The handle over descriptor `d`; it belongs to self.device, which every later call makes current."""
        self._desc, self._h = d, C.c_void_p()
        with torch.cuda.device(self.device):
            self._check(self._fn("create")(C.byref(d), C.byref(self._h)), f"fg_{self.FAMILY}_create")

    def _upload(self, inputs, state):
        """Every input of a host-array plan through _dev, in order (None stays None), then the state allocated on the
        device without a host copy (fill None: uninitialised).  Returns name -> tensor, or a list of two."""
        out = {}
        with torch.cuda.device(self.device):
            for k, a in inputs.items():
                if isinstance(a, list):
                    out[k] = [self._dev(x, _TORCH_DTYPES[x.dtype]) for x in a]
                else:
                    out[k] = None if a is None else self._dev(a, _TORCH_DTYPES[a.dtype])
            for k, (n, dt, fill) in state.items():
                dt = _TORCH_DTYPES[np.dtype(dt)]
                out[k] = (torch.empty(max(n, 1), dtype=dt, device=self.device) if fill is None
                          else torch.full((max(n, 1),), fill, dtype=dt, device=self.device))
        return out

    def _last_error(self):
        return (self._fn("last_error")(self._h) or b"").decode()

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            with torch.cuda.device(self.device):   # __del__ may run with any device current
                self._fn("destroy")(self._h)
                if getattr(self, "_trace", None) is not None and self._trace["h"] is not None:
                    self.lib.fg_trace_destroy(self._trace["h"])
            self._h = C.c_void_p()
            self._trace = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def init(self):
        with torch.cuda.device(self.device):
            self._check(self._fn("init")(self._h, self._stream()), f"fg_{self.FAMILY}_init")
        return self

    def step(self, n_cycles=1):
        """n_cycles cycles of fg_<FAMILY>_step.  With a trace started, a full trace block is moved aside and the trace
        restarted whenever more cycles follow, so every cycle is recorded."""
        n = int(n_cycles)
        with torch.cuda.device(self.device):
            while True:
                k = n
                tr = getattr(self, "_trace", None)
                if tr is not None and tr["h"] is not None:
                    if self._trace_rows() >= tr["capacity"] and n > 0:
                        self._trace_rotate()
                    k = min(n, tr["capacity"] - self._trace_rows())
                self._check(self._fn("step")(self._h, k, self._stream()), f"fg_{self.FAMILY}_step")
                n -= k
                if n <= 0:
                    break
        return self

    @property
    def launch_count(self):
        return int(self._fn("launch_count")(self._h))

    def solution_cost(self, infinity=float("inf"), unary=None):
        """(cost, violations) of the current assignment, reduced on the device (pydcop/dcop/dcop.py:319-367;
        `infinity` as `pydcop solve -i`).  `unary`: the variables' own costs in canonical order (MaxSum: WITHOUT its
        noise); default: variable costs are not added."""
        with torch.cuda.device(self.device):
            out = self._solution_cost(self._assignment(), infinity, unary).cpu().numpy()
        return float(out[0]), int(out[1])

    def solution_costs_segmented(self, seg_factor, seg_var, n_seg, infinity=float("inf"), unary=None):
        """(cost float64[n_seg], violations int64[n_seg]) of the current assignment per segment, reduced on the device
        (fg_solution_cost_segmented): what solution_cost computes over the factors and variables of each segment.
        seg_factor / seg_var: the segment (problem of a batch) of every factor and variable, canonical order."""
        with torch.cuda.device(self.device):
            seg = self._segments(seg_factor, seg_var, n_seg)
            out = self._solution_cost(self._assignment(), infinity, unary, seg=seg).cpu().numpy().reshape(-1, 2)
        return out[:, 0].copy(), out[:, 1].astype(np.int64)

    def _segments(self, seg_factor, seg_var, n_seg):
        """(factor segment, variable segment, n_seg) on the device in internal order, from canonical seg_factor /
        seg_var."""
        L = self.layout
        f_int = np.zeros(max(L.n_factors, 1), dtype=np.int32)
        f_int[L.factor_perm] = np.asarray(seg_factor, dtype=np.int32)
        v_int = _per_var(L, np.asarray(seg_var, dtype=np.int32)[L.var_order], np.int32)
        return self._dev(f_int, torch.int32), self._dev(v_int, torch.int32), int(n_seg)

    def start_trace(self, capacity, infinity=float("inf"), unary=None, seg=None, best=False, rows=True):
        """Record (cost, violations) of the current values after every cycle step() runs from now on, on the device
        and without synchronising (fg_trace_*): solution_cost's sums, or with seg = (seg_factor, seg_var, n_seg) as
        in solution_costs_segmented, solution_costs_segmented's.  `capacity`: rows per trace block; a full block is
        moved aside on the device and the trace goes on, so any number of cycles is recorded.
        best: also keep each segment's best recorded cycle and its values on the device (fg_trace_set_best, in the
        engine's mode), read by best().  rows=False (with best): the rows are only scratch for the best; a full
        block is restarted without a copy and trace() has nothing to give."""
        self.stop_trace()
        L = self.layout
        with torch.cuda.device(self.device):
            self._cost_inputs()
            segd = None if seg is None else self._segments(*seg)
            n_seg = 1 if seg is None else segd[2]
            capacity = max(1, int(capacity))
            rows_kept = rows or not best
            rows = torch.zeros(capacity * n_seg * 2, dtype=torch.float64, device=self.device)
            stamp = torch.zeros(capacity + 1, dtype=torch.int64, device=self.device)
            un = self._unary_dev(unary)
            d = _cabi.FgTraceDesc()
            d.abi_version, d.precision = _cabi.FG_ABI_VERSION, PRECISIONS[self.precision][0]
            d.n_vars, d.n_classes = L.n_vars, len(L.classes)
            d.classes = C.cast(self._classes, C.POINTER(FgClass))
            fill_desc(d, {"tables": self.tables, "edge_var": self._edge_var_dev, "unary": un,
                          "unary_off": self._cost_unary_off, "factor_seg": None if segd is None else segd[0],
                          "var_seg": None if segd is None else segd[1], "rows": rows, "stamp": stamp},
                      {"n_seg": n_seg, "infinity": float(infinity), "capacity": capacity})
            h = C.c_void_p()
            rc = self.lib.fg_trace_create(C.byref(d), C.byref(h))
            if rc != _cabi.FG_OK:
                msg = (self.lib.fg_trace_last_error(h) or b"").decode()
                self.lib.fg_trace_destroy(h)
                raise EngineError(f"fg_trace_create failed (rc={rc}): {msg}")
            self._trace = {"h": h, "capacity": capacity, "n_seg": n_seg, "rows": rows, "stamp": stamp,
                           "keep": (un, segd), "done": [], "keep_rows": bool(rows_kept), "best": None}
            self._trace_check(self.lib.fg_trace_start(h, self._stream()), "fg_trace_start")
            if best:
                b = (torch.zeros(2 * n_seg, dtype=torch.float64, device=self.device),
                     torch.zeros(n_seg, dtype=torch.int64, device=self.device),
                     torch.zeros(max(L.n_vars, 1), dtype=torch.int32, device=self.device))
                self._trace_check(self.lib.fg_trace_set_best(h, int(getattr(self._desc, "mode_max", 0)), _ptr(b[0]),
                                                             _ptr(b[1]), _ptr(b[2]), self._stream()),
                                  "fg_trace_set_best")
                self._trace["best"] = b
            self._check(self._fn("set_trace")(self._h, h), f"fg_{self.FAMILY}_set_trace")
        return self

    def _trace_check(self, rc, what):
        if rc != _cabi.FG_OK:
            raise EngineError(f"{what} failed (rc={rc}): "
                              f"{(self.lib.fg_trace_last_error(self._trace['h']) or b'').decode()}")

    def _trace_rows(self):
        if self._trace["h"] is None:   # stopped
            return self._trace["stopped_rows"]
        n = C.c_int64()
        self.lib.fg_trace_rows(self._trace["h"], C.byref(n))
        return n.value

    def _trace_rotate(self):
        """A full block: its rows and stamps copied aside on the stream (not when the rows are only the best's
        scratch), the trace restarted behind them; the best is kept outside the rows and survives."""
        tr = self._trace
        if tr["keep_rows"]:
            tr["done"].append((tr["rows"].clone(), tr["stamp"].clone(), self._trace_rows()))
        self._trace_check(self.lib.fg_trace_start(tr["h"], self._stream()), "fg_trace_start")

    def trace(self):
        """The cycles recorded since start_trace: cost float64[rows, n_seg], violation int64[rows, n_seg] and time
        float64[rows], seconds on the device's global timer from start_trace to the end of each row's record.
        Synchronises (it is the only call of a trace that does)."""
        tr = self._trace
        if tr is None:
            raise EngineError("no trace started")
        if not tr["keep_rows"]:
            raise EngineError("the trace keeps no rows: it was started with rows=False")
        with torch.cuda.device(self.device):
            blocks = tr["done"] + [(tr["rows"], tr["stamp"], self._trace_rows())]
            t0 = int(blocks[0][1][0].item())
            rows = [r.view(-1, tr["n_seg"], 2)[:n].cpu().numpy() for r, _, n in blocks]
            stamps = [s[1:n + 1].cpu().numpy() for _, s, n in blocks]
        out = np.concatenate(rows) if rows else np.zeros((0, tr["n_seg"], 2))
        return {"cost": out[:, :, 0].copy(), "violation": out[:, :, 1].astype(np.int64),
                "time": (np.concatenate(stamps).astype(np.int64) - t0) * 1e-9}

    def best(self):
        """The best cycle of each segment since start_trace(best=True) (fg_trace_set_best's rule: fewer violations,
        then a strictly better cost in the engine's mode, ties to the earlier cycle): cycle int64[n_seg] (the trace's
        numbering, 1 = the first cycle recorded; 0 = none), cost float64[n_seg] and violation int64[n_seg] (that
        row's), and value, the values after that cycle in canonical variable order (each variable's from its own
        segment's best cycle).  Synchronises; still readable after stop_trace."""
        tr = self._trace
        if tr is None or tr["best"] is None:
            raise EngineError("no best kept: start_trace(best=True) first")
        with torch.cuda.device(self.device):
            b, cycle, value = (t.cpu().numpy() for t in tr["best"])
        b = b.reshape(-1, 2)
        return {"cycle": cycle.astype(np.int64), "cost": b[:, 0].copy(), "violation": b[:, 1].astype(np.int64),
                "value": self.layout.vars_to_canonical(value[:self.layout.n_vars])}

    def stop_trace(self):
        """Detach the trace: the step loop is the plain one again.  trace() still reads what was recorded."""
        tr = getattr(self, "_trace", None)
        if tr is None or tr["h"] is None:
            return
        with torch.cuda.device(self.device):
            self._check(self._fn("set_trace")(self._h, None), f"fg_{self.FAMILY}_set_trace")
            tr["stopped_rows"] = self._trace_rows()
            self.lib.fg_trace_destroy(tr["h"])
        tr["h"] = None

    def _dev(self, a, dtype):
        a = np.ascontiguousarray(a)
        if not a.flags.writeable:      # e.g. a read-only memory map of the binary container
            a = a.copy()
        t = torch.from_numpy(a).to(device=self.device, dtype=dtype)
        self.h2d_bytes = getattr(self, "h2d_bytes", 0) + t.numel() * t.element_size()   # what crossed PCIe / C2C
        return t

    def _dev_tables(self, L, dtype):
        """L.tables on the device.  A layout that deferred its table permutation (one class; FactorGraphLayout.table_rows)
        and was not read on the host yet is permuted on the device by fg_gather_rows: the caller's array is uploaded as
        it is, without a host copy."""
        if L.table_rows is None or L._tables is not None:
            return self._dev(L.tables, dtype)
        src = self._dev(L.table_src, dtype)
        rows = self._dev(L.table_rows, torch.int64)
        out = torch.zeros(max(int(L.table_total), 1), dtype=dtype, device=self.device)
        n = len(L.table_rows)
        rc = self.lib.fg_gather_rows(PRECISIONS[self.precision][0], _ptr(out), _ptr(src), _ptr(rows), n,
                                     int(L.table_src.size // n), self._stream())
        self._check(rc, "fg_gather_rows")
        return out

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check(self, rc, what):
        if rc != _cabi.FG_OK:
            raise EngineError(f"{what} failed (rc={rc}): {self._last_error()}")

    def _solution_cost(self, value_tensor, infinity=float("inf"), unary=None, n_vars=None, factor_skip=None,
                       var_skip=None, seg=None):
        """(cost, violations) of `value_tensor` (internal variable order) as LOCAL sums, on the device:
        pydcop/dcop/dcop.py:319-367 — an entry equal to `infinity` is a violation, the others are
        summed, constraints and variable costs alike.  `unary`: the variables' own costs in CANONICAL
        order (default: none are added); n_vars: leading variables that count (a shard's own ones);
        factor_skip / var_skip: uint8 device tensors in internal order, non-zero = owned by another rank;
        seg: (factor segment, variable segment, n_seg), int32 device tensors in internal order, for n_seg
        (cost, violations) pairs (fg_solution_cost_segmented)."""
        L = self.layout
        prec = PRECISIONS[self.precision][0]
        with torch.cuda.device(self.device):
            self._cost_inputs()
            out = self._cost_out if seg is None else torch.zeros(2 * seg[2], dtype=torch.float64, device=self.device)
            un = self._unary_dev(unary)
            args = (prec, len(L.classes), C.cast(self._classes, C.POINTER(FgClass)), _ptr(self.tables),
                    _ptr(self._edge_var_dev), _ptr(value_tensor), _ptr(un), _ptr(self._cost_unary_off),
                    int(L.n_vars if n_vars is None else n_vars), _ptr(factor_skip), _ptr(var_skip))
            if seg is None:
                rc = self.lib.fg_solution_cost(*args, float(infinity), _ptr(out), self._stream())
            else:
                rc = self.lib.fg_solution_cost_segmented(*args, _ptr(seg[0]), _ptr(seg[1]), seg[2], float(infinity),
                                                         _ptr(out), self._stream())
            self._check(rc, "fg_solution_cost" if seg is None else "fg_solution_cost_segmented")
            return out


    def _cost_inputs(self):
        """The device arrays of the cost reductions the engine's descriptor does not hold, made once."""
        if not hasattr(self, "_cost_out"):
            L = self.layout
            self._edge_var_dev = self._dev(L.edge_var, torch.int32)
            self._cost_out = torch.zeros(2, dtype=torch.float64, device=self.device)
            self._cost_unary_off = self._dev(L.unary_off, torch.int64)

    def _unary_dev(self, unary):
        """The variables' own costs `unary` (canonical order) on the device in internal order (class-major, padded
        bases), in the engine's precision; None for None."""
        if unary is None:
            return None
        L = self.layout
        un_host = np.zeros(max(int(L.unary_off[-1]), 1))
        cu = np.asarray(unary, dtype=np.float64).reshape(-1)
        dom = L.dom_size.astype(np.int64)
        c_off = np.concatenate([[0], np.cumsum(dom[L.var_perm])])[:-1]   # canonical offsets
        if len(cu):
            src = np.repeat(c_off[L.var_order], dom) + (np.arange(int(dom.sum())) - np.repeat(np.cumsum(dom) - dom, dom))
            dst = np.repeat(L.unary_off[:-1], dom) + (np.arange(int(dom.sum())) - np.repeat(np.cumsum(dom) - dom, dom))
            un_host[dst] = cu[src]
        return self._dev(un_host, PRECISIONS[self.precision][1])


class _CycleEngine(_EngineBase):
    """MaxSum and DSA: a cycle is computed into the other message / value buffer, then committed;
    fg_<family>_current reports (current buffer, cycle)."""

    def cycle_compute(self):
        with torch.cuda.device(self.device):
            self._check(self._fn("cycle_compute")(self._h, self._stream()), f"fg_{self.FAMILY}_cycle_compute")

    def cycle_commit(self):
        with torch.cuda.device(self.device):
            self._check(self._fn("cycle_commit")(self._h), f"fg_{self.FAMILY}_cycle_commit")

    def _current(self):
        b, c = C.c_int32(), C.c_int64()
        with torch.cuda.device(self.device):
            self._fn("current")(self._h, C.byref(b), C.byref(c))
        return b.value, c.value

    @property
    def cur(self):
        return self._current()[0]

    @property
    def cycle(self):
        return self._current()[1]


class MaxSumEngine(_CycleEngine):
    """All-edges-at-once synchronous MaxSum.

    Parameters mirror the reference's algo_params (pydcop/algorithms/maxsum.py:212-220); `noise`
    is applied by the caller to the instance's `unary` before packing (pydcop_b200.ingest.add_noise).
    State after `init()` is the reference's cycle 0 (on_start); each `step()` cycle is one
    synchronous round of every factor's and every variable's on_new_cycle.
    """
    FAMILY = "maxsum"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min",
                 damping=0.5, damping_nodes="both", stability=0.1, start_messages="leafs",
                 record_sent=True):
        L = layout
        tdt = self._open(layout, device, precision)
        if damping_nodes not in ("vars", "factors", "both", "none"):
            raise ValueError(f"invalid damping_nodes {damping_nodes!r}")
        if start_messages not in _cabi.START_MESSAGES:
            raise ValueError(f"invalid start_messages {start_messages!r}")
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        with torch.cuda.device(self.device):
            self.tables = self._dev_tables(L, tdt)
            self.unary = self._dev(L.unary, tdt)
            self.dom_size = self._dev(L.dom_size, torch.int32)
            self.unary_off = self._dev(L.unary_off, torch.int64)
            self.var_ptr = self._dev(L.var_ptr, torch.int32)
            self.var_qbase = self._dev(L.var_qbase, torch.int64)
            self.slot_roff = self._dev(L.slot_roff, torch.int64)
            self.edge_qoff = self._dev(L.edge_qoff, torch.int64)
            fits32 = max(L.n_msg, L.n_msg_q) < 2 ** 32
            # uint32 offsets, stored as int32 bit patterns (torch has no uint32 arithmetic)
            self.slot_roff32 = self._dev(L.slot_roff.astype(np.uint32).view(np.int32), torch.int32) if fits32 else None
            self.edge_qoff32 = self._dev(L.edge_qoff.astype(np.uint32).view(np.int32), torch.int32) if fits32 else None
            self.slot_edge = self._dev(L.slot_edge, torch.int32)
            self.slot_var = self._dev(L.slot_var, torch.int32)
            self.init_value = self._dev(L.init_value, torch.int32)
            z = lambda n, dt: torch.zeros(max(int(n), 1), dtype=dt, device=self.device)  # noqa
            self.q = [z(L.n_msg_q, tdt), z(L.n_msg_q, tdt)]
            self.r = [z(L.n_msg, tdt), z(L.n_msg, tdt)]
            self.q_valid, self.r_valid = z(L.n_edges, torch.uint8), z(L.n_edges, torch.uint8)
            self.q_cnt, self.r_cnt = z(L.n_edges, torch.uint8), z(L.n_edges, torch.uint8)
            self.q_sent = z(L.n_edges, torch.uint8) if record_sent else None
            self.r_sent = z(L.n_edges, torch.uint8) if record_sent else None
            self.value = z(L.n_vars, torch.int32)
            self.value_cost = z(L.n_vars, tdt)
        self._classes = _class_array(L)
        d = fill_header(FgMaxSumDesc(), precision, L, self._classes)
        d.n_msg_r, d.n_msg_q = L.n_msg, L.n_msg_q
        d.uniform_dom, d.max_degree = L.uniform_dom, L.max_degree
        self._varclasses = _varclass_array(L)
        d.n_varclasses = len(L.var_classes)
        d.varclasses = C.cast(self._varclasses, C.POINTER(FgVarClass))
        fill_desc(d, {k: getattr(self, k) for k in (
            "tables", "unary", "dom_size", "unary_off", "var_ptr", "var_qbase", "slot_roff", "edge_qoff", "slot_roff32",
            "edge_qoff32", "slot_edge", "slot_var", "init_value", "q", "r", "q_valid", "r_valid", "q_cnt", "r_cnt",
            "q_sent", "r_sent", "value", "value_cost")})
        d.mode_max = int(mode == "max")
        d.damp_vars = int(damping_nodes in ("vars", "both"))
        d.damp_factors = int(damping_nodes in ("factors", "both"))
        d.start_messages = _cabi.START_MESSAGES[start_messages]
        d.damping, d.stability = float(damping), float(stability)
        self._create(d)

    KERNEL_FAMILIES = {-1: "ghost", 0: "generic", 1: "pipe", 2: "warp", 3: "tiled_rt"}

    def kernel_plan(self):
        """Kernel family of every factor class (fg_maxsum_kernel_plan), as a list of names."""
        n = len(self.layout.classes)
        out = (C.c_int32 * max(n, 1))()
        with torch.cuda.device(self.device):
            rc = self.lib.fg_maxsum_kernel_plan(self._h, out, n)
        if rc != 0:
            raise EngineError(f"fg_maxsum_kernel_plan rc={rc}")
        return [self.KERNEL_FAMILIES[int(out[i])] for i in range(n)]

    def table_widths(self):
        """Bytes per stored table entry the factor side reads for every factor class (fg_maxsum_table_width):
        1 where the warp kernel reads the engine's 8-bit copy of integer tables, else 4 (f32) or 8 (f64)."""
        n = len(self.layout.classes)
        out = (C.c_int32 * max(n, 1))()
        with torch.cuda.device(self.device):
            rc = self.lib.fg_maxsum_table_width(self._h, out, n)
        if rc != 0:
            raise EngineError(f"fg_maxsum_table_width rc={rc}")
        return [int(out[i]) for i in range(n)]

    # -- readback (canonical edge order) -----------------------------------------------------
    def messages(self):
        """(q, r) receiver-side message state as float64 numpy arrays in canonical edge order."""
        g = torch.from_numpy(self.layout.message_gather_index()).to(self.device)
        gq = torch.from_numpy(self.layout.message_gather_index_q()).to(self.device)
        cur = self.cur
        q = self.q[cur][gq].double().cpu().numpy() if g.numel() else np.zeros(0)
        r = self.r[cur][g].double().cpu().numpy() if g.numel() else np.zeros(0)
        return q, r

    def flags(self):
        """dict of canonical-edge-order numpy arrays: q_valid, r_valid, q_sent, r_sent, q_cnt, r_cnt."""
        L = self.layout
        out = {"q_valid": L.edges_to_canonical(self.q_valid.cpu().numpy()[:L.n_edges]),
               "r_valid": L.edges_to_canonical(self.r_valid.cpu().numpy()[:L.n_edges]),
               "r_cnt": L.edges_to_canonical(self.r_cnt.cpu().numpy()[:L.n_edges]),
               "q_cnt": L.slots_to_canonical_edges(self.q_cnt.cpu().numpy()[:L.n_edges])}
        if self.q_sent is not None:
            out["q_sent"] = L.slots_to_canonical_edges(self.q_sent.cpu().numpy()[:L.n_edges])
            out["r_sent"] = L.edges_to_canonical(self.r_sent.cpu().numpy()[:L.n_edges])
        return out

    def _assignment(self):
        return self.value

    def values(self):
        """(value index, reported cost) per variable, in the caller's canonical variable order."""
        L = self.layout
        n = L.n_vars
        return (L.vars_to_canonical(self.value[:n].cpu().numpy()),
                L.vars_to_canonical(self.value_cost[:n].double().cpu().numpy()))


def dsa_row_stride(d: int, elem: int) -> int:
    """Elements between two rows of an oriented table: the next power of two >= d, whole 128-byte lines above 128
    bytes (csrc/row_load.cuh::fg_row_stride, the same rule): the one row a slot reads per cycle then costs one or two
    whole DRAM lines."""
    p2 = 1
    while p2 < d:
        p2 *= 2
    line = 128 // elem
    return -(-d // line) * line if p2 * elem > 128 else p2


def dsa_fast_arrays(layout: FactorGraphLayout, tables: torch.Tensor, mode="min"):
    """Arrays of the DSA fast path, or None when the instance does not qualify (every constraint
    binary over ONE domain size).  Per slot (variable v, incident constraint c, neighbour u) the
    table of c is read ORIENTED so that row y = value of u is contiguous over v's values: slots at
    scope position 1 read the table as stored, slots at position 0 read a transposed copy; rows are
    stored with stride dsa_row_stride (each row on its own cache-line slot).
    Returns (tables_or, slot_tab, slot_nbr, slot_opt, D) as tensors on `tables.device`."""
    L = layout
    if not (len(L.classes) == 1 and L.classes[0].arity == 2 and L.classes[0].dom[0] == L.classes[0].dom[1]
            and L.n_edges and not L.classes[0].tag):
        return None
    dev = tables.device
    c0 = L.classes[0]
    D = c0.dom[0]
    S = D * D
    nF = c0.n_factors
    t = tables[c0.table_base:c0.table_base + nF * S].view(nF, D, D)
    RS = dsa_row_stride(D, t.element_size())
    SP = D * RS                                     # elements per padded table
    tables_or = torch.zeros(2 * nF * SP, dtype=t.dtype, device=dev)
    tv = tables_or.view(2, nF, D, RS)
    tv[0, :, :, :D] = t
    tv[1, :, :, :D] = t.transpose(1, 2)
    opt = (t.reshape(nF, S).max(dim=1).values if mode == "max" else t.reshape(nF, S).min(dim=1).values)
    e = L.slot_edge.astype(np.int64) - c0.first_edge
    f, j = e // 2, e % 2
    # position 1 (me second): T[y][x] is already row-contiguous; position 0: transposed copy
    slot_tab = np.where(j == 1, f * SP, nF * SP + f * SP).astype(np.int64)
    slot_nbr = L.edge_var[c0.first_edge + f * 2 + (1 - j)].astype(np.int32)
    return (tables_or, torch.from_numpy(np.ascontiguousarray(slot_tab)).to(dev),
            torch.from_numpy(np.ascontiguousarray(slot_nbr)).to(dev),
            opt[torch.from_numpy(f).to(dev)].contiguous(), D)


def dsa_plan(layout: FactorGraphLayout, precision="f32", mode="min", probability=0.7, p_mode="fixed", variant="B",
             stop_cycle=0, seed=0, isolated_value=None, var_global_id=None, frozen=None, var_costs=False,
             var_seed=None, var_pset=None, psets=None):
    """DsaEngine's host-array plan for the generic kernels (inputs, state, scalar descriptor fields), as mgm_plan;
    `value` is the double buffer, its second half uploaded as zeros.  The oriented-table and active-row arrays are
    DsaEngine's own.  frozen (canonical order): ghost variables of a shard, has_nbr = 2 (never written by the local
    kernels); var_costs: A-DSA's var_cost / unary_off.  var_pset (canonical order) / psets (checked parameter dicts):
    the parameter set of every variable of a union; `prob` then holds each variable's own set's probability and
    p_mode, and the kernels read its variant."""
    L = layout
    pset = _pset_index(L, var_pset, psets)
    dt = PRECISIONS[precision][2]
    if variant not in _cabi.DSA_VARIANTS:
        raise ValueError(f"invalid variant {variant!r}")
    if p_mode not in ("fixed", "arity"):
        raise ValueError(f"invalid p_mode {p_mode!r}")
    arity = np.array([c.arity for c in L.classes], dtype=np.int64)
    n_count = np.zeros(L.n_vars, dtype=np.int64)
    if L.n_edges:
        np.add.at(n_count, L.slot_var, arity[L.edge_class[L.slot_edge]] - 1)
    has_nbr = (n_count > 0).astype(np.uint8)
    if frozen is not None:   # 2 = ghost of another rank's variable: never written by the local kernels
        has_nbr[np.asarray(frozen, dtype=bool)[L.var_order]] = 2
    with np.errstate(divide="ignore"):   # p_mode arity, dsa.py:257-260: 1 / n_count * 1.2
        by_count = np.where(n_count > 0, 1.0 / np.maximum(n_count, 1) * 1.2, 0.0)
    if pset is not None:   # each variable's own set's p_mode and probability
        by_arity = np.array([p.get("p_mode", "fixed") == "arity" for p in psets])[pset[:L.n_vars]]
        prob = np.where(by_arity, by_count, np.array([float(p["probability"]) for p in psets])[pset[:L.n_vars]])
    elif p_mode == "arity":
        prob = by_count
    else:
        prob = np.full(L.n_vars, float(probability))
    # isolated variables (dsa.py:278-289): argopt of (own cost, value), tuple order
    if isolated_value is not None:   # given in canonical order
        isolated_value = np.asarray(isolated_value, dtype=np.int32)[L.var_order]
    else:
        isolated_value = np.zeros(L.n_vars, dtype=np.int32)
        for v in np.nonzero(n_count == 0)[0]:  # (frozen ghosts are filled by the exchange)
            c = L.unary[L.unary_off[v]:L.unary_off[v] + L.dom_size[v]]
            if mode == "min":
                isolated_value[v] = int(np.argmin(c))
            else:
                isolated_value[v] = int(len(c) - 1 - np.argmax(c[::-1]))
    i32 = lambda a: np.ascontiguousarray(a, np.int32)  # noqa: E731
    inputs = dict(tables=np.ascontiguousarray(L.tables, dt), dom_size=i32(L.dom_size), var_id=i32(L.var_order),
                  edge_var=i32(L.edge_var), edge_class=i32(L.edge_class), var_ptr=i32(L.var_ptr),
                  slot_edge=i32(L.slot_edge), has_nbr=has_nbr, prob=np.ascontiguousarray(prob, np.float64),
                  value=[_per_var(L, isolated_value, np.int32), np.zeros(max(L.n_vars, 1), np.int32)],
                  var_cost=np.ascontiguousarray(L.unary, dt) if var_costs else None,
                  unary_off=np.ascontiguousarray(L.unary_off, np.int64) if var_costs else None)
    _set_global_ids(inputs, L, var_global_id, var_seed)
    state = dict(con_opt=(L.n_factors, dt, 0), value_cost=(L.n_vars, dt, 0))
    scalars = dict(mode_max=int(mode == "max"), variant=_cabi.DSA_VARIANTS[variant], stop_cycle=int(stop_cycle),
                   seed=_seed(seed))
    _set_psets(inputs, scalars, pset, psets, _cabi.FgDsaPset, lambda p: dict(variant=_cabi.DSA_VARIANTS[p["variant"]]))
    return inputs, state, scalars


class DsaEngine(_CycleEngine):
    """All-variables-at-once DSA-A/B/C (pydcop/algorithms/dsa.py:130-135 parameters)."""
    FAMILY = "dsa"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min",
                 probability=0.7, p_mode="fixed", variant="B", stop_cycle=0, seed=0,
                 isolated_value=None, var_global_id=None, frozen=None, var_costs=False, var_seed=None,
                 var_pset=None, psets=None):
        """var_costs: A-DSA's decision (pydcop/algorithms/adsa.py:344-377: every candidate value carries the
        variable's own cost, the current cost does not); False: DSA.
        var_global_id / frozen (canonical order) serve the multi-GPU partition
        (pydcop_b200/multigpu_dsa.py): the Philox counter of each variable when the layout is a
        shard of a larger problem, and the ghost variables whose value is only copied through.
        var_seed (canonical order): the Philox key of each variable when the layout holds several problems with
        seeds of their own (pydcop_b200.batch); default: `seed` for every variable.
        var_pset / psets: the parameter set of each variable (canonical order) when the layout holds several problems
        with parameters of their own, as dsa_plan; default: the scalar parameters for every variable."""
        L = layout
        tdt = self._open(layout, device, precision)
        inputs, state, scalars = dsa_plan(L, precision, mode, probability, p_mode, variant, stop_cycle, seed,
                                          isolated_value, var_global_id, frozen, var_costs, var_seed, var_pset, psets)
        self.has_nbr_host = inputs["has_nbr"]
        value0, _ = inputs.pop("value")
        t = self._upload(inputs, state)
        with torch.cuda.device(self.device):   # the second buffer starts as zeros on the device, nothing to copy
            t["value"] = [self._dev(value0, torch.int32), torch.zeros(len(value0), dtype=torch.int32, device=self.device)]
        self.__dict__.update(t)
        # fast path: every constraint binary over ONE domain size -> oriented tables, one contiguous
        # row per incidence (transposed copy for scope position 0)
        self.tables_or = self.slot_nbr = self.slot_tab = self.slot_opt = None
        fast_dom = 0
        with torch.cuda.device(self.device):
            fast = dsa_fast_arrays(L, self.tables, mode)
        self.row_cache = self.slot_last = None
        if fast is not None:
            self.tables_or, self.slot_tab, self.slot_nbr, self.slot_opt, fast_dom = fast
            with torch.cuda.device(self.device):   # active-row array (csrc/dsa_cached.cuh): L.n_edges rows of fast_dom costs
                self.row_cache = torch.zeros(max(L.n_edges * fast_dom, 4), dtype=tdt, device=self.device)
                self.slot_last = torch.full((max(L.n_edges, 1),), 255, dtype=torch.uint8, device=self.device)
        self._classes = _class_array(L)
        d = fill_desc(fill_header(FgDsaDesc(), precision, L, self._classes), t, scalars)
        fill_desc(d, {k: getattr(self, k) for k in ("tables_or", "slot_nbr", "slot_tab", "slot_opt", "row_cache",
                                                    "slot_last")})
        d.fast_dom = fast_dom
        self._create(d)

    def _assignment(self):
        return self.value[self.cur]

    def values(self):
        """Current value index per variable, canonical variable order."""
        L = self.layout
        return L.vars_to_canonical(self.value[self.cur][:L.n_vars].cpu().numpy())


def distinct_neighbours(layout: FactorGraphLayout):
    """CSR (nbr_ptr, nbr_idx) of every variable's DISTINCT neighbours (the other variables of its
    constraints, mgm.py:245-252) in internal variable ids, each list in order of first appearance
    over the variable's constraints (node.constraints order, then scope order) — the order the
    oracle uses, so neighbour costs are added in the same sequence."""
    L = layout
    V, E = L.n_vars, L.n_edges
    if not E:
        return np.zeros(V + 1, dtype=np.int32), np.zeros(1, dtype=np.int32)
    arity = np.array([c.arity for c in L.classes], dtype=np.int64)
    first_edge = np.array([c.first_edge for c in L.classes], dtype=np.int64)
    e = L.slot_edge.astype(np.int64)
    cl = L.edge_class[e].astype(np.int64)
    a = arity[cl]
    e0 = first_edge[cl] + ((e - first_edge[cl]) // a) * a
    A = int(arity.max())
    vs, seqs, us = [], [], []
    slot = np.arange(E, dtype=np.int64)
    for j in range(A):
        m = a > j
        u = L.edge_var[(e0 + j)[m]].astype(np.int64)
        v = L.slot_var[m].astype(np.int64)
        keep = u != v
        vs.append(v[keep])
        us.append(u[keep])
        seqs.append((slot[m] * A + j)[keep])
    v, u, seq = np.concatenate(vs), np.concatenate(us), np.concatenate(seqs)
    o = np.lexsort((seq, u, v))            # by (v, u), earliest occurrence first
    v, u, seq = v[o], u[o], seq[o]
    first = np.ones(len(v), dtype=bool)
    first[1:] = (v[1:] != v[:-1]) | (u[1:] != u[:-1])
    v, u, seq = v[first], u[first], seq[first]
    o = np.lexsort((seq, v))               # back to first-appearance order inside each variable
    v, u = v[o], u[o]
    ptr = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(v, minlength=V), out=ptr[1:])
    return ptr, (u.astype(np.int32) if len(u) else np.zeros(1, dtype=np.int32))


def mgm_host_arrays(layout: FactorGraphLayout, mode="min", var_rank=None, isolated_value=None):
    """Everything MgmEngine derives on the host, in the layout's INTERNAL variable order: the
    neighbour CSR, name ranks, and the preset value / cost of the variables without neighbours
    (mgm.py:285-294: optimal_cost_value, then finished)."""
    L = layout
    nbr_ptr, nbr_idx = distinct_neighbours(L)
    has_nbr = np.diff(nbr_ptr) > 0
    rank = (np.arange(L.n_vars, dtype=np.int32) if var_rank is None
            else np.asarray(var_rank, dtype=np.int32))[L.var_order]
    value0 = np.zeros(L.n_vars, dtype=np.int32)
    cost0 = np.zeros(L.n_vars, dtype=np.float64)
    iso = np.nonzero(~has_nbr)[0]
    if isolated_value is not None:
        value0[iso] = np.asarray(isolated_value, dtype=np.int32)[L.var_order][iso]
    for v in iso:
        c = L.unary[L.unary_off[v]:L.unary_off[v] + L.dom_size[v]]
        if isolated_value is None:
            value0[v] = int(np.argmin(c)) if mode == "min" else int(len(c) - 1 - np.argmax(c[::-1]))
        cost0[v] = c[value0[v]]
    return dict(nbr_ptr=nbr_ptr, nbr_idx=nbr_idx, has_nbr=has_nbr, var_rank=rank.astype(np.int32),
                value0=value0, cost0=cost0)


def _per_var(layout, a, dtype):
    """A per-variable input: `a` in `dtype`, or one zero without variables."""
    return np.ascontiguousarray(a, dtype) if layout.n_vars else np.zeros(1, dtype)


def _neighbourhood_inputs(layout, dt, h):
    """The constraint tables and the neighbourhood arrays MGM, MGM-2 and GDBA all upload (h: mgm_host_arrays)."""
    L = layout
    i32 = lambda a: np.ascontiguousarray(a, np.int32)  # noqa: E731
    return dict(tables=np.ascontiguousarray(L.tables, dt), dom_size=i32(L.dom_size), var_id=i32(L.var_order),
                var_rank=i32(h["var_rank"]), edge_var=i32(L.edge_var), edge_class=i32(L.edge_class),
                var_ptr=i32(L.var_ptr), slot_edge=i32(L.slot_edge), nbr_ptr=i32(h["nbr_ptr"]),
                nbr_idx=i32(h["nbr_idx"]), init_value=i32(L.init_value))


def _seed(seed):
    return int(seed) & (2 ** 64 - 1)


def _var_seeds(layout, var_seed):
    """var_seed (canonical order, any ints) as uint64 in internal order, each masked as _seed masks the scalar seed."""
    keys = (np.asarray(var_seed, dtype=object) & (2 ** 64 - 1)).astype(np.uint64)
    return _per_var(layout, keys[layout.var_order], np.uint64)


def _set_global_ids(inputs, layout, var_global_id, var_seed=None):
    """Replace the uploaded var_id (the canonical index) by var_global_id (canonical order), the Philox counter of
    every variable when the layout is part of a larger problem (a shard) or one problem of a union (a batch).  Add
    var_seed (canonical order), the Philox key of every variable when the problems of a union have seeds of their
    own; without it the descriptor's dev_var_seed stays NULL and every draw is keyed by the scalar seed."""
    if var_global_id is not None:
        inputs["var_id"] = _per_var(layout, np.asarray(var_global_id, dtype=np.int32)[layout.var_order], np.int32)
    if var_seed is not None:
        inputs["var_seed"] = _var_seeds(layout, var_seed)
    return inputs


def _pset_index(layout, var_pset, psets):
    """var_pset (canonical order): the parameter set of every variable, an index into `psets` (a list of checked
    parameter dicts), as uint16 in internal order; None when neither is given."""
    if var_pset is None and psets is None:
        return None
    if var_pset is None or psets is None or not 1 <= len(psets) <= _cabi.FG_MAX_PSETS:
        raise ValueError(f"var_pset and psets go together, with 1 to {_cabi.FG_MAX_PSETS} parameter sets")
    vp = np.asarray(var_pset, dtype=np.int64)
    if vp.shape != (layout.n_vars,) or (vp < 0).any() or (vp >= len(psets)).any():
        raise ValueError(f"var_pset must hold one index into the {len(psets)} parameter sets per variable")
    return _per_var(layout, vp[layout.var_order], np.uint16)


def _set_psets(inputs, scalars, index, psets, struct, fields):
    """Add a union's parameter sets to a plan: `index` (_pset_index) as dev_var_pset, and the host table of `struct`
    (fields(params) -> its field values) as psets / n_psets.  Nothing without an index: the plan is the plan of the
    scalar parameters."""
    if index is None:
        return inputs, scalars
    inputs["var_pset"] = index
    table = (struct * len(psets))(*[struct(**fields(p)) for p in psets])
    scalars.update(psets=table, n_psets=len(psets))   # a descriptor holding the table keeps it alive (ctypes)
    return inputs, scalars


def mgm_plan(layout: FactorGraphLayout, precision="f32", mode="min", stop_cycle=0, seed=0, var_rank=None,
             isolated_value=None, var_global_id=None, var_seed=None):
    """MgmEngine's host-array plan: (inputs: name -> array in its final dtype, in upload order; state: name ->
    (length, dtype, fill); the descriptor's scalar fields).  Every name is a dev_<name> field of fg_mgm_desc_t.
    var_global_id (canonical order): the Philox counter of every variable (default: the canonical index); var_seed
    (canonical order): the Philox key of every variable (default: `seed` for all)."""
    L = layout
    dt = PRECISIONS[precision][2]
    h = mgm_host_arrays(L, mode, var_rank, isolated_value)
    nb = _neighbourhood_inputs(L, dt, h)
    inputs = dict(tables=nb.pop("tables"), unary=np.ascontiguousarray(L.unary, dt),
                  unary_off=np.ascontiguousarray(L.unary_off, np.int64), **nb,
                  value=_per_var(L, h["value0"], np.int32), cost=_per_var(L, h["cost0"], dt),
                  has_cost=_per_var(L, ~h["has_nbr"], np.uint8))
    _set_global_ids(inputs, L, var_global_id, var_seed)
    state = dict(gain=(L.n_vars, dt, 0), new_value=(L.n_vars, np.int32, 0))
    return inputs, state, dict(mode_max=int(mode == "max"), stop_cycle=int(stop_cycle), seed=_seed(seed))


class _LocalSearchEngine(_EngineBase):
    """MGM, MGM-2 and GDBA: fg_<family>_current reports (round, finished); each variable's cost is known once
    has_cost is set."""

    def _current(self):
        c, f = C.c_int64(), C.c_int32()
        with torch.cuda.device(self.device):
            self._fn("current")(self._h, C.byref(c), C.byref(f))
        return c.value, bool(f.value)

    @property
    def cycle(self):
        return self._current()[0]

    @property
    def finished(self):
        return self._current()[1]

    def values(self):
        """(value index, current cost or NaN while the reference's is None) per variable,
        canonical variable order."""
        L = self.layout
        n = L.n_vars
        cost = self.cost[:n].double().cpu().numpy()
        cost[self.has_cost[:n].cpu().numpy() == 0] = np.nan
        return L.vars_to_canonical(self._assignment()[:n].cpu().numpy()), L.vars_to_canonical(cost)


class MgmEngine(_LocalSearchEngine):
    """All-variables-at-once MGM (pydcop/algorithms/mgm.py; parameters :78-81).

    var_rank       canonical order: position of each variable's NAME in sorted order, the
                   lexicographic tie break of mgm.py:574-583 (default: the canonical index)
    isolated_value canonical order: value index of the variables without neighbours
                   (optimal_cost_value over the real domain values, relations.py:1641-1669);
                   default: argopt of the own cost with ties broken on the value index
    var_global_id  canonical order: the Philox counter of each variable when the layout holds several problems
                   (pydcop_b200.batch; default: the canonical index)
    var_seed       canonical order: the Philox key of each variable when those problems have seeds of their own
                   (default: `seed` for every variable)
    `break_mode` is accepted for the reference's signature; its 'random' branch is dead code in
    the reference (mgm.py:541 compares with the `random` module) and both settings act as 'lexic'.
    """
    FAMILY = "mgm"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min",
                 stop_cycle=0, seed=0, break_mode="lexic", var_rank=None, isolated_value=None, var_global_id=None,
                 var_seed=None):
        L = layout
        tdt = self._open(layout, device, precision)
        if break_mode not in ("lexic", "random"):
            raise ValueError(f"invalid break_mode {break_mode!r}")
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        inputs, state, scalars = mgm_plan(L, precision, mode, stop_cycle, seed, var_rank, isolated_value,
                                          var_global_id, var_seed)
        self.has_nbr_host = np.diff(inputs["nbr_ptr"]) > 0
        t = self._upload(inputs, state)
        self.__dict__.update(t)
        self._classes = _class_array(L)
        d = fill_desc(fill_header(FgMgmDesc(), precision, L, self._classes), t, scalars)
        # the fast value-phase kernel on the DSA fast-path arrays (binary constraints over one domain size
        # in {4, 8, 10, 16, 20}), 2 incidences per trip by default.  PYDCOP_B200_MGM_FAST=0|2|4
        self.fast_chunk = 0
        chunk = int(os.environ.get("PYDCOP_B200_MGM_FAST", "2") or 0)
        if chunk in (2, 4):
            with torch.cuda.device(self.device):
                fast = dsa_fast_arrays(L, self.tables, mode)
            if fast is not None and fast[4] in (4, 8, 10, 16, 20):
                self.tables_or, self.slot_tab, self.slot_nbr, _, fast_dom = fast
                d.fast_dom, d.fast_chunk = fast_dom, chunk
                self.fast_chunk = chunk
                self.row_cache = self.slot_last = None
                if os.environ.get("PYDCOP_B200_MGM_CACHE", "1") != "0":   # active-row array (csrc/mgm_cached_kernels.cuh)
                    with torch.cuda.device(self.device):
                        self.row_cache = torch.zeros(max(L.n_edges * fast_dom, 4), dtype=tdt, device=self.device)
                        self.slot_last = torch.full((max(L.n_edges, 1),), 255, dtype=torch.uint8, device=self.device)
                fill_desc(d, {k: getattr(self, k) for k in ("tables_or", "slot_nbr", "slot_tab", "row_cache",
                                                            "slot_last")})
        self._create(d)

    def _assignment(self):
        return self.value

    def gains(self):
        """(gain, intended value) of the last round per variable, canonical order."""
        L = self.layout
        n = L.n_vars
        return (L.vars_to_canonical(self.gain[:n].double().cpu().numpy()),
                L.vars_to_canonical(self.new_value[:n].cpu().numpy()))


def mgm2_offer_offsets(layout: FactorGraphLayout, nbr_ptr, nbr_idx):
    """Start of every variable's MGM-2 offer table (internal order) and the total size: an offerer
    writes dom(v) x dom(partner) gains, so v gets dom(v) x max dom of its neighbours entries (none
    without neighbours)."""
    L = layout
    dom = L.dom_size.astype(np.int64)
    deg = np.diff(nbr_ptr).astype(np.int64)
    widest = np.zeros(L.n_vars, dtype=np.int64)
    if len(nbr_idx) and int(nbr_ptr[-1]):
        owner = np.repeat(np.arange(L.n_vars), deg)
        np.maximum.at(widest, owner, dom[nbr_idx[:int(nbr_ptr[-1])]])
    size = dom * widest
    off = np.zeros(L.n_vars + 1, dtype=np.int64)
    np.cumsum(size, out=off[1:])
    return off[:-1].copy(), int(off[-1])


def mgm2_plan(layout: FactorGraphLayout, precision="f32", mode="min", threshold=0.5, favor="unilateral",
              stop_cycle=0, seed=0, var_rank=None, var_global_id=None, var_seed=None, var_pset=None, psets=None):
    """Mgm2Engine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan.  var_global_id (canonical
    order): the Philox counter of every variable when the layout is a shard of a larger problem; var_seed as
    mgm_plan; var_pset / psets as dsa_plan (the kernels read each variable's threshold and favor)."""
    L = layout
    pset = _pset_index(L, var_pset, psets)
    dt = PRECISIONS[precision][2]
    h = mgm_host_arrays(L, mode, var_rank)
    offer_off, offer_size = mgm2_offer_offsets(L, h["nbr_ptr"], h["nbr_idx"])
    inputs = _set_global_ids(dict(**_neighbourhood_inputs(L, dt, h), offer_off=_per_var(L, offer_off, np.int64)),
                             L, var_global_id, var_seed)
    n = L.n_vars
    state = dict(value=(n, np.int32, 0), potential_value=(n, np.int32, 0), answer_value=(n, np.int32, 0),
                 partner=(n, np.int32, -1), cost=(n, dt, 0), gain=(n, dt, 0), local_cost=(n, dt, 0),
                 answer_gain=(n, dt, 0), has_cost=(n, np.uint8, 0), offerer=(n, np.uint8, 0),
                 committed=(n, np.uint8, 0), go=(n, np.uint8, 0), answer=(n, np.uint8, 0),
                 offer=(offer_size, dt, 0))
    scalars = dict(mode_max=int(mode == "max"), favor=_cabi.MGM2_FAVORS[favor], threshold=float(threshold),
                   stop_cycle=int(stop_cycle or 0), seed=_seed(seed))
    _set_psets(inputs, scalars, pset, psets, _cabi.FgMgm2Pset,
               lambda p: dict(threshold=float(p["threshold"]), favor=_cabi.MGM2_FAVORS[p["favor"]]))
    return inputs, state, scalars


class Mgm2Engine(_LocalSearchEngine):
    """All-variables-at-once MGM-2 (pydcop/algorithms/mgm2.py; parameters :139-143).

    threshold  a variable offers a coordinated move when its draw u < threshold
    favor      unilateral | no | coordinated: what a receiver does when its best offer's global gain
               EQUALS its best unilateral gain (mgm2.py:818-822)
    var_rank   canonical order: position of each variable's NAME in sorted order, the lexicographic
               tie break of mgm2.py:944-949 (default: the canonical index)
    var_global_id  canonical order: the Philox counter of each variable when the layout is one rank's shard
               of a larger problem (pydcop_b200/multigpu_mgm2.py; default: the canonical index)
    var_seed   canonical order: the Philox key of each variable, as MgmEngine (default: `seed` for every variable)
    var_pset, psets  the parameter set of each variable (canonical order) and the sets, as DsaEngine
    Variable costs are not part of MGM-2's costs (assignment_cost without them); a variable without
    neighbours takes a drawn value among its best over its unary constraints on the device.
    """
    FAMILY = "mgm2"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min",
                 threshold=0.5, favor="unilateral", stop_cycle=0, seed=0, var_rank=None, var_global_id=None,
                 var_seed=None, var_pset=None, psets=None):
        L = layout
        self._open(layout, device, precision)
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        if favor not in _cabi.MGM2_FAVORS:
            raise ValueError(f"invalid favor {favor!r}: expected one of {sorted(_cabi.MGM2_FAVORS)}")
        inputs, state, scalars = mgm2_plan(L, precision, mode, threshold, favor, stop_cycle, seed, var_rank,
                                           var_global_id, var_seed, var_pset, psets)
        self.nbr_ptr_host, self.nbr_idx_host = inputs["nbr_ptr"], inputs["nbr_idx"]
        self.has_nbr_host = np.diff(self.nbr_ptr_host) > 0
        self.offer_bytes = state["offer"][0] * np.dtype(self.np_dtype).itemsize
        t = self._upload(inputs, state)
        self.__dict__.update(t)
        self._classes = _class_array(L)
        self._create(fill_desc(fill_header(_cabi.FgMgm2Desc(), precision, L, self._classes), t, scalars))

    def _assignment(self):
        return self.value

    def record(self):
        """State of the last cycle per variable, canonical order: local_cost and gain (NaN without
        neighbours), offerer, partner (position in the variable's neighbour list, or -1), committed,
        potential_value (-1 without neighbours), go."""
        L = self.layout
        n = L.n_vars
        conn = self.has_nbr_host[:n]
        host = lambda t: t[:n].cpu().numpy()  # noqa: E731
        partner = host(self.partner)
        pos = np.full(n, -1, dtype=np.int32)
        for v in np.nonzero(partner >= 0)[0]:
            row = self.nbr_idx_host[self.nbr_ptr_host[v]:self.nbr_ptr_host[v + 1]]
            pos[v] = int(np.nonzero(row == partner[v])[0][0])
        out = dict(local_cost=np.where(conn, host(self.local_cost).astype(np.float64), np.nan),
                   gain=np.where(conn, host(self.gain).astype(np.float64), np.nan),
                   offerer=host(self.offerer), partner=pos, committed=host(self.committed),
                   potential_value=np.where(conn, host(self.potential_value), -1).astype(np.int32),
                   go=host(self.go))
        return {k: L.vars_to_canonical(v) for k, v in out.items()}

    # -- one rank of a sharded problem (pydcop_b200/multigpu_mgm2.py; fg_mgm2_shard_*) --

    def shard_attach(self, arrays):
        """Upload a shard plan (multigpu_mgm2.Mgm2Shard.plan_arrays: host arrays, internal order) and allocate the
        exchange buffers send_buf[x] / recv_buf[x] in the run's precision."""
        tdt = PRECISIONS[self.precision][1]
        with torch.cuda.device(self.device):
            dev = {k: self._dev(a, _TORCH_DTYPES[np.asarray(a).dtype]) for k, a in arrays.items()
                   if not isinstance(a, list)}
            lists = [{k: self._dev(a, _TORCH_DTYPES[np.asarray(a).dtype]) for k, a in x.items()}
                     for x in arrays["x"]]
            self.send_buf = [torch.zeros(max(int(x["send_off"][-1]), 1), dtype=tdt, device=self.device)
                             for x in arrays["x"]]
            self.recv_buf = [torch.zeros(max(int(x["recv_off"][-1]), 1), dtype=tdt, device=self.device)
                             for x in arrays["x"]]
        plan = _cabi.FgMgm2ShardPlan()
        for i, x in enumerate(lists):
            p = plan.x[i]
            p.n_send, p.n_recv = len(arrays["x"][i]["send_var"]), len(arrays["x"][i]["recv_var"])
            p.dev_send_var, p.dev_recv_var = _ptr(x["send_var"]), _ptr(x["recv_var"])
            p.dev_send_off, p.dev_recv_off = _ptr(x["send_off"]), _ptr(x["recv_off"])
            p.dev_send_buf, p.dev_recv_buf = _ptr(self.send_buf[i]), _ptr(self.recv_buf[i])
        for k in ("ghost", "send_peer", "owner_rank", "owner_local"):
            setattr(plan, "dev_" + k, _ptr(dev[k]))
        self._shard_keep, self._shard_plan = (dev, lists), plan
        self._shard_call("attach", C.byref(plan), None)

    def shard_attach_peer(self, peer):
        """Add the NVLink transport (a filled _cabi.FgMgm2PeerPlan) to the attached shard plan."""
        self._shard_peer = peer
        self._shard_call("attach", C.byref(self._shard_plan), C.byref(peer))

    def _shard_call(self, name, *args, stream=False):
        with torch.cuda.device(self.device):
            a = list(args) + ([self._stream()] if stream else [])
            self._check(getattr(self.lib, f"fg_mgm2_shard_{name}")(self._h, *a), f"fg_mgm2_shard_{name}")

    def shard_init(self):
        self._shard_call("init", stream=True)

    def shard_phase(self, x):
        self._shard_call("phase", int(x), stream=True)

    def shard_unpack(self, x):
        self._shard_call("unpack", int(x), stream=True)

    def shard_step(self, n_cycles):
        self._shard_call("step", int(n_cycles), stream=True)


def gdba_host_arrays(layout: FactorGraphLayout, nbr_ptr, increase_mode="E", violation="NZ"):
    """GDBA's host-side arrays, internal order:
    mod_off   per slot, start of its modifier table (increase modes E / R / C; -1 where the slot's constraint
              does not span {variable} + all its neighbours, so the reference never reads what those modes
              write there), None with T (one count per slot)
    mod_size  int32 elements of the modifier array
    viol_ref  per internal factor, the min (NM) or max (MX) of its base table, None with NZ
    canon_slot  canonical slot (var_ptr / var_con order) of every internal slot, and canon_mod_off the
              start of every canonical slot's entries in the flattened `modifiers()` view."""
    L = layout
    E = L.n_edges
    arity = np.array([c.arity for c in L.classes], dtype=np.int64)
    tsize = np.array([c.table_size for c in L.classes], dtype=np.int64)
    cls = L.edge_class[L.slot_edge].astype(np.int64) if E else np.zeros(0, np.int64)
    deg = np.diff(nbr_ptr).astype(np.int64)
    slot_deg = np.repeat(deg, np.diff(L.var_ptr))
    slot_size = tsize[cls]
    if increase_mode == "T":
        mod_off, mod_size = None, E
    else:
        span = (slot_deg > 0) & (arity[cls] == slot_deg + 1)
        size = np.where(span, slot_size, 0)
        start = np.cumsum(size) - size
        mod_off = np.where(span, start, -1).astype(np.int64)
        mod_size = int(size.sum())
    viol_ref = None
    if violation != "NZ" and L.n_factors:
        viol_ref = np.zeros(L.n_factors, dtype=np.float64)
        for c in L.classes:
            t = L.tables[c.table_base:c.table_base + c.n_factors * c.table_size].reshape(c.n_factors, c.table_size)
            viol_ref[c.first_factor:c.first_factor + c.n_factors] = t.min(1) if violation == "NM" else t.max(1)
    pos = np.empty(E, dtype=np.int64)
    pos[L.canon_var_edge] = np.arange(E)
    canon_slot = pos[L.slot_canon_edge] if E else np.zeros(0, np.int64)
    canon_size = np.zeros(E, dtype=np.int64)
    canon_size[canon_slot] = slot_size
    canon_mod_off = np.concatenate([[0], np.cumsum(canon_size)]).astype(np.int64)
    return dict(mod_off=mod_off, mod_size=int(mod_size), viol_ref=viol_ref, canon_slot=canon_slot,
                canon_mod_off=canon_mod_off)


def gdba_modifiers_view(h, mods, base_mod, increase_mode):
    """Flattened modifiers as reads see them (canonical variable, slot and table entry order) from the
    int32 counts `mods` laid out by gdba_host_arrays `h`."""
    off = h["canon_mod_off"]
    out = np.full(int(off[-1]), base_mod, dtype=np.int32)
    for s, cs in enumerate(h["canon_slot"]):
        a, b = off[cs], off[cs + 1]
        if increase_mode == "T":
            out[a:b] += mods[s]
        elif h["mod_off"][s] >= 0:
            out[a:b] += mods[h["mod_off"][s]:h["mod_off"][s] + (b - a)]
    return out


def gdba_plan(layout: FactorGraphLayout, precision="f32", mode="min", modifier="A", violation="NZ", increase_mode="E",
              stop_cycle=0, seed=0, var_rank=None, isolated_value=None, var_global_id=None, var_seed=None,
              var_pset=None, psets=None):
    """GdbaEngine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan; `value` is the double
    buffer, and viol_ref / mod_off are None where the modes do not read them.  var_pset / psets as dsa_plan (the
    kernels read each variable's modifier and violation mode; a factor's viol_ref is its variables' set's)."""
    L = layout
    dt = PRECISIONS[precision][2]
    pset = _pset_index(L, var_pset, psets)
    h = mgm_host_arrays(L, mode, var_rank, isolated_value)
    g = gdba_host_arrays(L, h["nbr_ptr"], increase_mode, violation)
    if pset is not None:
        g["viol_ref"] = _gdba_viol_ref(L, pset, [p["violation"] for p in psets])
    nb = _neighbourhood_inputs(L, dt, h)
    value0 = _per_var(L, h["value0"], np.int32)
    inputs = dict(tables=nb.pop("tables"), unary=np.ascontiguousarray(L.unary, dt),
                  unary_off=np.ascontiguousarray(L.unary_off, np.int64),
                  viol_ref=None if g["viol_ref"] is None else np.ascontiguousarray(g["viol_ref"], dt), **nb,
                  value=[value0, value0.copy()], cost=_per_var(L, h["cost0"], dt), has_cost=_per_var(L, ~h["has_nbr"], np.uint8),
                  mod_off=None if g["mod_off"] is None else np.ascontiguousarray(g["mod_off"], np.int64))
    _set_global_ids(inputs, L, var_global_id, var_seed)
    n = L.n_vars
    state = dict(improve=(n, dt, 0), new_value=(n, np.int32, 0), breakout=(n, np.uint8, 0),
                 violated=(L.n_edges, np.uint8, 0), mod=(g["mod_size"], np.int32, 0))
    scalars = dict(mode_max=int(mode == "max"), modifier=_cabi.GDBA_MODIFIERS[modifier],
                   violation=_cabi.GDBA_VIOLATIONS[violation], increase_mode=_cabi.GDBA_INCREASE_MODES[increase_mode],
                   mod_size=g["mod_size"], stop_cycle=int(stop_cycle or 0), seed=_seed(seed))
    _set_psets(inputs, scalars, pset, psets, _cabi.FgGdbaPset,
               lambda p: dict(modifier=_cabi.GDBA_MODIFIERS[p["modifier"]],
                              violation=_cabi.GDBA_VIOLATIONS[p["violation"]]))
    return inputs, state, scalars


def _gdba_viol_ref(layout, pset, violations):
    """viol_ref of a union whose variables have parameter sets (pset: internal order, violations: each set's mode):
    per internal factor, the min (NM) or max (MX) of its base table by the set of its first variable (every variable of
    a factor is of one problem, so of one set); None when every set is NZ."""
    L = layout
    code = np.array([_cabi.GDBA_VIOLATIONS[v] for v in violations])
    if not L.n_factors or not code.any():
        return None
    out = np.zeros(L.n_factors, dtype=np.float64)
    for c in L.classes:
        t = L.tables[c.table_base:c.table_base + c.n_factors * c.table_size].reshape(c.n_factors, c.table_size)
        first = L.edge_var[c.first_edge + np.arange(c.n_factors, dtype=np.int64) * c.arity]
        mx = code[pset[first]] == _cabi.GDBA_VIOLATIONS["MX"]
        out[c.first_factor:c.first_factor + c.n_factors] = np.where(mx, t.max(1), t.min(1))
    return out


class GdbaEngine(_LocalSearchEngine):
    """All-variables-at-once GDBA (pydcop/algorithms/gdba.py; parameters :181-185).

    modifier       A (base + m, m from 0) | M (base * m, m from 1)
    violation      NZ (entry != 0) | NM (entry != table min) | MX (entry == table max), on the base table
    increase_mode  E | R | C | T: which modifiers a breakout raises (E / R / C only on a constraint that spans
                   the variable's neighbourhood, where the reference reads them; T every entry)
    stop_cycle     0 = run forever; else rounds stop when round + 1 >= stop_cycle (mgm_gpu's convention;
                   the reference has none)
    var_rank       canonical order: position of each variable's NAME in sorted order, the tie break of
                   gdba.py:657-658 (default: the canonical index)
    isolated_value canonical order: value index of the variables without neighbours (optimal_cost_value);
                   default: argopt of the own cost with ties broken on the value index
    var_global_id  canonical order: the Philox counter of each variable (default: the canonical index), as MgmEngine
    var_seed       canonical order: the Philox key of each variable (default: `seed` for every variable), as MgmEngine
    var_pset, psets  the parameter set of each variable (canonical order) and the sets, as DsaEngine; `modifiers()`
                   reads with the scalar modifier's base
    """
    FAMILY = "gdba"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min", modifier="A",
                 violation="NZ", increase_mode="E", stop_cycle=0, seed=0, var_rank=None, isolated_value=None,
                 var_global_id=None, var_seed=None, var_pset=None, psets=None):
        L = layout
        self._open(layout, device, precision)
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        for name, v, ok in (("modifier", modifier, _cabi.GDBA_MODIFIERS),
                            ("violation", violation, _cabi.GDBA_VIOLATIONS),
                            ("increase_mode", increase_mode, _cabi.GDBA_INCREASE_MODES)):
            if v not in ok:
                raise ValueError(f"invalid {name} {v!r}: expected one of {sorted(ok)}")
        self.modifier, self.violation, self.increase_mode = modifier, violation, increase_mode
        inputs, state, scalars = gdba_plan(L, precision, mode, modifier, violation, increase_mode, stop_cycle, seed,
                                           var_rank, isolated_value, var_global_id, var_seed, var_pset, psets)
        self.nbr_ptr_host = inputs["nbr_ptr"]
        self.has_nbr_host = np.diff(self.nbr_ptr_host) > 0
        self.modifier_bytes = scalars["mod_size"] * 4
        t = self._upload(inputs, state)
        self.__dict__.update(t)
        self._classes = _class_array(L)
        self._create(fill_desc(fill_header(_cabi.FgGdbaDesc(), precision, L, self._classes), t, scalars))

    @functools.cached_property
    def gh(self):
        """gdba_host_arrays of the layout: where each slot's modifiers are, for the canonical readback."""
        return gdba_host_arrays(self.layout, self.nbr_ptr_host, self.increase_mode, self.violation)

    def _assignment(self):
        return self.value[self.cycle % 2]

    def record(self):
        """State of the last round, canonical order: improve (NaN without neighbours), new_value (-1
        without neighbours), violated per canonical slot, breakout, modifiers (see `modifiers`)."""
        L = self.layout
        n = L.n_vars
        conn = self.has_nbr_host[:n]
        host = lambda t: t[:n].cpu().numpy()  # noqa: E731
        viol = np.zeros(L.n_edges, dtype=np.uint8)
        viol[self.gh["canon_slot"]] = self.violated[:L.n_edges].cpu().numpy()
        return dict(improve=L.vars_to_canonical(np.where(conn, host(self.improve).astype(np.float64), np.nan)),
                    new_value=L.vars_to_canonical(np.where(conn, host(self.new_value), -1).astype(np.int32)),
                    violated=viol, breakout=L.vars_to_canonical(host(self.breakout)), modifiers=self.modifiers())

    def modifiers(self):
        """Every modifier as a read sees it, flattened: canonical variable, its slots in node.constraints
        order, the constraint's table entries."""
        return gdba_modifiers_view(self.gh, self.mod.cpu().numpy(), 0 if self.modifier == "A" else 1,
                                   self.increase_mode)


DBA_MODE_ERROR = "DBA is a constraint **satisfaction** algorithm and only support minimization objective"
DBA_LIVE = 2 ** 31 - 1     # finish_phase of a variable that has not finished


def canonical_slot(layout: FactorGraphLayout):
    """Canonical slot (var_ptr / var_con order) of every internal slot."""
    L = layout
    pos = np.empty(L.n_edges, dtype=np.int64)
    pos[L.canon_var_edge] = np.arange(L.n_edges)
    return pos[L.slot_canon_edge] if L.n_edges else np.zeros(0, np.int64)


def dba_bit_offsets(layout: FactorGraphLayout):
    """First uint32 word of every internal slot's violation bit rows, and the total after the last: slot s of
    variable v owns table_size / dom(v) rows of ceil(dom(v) / 32) words (csrc/dba_kernels.cuh)."""
    L = layout
    if not L.n_edges:
        return np.zeros(1, dtype=np.int64)
    tsize = np.array([c.table_size for c in L.classes], dtype=np.int64)
    d = L.dom_size[L.slot_var].astype(np.int64)
    words = tsize[L.edge_class[L.slot_edge]] // d * ((d + 31) // 32)
    if int(words.max()) >= 2 ** 32:
        raise ValueError("a constraint with 2^32 or more bit-row words per variable")
    return np.concatenate([[0], np.cumsum(words)]).astype(np.int64)


def dba_plan(layout: FactorGraphLayout, precision="f32", infinity=10000, max_distance=50, stop_cycle=0, seed=0,
             var_rank=None):
    """DbaEngine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan; `value` is the double
    buffer and `bits` the violation bit rows fg_dba_init fills from `tables`."""
    L = layout
    dt = PRECISIONS[precision][2]
    h = mgm_host_arrays(L, "min", var_rank)
    nb = _neighbourhood_inputs(L, dt, h)
    nb.pop("init_value")                      # dba.py:341-349 ignores initial values
    bit_off = dba_bit_offsets(L)
    value0 = _per_var(L, np.zeros(L.n_vars), np.int32)
    inputs = dict(**nb, bit_off=bit_off, value=[value0, value0.copy()])
    n, E = L.n_vars, L.n_edges
    state = dict(bits=(int(bit_off[-1]), np.int32, None), cost=(n, np.int64, 0), has_cost=(n, np.uint8, 0),
                 eval=(n, np.int64, 0), improve=(n, np.int64, 0), counter=(n, np.int32, 0),
                 counter_own=(n, np.int32, 0), new_value=(n, np.int32, -1), can_move=(n, np.uint8, 0),
                 qlm=(n, np.uint8, 0), consistent=(n, np.uint8, 0), finish_phase=(n, np.int32, DBA_LIVE),
                 weight=(E, np.int32, 1), violated=(E, np.uint8, 0), status=(2, np.int32, 0),
                 unresolved=(1, np.int32, 0))
    return inputs, state, dict(n_words=int(bit_off[-1]), infinity=int(infinity), max_distance=int(max_distance),
                               stop_cycle=int(stop_cycle or 0), n_live=int(h["has_nbr"].sum()), seed=_seed(seed))


class DbaEngine(_LocalSearchEngine):
    """All-variables-at-once DBA (pydcop/algorithms/dba.py; parameters :265-268).

    infinity      a constraint is violated where its entry is >= infinity (compared in the tables' precision)
    max_distance  a variable stops when its termination counter reaches it (0: never)
    stop_cycle    0 = run until every variable with neighbours has finished; else rounds also stop when
                  round + 1 >= stop_cycle (gdba_gpu's convention)
    var_rank      canonical order: position of each variable's NAME in sorted order, the tie break of
                  dba.py:515 (default: the canonical index)
    `cycle` is the number of rounds that changed the state, `finished` is true once every variable with
    neighbours has finished (or at stop_cycle); `unresolved` counts the rounds in which a variable could improve
    but had no value below infinity, where the reference raises on random.choice([]): it keeps its value.
    """
    FAMILY = "dba"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min", infinity=10000,
                 max_distance=50, stop_cycle=0, seed=0, var_rank=None):
        if mode != "min":
            raise ValueError(DBA_MODE_ERROR)
        if int(max_distance) < 0:
            raise ValueError(f"invalid max_distance {max_distance!r}: must be >= 0")
        L = layout
        self._open(layout, device, precision)
        inputs, state, scalars = dba_plan(L, precision, infinity, max_distance, stop_cycle, seed, var_rank)
        self.has_nbr_host = np.diff(inputs["nbr_ptr"]) > 0
        self.bit_row_bytes = scalars["n_words"] * 4
        t = self._upload(inputs, state)
        self.__dict__.update({k: v for k, v in t.items() if k != "unresolved"})
        self.unresolved_dev = t["unresolved"]
        self._classes = _class_array(L)
        self._create(fill_desc(fill_header(_cabi.FgDbaDesc(), precision, L, self._classes), t, scalars))

    @functools.cached_property
    def _canon_slot(self):
        return canonical_slot(self.layout)

    def _assignment(self):
        return self.value[self.cycle % 2]

    @property
    def unresolved(self):
        return int(self.unresolved_dev.item())

    def finished_vars(self):
        """Per variable, canonical order: it has finished (stopped, or reached by the End flood)."""
        n = self.layout.n_vars
        return self.layout.vars_to_canonical(self.finish_phase[:n].cpu().numpy() != DBA_LIVE)

    def record(self):
        """State after the last round, canonical order: per variable eval, improve, new_value (-1 without a draw),
        can_move, qlm, consistent, counter (as posted with the improve message) and finish_phase (DBA_LIVE while
        live; phases: ok of round k = 2k, improve = 2k + 1); per canonical slot violated and weight; and the
        unresolved count and bit_row_bytes."""
        L = self.layout
        n, E = L.n_vars, L.n_edges
        var = lambda t: L.vars_to_canonical(t[:n].cpu().numpy())  # noqa: E731

        def slots(t):
            out = np.zeros(E, dtype=t.cpu().numpy().dtype)
            out[self._canon_slot] = t[:E].cpu().numpy()
            return out
        out = {k: var(self.__dict__[k]) for k in ("eval", "improve", "new_value", "can_move", "qlm", "consistent",
                                                  "counter", "finish_phase")}
        out.update(violated=slots(self.violated), weight=slots(self.weight), unresolved=self.unresolved,
                   bit_row_bytes=self.bit_row_bytes)
        return out


def mixeddsa_hard_factors(layout: FactorGraphLayout, tables):
    """Per internal factor: its table holds a +inf or -inf entry (mixeddsa.py:219), tested on `tables`, the layout's
    tables in the run's precision (an f64 entry above the f32 range is therefore hard in f32 only)."""
    L = layout
    hard = np.zeros(L.n_factors, dtype=bool)
    for c in L.classes:
        if c.n_factors:
            t = tables[c.table_base:c.table_base + c.n_factors * c.table_size].reshape(c.n_factors, c.table_size)
            hard[c.first_factor:c.first_factor + c.n_factors] = np.isinf(t).any(1)
    return hard


def mixeddsa_slots(layout: FactorGraphLayout, hard):
    """(slot_edge, soft_end): every variable's slots reordered to its soft constraints, then its hard ones, each in
    node.constraints order, and where its soft slots end (csrc/mixeddsa_kernels.cuh sums them in that order)."""
    L = layout
    V, E = L.n_vars, L.n_edges
    soft_end = np.asarray(L.var_ptr[:-1], dtype=np.int32).copy()
    if not E:
        return np.zeros(1, dtype=np.int32), soft_end
    arity = np.array([c.arity for c in L.classes], dtype=np.int64)
    first_edge = np.array([c.first_edge for c in L.classes], dtype=np.int64)
    first_factor = np.array([c.first_factor for c in L.classes], dtype=np.int64)
    e = L.slot_edge.astype(np.int64)
    cl = L.edge_class[e].astype(np.int64)
    slot_hard = hard[first_factor[cl] + (e - first_edge[cl]) // arity[cl]]
    order = np.lexsort((np.arange(E), slot_hard, L.slot_var))
    soft_end += np.bincount(L.slot_var[~slot_hard], minlength=V).astype(np.int32)
    return np.ascontiguousarray(L.slot_edge[order], np.int32), soft_end


def mixeddsa_plan(layout: FactorGraphLayout, precision="f32", mode="min", proba_hard=0.7, proba_soft=0.5, variant="B",
                  stop_cycle=0, seed=0, var_global_id=None, var_seed=None, var_pset=None, psets=None):
    """MixedDsaEngine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan; `value` is the double
    buffer, `slot_edge` the soft-then-hard slot order of mixeddsa_slots, `con_opt` written by fg_mixeddsa_init.
    var_pset / psets as dsa_plan (the kernels read each variable's probabilities and variant)."""
    L = layout
    pset = _pset_index(L, var_pset, psets)
    dt = PRECISIONS[precision][2]
    with np.errstate(over="ignore"):     # an f64 entry above the f32 range becomes inf: hard in f32 (mixeddsa.py:219)
        tables = np.ascontiguousarray(L.tables, dt)
    slot_edge, soft_end = mixeddsa_slots(L, mixeddsa_hard_factors(L, tables))
    nbr_ptr, nbr_idx = distinct_neighbours(L)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)  # noqa: E731
    value0 = _per_var(L, np.zeros(L.n_vars), np.int32)
    inputs = dict(tables=tables, unary=np.ascontiguousarray(L.unary, dt),
                  unary_off=np.ascontiguousarray(L.unary_off, np.int64), dom_size=i32(L.dom_size),
                  var_id=i32(L.var_order), edge_var=i32(L.edge_var), edge_class=i32(L.edge_class),
                  var_ptr=i32(L.var_ptr), slot_edge=slot_edge, soft_end=_per_var(L, soft_end, np.int32),
                  nbr_ptr=i32(nbr_ptr), nbr_idx=i32(nbr_idx), init_value=i32(L.init_value),
                  value=[value0, value0.copy()])
    _set_global_ids(inputs, L, var_global_id, var_seed)
    n = L.n_vars
    state = dict(con_opt=(L.n_factors, dt, 0), cost=(n, dt, 0), has_cost=(n, np.uint8, 0),
                 h_best=(n, np.int32, -1), branch=(n, np.uint8, 0))
    scalars = dict(proba_hard=float(proba_hard), proba_soft=float(proba_soft), mode_max=int(mode == "max"),
                   variant=_cabi.MIXEDDSA_VARIANTS[variant], stop_cycle=int(stop_cycle or 0), seed=_seed(seed))
    _set_psets(inputs, scalars, pset, psets, _cabi.FgMixedDsaPset,
               lambda p: dict(proba_hard=float(p["proba_hard"]), proba_soft=float(p["proba_soft"]),
                              variant=_cabi.MIXEDDSA_VARIANTS[p["variant"]]))
    return inputs, state, scalars


class MixedDsaEngine(_LocalSearchEngine):
    """All-variables-at-once MixedDSA (pydcop/algorithms/mixeddsa.py, MixedDsaComputation; parameters :119-124).

    proba_hard  probability of a move that lowers the number of violated hard constraints, or of a sideways move
                while some remain violated
    proba_soft  probability of a move that only improves the soft cost, or of a sideways move away from a violated
                soft constraint (variants B and C)
    variant     A | B | C; C behaves as B (its own branch in the reference is unreachable)
    stop_cycle  0 = run forever; else the run ends after stop_cycle rounds (dsa_gpu's convention, dsa.py:352)
    var_global_id  canonical order: the Philox counter of each variable (default: the canonical index), as MgmEngine
    var_seed    canonical order: the Philox key of each variable (default: `seed` for every variable), as MgmEngine
    var_pset, psets  the parameter set of each variable (canonical order) and the sets, as DsaEngine
    `values()` reports the cost of the last move (inf while a hard constraint stays violated), NaN before the first
    one; `record()` the best H and the branch of the last round.
    """
    FAMILY = "mixeddsa"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f32", mode="min", proba_hard=0.7,
                 proba_soft=0.5, variant="B", stop_cycle=0, seed=0, var_global_id=None, var_seed=None,
                 var_pset=None, psets=None):
        L = layout
        self._open(layout, device, precision)
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        if variant not in _cabi.MIXEDDSA_VARIANTS:
            raise ValueError(f"invalid variant {variant!r}: expected one of {sorted(_cabi.MIXEDDSA_VARIANTS)}")
        if int(stop_cycle or 0) < 0:
            raise ValueError(f"invalid stop_cycle {stop_cycle!r}: must be >= 0")
        inputs, state, scalars = mixeddsa_plan(L, precision, mode, proba_hard, proba_soft, variant, stop_cycle, seed,
                                               var_global_id, var_seed, var_pset, psets)
        t = self._upload(inputs, state)
        self.__dict__.update(t)
        self._classes = _class_array(L)
        self._create(fill_desc(fill_header(_cabi.FgMixedDsaDesc(), precision, L, self._classes), t, scalars))

    def _assignment(self):
        return self.value[self.cycle % 2]

    def record(self):
        """State of the last round, canonical order: h_best (-1 where the variable did not evaluate) and branch
        (MIXEDDSA_BRANCH_* | MIXEDDSA_MOVED)."""
        L = self.layout
        n = L.n_vars
        return dict(h_best=L.vars_to_canonical(self.h_best[:n].cpu().numpy()),
                    branch=L.vars_to_canonical(self.branch[:n].cpu().numpy()))


def dpop_plan(layout: FactorGraphLayout, tree, sched, precision="f64", mode="min"):
    """DpopEngine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan, for the pseudo-tree
    `tree` and its pseudotree.schedule `sched`; the scalars carry the launch lists."""
    from . import pseudotree as pt
    L = layout
    dt = PRECISIONS[precision][2]
    terms = pt.terms(tree, L)
    arena = terms.pop("arena_size")
    inputs = dict(tables=np.ascontiguousarray(L.tables, dt), unary=np.ascontiguousarray(L.unary, dt), **terms,
                  **{k: getattr(sched, k) for k in ("util_nodes", "util_seg_ptr", "value_nodes", "value_seg_ptr")})
    state = dict(arena=(arena, dt, None), value=(L.n_vars, np.int32, 0), cost=(L.n_vars, dt, 0),
                 unresolved=(1, np.int32, 0))
    launches = lambda ls: C.cast((_cabi.FgDpopLaunch * max(1, len(ls)))(*[_cabi.FgDpopLaunch(*l, 0) for l in ls]),  # noqa: E731
                                 C.POINTER(_cabi.FgDpopLaunch))
    return inputs, state, dict(
        n_vars=L.n_vars, mode_max=int(mode == "max"), n_terms=len(terms["term_kind"]),
        n_tdims=len(terms["tdim_pos"]), arena_size=arena, n_util_segs=len(sched.util_seg_ptr) - 1,
        n_value_segs=len(sched.value_seg_ptr) - 1, n_util_launches=len(sched.util_launches),
        n_value_launches=len(sched.value_launches), util_launches=launches(sched.util_launches),
        value_launches=launches(sched.value_launches), max_sep=max((len(s) for s in tree.sep), default=0))


class DpopEngine(_EngineBase):
    """DPOP (pydcop/algorithms/dpop.py) on a pseudo-tree (pydcop_b200.pseudotree): one `step()` runs the
    UTIL phase bottom-up and the VALUE phase top-down as a fixed, host-computed sequence of launches
    (pseudotree.schedule), after which `finished` is true.  Every node's UTIL stays in one arena.

    tree  a completed PseudoTree over the layout's canonical variables and constraints (build_tree, or
          tree_from_links on the plugin path)
    """
    FAMILY = "dpop"

    def __init__(self, layout: FactorGraphLayout, tree, device=None, precision="f64", mode="min"):
        from . import pseudotree as pt
        L = layout
        self._open(layout, device, precision)
        self.tree = tree
        if mode not in ("min", "max"):
            raise ValueError(f"invalid mode {mode!r}")
        if tree.n_vars != L.n_vars or len(tree.owner) != L.n_factors:
            raise ValueError("the pseudo-tree does not match the layout")
        elem = np.dtype(self.np_dtype).itemsize
        self._util_off, arena = pt.arena_layout(tree)
        big_u, big_sep = pt.largest_separator(tree)
        self.util_bytes = arena * elem
        free, _ = torch.cuda.mem_get_info(self.device)
        if self.util_bytes > free:
            names = ", ".join(str(v) for v in big_sep)
            raise EngineError(
                f"DPOP needs {self.util_bytes} bytes of UTIL tables but {free} bytes of device memory are free; "
                f"the largest separator is that of variable {big_u}: {len(big_sep)} variables [{names}] "
                f"({tree.util_size[big_u]} entries)")
        max_sep = max((len(s) for s in tree.sep), default=0)
        if max_sep > pt.MAX_SEP:
            raise EngineError(f"a separator of {max_sep} variables: the kernels decode at most {pt.MAX_SEP}")
        self.sched = pt.schedule(tree)
        inputs, state, scalars = dpop_plan(L, tree, self.sched, precision, mode)
        self.dev = self._upload(inputs, state)
        self.arena, self.value, self.cost = self.dev["arena"], self.dev["value"], self.dev["cost"]
        self.tables, self.unresolved_dev = self.dev["tables"], self.dev["unresolved"]
        self._classes = _class_array(L)
        d = _cabi.FgDpopDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, PRECISIONS[precision][0]
        self._done = False
        self._create(fill_desc(d, self.dev, scalars))

    def init(self):
        self._done = False
        return self

    def step(self, n_cycles=1):
        """Both phases (DPOP is not iterative: further steps do nothing)."""
        if not self._done and n_cycles > 0:
            with torch.cuda.device(self.device):
                self._check(self.lib.fg_dpop_run(self._h, self._stream()), "fg_dpop_run")
            self._done = True
        return self

    @property
    def finished(self):
        return self._done

    @property
    def cycle(self):
        return 0

    @property
    def unresolved(self):
        """Nodes where no value reached the best (the reference raises IndexError there)."""
        return int(self.unresolved_dev.item())

    def values(self):
        """(value index, the chosen value's joined entry — the reference's reported cost) per variable,
        canonical order."""
        n = self.layout.n_vars
        return self.value[:n].cpu().numpy(), self.cost[:n].double().cpu().numpy()

    def util(self, var):
        """(separator as canonical variable indices, root side first; the UTIL table shaped by their
        domain sizes) of canonical variable `var`."""
        off = self._util_off
        sep = self.tree.sep[var]
        n = self.tree.util_size[var]
        shape = tuple(int(self.layout.canon_dom_size[v]) for v in sep)
        return sep, self.arena[off[var]:off[var] + n].double().cpu().numpy().reshape(shape)

    def _assignment(self):
        """The canonical-order values in the layout's internal order."""
        L = self.layout
        return (self.value[:max(L.n_vars, 1)][torch.as_tensor(L.var_order.astype(np.int64), device=self.device)]
                .contiguous() if L.n_vars else self.value)


def syncbb_plan(layout: FactorGraphLayout, precision="f64", mode="min", var_rank=None, factor_names=None):
    """SyncbbEngine's host-array plan (inputs, state, scalar descriptor fields), as mgm_plan, in CHAIN order (the
    variables sorted by name, `var_rank`; default: the canonical index).  Per chain position p: its earlier
    neighbours sorted by chain position, and per (p, neighbour u) one pair table laid out [val_u][x], every binary
    constraint of p on u added from 0 in node.constraints order in the tables' precision (relations.py:1513-1530 sums
    the same terms in that order).  Unary constraints and variable costs are not part of the plan (syncbb.py reads
    neither); a constraint of arity > 2 raises ValueError naming it (`factor_names`: canonical factor names)."""
    L = layout
    dt = PRECISIONS[precision][2]
    V = L.n_vars
    if V < 2:
        raise ValueError(f"SyncBB needs at least two variables, got {V}: with one, the reference's first variable "
                         "posts its start message to no next variable (syncbb.py:210) and never finishes")
    if mode not in ("min", "max"):
        raise ValueError(f"invalid mode {mode!r}")
    rank = np.arange(V) if var_rank is None else np.asarray(var_rank, dtype=np.int64)
    chain = np.argsort(rank, kind="stable")
    pos = np.empty(V, dtype=np.int64)
    pos[chain] = np.arange(V)
    inv_factor = np.empty(L.n_factors, dtype=np.int64)
    inv_factor[L.factor_perm] = np.arange(L.n_factors)
    for c in L.classes:
        if c.arity > 2:
            f = int(inv_factor[c.first_factor])
            name = factor_names[f] if factor_names is not None else f"#{f}"
            raise ValueError(f"constraint {name} has arity {c.arity}: SyncBB supports binary constraints only "
                             "(syncbb.py:456)")
    edge_class = np.asarray(L.edge_class)
    pair = {}                                   # (p, q) -> [val_u][x] table
    for v in range(V):
        p = int(pos[v])
        for e in L.canon_var_edge[L.canon_var_ptr[v]:L.canon_var_ptr[v + 1]]:   # node.constraints order
            ie = int(L.edge_perm[e])
            c = L.classes[int(edge_class[ie])]
            if c.arity != 2:
                continue
            fl, j = divmod(ie - c.first_edge, 2)
            u = int(L.var_order[L.edge_var[c.first_edge + 2 * fl + 1 - j]])
            q = int(pos[u])
            if q >= p:
                continue
            t = np.asarray(L.tables[c.table_base + fl * c.table_size:c.table_base + (fl + 1) * c.table_size],
                           dtype=dt).reshape(c.dom[0], c.dom[1])
            t = t.T if j == 0 else t            # [val_u][x]
            pair[(p, q)] = (pair.get((p, q), dt(0)) + t).astype(dt)
    keys = sorted(pair)
    elt_ptr = np.zeros(V + 1, dtype=np.int32)
    np.add.at(elt_ptr, np.array([k[0] + 1 for k in keys], dtype=np.int64), 1)
    elt_ptr = np.cumsum(elt_ptr).astype(np.int32)
    sizes = np.array([pair[k].size for k in keys], dtype=np.int64)
    elt_tab = np.concatenate([[0], np.cumsum(sizes)])[:-1].astype(np.int64)
    tabs = np.concatenate([pair[k].reshape(-1) for k in keys]).astype(dt) if keys else np.zeros(0, dt)
    dom = np.asarray(L.canon_dom_size, dtype=np.int32)[chain]
    inputs = dict(dom=dom, elt_ptr=elt_ptr, elt_pos=np.array([k[1] for k in keys], dtype=np.int32),
                  elt_tab=elt_tab, pair=tabs)
    state = dict(ub=(V, dt, None), sel=(V, np.int32, None), path_val=(V, np.int32, None),
                 path_cost=(V, dt, None), path_sum=(V, dt, None), path_comp=(V, dt, None),
                 msg=(4, np.int32, 0), msg_ub=(1, dt, None), count=(2, np.int64, 0), cycles=(V, np.int64, None))
    return inputs, state, dict(n_vars=V, mode_max=int(mode == "max"), n_elts=len(keys), n_pair=int(tabs.size))


SYNCBB_TYPES = ("forward", "backward", "terminate")


class SyncbbEngine(_EngineBase):
    """SyncBB (pydcop/algorithms/syncbb.py): the whole branch-and-bound search in one resident CTA, one message per
    step (forward, backward or terminate).  `step(n)` enqueues one launch that delivers up to n messages; the state
    stays on the device, so a run may be split anywhere.  `finished` once the last variable received its terminate
    message; `values()` is each variable's last value selection (-1 for one that never selected).

    var_rank      position of each variable's NAME in sorted order: the chain (default: the canonical index)
    factor_names  canonical constraint names, for the arity error
    """
    FAMILY = "syncbb"

    def __init__(self, layout: FactorGraphLayout, device=None, precision="f64", mode="min", var_rank=None,
                 factor_names=None):
        L = layout
        inputs, state, scalars = syncbb_plan(L, precision, mode, var_rank, factor_names)
        self._open(layout, device, precision)
        self.mode = mode
        self.chain = np.argsort(np.arange(L.n_vars) if var_rank is None else np.asarray(var_rank), kind="stable")
        self.dev = self._upload(inputs, state)
        self._classes = _class_array(L)
        d = _cabi.FgSyncbbDesc()
        d.abi_version, d.precision = _cabi.FG_ABI_VERSION, PRECISIONS[precision][0]
        self._create(fill_desc(d, self.dev, scalars))

    def step(self, n_steps=1):
        with torch.cuda.device(self.device):
            self._check(self.lib.fg_syncbb_step(self._h, int(n_steps), self._stream()), "fg_syncbb_step")
        return self

    def _current(self):
        s, m, f = C.c_int64(), C.c_int64(), C.c_int32()
        with torch.cuda.device(self.device):
            self._check(self.lib.fg_syncbb_current(self._h, C.byref(s), C.byref(m), C.byref(f)), "fg_syncbb_current")
        return s.value, m.value, bool(f.value)

    @property
    def steps(self):
        """Messages delivered."""
        return self._current()[0]

    @property
    def messages(self):
        """Messages posted: forward, backward and terminate, the first variable's start message included."""
        return self._current()[1]

    @property
    def finished(self):
        return self._current()[2]

    @property
    def cycle(self):
        """What the reference's orchestrated run reports as `cycle`: the largest per-variable new_cycle count
        (orchestrator.py:1243-1258 over agents.py:733)."""
        return int(self.dev["cycles"][:self.layout.n_vars].max().item())

    def cycle_counts(self):
        """Each variable's new_cycle count (messages it received, plus one for the first variable's start),
        canonical order."""
        return self._canonical(self.dev["cycles"][:self.layout.n_vars].cpu().numpy())

    def _canonical(self, a):
        out = np.empty_like(a)
        out[self.chain] = a
        return out

    def values(self):
        """Each variable's last value selection (domain index, -1: none), canonical order."""
        return self._canonical(self.dev["sel"][:self.layout.n_vars].cpu().numpy())

    def bounds(self):
        """Each variable's upper_bound, canonical order."""
        return self._canonical(self.dev["ub"][:self.layout.n_vars].cpu().numpy())

    def message(self):
        """The message in flight: (type 0 forward / 1 backward / 2 terminate, receiver as canonical index, path
        length, bound carried, finished)."""
        m = self.dev["msg"].cpu().numpy()
        return int(m[0]), int(self.chain[m[1]]), int(m[2]), self.dev["msg_ub"][0].item(), bool(m[3])

    def _assignment(self):
        """The canonical-order values in the layout's internal order (a variable without a value reads 0)."""
        L = self.layout
        canon = torch.as_tensor(np.maximum(self.values(), 0).astype(np.int32), device=self.device)
        return canon[torch.as_tensor(L.var_order.astype(np.int64), device=self.device)].contiguous()

    @property
    def tables(self):
        """The full tables, uploaded on first use: only the solution cost reads them."""
        if not hasattr(self, "_tables"):
            self._tables = self._dev(self.layout.tables, PRECISIONS[self.precision][1])
        return self._tables


def make_engine(kind, layout: FactorGraphLayout, params, *, mode="min", precision="f32", device=None, seed=0,
                var_rank=None, isolated_value=None, tree=None, var_global_id=None, var_seed=None, var_pset=None,
                psets=None):
    """The single-GPU engine of algorithm `kind` (a value of solve.ALGOS) over `layout`.  `params`: its algorithm
    parameters, the missing ones taking solve.DEFAULTS; var_rank / isolated_value / var_global_id in canonical order
    as the engines take them (var_rank None: the canonical index; var_global_id None: the canonical index as every
    Philox counter, ignored by the families without draws: MaxSum, DPOP, SyncBB); var_seed in canonical order: the
    Philox key of every variable (None: `seed` for all; DBA, MaxSum, DPOP and SyncBB take none and refuse one);
    var_pset / psets: the parameter set of every variable (canonical order) and the sets (checked parameter dicts)
    for DSA, A-DSA, MGM-2, GDBA and MixedDSA (None: `params` for all; the other families refuse them).
    tree: DPOP's pseudo-tree.  MaxSum records no sent flags."""
    from .solve import DEFAULTS
    p = dict(DEFAULTS[kind], **params)
    if var_seed is not None and kind in ("syncbb", "dba", "dpop", "maxsum"):
        raise ValueError(f"{kind} takes no per-variable seeds")
    if (var_pset is not None or psets is not None) and kind in ("syncbb", "dba", "dpop", "maxsum", "mgm"):
        raise ValueError(f"{kind} takes no per-variable parameter sets")
    if kind == "syncbb":
        return SyncbbEngine(layout, device=device, precision=precision, mode=mode, var_rank=var_rank)
    if kind == "dba":
        return DbaEngine(layout, device=device, precision=precision, mode=mode, infinity=p["infinity"],
                         max_distance=p["max_distance"], stop_cycle=p["stop_cycle"], seed=seed, var_rank=var_rank)
    if kind == "dpop":
        return DpopEngine(layout, tree=tree, device=device, precision=precision, mode=mode)
    if kind == "mixeddsa":
        return MixedDsaEngine(layout, device=device, precision=precision, mode=mode, proba_hard=p["proba_hard"],
                              proba_soft=p["proba_soft"], variant=p["variant"], stop_cycle=p["stop_cycle"], seed=seed,
                              var_global_id=var_global_id, var_seed=var_seed, var_pset=var_pset, psets=psets)
    if kind == "gdba":
        return GdbaEngine(layout, device=device, precision=precision, mode=mode, modifier=p["modifier"],
                          violation=p["violation"], increase_mode=p["increase_mode"], stop_cycle=p["stop_cycle"],
                          seed=seed, var_rank=var_rank, isolated_value=isolated_value, var_global_id=var_global_id,
                          var_seed=var_seed, var_pset=var_pset, psets=psets)
    if kind == "mgm2":
        return Mgm2Engine(layout, device=device, precision=precision, mode=mode, threshold=p["threshold"],
                          favor=p["favor"], stop_cycle=p["stop_cycle"], seed=seed, var_rank=var_rank,
                          var_global_id=var_global_id, var_seed=var_seed, var_pset=var_pset, psets=psets)
    if kind == "mgm":
        return MgmEngine(layout, device=device, precision=precision, mode=mode, stop_cycle=p["stop_cycle"], seed=seed,
                         break_mode=p["break_mode"], var_rank=var_rank, isolated_value=isolated_value,
                         var_global_id=var_global_id, var_seed=var_seed)
    if kind == "maxsum":
        return MaxSumEngine(layout, device=device, precision=precision, mode=mode, damping=p["damping"],
                            damping_nodes=p["damping_nodes"], stability=p["stability"],
                            start_messages=p["start_messages"], record_sent=False)
    return DsaEngine(layout, device=device, precision=precision, mode=mode, probability=p["probability"],
                     p_mode=p.get("p_mode", "fixed"), variant=p["variant"], stop_cycle=p["stop_cycle"], seed=seed,
                     isolated_value=isolated_value, var_global_id=var_global_id, var_seed=var_seed,
                     var_costs=(kind == "adsa"), var_pset=var_pset, psets=psets)   # A-DSA: candidates carry own costs
