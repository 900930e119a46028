"""Graph operators with the reference's `ntsGraphOp` interface (core/ntsBaseOp.hpp:24-48):
constructed from `(PartitionedGraph, active)`, `forward(x)` / `forward(x, w)`, `backward(grad)`,
`get_additional_grad()`; outputs are freshly allocated zero tensors the kernels accumulate into
(NtsScheduler::NewKeyTensor / NewLeafTensor, core/NtsScheduler.hpp:378-394), except ForwardSingleGPUfuseOp's, which
its aggregation writes without a zero fill.

Every operator calls the sm_90a kernels through the C ABI (`_lib.call`); tensors only provide device
memory and the current CUDA stream.  There is no CPU path: a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
import time as _time

import torch

from . import _lib
from ._lib import stream as _stream


def row_pitched(t):
    """True for a 2-D tensor whose rows are contiguous and start a row pitch >= its width apart (a contiguous tensor,
    or a column slice t[:, :F] of one)."""
    return t.dim() == 2 and (t.is_contiguous() or (t.stride(1) == 1 and t.stride(0) >= t.shape[1]))


_F32 = (torch.float32,)
_F32_BF16 = (torch.float32, torch.bfloat16)


def _check_input(t, name="input", pitched=False, dtypes=_F32):
    """A 2-D CUDA tensor of one of `dtypes` (the gathered operand of BF16 gathers may be bfloat16 as well:
    _gathered_dtypes).  pitched=True: also accept row-pitched tensors (row_pitched), for operators that pass the row
    pitch on."""
    if not t.is_cuda:
        raise _lib.NtsError("%s must be a CUDA tensor (libnts_b200 has no CPU fallback)" % name)
    if t.dtype not in dtypes or t.dim() != 2:
        raise _lib.NtsError("%s must be a 2-D %s tensor" % (name, " or ".join(str(d)[len("torch."):] for d in dtypes)))
    if not (t.is_contiguous() or (pitched and row_pitched(t))):
        # the reference borrows packed_accessor storage (core/NtsScheduler.hpp:505-515): contiguous only
        raise _lib.NtsError("%s must be contiguous" % name + (" or row-pitched" if pitched else ""))
    return t


def _check_gather_dtype(gather_dtype):
    """The gathered-operand options: None (FP32 gathers) or torch.bfloat16 (BF16 gathers, FP32 accumulation)."""
    if gather_dtype is not None and gather_dtype != torch.bfloat16:
        raise _lib.NtsError("gather_dtype must be None or torch.bfloat16, not %s" % (gather_dtype,))
    return gather_dtype


def _gathered_dtypes(gather_dtype):
    """The types a gathered operand may have: float32, and with BF16 gathers bfloat16 as well (used as is)."""
    return _F32 if gather_dtype is None else _F32_BF16


_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1}   # NTS_DTYPE_F32 / NTS_DTYPE_BF16 of include/nts_b200.h
PLAN_OVERWRITE, PLAN_COPY_INPUT = 1, 2                # NTS_PLAN_OVERWRITE / NTS_PLAN_COPY_INPUT


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class KernelTimer:
    """Optional CUDA-event bracket around every aggregation launch (bench.py's live roofline measurement).
    Events are recorded on the stream the kernel is launched on; nothing is synchronised until `summary()`."""

    def __init__(self):
        self.records = []  # (tag, F, edges, rows, start, stop)

    def bracket(self, tag, F, edges, rows):
        start = torch.cuda.Event(enable_timing=True)
        stop = torch.cuda.Event(enable_timing=True)
        self.records.append((tag, int(F), int(edges), int(rows), start, stop))
        return start, stop

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for tag, F, edges, rows, a, b in self.records:
            d = out.setdefault((tag, F), {"calls": 0, "ms": 0.0, "edges": 0, "rows": 0})
            d["calls"] += 1
            d["ms"] += a.elapsed_time(b)
            d["edges"] += edges
            d["rows"] += rows
        return out


_timer = None


def set_kernel_timer(timer):
    global _timer
    _timer = timer


class _timed:
    """`with _timed(tag, F, edges, rows): launch` - CUDA events around the launch when a KernelTimer is installed."""

    def __init__(self, tag, F, edges, rows):
        self.ev = _timer.bracket(tag, F, edges, rows) if _timer else None

    def __enter__(self):
        if self.ev:
            self.ev[0].record()

    def __exit__(self, *exc):
        if self.ev:
            self.ev[1].record()
        return False


def segment_gather_sum(out, x, weight, indices, offsets, index_base, n_rows, n_edges):
    """out[r,:] += sum_e x[indices[e]-index_base,:] * weight[e]  (nts_segment_gather_sum)."""
    _lib.call("nts_segment_gather_sum", _ptr(x), _ptr(out), _ptr(weight), _ptr(indices), _ptr(offsets),
              int(index_base), int(n_rows), int(n_edges), int(x.shape[1]), _stream())
    return out


class GatherPlan:
    """nts_gather_plan (include/nts_b200.h): one chunk direction preprocessed once for repeated aggregation -
    source-slab bucketing (L2 residency), interleaved (row, weight) pairs, 16-byte aligned gathers."""

    def __init__(self, offsets, indices, weight, index_base, n_rows, n_edges, gather_rows, slabs, slot_of=None,
                 tune_for=0, hubs=(0, 0), gather_dtype=None, tune_accumulate=True):
        """slabs > 0: that many source slabs and hubs = (hub columns, hub rows) dense blocks
        (nts_gather_plan_create_hybrid); slabs == 0: slab and hub counts are MEASURED for feature width `tune_for`
        (nts_gather_plan_create_tuned_ex), timed as BF16 gathers when gather_dtype is torch.bfloat16, and as
        overwriting runs (`run(..., accumulate=False)`) when tune_accumulate is False.  build_s is the one-time
        construction (and tuning) time."""
        L = _lib.load()
        _check_gather_dtype(gather_dtype)
        t0 = _time.perf_counter()
        if slabs > 0:
            self.handle = L.nts_gather_plan_create_hybrid(_ptr(offsets), _ptr(indices), _ptr(weight), _ptr(slot_of),
                                                          int(index_base), int(n_rows), int(n_edges),
                                                          int(gather_rows), int(slabs), int(hubs[0]), int(hubs[1]),
                                                          _stream())
        else:
            self.handle = L.nts_gather_plan_create_tuned_ex(
                _ptr(offsets), _ptr(indices), _ptr(weight), _ptr(slot_of), int(index_base), int(n_rows), int(n_edges),
                int(gather_rows), int(tune_for), _DTYPE_CODE[gather_dtype or torch.float32],
                0 if tune_accumulate else PLAN_OVERWRITE, _stream())
        self.build_s = _time.perf_counter() - t0      # create synchronises the stream
        _lib.checked(self.handle, "gather plan construction")
        self.slabs = int(L.nts_gather_plan_slabs(self.handle))
        hc, hr = C.c_int(0), C.c_int(0)
        _lib.call("nts_gather_plan_hubs", self.handle, C.byref(hc), C.byref(hr))
        self.hub_cols, self.hub_rows = hc.value, hr.value
        self.n_rows, self.n_edges = int(n_rows), int(n_edges)

    @property
    def overlap(self):
        """True when the hub-row block runs inside the slab launches (nts_gather_plan_overlap)."""
        return bool(_lib.load().nts_gather_plan_overlap(self.handle))

    def set_overlap(self, overlap):
        _lib.call("nts_gather_plan_set_overlap", self.handle, int(bool(overlap)))

    def key(self):
        """What decides the plan's arrays and schedule besides the chunk direction: plans with equal keys are
        interchangeable."""
        return ((self.slabs,) + ((self.hub_cols, self.hub_rows) if self.hub_cols or self.hub_rows else ())
                + (("overlap",) if self.overlap else ()))

    def run(self, x, out, gather_dtype=None, accumulate=True):
        """out += A x, or out = A x with accumulate=False (out may then hold anything, NaN included).  x may be
        row-pitched (a column slice x[:, :F] of a wider tensor): its row pitch is passed on, and where the pitch allows
        it the rows are gathered in place.  gather_dtype=torch.bfloat16: the rows of x (float32 or bfloat16) are
        gathered as BF16 with FP32 accumulation (nts_gather_plan_run_bf16_ex); a bfloat16 x needs that option."""
        if not row_pitched(x):
            raise _lib.NtsError("the gathered input must have contiguous rows (unit column stride)")
        F = int(x.shape[1])
        ld = F if x.is_contiguous() else int(x.stride(0))
        flags = 0 if accumulate else PLAN_OVERWRITE
        # an in-place gather reads all ld values of the last row too: without storage behind them, gather a copy
        if ld != F and (x.storage_offset() + x.shape[0] * ld) * x.element_size() > x.untyped_storage().nbytes():
            flags |= PLAN_COPY_INPUT
        if _check_gather_dtype(gather_dtype) is not None:
            if x.dtype not in _DTYPE_CODE:
                raise _lib.NtsError("BF16 gathers take a float32 or bfloat16 input, not %s" % x.dtype)
            _lib.call("nts_gather_plan_run_bf16_ex", self.handle, _ptr(x), _DTYPE_CODE[x.dtype], ld, _ptr(out), F,
                      flags, _stream())
            return out
        if x.dtype == torch.bfloat16:
            raise _lib.NtsError("a bfloat16 input needs gather_dtype=torch.bfloat16")
        _lib.call("nts_gather_plan_run_ex", self.handle, _ptr(x), ld, _ptr(out), F, flags, _stream())
        return out

    def bytes(self):
        return int(_lib.load().nts_gather_plan_bytes(self.handle))

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _lib.load().nts_gather_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


# Plan policy: "auto" preprocesses chunks with at least PLAN_MIN_EDGES edges on first use (the arrays of a chunk are
# immutable, like the reference's CopyGraphToDevice uploads); "off" always takes the plain kernel on the reference
# layout; "on" plans every chunk.  NTS_PLAN / NTS_PLAN_SLABS are measurement overrides.
import os as _os

PLAN_MIN_EDGES = 1 << 20
_plan_mode = {"0": "off", "1": "on"}.get(_os.environ.get("NTS_PLAN", ""), "auto")
_plan_slabs = int(_os.environ.get("NTS_PLAN_SLABS", "0"))


def set_plan_mode(mode, slabs=0):
    """mode in {"auto", "on", "off"}; slabs > 0 forces the slab count (0 = nts_gather_plan_pick_slabs)."""
    global _plan_mode, _plan_slabs
    if mode not in ("auto", "on", "off"):
        raise ValueError("plan mode must be auto, on or off")
    _plan_mode, _plan_slabs = mode, int(slabs)


def _chunk_direction(chunk, direction):
    """(offsets, indices, weight, index base, output rows, gathered rows) of one chunk direction: the CSC for "fwd"
    (Y = A X), the CSR for "bwd" (dX = A^T dY)."""
    if direction == "fwd":
        return (chunk.column_offset_gpu, chunk.row_indices_gpu, chunk.edge_weight_forward_gpu, chunk.src_range[0],
                chunk.batch_size_forward, chunk.batch_size_backward)
    return (chunk.row_offset_gpu, chunk.column_indices_gpu, chunk.edge_weight_backward_gpu, chunk.dst_range[0],
            chunk.batch_size_backward, chunk.batch_size_forward)


def _chunk_plan(chunk, direction, F, gather_dtype=None):
    """The GatherPlan of one chunk direction for feature width F, or None when the plain kernel should run.
    BF16 gathers exist only in nts_gather_plan: with gather_dtype=torch.bfloat16 every chunk gets a plan, whatever its
    size or the plan mode, tuned per (width, type).  Measured plans are timed as overwriting runs, the mode
    ForwardSingleGPUfuseOp runs them in."""
    if gather_dtype is None and (_plan_mode == "off" or (_plan_mode == "auto" and chunk.edge_size < PLAN_MIN_EDGES)):
        return None
    plans = chunk.__dict__.setdefault("_gather_plans", {})      # (direction, slabs[, hub cols, hub rows]) -> plan
    tuned = chunk.__dict__.setdefault("_gather_plan_for", {})   # (direction, F[, "bf16"]) -> plan picked by measurement
    key = (direction, _plan_slabs) if _plan_slabs else (direction, "F", int(F))
    if gather_dtype is not None and not _plan_slabs:
        key += ("bf16",)
    plan = plans.get(key) if _plan_slabs else tuned.get(key)
    if plan is None:
        offsets, indices, weight, index_base, n_rows, gather_rows = _chunk_direction(chunk, direction)
        plan = GatherPlan(offsets, indices, weight, index_base, n_rows, chunk.edge_size, gather_rows, _plan_slabs,
                          tune_for=int(F), gather_dtype=gather_dtype, tune_accumulate=False)
        share = (direction,) + plan.key()
        if share in plans:     # another width already settled on these slab and hub counts: share the arrays
            plan = plans[share]
        plans[share] = plan
        if not _plan_slabs:
            tuned[key] = plan
    return plan


def _bf16_plan(chunk, direction, F, with_weight, gather_dtype):
    if _check_gather_dtype(gather_dtype) is None:
        return _chunk_plan(chunk, direction, F) if with_weight else None
    if not with_weight:
        raise _lib.NtsError("BF16 gathers always apply the edge weights (with_weight=True)")
    return _chunk_plan(chunk, direction, F, gather_dtype)


def _plain_operands(out, x, accumulate):
    """The plain kernels accumulate into out and read contiguous rows."""
    if not accumulate:
        out.zero_()
    return x.contiguous()


def _gather_chunk(direction, chunk, out, x, with_weight, gather_dtype, accumulate):
    """One chunk direction (_chunk_direction) through its plan, or the plain kernel on the reference layout."""
    plan = _bf16_plan(chunk, direction, x.shape[1], with_weight, gather_dtype)
    offsets, indices, weight, _, n_rows, _ = _chunk_direction(chunk, direction)
    with _timed(direction, x.shape[1], chunk.edge_size, n_rows):
        if plan is not None:
            return plan.run(x, out, gather_dtype, accumulate)
        x = _plain_operands(out, x, accumulate)
        # the plain entries take the CSC as (row_indices, column_offset) and the CSR as (row_offset, column_indices)
        entry, a, b = (("nts_gather_by_dst_from_src", indices, offsets) if direction == "fwd" else
                       ("nts_gather_by_src_from_dst", offsets, indices))
        _lib.call(entry, _ptr(x), _ptr(out), _ptr(weight), _ptr(a), _ptr(b), chunk.src_range[0], chunk.src_range[1],
                  chunk.dst_range[0], chunk.dst_range[1], chunk.edge_size, n_rows, int(x.shape[1]),
                  1 if with_weight else 0, _stream())
    return out


def gather_by_dst_from_src(chunk, out, x, with_weight=True, gather_dtype=None, accumulate=True):
    """NtsScheduler::GatherByDstFromSrc (core/NtsScheduler.hpp:151-191) on one chunk: out += A x, or out = A x with
    accumulate=False.  x may be row-pitched (GatherPlan.run).  gather_dtype=torch.bfloat16: x (float32 or bfloat16)
    is gathered as BF16 rows with FP32 accumulation (GatherPlan.run)."""
    return _gather_chunk("fwd", chunk, out, x, with_weight, gather_dtype, accumulate)


def gather_by_src_from_dst(chunk, out, grad, with_weight=True, gather_dtype=None, accumulate=True):
    """NtsScheduler::GatherBySrcFromDst (core/NtsScheduler.hpp:257-293) on one chunk (accumulate and gather_dtype as
    in gather_by_dst_from_src: the gathered output gradient is rounded to BF16, dX accumulates in FP32)."""
    return _gather_chunk("bwd", chunk, out, grad, with_weight, gather_dtype, accumulate)


class ntsGraphOp:
    """core/ntsBaseOp.hpp:24-48."""

    def __init__(self, partitioned_graph, active=None):
        self.partitioned_graph_ = partitioned_graph
        self.active_ = active

    def forward(self, f_input, f_input1=None):
        raise NotImplementedError

    def backward(self, output_grad):
        raise NotImplementedError

    def get_additional_grad(self):
        raise NotImplementedError("get_additional_grad is not implemented")


class ForwardSingleGPUfuseOp(ntsGraphOp):
    """core/ntsSingleGPUFusedGraphOp.hpp:48-71 -> Graph::forward_single / backward_single
    (core/graph.hpp:3805-3855): Y = A X on chunk 0, dX = A^T dY, no communication.

    gather_dtype=torch.bfloat16: the gathered operand (X forward, dY backward) is rounded to BF16 and accumulated in
    FP32; forward takes a float32 or bfloat16 X, Y and dX are float32, backward takes a float32 dY.

    X and dY may be row-pitched (a column slice of a wider tensor, ops.row_pitched): a planned run passes the pitch on
    and gathers the rows in place when it is a multiple of 16 bytes.  Y and dX are freshly allocated and written by
    overwriting runs (GatherPlan.run(..., accumulate=False)), never zero-filled first."""

    def __init__(self, partitioned_graph, active=None, gather_dtype=None):
        super().__init__(partitioned_graph, active)
        self.gather_dtype = _check_gather_dtype(gather_dtype)

    def forward(self, f_input, f_input1=None):
        x = _check_input(f_input, "input", True, _gathered_dtypes(self.gather_dtype))
        c = self.partitioned_graph_.graph_chunks[0]
        y = torch.empty((c.batch_size_forward, x.shape[1]), dtype=torch.float32, device=x.device)
        return gather_by_dst_from_src(c, y, x, gather_dtype=self.gather_dtype, accumulate=False)

    def backward(self, f_output_grad):
        g = _check_input(f_output_grad, "output_grad", pitched=True)
        c = self.partitioned_graph_.graph_chunks[0]
        dx = torch.empty((c.batch_size_backward, g.shape[1]), dtype=torch.float32, device=g.device)
        return gather_by_src_from_dst(c, dx, g, gather_dtype=self.gather_dtype, accumulate=False)


class MiniBatchFuseOp(ntsGraphOp):
    """core/ntsMiniBatchGraphOp.hpp:61-131 on one block of a sample (sample.SampledSubgraph): forward
    Y[n_dst, F] = sum_e w_e X[src_local(e)], backward dX[n_src, F] over the transposed block, both through K1
    (nts_segment_gather_sum) on the block's own arrays - a block changes every step, so nothing is planned.

    table=True: X is the whole [V, F] feature table and the forward gathers by the block's global source ids
    (row_global), so the table rows of the block's sources are never copied out first; the table must have at least
    the graph's V rows (sampled_subgraph.vertices).  Such an op has no backward: it is the first graph op of the
    model, which the tape never back-propagates.

    gather_dtype=torch.bfloat16: both directions gather BF16 rows with FP32 accumulation (nts_segment_gather_sum_bf16);
    Y and dX stay float32.  A bfloat16 X (the table or local rows) is used as it is: rows of a pitch ld % 8 == 0
    (ld >= F, e.g. a [:, :F] view of [n, ld] rows), 16-byte aligned.  A float32 X, and dY in the backward, are rounded
    once into pitched scratch rows (nts_rows_to_bf16)."""

    def __init__(self, sampled_subgraph, hop, table=False, gather_dtype=None):
        super().__init__(sampled_subgraph, None)
        self.block = sampled_subgraph.blocks[hop]
        self.hop, self.table = int(hop), bool(table)
        self.gather_dtype = _check_gather_dtype(gather_dtype)
        self.vertices = getattr(sampled_subgraph, "vertices", None)
        if self.table and (self.block.row_global is None or self.vertices is None):
            raise _lib.NtsError("table=True needs the block's global source ids (row_global) and the graph's vertex "
                                "count (SampledSubgraph.vertices)")

    def forward(self, f_input, f_input1=None):
        b = self.block
        if self.gather_dtype is None:
            x = _check_input(f_input, "input")
        else:
            x = _check_bf16_operand(_check_input(f_input, "input", True, _F32_BF16), "input")
        if self.table and x.shape[0] < self.vertices:
            raise _lib.NtsError("the feature table has %d rows, the sampled graph has %d vertices"
                                % (x.shape[0], self.vertices))
        if not self.table and x.shape[0] != b.n_src:
            raise _lib.NtsError("input has %d rows, hop %d has %d sources" % (x.shape[0], self.hop, b.n_src))
        y = torch.zeros((b.n_dst, x.shape[1]), dtype=torch.float32, device=x.device)
        idx = b.row_global if self.table else b.row_indices
        return self._k1(y, x, b.weight, idx, b.column_offset, b.n_dst, "minibatch_fwd")

    def backward(self, f_output_grad):
        if self.table:
            raise _lib.NtsError("a table gather (table=True) has no backward")
        g = _check_input(f_output_grad, "output_grad")
        b = self.block
        if g.shape[0] != b.n_dst:
            raise _lib.NtsError("output_grad has %d rows, hop %d has %d destinations" % (g.shape[0], self.hop, b.n_dst))
        dx = torch.zeros((b.n_src, g.shape[1]), dtype=torch.float32, device=g.device)
        return self._k1(dx, g, b.weight_backward, b.column_indices, b.row_offset, b.n_src, "minibatch_bwd")

    def _k1(self, out, x, weight, indices, offsets, n_rows, tag):
        """out += the block's gather-sum of x (K1 on FP32 rows, or on BF16 rows under tag + "_bf16")."""
        n_edges = self.block.n_edges
        if self.gather_dtype is None:
            with _timed(tag, x.shape[1], n_edges, n_rows):
                return segment_gather_sum(out, x, weight, indices, offsets, 0, n_rows, n_edges)
        r = _bf16_rows(x, "minibatch_bf16_round")
        return segment_gather_sum_bf16(out, (r, int(r.stride(0))), weight, indices, offsets, n_rows, n_edges,
                                       tag + "_bf16")


def _check_bf16_operand(t, name):
    """A bfloat16 operand of K1 on BF16 rows must already have its layout: row pitch % 8 == 0, 16-byte aligned."""
    if t.dtype == torch.bfloat16 and (t.stride(0) % 8 != 0 or t.data_ptr() % 16 != 0):
        raise _lib.NtsError("a bfloat16 %s needs rows of a pitch that is a multiple of 8 values (e.g. a [:, :F] view "
                            "of [n, 8*ceil(F/8)] rows), 16-byte aligned; got pitch %d" % (name, t.stride(0)))
    return t


def _bf16_rows(t, tag, ld=None):
    """A bfloat16 t as it is; a float32 t (of unit column stride) rounded once into [n, ld] BF16 rows (by default
    ld = 8*ceil(F/8)), the columns past F zero."""
    if t.dtype == torch.bfloat16:
        return t
    n, F = t.shape
    ld = (F + 7) // 8 * 8 if ld is None else int(ld)
    r = torch.empty((n, ld), dtype=torch.bfloat16, device=t.device)
    with _timed(tag, F, 0, n):
        _lib.call("nts_rows_to_bf16", _ptr(t), _DTYPE_CODE[torch.float32], int(t.stride(0)), _ptr(r), n, F, ld,
                  _stream())
    return r


def segment_gather_sum_bf16(out, rows, weight, indices, offsets, n_rows, n_edges, tag="segment_gather_sum_bf16"):
    """out[r,:F] += sum_e float(x[indices[e],:F]) * weight[e] for rows = (x, ld): BF16 rows of pitch ld
    (nts_segment_gather_sum_bf16)."""
    x, ld = rows
    with _timed(tag, out.shape[1], n_edges, n_rows):
        _lib.call("nts_segment_gather_sum_bf16", _ptr(x), ld, _ptr(out), _ptr(weight), _ptr(indices), _ptr(offsets),
                  int(n_rows), int(n_edges), int(out.shape[1]), _stream())
    return out


class ForwardGPUfuseOp(ntsGraphOp):
    """core/ntsDistGPUFusedGraphOp.hpp:48-90: the distributed fused GCN aggregation.  The reference drives it
    through Graph::sync_compute_decoupled / compute_sync_decoupled with host-staged MPI messages
    (core/graph.hpp:3455-3719); here the exchange is device-resident (neutronstarlite_b200.exchange)."""

    def __init__(self, partitioned_graph, active=None, exchange=None, gather_dtype=None):
        super().__init__(partitioned_graph, active)
        self.gather_dtype = _check_gather_dtype(gather_dtype)
        if exchange is None:
            from .exchange import default_exchange
            exchange = default_exchange(partitioned_graph)
        self.exchange = exchange

    def forward(self, f_input, f_input1=None):
        x = _check_input(f_input, "input", dtypes=_gathered_dtypes(self.gather_dtype))
        if self.gather_dtype is None:
            return self.exchange.forward(x)
        return self.exchange.forward(x, gather_dtype=self.gather_dtype)

    def backward(self, f_output_grad):
        g = _check_input(f_output_grad, "output_grad")
        if self.gather_dtype is None:
            return self.exchange.backward(g)
        return self.exchange.backward(g, gather_dtype=self.gather_dtype)


# ---- edge-granular operators (core/ntsDistGPUGraphOp.hpp) ------------------------------------------------------
class _EdgeOp(ntsGraphOp):
    def _topo(self):
        pg = self.partitioned_graph_
        if pg.column_offset_gpu is None or pg.row_indices_gpu is None:
            raise _lib.NtsError("whole-partition CSC missing: call PartitionedGraph.generate_all(dist=True, device=...)")
        return pg


class DistGPUGetDepNbrOp(ntsGraphOp):
    """core/ntsDistGPUGraphOp.hpp:48-143: fetch the feature rows of every (local or remote) source of a local
    in-edge into the mirror matrix [owned_mirrors, F]; backward returns mirror gradients to the owners.
    Device-resident here (f4 of SURVEY 8f): no .cpu()/MPI/.cuda() round trip."""

    def __init__(self, partitioned_graph, active=None, exchange=None):
        super().__init__(partitioned_graph, active)
        if exchange is None:
            from .exchange import default_exchange
            exchange = default_exchange(partitioned_graph)
        self.exchange = exchange

    def forward(self, f_input, f_input1=None):
        return self.exchange.fetch_mirrors(_check_input(f_input))

    def backward(self, f_output_grad):
        return self.exchange.return_mirror_grads(_check_input(f_output_grad, "output_grad"))


class DistGPUScatterSrc(_EdgeOp):
    """core/ntsDistGPUGraphOp.hpp:100-176: mirror [M,F] -> edge messages [E_p,F]."""

    def forward(self, f_input, f_input1=None):
        pg = self._topo()
        x = _check_input(f_input)
        msg = torch.zeros((pg.owned_edges, x.shape[1]), dtype=torch.float32, device=x.device)
        _lib.call("nts_scatter_src_mirror_to_msg", _ptr(msg), _ptr(x), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), _ptr(pg.mirror_index_gpu), pg.owned_vertices, x.shape[1], _stream())
        return msg

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        out = torch.zeros((pg.owned_mirrors, g.shape[1]), dtype=torch.float32, device=g.device)
        _lib.call("nts_gather_msg_to_src_mirror", _ptr(out), _ptr(g), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), _ptr(pg.mirror_index_gpu), pg.owned_vertices, g.shape[1], _stream())
        return out


class DistGPUScatterDst(_EdgeOp):
    """core/ntsDistGPUGraphOp.hpp:178-238: local vertices [V_p,F] -> edge messages [E_p,F]."""

    def forward(self, f_input, f_input1=None):
        pg = self._topo()
        x = _check_input(f_input)
        msg = torch.zeros((pg.owned_edges, x.shape[1]), dtype=torch.float32, device=x.device)
        _lib.call("nts_scatter_dst_to_msg", _ptr(msg), _ptr(x), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), pg.owned_vertices, x.shape[1], _stream())
        return msg

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        out = torch.zeros((pg.owned_vertices, g.shape[1]), dtype=torch.float32, device=g.device)
        _lib.call("nts_gather_msg_to_dst", _ptr(out), _ptr(g), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), pg.owned_vertices, g.shape[1], _stream())
        return out


class DistGPUAggregateDst(_EdgeOp):
    """core/ntsDistGPUGraphOp.hpp:240-300: edge messages [E_p,F] -> sum per destination [V_p,F]."""

    def forward(self, f_input, f_input1=None):
        pg = self._topo()
        m = _check_input(f_input)
        out = torch.zeros((pg.owned_vertices, m.shape[1]), dtype=torch.float32, device=m.device)
        _lib.call("nts_gather_msg_to_dst", _ptr(out), _ptr(m), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), pg.owned_vertices, m.shape[1], _stream())
        return out

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        msg = torch.zeros((pg.owned_edges, g.shape[1]), dtype=torch.float32, device=g.device)
        _lib.call("nts_scatter_dst_to_msg", _ptr(msg), _ptr(g), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), pg.owned_vertices, g.shape[1], _stream())
        return msg


class DistGPUEdgeSoftMax(_EdgeOp):
    """core/ntsDistGPUGraphOp.hpp:302-361; numerics follow the CPU operator DistEdgeSoftMax
    (core/ntsDistCPUGraphOp.hpp:442-492): column-wise, max-subtracted."""

    def __init__(self, partitioned_graph, active=None):
        super().__init__(partitioned_graph, active)
        self.IntermediateResult = None

    def forward(self, f_input, f_input1=None):
        pg = self._topo()
        m = _check_input(f_input)
        out = torch.zeros_like(m)
        self.IntermediateResult = torch.zeros_like(m)
        _lib.call("nts_edge_softmax_forward", _ptr(out), _ptr(m), _ptr(self.IntermediateResult),
                  _ptr(pg.row_indices_gpu), _ptr(pg.column_offset_gpu), pg.owned_vertices, m.shape[1], _stream())
        return out

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        out = torch.zeros_like(g)
        _lib.call("nts_edge_softmax_backward", _ptr(out), _ptr(g), _ptr(self.IntermediateResult),
                  _ptr(pg.row_indices_gpu), _ptr(pg.column_offset_gpu), pg.owned_vertices, g.shape[1], _stream())
        return out


class DistGPUAggregateDstFuseWeight(_EdgeOp):
    """GPU twin of DistAggregateDstFuseWeight (core/ntsDistCPUGraphOp.hpp:499-594), the fused GAT aggregation
    of toolkits/GAT_CPU_DIST_OPTM.hpp:196-241: y[d,:] = sum_e a[e] * mirror[MirrorIndex[src(e)],:], never
    materialising an [E,F] message.  backward returns d_mirror; `get_additional_grad()` returns d_a [E,1]."""

    def __init__(self, partitioned_graph, active=None):
        super().__init__(partitioned_graph, active)
        self._mirror = None
        self._a = None
        self.e_weight_grad = None

    def forward(self, f_input, e_weight=None):
        pg = self._topo()
        x = _check_input(f_input)
        a = _check_input(e_weight, "edge weight")
        self._mirror, self._a = x, a
        heads = int(a.shape[1])  # [E, H]: head h weights columns [h*D, (h+1)*D); H = 1 is the reference's operator
        out = torch.zeros((pg.owned_vertices, x.shape[1]), dtype=torch.float32, device=x.device)
        _lib.call("nts_segment_gather_sum_heads", _ptr(x), _ptr(out), _ptr(a), _ptr(pg.row_indices_gpu),
                  _ptr(pg.column_offset_gpu), _ptr(pg.mirror_index_gpu), 0, pg.owned_vertices, pg.owned_edges,
                  x.shape[1], heads, _stream())
        return out

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        dm = torch.zeros((pg.owned_mirrors, g.shape[1]), dtype=torch.float32, device=g.device)
        self.e_weight_grad = torch.zeros_like(self._a)
        _lib.call("nts_aggregate_dst_fuse_weight_backward_heads", _ptr(dm), _ptr(self.e_weight_grad),
                  _ptr(self._mirror), _ptr(self._a), _ptr(g), _ptr(pg.row_indices_gpu), _ptr(pg.column_offset_gpu),
                  _ptr(pg.mirror_index_gpu), pg.owned_vertices, g.shape[1], int(self._a.shape[1]), _stream())
        return dm

    def get_additional_grad(self):
        return self.e_weight_grad


class _FusedGAT:
    """The K7 launches of one GAT layer on one topology, shared by DistGPUFusedGATOp (a partition's CSC and its
    mirror-slot CSR) and MiniBatchGATOp (a sampled block and its transposed block).  Edge e of destination d
    (column_offset[d] <= e < column_offset[d+1]) reads row slots[e] of the gathered matrix, which has n_src rows; the
    two-pass backward lists the out-edges of every row in (slot_row_offset, slot_column_indices), edges of a row in
    edge order.  forward(x, s, d) runs the statistics and the aggregation and keeps what the backward needs;
    backward_two_pass(g, slot_row_offset, slot_column_indices) and backward_one_pass(g, row_indices, mirror_index)
    return (dx, ds, dd)."""

    def __init__(self, column_offset, slots, n_dst, n_src, n_edges, slope, gather_dtype):
        self.column_offset, self.slots = column_offset, slots
        self.n_dst, self.n_src, self.n_edges = int(n_dst), int(n_src), int(n_edges)
        self.slope, self.gather_dtype = slope, gather_dtype
        self.saved = None

    def forward(self, x, s, d):
        H, F = int(s.shape[1]), int(x.shape[1])
        seg_max = torch.empty((self.n_dst, H), dtype=torch.float32, device=x.device)
        seg_sum = torch.empty_like(seg_max)
        with _timed("gat_stats", F, self.n_edges, self.n_dst):
            _lib.call("nts_gat_softmax_stats", _ptr(seg_max), _ptr(seg_sum), _ptr(s), _ptr(d), _ptr(self.slots),
                      _ptr(self.column_offset), 0, self.n_dst, H, self.slope, _stream())
        if self.gather_dtype is None:
            # odd single-head width (the 41-wide output layer of config D): gather from a copy padded to a multiple
            # of 4 columns so that the kernel uses 16-byte loads and packed virtual warps instead of 4-byte gathers
            # (11.9 -> ~4 ms per call on config D); the zero columns are dropped again below
            ld = (F + 3) // 4 * 4 if H == 1 else F
            rows = x if ld == F else torch.nn.functional.pad(x, (0, ld - F))
            entry, widths = "nts_gat_fused_aggregate_forward", (ld,)
        else:
            # rows of ld = ceil(F/8)*8 BF16 values: 16-byte chunks of 8, and for the 41-wide layer this replaces the
            # padded FP32 copy of the FP32 path; out shares the row stride and loses its zero pad columns below
            ld = (F + 7) // 8 * 8
            rows = self._to_bf16_rows(x, ld)
            entry, widths = "nts_gat_fused_aggregate_forward_bf16", (F, ld)
        out = torch.zeros((self.n_dst, ld), dtype=torch.float32, device=x.device)
        with _timed("gat_fwd", F, self.n_edges, self.n_dst):
            _lib.call(entry, _ptr(rows), _ptr(out), _ptr(s), _ptr(d), _ptr(seg_max), _ptr(seg_sum), _ptr(self.slots),
                      _ptr(self.column_offset), 0, self.n_dst, self.n_edges, *widths, H, self.slope, _stream())
        if ld != F:
            out = out[:, :F].contiguous()
        # what the backward gathers: x, or m~ = bf16(x) (the FP32 input is then not kept)
        self.saved = (x if self.gather_dtype is None else rows, s, d, seg_max, seg_sum, out)
        return out

    @staticmethod
    def _to_bf16_rows(t, ld):
        """bf16(t) as rows of ld values, the columns past t's width zero: K7's one rounding of its gathered operand."""
        return _bf16_rows(t, "gat_bf16_round", ld)

    def _grads(self, g):
        """(out_dot_g, dm, ds, dd) for the gathered output gradient g (float32, or BF16 rows g~ = bf16(grad_out)):
        out_dot_g[d, h] = <out[d,h], g[d,h]> = sum_e a[e,h] <x[slot(e),h], g[d,h]>, so the softmax backward needs no
        edge pass, and zeroed gradients, dm as wide as the gathered rows."""
        rows, s, d, _, _, out = self.saved
        H, F = int(s.shape[1]), int(out.shape[1])
        o = out.detach()
        # <out, g~>, not <out, g>: the BF16 passes rely on sum_e a <m~, g~> == <out, g~>; mixing g and g~ would bias
        # the score gradients by about 2^-8
        out_dot_g = (o * (g if g.dtype == torch.float32 else g[:, :F].float())).view(-1, H, F // H).sum(-1).contiguous()
        if rows.dtype == torch.float32:
            dm = torch.zeros_like(rows)
        else:
            dm = torch.zeros(rows.shape, dtype=torch.float32, device=g.device)
        return out_dot_g, dm, torch.zeros_like(s), torch.zeros_like(d)

    def backward_two_pass(self, g, slot_off, slot_dst):
        """No per-edge atomics: a destination-major and a source-major pass, each with register accumulators."""
        rows, s, d, seg_max, seg_sum, out = self.saved
        H, F = int(s.shape[1]), int(out.shape[1])
        if self.gather_dtype is None:
            gk, entry, widths = g, "nts_gat_fused_aggregate_backward_two_pass", (F,)
        else:
            gk = self._to_bf16_rows(g, rows.shape[1])
            entry, widths = "nts_gat_fused_aggregate_backward_two_pass_bf16", (F, int(rows.shape[1]))
        out_dot_g, dm, ds, dd = self._grads(gk)
        pack = torch.empty((self.n_dst, H, 4), dtype=torch.float32, device=g.device)
        with _timed("gat_bwd", F, 2 * self.n_edges, self.n_dst):
            _lib.call(entry, _ptr(dm), _ptr(ds), _ptr(dd), _ptr(pack), _ptr(rows), _ptr(s), _ptr(d), _ptr(seg_max),
                      _ptr(seg_sum), _ptr(out_dot_g), _ptr(gk), _ptr(self.slots), _ptr(self.column_offset), 0,
                      _ptr(slot_off), _ptr(slot_dst), self.n_dst, rows.shape[0], *widths, H, self.slope, _stream())
        if dm.shape[1] != F:
            dm = dm[:, :F].contiguous()
        return dm, ds, dd

    def backward_one_pass(self, g, row_indices, mirror_index):
        """The FP32 backward with per-edge atomics, on the CSC's row_indices and their mirror slots."""
        x, s, d, seg_max, seg_sum, out = self.saved
        out_dot_g, dm, ds, dd = self._grads(g)
        _lib.call("nts_gat_fused_aggregate_backward", _ptr(dm), _ptr(ds), _ptr(dd), _ptr(x), _ptr(s), _ptr(d),
                  _ptr(seg_max), _ptr(seg_sum), _ptr(out_dot_g), _ptr(g), _ptr(row_indices), _ptr(self.column_offset),
                  _ptr(mirror_index), self.n_dst, x.shape[1], int(s.shape[1]), self.slope, _stream())
        return dm, ds, dd


class DistGPUFusedGATOp(_EdgeOp):
    """K7: the whole attention + aggregation of one GAT layer in two kernels forward and two passes backward, never
    materialising an edge-sized tensor (toolkits/GAT_CPU_DIST_OPTM.hpp:196-241 keeps [E,1] logits / attention;
    toolkits/GAT_GPU_DIST.hpp:187-219 keeps four [E,F] messages).

        forward(mirror [M, H*D], src_score [M, H], dst_score [V, H]) -> out [V, H*D]
            a[e,h] = softmax over the in-edges of dst(e) of leaky_relu(src_score[slot(e),h] + dst_score[dst(e),h])
            out[d, hD:(h+1)D] = sum_e a[e,h] * mirror[slot(e), hD:(h+1)D]
        backward(grad_out) -> (d_mirror, d_src_score, d_dst_score)

    gather_dtype=torch.bfloat16: the aggregation and both backward passes gather BF16 rows with FP32 accumulation.  The
    forward rounds the FP32 mirror once into m~ = bf16(mirror), the backward rounds grad_out once into g~; the layer then
    computes the FP32 layer's function and gradients at m~ and g~ (include/nts_b200.h).  Scores, softmax statistics,
    out, d_mirror and the score gradients stay float32.  Needs two_pass_backward=True, and with heads > 1 a head width
    D that is a multiple of 8; other shapes raise NtsError.
    """

    def __init__(self, partitioned_graph, active=None, negative_slope=0.2, two_pass_backward=True, gather_dtype=None):
        super().__init__(partitioned_graph, active)
        self.slope = float(negative_slope)
        self.two_pass_backward = bool(two_pass_backward)
        self.gather_dtype = _check_gather_dtype(gather_dtype)
        if self.gather_dtype is not None and not self.two_pass_backward:
            raise _lib.NtsError("BF16 gathers of the fused GAT layer need two_pass_backward=True")
        self._k7 = None

    @staticmethod
    def slot_indices(pg):
        """row_indices with the MirrorIndex lookup already applied (mirror slot of every CSC edge), cached on the
        graph: the kernels then skip one dependent load per edge (the C ABI accepts mirror_index = NULL for this)."""
        cached = getattr(pg, "_slot_indices_gpu", None)
        if cached is None:
            cached = pg.mirror_index_gpu[pg.row_indices_gpu.long()].to(torch.int32).contiguous()
            pg._slot_indices_gpu = cached
        return cached

    @staticmethod
    def slot_csr(pg):
        """Out-edges of every mirror slot: (slot_row_offset [M+1], slot_column_indices [E], local destination ids) -
        the CSR twin of the whole-partition CSC, built once per PartitionedGraph on the device and cached on it."""
        cached = getattr(pg, "_slot_csr_gpu", None)
        if cached is not None:
            return cached
        col = pg.column_offset_gpu.long()
        V, M = pg.owned_vertices, pg.owned_mirrors
        slot = DistGPUFusedGATOp.slot_indices(pg).long()
        dst = torch.repeat_interleave(torch.arange(V, device=col.device), col[1:V + 1] - col[:V])
        order = torch.sort(slot, stable=True).indices
        csr_dst = dst[order].to(torch.int32).contiguous()
        off = torch.zeros(M + 1, dtype=torch.int64, device=col.device)
        off[1:] = torch.cumsum(torch.bincount(slot, minlength=M), 0)
        pg._slot_csr_gpu = (off.to(torch.int32).contiguous(), csr_dst)
        return pg._slot_csr_gpu

    def forward(self, mirror, src_score, dst_score):
        pg = self._topo()
        x = _check_input(mirror, "mirror")
        s = _check_input(src_score, "src_score")
        d = _check_input(dst_score, "dst_score")
        self._k7 = _FusedGAT(pg.column_offset_gpu, self.slot_indices(pg), pg.owned_vertices, x.shape[0],
                             pg.owned_edges, self.slope, self.gather_dtype)
        return self._k7.forward(x, s, d)

    @property
    def _saved(self):
        """(mirror or m~, src_score, dst_score, seg_max, seg_sum, out) of the last forward; None before the first."""
        return None if self._k7 is None else self._k7.saved

    def backward(self, f_output_grad):
        pg = self._topo()
        g = _check_input(f_output_grad, "output_grad")
        if self.two_pass_backward:
            return self._k7.backward_two_pass(g, *self.slot_csr(pg))
        return self._k7.backward_one_pass(g, pg.row_indices_gpu, pg.mirror_index_gpu)


# the refusal of nts_gat_fused_aggregate_forward_bf16 (check_gat_bf16_layout) for a head width D % 8 != 0
BF16_HEAD_WIDTH_ERROR = ("BF16 rows with heads > 1 need a head width D % 8 == 0 (a 16-byte chunk never straddles two "
                         "heads) and ld == feature_size")


def gat_bf16_shape_error(feature_size, heads):
    """Why the BF16 K7 entries refuse a layer of feature_size = heads * D columns (gathered as rows of
    ld = ceil(F/8)*8 BF16 values, as _FusedGAT does), or None when both accept it.  The entries give the verdict
    themselves: both check layout and shape before their batch_size == 0 return, so a call with batch 0 and null
    pointers does no device work.  Returns "<entry>: <its error message>"."""
    F, H = int(feature_size), int(heads)
    ld = (F + 7) // 8 * 8
    lib = _lib.load()
    # (pointers, then batch 0 and 0 edges / mirror rows, F, ld, H, slope, stream)
    for name, n_ptrs in (("nts_gat_fused_aggregate_forward_bf16", 9),
                         ("nts_gat_fused_aggregate_backward_two_pass_bf16", 16)):
        if getattr(lib, name)(*([None] * n_ptrs), 0, 0, F, ld, H, 0.2, None) != 0:
            return "%s: %s" % (name, _lib.last_error())
    return None


class MiniBatchGATOp(ntsGraphOp):
    """K7 on one block of a sample whose sources include its destinations (sample.NeighborSampler(...,
    include_dst=True)): the GAT layer of DistGPUFusedGATOp with the block as topology.  Edge e of local destination d
    reads source row row_indices[e] (local ids: the block's slots, no mirror lookup); the two-pass backward walks the
    transposed block (row_offset, column_indices), whose edges of a source are in edge order.

        forward(x_trans [n_src, H*D], src_score [n_src, H], dst_score [n_dst, H]) -> out [n_dst, H*D]
        backward(grad_out [n_dst, H*D]) -> (d_x_trans, d_src_score, d_dst_score)

    The caller forms dst_score from the destinations' own rows, x_trans[block.dst_pos]; a block without dst_pos is
    refused.  A destination without kept edges gets a zero output row and zero gradients.  gather_dtype=torch.bfloat16
    gathers BF16 rows with FP32 accumulation exactly as DistGPUFusedGATOp does, with the same shape limits."""

    def __init__(self, sampled_subgraph, hop, negative_slope=0.2, gather_dtype=None):
        super().__init__(sampled_subgraph, None)
        self.hop = int(hop)
        self.block = sampled_subgraph.blocks[self.hop]
        if self.block.dst_pos is None:
            raise _lib.NtsError("MiniBatchGATOp needs a block whose sources include its destinations (dst_pos): "
                                "sample with NeighborSampler(..., include_dst=True)")
        self.slope = float(negative_slope)
        self.gather_dtype = _check_gather_dtype(gather_dtype)
        self._k7 = None

    def forward(self, x_trans, src_score, dst_score):
        b = self.block
        x = _check_input(x_trans, "x_trans")
        s = _check_input(src_score, "src_score")
        d = _check_input(dst_score, "dst_score")
        if x.shape[0] != b.n_src or s.shape[0] != b.n_src:
            raise _lib.NtsError("x_trans and src_score need %d rows (hop %d sources), got %d and %d"
                                % (b.n_src, self.hop, x.shape[0], s.shape[0]))
        if d.shape[0] != b.n_dst:
            raise _lib.NtsError("dst_score needs %d rows (hop %d destinations), got %d"
                                % (b.n_dst, self.hop, d.shape[0]))
        H, F = int(s.shape[1]), int(x.shape[1])
        if d.shape[1] != H or H < 1 or F % H != 0:
            raise _lib.NtsError("scores need the same head count, and x_trans a width that is a multiple of it")
        if b.n_edges == 0:
            # no edge anywhere in the block: every output row is an empty sum, and no K7 entry runs.  A BF16 shape
            # that the entries refuse (nts_gat_fused_aggregate_forward_bf16) is refused here with their words
            if self.gather_dtype is not None and H > 1 and (F // H) % 8 != 0:
                raise _lib.NtsError(BF16_HEAD_WIDTH_ERROR)
            self._shapes = (x, s, d)
            return torch.zeros((b.n_dst, F), dtype=torch.float32, device=x.device)
        self._k7 = _FusedGAT(b.column_offset, b.row_indices, b.n_dst, b.n_src, b.n_edges, self.slope,
                             self.gather_dtype)
        return self._k7.forward(x, s, d)

    def backward(self, f_output_grad):
        b = self.block
        g = _check_input(f_output_grad, "output_grad")
        if g.shape[0] != b.n_dst:
            raise _lib.NtsError("output_grad has %d rows, hop %d has %d destinations" % (g.shape[0], self.hop, b.n_dst))
        if self._k7 is None:
            x, s, d = self._shapes
            return torch.zeros_like(x), torch.zeros_like(s), torch.zeros_like(d)
        return self._k7.backward_two_pass(g, b.row_offset, b.column_indices)
