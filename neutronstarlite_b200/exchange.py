"""Device-resident partition-boundary exchange: the replacement for the reference's host-staged MPI ring
(`Graph::sync_compute_decoupled` / `compute_sync_decoupled`, core/graph.hpp:3455-3719, and `NtsGraphCommunicator`,
comm/network.cpp:159-844).

What moves, and when (rank p of P, partition i -> chunk i = edges src in part i -> dst in part p):

  forward   Y_p = sum_i A_{p<-i} X_i.  Rank p needs, from every other rank i, only the rows of X_i that are sources
            of chunk i (`source_active`, core/PartitionedGraph.hpp:397) - M_{p<-i} dense rows, no (vid,row) records.
            They land in a staging buffer indexed by a compact slot; chunk i's CSC indices are remapped to slots
            once at setup, so the aggregation kernel consumes the received rows with no unpack pass.  The local
            chunk (i == p) aggregates while the rows are in flight; remote chunks follow in the reference's ring
            order (p+1, p+2, ... mod P; core/graph.hpp:3678-3683).
  backward  dX_p = sum_j A_{j<-p}^T dY_j.  Rank p computes, per chunk i, the partial gradients of the ACTIVE sources
            only (CSR compacted to active rows -> [M_{p<-i}, F], written straight into the send staging), ships them
            to i, and adds what it receives for its own rows with one unique-row scatter-add per peer
            (replaces aggregate_data_buffer_debug's per-element atomics, cuda/ntsCUDATransferKernel.cuh:49-68).

Transports:
  "nccl"  one all-to-all(v) of the packed rows (torch.distributed / NCCL over NVLink) on a side stream, then ONE
          launch over the merged CSC of all remote chunks - the baseline.
  "p2p"   the peer-memory engine (csrc/nts_exchange.cu), no packing and no NCCL on the data path: the OWNER of a row
          stores it straight into the reader's CUDA-IPC receive window over NVLink (one persistent push kernel per
          call, ring order), raises an epoch flag (`st.release.sys`), and the reader aggregates chunk (p+s) as soon
          as the rows of partition (p+s) have landed - the reference's per-chunk pipeline (core/graph.hpp:3678-3719)
          with the host staging removed.  Backward: per-chunk partials pushed to the owner while the next chunk
          computes.  Big chunks run through nts_gather_plan (slab count measured per width).

gather_dtype=torch.bfloat16 (both transports): the gathered operand is rounded to BF16 once per call by its owner,
forward rows travel as BF16 (half the bytes), every chunk gathers through a plan tuned per (width, type) and
accumulates in FP32; backward partial gradients stay FP32.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from . import ops


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class ExchangePlan:
    """Setup-time index structures (per PartitionedGraph).  Backend-agnostic: built with torch ops on whatever
    device the chunk arrays live on and torch.distributed collectives (works with gloo on CPU tensors)."""

    def __init__(self, pg, group=None, merged=True):
        """merged = also build the one-launch CSC / compact CSR over ALL remote chunks (what the NCCL transport
        aggregates from); the peer-memory engine works per chunk and skips it."""
        self.pg = pg
        self.P = pg.partitions
        self.p = pg.partition_id
        self.group = group
        P, p = self.P, self.p
        chunks = pg.graph_chunks
        dev = chunks[0].column_offset_gpu.device if chunks[0].column_offset_gpu is not None else torch.device("cpu")
        self.device = dev
        self.need = [None] * P            # need[i]: int32 local ids (within partition i) of the rows of X_i I read
        self.csc_slots = [None] * P       # chunk i's row_indices remapped to staging slots (int32 [E_i])
        self.csr_offsets_compact = [None] * P  # chunk i's row_offset restricted to active rows (int32 [M_i+1])
        for i in range(P):
            c = chunks[i]
            ro = self._arr(c, "row_offset").to(torch.int64)
            deg = ro[1:] - ro[:-1]
            active = torch.nonzero(deg > 0).view(-1)
            self.need[i] = active.to(torch.int32)
            if i != p:
                slot_of = torch.zeros(c.batch_size_backward, dtype=torch.int32, device=dev)
                slot_of[active] = torch.arange(active.numel(), dtype=torch.int32, device=dev)
                ri = self._arr(c, "row_indices").to(torch.int64) - c.src_range[0]
                self.csc_slots[i] = slot_of[ri] if ri.numel() else torch.zeros(0, dtype=torch.int32, device=dev)
                self.csr_offsets_compact[i] = torch.cat([ro[active], ro[-1:]]).to(torch.int32)
        self.need_count = [int(n.numel()) for n in self.need]
        # tell every peer which of its rows I need (forward) == which rows it will get gradients for (backward)
        self.send_rows = [None] * P
        counts_in = torch.tensor([self.need_count[i] if i != p else 0 for i in range(P)], dtype=torch.int64)
        counts_out = torch.zeros(P, dtype=torch.int64)
        if P > 1:
            cdev = dev if dist.get_backend(group) == "nccl" else torch.device("cpu")
            ci, co = counts_in.to(cdev), counts_out.to(cdev)
            dist.all_to_all_single(co, ci, group=group)
            counts_out = co.cpu()
            send = torch.cat([self.need[i] if i != p else self.need[i][:0] for i in range(P)]).to(cdev)
            recv = torch.zeros(int(counts_out.sum()), dtype=torch.int32, device=cdev)
            dist.all_to_all_single(recv, send, output_split_sizes=counts_out.tolist(),
                                   input_split_sizes=counts_in.tolist(), group=group)
            pos = 0
            for j in range(P):
                n = int(counts_out[j])
                self.send_rows[j] = recv[pos:pos + n].to(dev)
                pos += n
        self.send_count = [0 if r is None else int(r.numel()) for r in self.send_rows]
        if P == 1:
            self.send_rows = [None]
        self.recv_total = sum(self.need_count[i] for i in range(P) if i != p)
        self.send_total = sum(self.send_count[j] for j in range(P) if j != p)
        rows = [self.send_rows[j] for j in range(P) if j != p and self.send_rows[j] is not None]
        self.send_rows_all = torch.cat(rows).contiguous() if rows else torch.zeros(0, dtype=torch.int32, device=dev)
        self.remote_edges = sum(int(chunks[i].edge_size) for i in range(P) if i != p)
        self.remote_col_offset = self.remote_slots = self.remote_w = None
        self.bwd_offsets = self.bwd_indices = self.bwd_w = None
        self.recv_offs = np.concatenate([[0], np.cumsum([self.need_count[i] if i != p else 0 for i in range(P)])])
        if merged:
            self._merge_remote()

    def _merge_remote(self):
        """One CSC over ALL remote chunks (sources = slots of the single receive staging buffer) and one compact CSR
        over all remote chunks (rows = the send staging layout): the remote part of an aggregation is then ONE kernel
        launch instead of P-1 (at 8 GPUs the per-chunk kernels are ~0.1-0.3 ms, i.e. launch-bound)."""
        P, p, dev = self.P, self.p, self.device
        chunks = self.pg.graph_chunks
        self.recv_offs = np.concatenate([[0], np.cumsum([self.need_count[i] if i != p else 0 for i in range(P)])])
        self.remote_edges = 0
        self.remote_col_offset = self.remote_slots = self.remote_w = None
        self.bwd_offsets = self.bwd_indices = self.bwd_w = None
        self.send_rows_all = None
        if P == 1:
            return
        Vp = self.pg.owned_vertices
        dsts, slots, ws, b_off, b_idx, b_w = [], [], [], [], [], []
        edge_base = 0
        for i in range(P):
            if i == p:
                continue
            c = chunks[i]
            if c.edge_size:
                co = self._arr(c, "column_offset").to(torch.int64)
                dsts.append(torch.repeat_interleave(torch.arange(Vp, device=dev), co[1:] - co[:-1]))
                slots.append(self.csc_slots[i].to(torch.int64) + int(self.recv_offs[i]))
                ws.append(self._farr(c, "edge_weight_forward"))
                b_idx.append(self._arr(c, "column_indices"))
                b_w.append(self._farr(c, "edge_weight_backward"))
            b_off.append(self.csr_offsets_compact[i][:-1].to(torch.int64) + edge_base)
            edge_base += c.edge_size
        self.remote_edges = edge_base
        if edge_base:
            dst = torch.cat(dsts)
            order = torch.argsort(dst, stable=True)
            self.remote_slots = torch.cat(slots)[order].to(torch.int32)
            self.remote_w = torch.cat(ws)[order].contiguous()
            col = torch.zeros(Vp + 1, dtype=torch.int64, device=dev)
            col[1:] = torch.cumsum(torch.bincount(dst, minlength=Vp), 0)
            self.remote_col_offset = col.to(torch.int32)
            self.bwd_indices = torch.cat(b_idx).contiguous()
            self.bwd_w = torch.cat(b_w).contiguous()
        self.bwd_offsets = torch.cat(b_off + [torch.tensor([edge_base], dtype=torch.int64, device=dev)]).to(torch.int32)
        rows = [self.send_rows[j] for j in range(P) if j != p and self.send_rows[j] is not None]
        self.send_rows_all = torch.cat(rows).contiguous() if rows else torch.zeros(0, dtype=torch.int32, device=dev)

    @staticmethod
    def _farr(c, name):
        g = getattr(c, name + "_gpu")
        if g is not None:
            return g
        return torch.from_numpy(getattr(c, name))

    @staticmethod
    def _arr(c, name):
        g = getattr(c, name + "_gpu")
        if g is not None:
            return g
        return torch.from_numpy(getattr(c, name).view(np.int32))

    def push_offsets(self):
        """(fwd_push_offset[P], bwd_push_offset[P]) of nts_exchange_desc: where MY rows start inside rank j's receive
        staging (rows it reads from the partitions before mine) and where MY partial gradients start inside rank i's
        gradient staging (rows the ranks before me return to i).  Needs every rank's need counts."""
        P, p = self.P, self.p
        if P == 1:
            return [0], [0]
        mine = [self.need_count[i] if i != p else 0 for i in range(P)]
        allc = [None] * P
        dist.all_gather_object(allc, mine, group=self.group)
        fwd = [int(sum(allc[j][i] for i in range(p) if i != j)) if j != p else 0 for j in range(P)]
        bwd = [int(sum(allc[j][i] for j in range(p) if j != i)) if i != p else 0 for i in range(P)]
        return fwd, bwd

    def ring(self):
        """Remote chunks in the reference's processing order: (p+1), (p+2), ... mod P."""
        return [(self.p + s) % self.P for s in range(1, self.P)]


class GpuExchange:
    """Forward / backward drivers of the distributed fused aggregation on one GPU per rank."""

    def __init__(self, pg, transport="nccl", group=None, n_buffers=None):
        if not torch.cuda.is_available():
            raise _lib.NtsError("GpuExchange needs a CUDA device (libnts_b200 has no CPU fallback)")
        self.pg = pg
        self.P, self.p = pg.partitions, pg.partition_id
        self.group = group
        self.plan = ExchangePlan(pg, group, merged=(transport != "p2p"))
        self.transport = transport
        self.device = self.plan.device
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._staging = {}
        self._p2p = None
        if transport == "p2p" and self.P > 1:
            import os
            nb = n_buffers if n_buffers else int(os.environ.get("NTS_EXCHANGE_BUFFERS", "2"))
            self._p2p = _PeerWindows(self, n_buffers=nb)
        elif transport not in ("nccl", "p2p"):
            raise ValueError("transport must be 'nccl' or 'p2p'")

    def close(self):
        """Release the engine (its IPC mappings of the peers' windows) - collective in effect: call it on every rank
        before the process group goes away."""
        if self._p2p is not None:
            self._p2p.close()
            self._p2p = None

    # ---- buffers ---------------------------------------------------------------------------------------------
    def _buf(self, key, rows, F, dtype=torch.float32):
        t = self._staging.get((key, F))
        if t is None or t.shape[0] < rows:
            t = torch.empty((max(rows, 1), F), dtype=dtype, device=self.device)
            self._staging[(key, F)] = t
        return t[:rows]

    # ---- forward -----------------------------------------------------------------------------------------------
    def _merged_plan(self, direction, F):
        """BF16 gathers on the NCCL transport: the merged remote CSC (forward) / compact CSR (backward) as one
        nts_gather_plan tuned for BF16 rows of width F (BF16 gathers exist only in plans), built once per width."""
        plans = self.__dict__.setdefault("_bf16_merged", {})
        pl = plans.get((direction, F))
        if pl is None:
            plan, Vp = self.plan, self.pg.owned_vertices
            if direction == "fwd":
                pl = ops.GatherPlan(plan.remote_col_offset, plan.remote_slots, plan.remote_w, 0, Vp,
                                    plan.remote_edges, plan.recv_total, 0, tune_for=F, gather_dtype=torch.bfloat16)
            else:
                pl = ops.GatherPlan(plan.bwd_offsets, plan.bwd_indices, plan.bwd_w,
                                    self.pg.graph_chunks[self.p].dst_range[0], plan.recv_total, plan.remote_edges,
                                    Vp, 0, tune_for=F, gather_dtype=torch.bfloat16)
            plans[(direction, F)] = pl
        return pl

    def forward(self, x, gather_dtype=None):
        """gather_dtype=torch.bfloat16: BF16 gathers with FP32 accumulation (ops.GatherPlan.run's contract); x may be
        float32 or bfloat16, the rows travel as BF16 on both transports."""
        pg, plan = self.pg, self.plan
        bf16 = ops._check_gather_dtype(gather_dtype) is not None
        F = x.shape[1]
        y = torch.zeros((pg.owned_vertices, F), dtype=torch.float32, device=x.device)
        if self.P == 1:
            return ops.gather_by_dst_from_src(pg.graph_chunks[0], y, x, gather_dtype=gather_dtype)
        if self._p2p is not None:
            return self._forward_p2p(x, y, bf16)
        if bf16:
            return self._forward_nccl_bf16(x, y)
        # pack the rows every peer needs (one launch over the concatenated row list), exchange on the side stream
        send = self._buf("fsend", plan.send_total, F)
        recv = self._buf("frecv", plan.recv_total, F)
        if plan.send_total:
            _lib.call("nts_gather_rows", _ptr(send), _ptr(x), _ptr(plan.send_rows_all), plan.send_total, F,
                      _lib.stream())
        self._all_to_all(recv, send, True, lambda: ops.gather_by_dst_from_src(pg.graph_chunks[self.p], y, x))
        self._aggregate_remote(y, recv)
        return y

    def _all_to_all(self, recv, send, forward, local):
        """One all_to_all_single of the packed rows with every peer on the side stream, while local() (the local
        chunk's aggregation) runs on the current stream; the current stream then waits for recv.  forward: send
        holds the rows each peer needs of this rank and recv the rows this rank needs; backward the other way round,
        with partial gradients."""
        plan, P, p = self.plan, self.P, self.p
        cur = torch.cuda.current_stream()
        self.comm_stream.wait_stream(cur)
        with torch.cuda.stream(self.comm_stream):
            sends = [plan.send_count[j] if j != p else 0 for j in range(P)]
            needs = [plan.need_count[i] if i != p else 0 for i in range(P)]
            dist.all_to_all_single(recv, send, output_split_sizes=needs if forward else sends,
                                   input_split_sizes=sends if forward else needs, group=self.group)
        local()
        cur.wait_stream(self.comm_stream)
        recv.record_stream(cur)

    def _forward_nccl_bf16(self, x, y):
        """x converted to BF16 once; the packed rows travel as BF16 (half the bytes); the local chunk and the merged
        remote chunks gather BF16 rows."""
        pg, plan = self.pg, self.plan
        F = x.shape[1]
        xb = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
        send = self._buf("fsend16", plan.send_total, F, torch.bfloat16)
        recv = self._buf("frecv16", plan.recv_total, F, torch.bfloat16)
        if plan.send_total:
            torch.index_select(xb, 0, plan.send_rows_all, out=send)
        self._all_to_all(recv, send, True, lambda: ops.gather_by_dst_from_src(pg.graph_chunks[self.p], y, xb,
                                                                              gather_dtype=torch.bfloat16))
        if plan.remote_edges:
            self._merged_plan("fwd", F).run(recv, y, torch.bfloat16)
        return y

    def _backward_nccl_bf16(self, g, dx):
        """dY converted to BF16 once locally; partial gradients are computed, sent and added in FP32."""
        pg, plan = self.pg, self.plan
        F = g.shape[1]
        gb = g.to(torch.bfloat16)
        send = self._buf("bsend", plan.recv_total, F)
        recv = self._buf("brecv", plan.send_total, F)
        send.zero_()
        if plan.remote_edges:
            self._merged_plan("bwd", F).run(gb, send, torch.bfloat16)
        self._all_to_all(recv, send, False, lambda: ops.gather_by_src_from_dst(pg.graph_chunks[self.p], dx, gb,
                                                                               gather_dtype=torch.bfloat16))
        if plan.send_total:
            _lib.call("nts_scatter_add_rows_atomic", _ptr(dx), _ptr(recv), _ptr(plan.send_rows_all), plan.send_total, F,
                      _lib.stream())
        return dx

    def _aggregate_remote(self, y, staged):
        """All remote chunks in one launch: merged CSC whose indices are slots of the receive staging buffer."""
        plan = self.plan
        if not plan.remote_edges:
            return
        with ops._timed("fwd", staged.shape[1], plan.remote_edges, self.pg.owned_vertices):
            _lib.call("nts_segment_gather_sum", _ptr(staged), _ptr(y), _ptr(plan.remote_w), _ptr(plan.remote_slots),
                      _ptr(plan.remote_col_offset), 0, self.pg.owned_vertices, plan.remote_edges, staged.shape[1],
                      _lib.stream())

    def _partial_remote(self, out_rows, g):
        """Partial gradients of the active sources of ALL remote chunks in one launch (merged compact CSR); the
        output rows are laid out exactly like the send staging buffer."""
        plan = self.plan
        if not plan.remote_edges:
            return
        with ops._timed("bwd", g.shape[1], plan.remote_edges, out_rows.shape[0]):
            _lib.call("nts_segment_gather_sum", _ptr(g), _ptr(out_rows), _ptr(plan.bwd_w), _ptr(plan.bwd_indices),
                      _ptr(plan.bwd_offsets), self.pg.graph_chunks[self.p].dst_range[0], out_rows.shape[0],
                      plan.remote_edges, g.shape[1], _lib.stream())

    # ---- mirror fetch / return (DistGPUGetDepNbrOp, core/ntsDistGPUGraphOp.hpp:48-143) ----------------------------
    def fetch_mirrors(self, x):
        """mirror[MirrorIndex[s], :] = X[s, :] for every source s of a local in-edge, [owned_mirrors, F].
        MirrorIndex numbers active sources in global-id order = partition order, so the mirror matrix is the
        concatenation over partitions i of the needed rows of partition i: exactly the output layout of one
        all-to-all(v) whose self segment carries this rank's own active rows.  (The reference moves the whole
        feature matrix to the host, through MPI and back, core/ntsDistGPUGraphOp.hpp:56-98.)"""
        plan, P, p = self.plan, self.P, self.p
        F = x.shape[1]
        st = _lib.stream()
        M = sum(plan.need_count)
        mirror = torch.zeros((M, F), dtype=torch.float32, device=x.device)
        if self._p2p is not None:   # the peer-memory engine: rows pushed into the receive windows, no NCCL
            self._p2p.reserve(F)
            _lib.call("nts_exchange_fetch_mirrors", self._p2p.handle, _ptr(x), _ptr(mirror), F, st)
            return mirror
        if P == 1:
            if M:
                _lib.call("nts_gather_rows", _ptr(mirror), _ptr(x), _ptr(plan.need[0]), M, F, st)
            return mirror
        rows_out = [plan.send_rows[j] if j != p else plan.need[p] for j in range(P)]
        n_out = [int(r.numel()) for r in rows_out]
        send = self._buf("msend", sum(n_out), F)
        pos = 0
        for j in range(P):
            if n_out[j]:
                _lib.call("nts_gather_rows", _ptr(send[pos:pos + n_out[j]]), _ptr(x), _ptr(rows_out[j]), n_out[j], F,
                          st)
            pos += n_out[j]
        dist.all_to_all_single(mirror, send, output_split_sizes=list(plan.need_count), input_split_sizes=n_out,
                               group=self.group)
        return mirror

    def return_mirror_grads(self, gm):
        """DistGPUGetDepNbrOp::backward: every mirror gradient goes back to the owner of the source vertex, who sums
        what arrives from all partitions (one unique-row scatter-add per sender)."""
        pg, plan, P, p = self.pg, self.plan, self.P, self.p
        F = gm.shape[1]
        st = _lib.stream()
        dx = torch.zeros((pg.owned_vertices, F), dtype=torch.float32, device=gm.device)
        if self._p2p is not None:
            self._p2p.reserve(F)
            _lib.call("nts_exchange_return_mirror_grads", self._p2p.handle, _ptr(gm.contiguous()), _ptr(dx), F, st)
            return dx
        if P == 1:
            if gm.shape[0]:
                _lib.call("nts_scatter_add_rows", _ptr(dx), _ptr(gm), _ptr(plan.need[0]), gm.shape[0], F, st)
            return dx
        rows_in = [plan.send_rows[j] if j != p else plan.need[p] for j in range(P)]
        n_in = [int(r.numel()) for r in rows_in]
        recv = self._buf("mrecv", sum(n_in), F)
        dist.all_to_all_single(recv, gm.contiguous(), output_split_sizes=n_in,
                               input_split_sizes=list(plan.need_count), group=self.group)
        pos = 0
        for j in range(P):
            if n_in[j]:
                _lib.call("nts_scatter_add_rows", _ptr(dx), _ptr(recv[pos:pos + n_in[j]]), _ptr(rows_in[j]), n_in[j],
                          F, st)
            pos += n_in[j]
        return dx

    # ---- backward ----------------------------------------------------------------------------------------------
    def backward(self, g, gather_dtype=None):
        pg, plan = self.pg, self.plan
        bf16 = ops._check_gather_dtype(gather_dtype) is not None
        F = g.shape[1]
        dx = torch.zeros((pg.owned_vertices, F), dtype=torch.float32, device=g.device)
        if self.P == 1:
            return ops.gather_by_src_from_dst(pg.graph_chunks[0], dx, g, gather_dtype=gather_dtype)
        if self._p2p is not None:
            return self._backward_p2p(g, dx, bf16)
        if bf16:
            return self._backward_nccl_bf16(g, dx)
        # partial gradients of the active sources of every remote chunk, written straight into the send staging
        send = self._buf("bsend", plan.recv_total, F)
        recv = self._buf("brecv", plan.send_total, F)
        send.zero_()
        self._partial_remote(send, g)
        self._all_to_all(recv, send, False, lambda: ops.gather_by_src_from_dst(pg.graph_chunks[self.p], dx, g))
        if plan.send_total:  # rows repeat across senders -> vector atomics, one launch
            _lib.call("nts_scatter_add_rows_atomic", _ptr(dx), _ptr(recv), _ptr(plan.send_rows_all), plan.send_total, F,
                      _lib.stream())
        return dx

    # ---- peer-memory transport: the C++ engine (csrc/nts_exchange.cu) --------------------------------------------------
    def _forward_p2p(self, x, y, bf16=False):
        self._p2p.reserve(x.shape[1], bf16)
        with ops._timed("fwd", x.shape[1], self.pg.owned_edges, self.pg.owned_vertices):
            if bf16:
                _lib.call("nts_exchange_forward_bf16", self._p2p.handle, _ptr(x), ops._DTYPE_CODE[x.dtype], _ptr(y),
                          x.shape[1], _lib.stream())
            else:
                _lib.call("nts_exchange_forward", self._p2p.handle, _ptr(x), _ptr(y), x.shape[1], _lib.stream())
        return y

    def _backward_p2p(self, g, dx, bf16=False):
        self._p2p.reserve(g.shape[1], bf16)
        with ops._timed("bwd", g.shape[1], self.pg.owned_edges, self.pg.owned_vertices):
            _lib.call("nts_exchange_backward_bf16" if bf16 else "nts_exchange_backward", self._p2p.handle, _ptr(g),
                      _ptr(dx), g.shape[1], _lib.stream())
        return dx


class _PeerWindows:
    """Control plane of the peer-memory transport: hands the plan arrays to the C++ engine and moves the IPC handles
    between ranks with torch.distributed; the data plane (windows, flags, streams, launch sequence) is
    `nts_exchange_*` in csrc/nts_exchange.cu."""

    def __init__(self, ex, n_buffers=2):
        import ctypes as C
        self.ex = ex
        P, p = ex.P, ex.p
        pg, plan = ex.pg, ex.plan
        L = _lib.load()
        self.n_buffers = int(n_buffers)
        fwd_off, bwd_off = plan.push_offsets()
        c = pg.graph_chunks[p]
        u32 = C.c_uint32 * P
        chunks = (_lib.ExchangeChunk * P)()
        for i in range(P):
            if i == p:
                continue
            ci = pg.graph_chunks[i]
            h = chunks[i]
            h.column_offset, h.slots = _ptr(ci.column_offset_gpu), _ptr(plan.csc_slots[i])
            h.weight_forward, h.weight_backward = _ptr(ci.edge_weight_forward_gpu), _ptr(ci.edge_weight_backward_gpu)
            h.row_offset_compact, h.column_indices = _ptr(plan.csr_offsets_compact[i]), _ptr(ci.column_indices_gpu)
            h.edges = int(ci.edge_size)
        self._keep = {
            "need_count": u32(*[plan.need_count[i] if i != p else 0 for i in range(P)]),
            "send_count": u32(*[plan.send_count[j] if j != p else 0 for j in range(P)]),
            "fwd_off": u32(*fwd_off), "bwd_off": u32(*bwd_off), "chunks": chunks,
        }
        d = _lib.ExchangeDesc()
        d.partitions, d.rank = P, p
        d.owned_vertices, d.dst_start = pg.owned_vertices, c.dst_range[0]
        d.local_column_offset, d.local_row_indices = _ptr(c.column_offset_gpu), _ptr(c.row_indices_gpu)
        d.local_row_offset, d.local_column_indices = _ptr(c.row_offset_gpu), _ptr(c.column_indices_gpu)
        d.local_weight_forward, d.local_weight_backward = _ptr(c.edge_weight_forward_gpu), _ptr(c.edge_weight_backward_gpu)
        d.local_edges = c.edge_size
        d.chunks = chunks
        d.need_count = self._keep["need_count"]
        d.send_count = self._keep["send_count"]
        d.send_rows_all = _ptr(plan.send_rows_all)
        d.fwd_push_offset = self._keep["fwd_off"]
        d.bwd_push_offset = self._keep["bwd_off"]
        d.local_need, d.local_need_count = _ptr(plan.need[p]), plan.need_count[p]
        self.handle = _lib.checked(L.nts_exchange_create(C.byref(d)), "nts_exchange_create")

    def _cpu_collective(self):
        return dist.get_backend(self.ex.group) != "nccl"

    def reserve(self, F, bf16=False):
        """Make the exported receive window large enough for feature width F (BF16 calls: padded BF16 rows forward,
        nts_exchange_required_floats_bf16) on EVERY rank.  Collective whenever a rank needs more than it has (all
        ranks always hold the same capacity: it is the max over ranks):
        release peers -> barrier -> reallocate -> all-gather of the IPC handles -> open -> barrier
        (the contract of nts_exchange_reserve, include/nts_b200.h)."""
        import ctypes as C
        L = _lib.load()
        ex = self.ex
        required = L.nts_exchange_required_floats_bf16 if bf16 else L.nts_exchange_required_floats
        seen = "_max_F16" if bf16 else "_max_F"       # every rank makes the same sequence of calls
        if required(self.handle, F) <= L.nts_exchange_capacity_floats(self.handle) and F <= getattr(self, seen, 0):
            return
        cdev = torch.device("cpu") if self._cpu_collective() else ex.device
        need = torch.tensor([required(self.handle, F)], dtype=torch.int64, device=cdev)
        dist.all_reduce(need, op=dist.ReduceOp.MAX, group=ex.group)
        setattr(self, seen, max(F, getattr(self, seen, 0)))
        if int(need.item()) <= L.nts_exchange_capacity_floats(self.handle):
            return
        _lib.call("nts_exchange_release_peers", self.handle)
        dist.barrier(group=ex.group)
        _lib.call("nts_exchange_reserve", self.handle, int(need.item()), self.n_buffers)
        wh, fh = C.create_string_buffer(64), C.create_string_buffer(64)
        _lib.call("nts_exchange_handles", self.handle, wh, fh)
        handles = [None] * ex.P
        dist.all_gather_object(handles, (bytes(wh.raw), bytes(fh.raw)), group=ex.group)
        _lib.call("nts_exchange_open_peers", self.handle, b"".join(h[0] for h in handles),
                  b"".join(h[1] for h in handles))
        dist.barrier(group=ex.group)

    def close(self):
        if getattr(self, "handle", None):
            _lib.load().nts_exchange_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def default_exchange(pg):
    """One exchange object per PartitionedGraph (created lazily by ForwardGPUfuseOp), kept ON the graph object so
    that it dies with it (an id()-keyed cache would hand a recycled id a stale plan)."""
    ex = pg.__dict__.get("_default_exchange")
    if ex is None:
        ex = GpuExchange(pg, transport="nccl")
        pg.__dict__["_default_exchange"] = ex
    return ex
