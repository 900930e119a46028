"""Host mirror of the reference's graph layout for the aggregation path.

  * `CSCSegment`       <-> `CSC_segment_pinned` (core/GraphSegment.h:52-139): one chunk "sources of partition i ->
                           destinations of this rank" as CSC + CSR with per-edge weights, host arrays plus the
                           `*_gpu` device copies made by `CopyGraphToDevice` (core/GraphSegment.cpp:178-220).
  * `PartitionedGraph` <-> `PartitionedGraph` (core/PartitionedGraph.hpp:60-143,295-420): the P chunks of a rank,
                           `MirrorIndex` / `owned_mirrors`, and the whole-partition CSC used by the edge operators.

All arrays are built by the C++ host routines of libnts_b200 (`nts_host_*`, nts_graph_host.cpp, through
`generate_all`) or on the GPU by `nts_graph_build` (nts_graph_build.cu), from a packed binary edge file
(`PartitionedGraph.from_edge_file`) or from edge tensors already on the device (`from_device_edges`); both produce
identical arrays (tests/test_graph_host.py, tests/test_graph_build_device.py).  The device builders fill only the
`*_gpu` arrays; the host arrays stay None.
"""
from __future__ import annotations

import os

import numpy as np

from . import _lib


def _ptr(a):
    return a.ctypes.data if a is not None else None


PAGESIZE = 1 << 10  # dep/gemini/constants.hpp


def partition_offsets_from_out_degree(out_degree_raw, n_edges, partitions):
    """The reference's vertex-chunk partitioner (core/graph.hpp:1185-1211) from the RAW (un-clamped) out-degree
    array: greedy prefix over out_degree + alpha, alpha = 12*(P+1); cut rounded down to PAGESIZE.  Pure host
    arithmetic on V integers (numpy); same result as nts_host_partition_offsets."""
    deg = np.asarray(out_degree_raw, dtype=np.int64)
    V = int(deg.shape[0])
    P = int(partitions)
    alpha = 12 * (P + 1)
    prefix = np.concatenate([[0], np.cumsum(deg + alpha)])
    off = np.zeros(P + 1, dtype=np.uint32)
    remained = int(n_edges) + V * alpha
    for i in range(P):
        left = P - i
        start = int(off[i])
        if left == 1:
            off[i + 1] = V
        else:
            expected = remained // left
            v_i = int(np.searchsorted(prefix[1:], prefix[start] + expected, side="right"))
            v_i = max(min(v_i, V - 1), start)
            off[i + 1] = (v_i // PAGESIZE) * PAGESIZE
        remained -= int(prefix[int(off[i + 1])] - prefix[start])
    return off


class HostGraph:
    """A packed binary edge list ({u32 src, u32 dst}, dep/gemini/type.hpp:100-106) plus the global
    artefacts every rank derives from it: clamped degrees and the partition offsets."""

    def __init__(self, edges, vertices):
        edges = np.ascontiguousarray(edges, dtype=np.uint32).reshape(-1, 2)
        self.edges = edges
        self.vertices = int(vertices)
        self.n_edges = int(edges.shape[0])
        self._deg = None

    @staticmethod
    def from_file(path, vertices):
        return HostGraph(np.fromfile(path, dtype=np.uint32).reshape(-1, 2), vertices)

    def degrees(self):
        """(out_degree_for_backward, in_degree_for_backward): with multiplicity, clamped to >= 1."""
        if self._deg is None:
            out_d = np.empty(self.vertices, dtype=np.uint32)
            in_d = np.empty(self.vertices, dtype=np.uint32)
            _lib.call("nts_host_degrees", _ptr(self.edges), self.n_edges, self.vertices, _ptr(out_d), _ptr(in_d))
            self._deg = (out_d, in_d)
        return self._deg

    def partition_offsets(self, partitions):
        po = np.empty(partitions + 1, dtype=np.uint32)
        _lib.call("nts_host_partition_offsets", _ptr(self.edges), self.n_edges, self.vertices, int(partitions), _ptr(po))
        return po


class CSCSegment:
    """Mirror of CSC_segment_pinned: field names follow core/GraphSegment.h:52-101."""

    def __init__(self):
        self.column_offset = None          # u32 [Vp+1], by local destination
        self.row_indices = None            # u32 [E], GLOBAL source id, ascending inside a destination
        self.edge_weight_forward = None    # f32 [E]
        self.row_offset = None             # u32 [Vi+1], by source local to partition i
        self.column_indices = None         # u32 [E], GLOBAL destination id
        self.edge_weight_backward = None   # f32 [E]
        self.source_active = None          # u8  [Vi] (bitmap in the reference)
        self.edge_size = 0
        self.batch_size_forward = 0        # Vp
        self.batch_size_backward = 0       # Vi
        self.src_range = (0, 0)
        self.dst_range = (0, 0)
        # device copies
        self.column_offset_gpu = None
        self.row_indices_gpu = None
        self.edge_weight_forward_gpu = None
        self.row_offset_gpu = None
        self.column_indices_gpu = None
        self.edge_weight_backward_gpu = None
        self.source_active_gpu = None      # u8 [Vi], filled by the device builders only

    def copy_graph_to_device(self, device):
        """CSC_segment_pinned::CopyGraphToDevice (core/GraphSegment.cpp:178-220)."""
        import torch

        def up(a, dt):
            if a is None:
                return None
            t = torch.from_numpy(np.ascontiguousarray(a).view(dt))
            return t.to(device, non_blocking=False)

        # +1 slack element like the reference (arrays are allocated edge_size+1) so 16-byte bulk copies of the
        # last tile never run past the allocation
        def up_pad(a, dt):
            if a is None:
                return None
            pad = np.zeros(a.shape[0] + 8, dtype=a.dtype)
            pad[: a.shape[0]] = a
            return up(pad, dt)[: a.shape[0]]

        self.column_offset_gpu = up(self.column_offset, np.int32)
        self.row_offset_gpu = up(self.row_offset, np.int32)
        self.row_indices_gpu = up_pad(self.row_indices, np.int32)
        self.column_indices_gpu = up_pad(self.column_indices, np.int32)
        self.edge_weight_forward_gpu = up_pad(self.edge_weight_forward, np.float32)
        self.edge_weight_backward_gpu = up_pad(self.edge_weight_backward, np.float32)
        return self


class PartitionedGraph:
    """Mirror of core/PartitionedGraph.hpp for one rank."""

    def __init__(self, host_graph, partitions=1, partition_id=0, partition_offset=None):
        self.graph = host_graph
        self.global_vertices = host_graph.vertices if host_graph is not None else 0
        self.partitions = int(partitions)
        self.partition_id = int(partition_id)
        if partition_offset is None and host_graph is not None:
            partition_offset = host_graph.partition_offsets(self.partitions)
        self.partition_offset = None if partition_offset is None else np.asarray(partition_offset, dtype=np.uint32)
        self.graph_chunks = []
        self.owned_vertices = 0
        self.owned_edges = 0
        self.owned_mirrors = 0
        self.MirrorIndex = None
        self.column_offset = None      # whole-partition CSC (GenerateWholeGraphTopo)
        self.row_indices = None
        self.device = None
        self.column_offset_gpu = None
        self.row_indices_gpu = None
        self.mirror_index_gpu = None
        if self.partition_offset is not None:
            self.owned_vertices = int(self.partition_offset[self.partition_id + 1] - self.partition_offset[self.partition_id])

    # -- GenerateAll (core/PartitionedGraph.hpp:80-104) ------------------------------------------------------
    def generate_all(self, device=None, dist=False):
        self.partition_to_chunks()
        if dist:
            self.generate_mirror_index()
            self.generate_whole_graph_topo()
        if device is not None:
            self.to_device(device)
        return self

    def partition_to_chunks(self):
        """PartitionToChunks (core/PartitionedGraph.hpp:324-420) through nts_host_build_chunk."""
        g = self.graph
        out_d, in_d = g.degrees()
        P, p = self.partitions, self.partition_id
        po = self.partition_offset
        counts = np.zeros(P, dtype=np.uint64)
        _lib.call("nts_host_chunk_edge_counts", _ptr(g.edges), g.n_edges, _ptr(po), P, p, _ptr(counts))
        self.graph_chunks = []
        Vp = int(po[p + 1] - po[p])
        for i in range(P):
            c = CSCSegment()
            Ei = int(counts[i])
            Vi = int(po[i + 1] - po[i])
            c.edge_size = Ei
            c.batch_size_forward = Vp
            c.batch_size_backward = Vi
            c.src_range = (int(po[i]), int(po[i + 1]))
            c.dst_range = (int(po[p]), int(po[p + 1]))
            c.column_offset = np.zeros(Vp + 1, dtype=np.uint32)
            c.row_offset = np.zeros(Vi + 1, dtype=np.uint32)
            c.row_indices = np.zeros(Ei, dtype=np.uint32)
            c.column_indices = np.zeros(Ei, dtype=np.uint32)
            c.edge_weight_forward = np.zeros(Ei, dtype=np.float32)
            c.edge_weight_backward = np.zeros(Ei, dtype=np.float32)
            c.source_active = np.zeros(Vi, dtype=np.uint8)
            _lib.call("nts_host_build_chunk", _ptr(g.edges), g.n_edges, g.vertices, _ptr(po), P, p, i,
                      _ptr(out_d), _ptr(in_d), _ptr(c.column_offset), _ptr(c.row_indices),
                      _ptr(c.edge_weight_forward), _ptr(c.row_offset), _ptr(c.column_indices),
                      _ptr(c.edge_weight_backward), _ptr(c.source_active))
            self.graph_chunks.append(c)
        self.owned_edges = int(counts.sum())
        return self.graph_chunks

    def generate_mirror_index(self):
        """generateMirrorIndex (core/PartitionedGraph.hpp:295-305)."""
        g = self.graph
        mi = np.zeros(g.vertices + 1, dtype=np.uint32)
        owned = np.zeros(1, dtype=np.uint32)
        _lib.call("nts_host_mirror_index", _ptr(g.edges), g.n_edges, g.vertices, _ptr(self.partition_offset),
                  self.partition_id, _ptr(mi), _ptr(owned))
        self.MirrorIndex = mi
        self.owned_mirrors = int(owned[0])
        return mi

    def generate_whole_graph_topo(self):
        """GenerateWholeGraphTopo (core/PartitionedGraph.hpp:105-143): CSC over ALL local in-edges = the P chunk
        CSCs merged per destination (chunks are ordered by source partition, sources ascend inside a chunk)."""
        Vp = self.owned_vertices
        if not self.graph_chunks:
            self.partition_to_chunks()
        deg = np.zeros(Vp, dtype=np.int64)
        for c in self.graph_chunks:
            deg += np.diff(c.column_offset.astype(np.int64))
        col = np.zeros(Vp + 1, dtype=np.uint32)
        np.cumsum(deg, out=col[1:])
        rows = np.zeros(int(col[-1]), dtype=np.uint32)
        cursor = col[:-1].astype(np.int64).copy()
        for c in self.graph_chunks:
            d = np.diff(c.column_offset.astype(np.int64))
            if c.edge_size == 0:
                continue
            dst_of_edge = np.repeat(np.arange(Vp, dtype=np.int64), d)
            within = np.arange(c.edge_size, dtype=np.int64) - np.repeat(c.column_offset[:-1].astype(np.int64), d)
            rows[cursor[dst_of_edge] + within] = c.row_indices
            cursor += d
        self.column_offset = col
        self.row_indices = rows
        self.owned_edges = int(col[-1])
        return col, rows

    def to_device(self, device):
        import torch

        self.device = torch.device(device)
        for c in self.graph_chunks:
            c.copy_graph_to_device(self.device)
        if self.column_offset is not None:
            self.column_offset_gpu = torch.from_numpy(self.column_offset.view(np.int32)).to(self.device)
            pad = np.zeros(self.row_indices.shape[0] + 8, dtype=np.uint32)
            pad[: self.row_indices.shape[0]] = self.row_indices
            self.row_indices_gpu = torch.from_numpy(pad.view(np.int32)).to(self.device)[: self.row_indices.shape[0]]
        if self.MirrorIndex is not None:
            self.mirror_index_gpu = torch.from_numpy(self.MirrorIndex.view(np.int32)).to(self.device)
        return self

    # -- device-side construction (nts_graph_build, csrc/nts_graph_build.cu) -------------------------------------
    @staticmethod
    def from_edge_file(path, vertices, partitions=1, partition_id=0, device=None, dist=False, partition_offset=None,
                       block_edges=1 << 26):
        """Build the chunks of one rank on the GPU from a packed binary edge file ({u32 src, u32 dst} records,
        dep/gemini/type.hpp:100-106).  The file is streamed twice in blocks of `block_edges` records (degrees, then
        the edges this rank owns), so no process holds the edge list in host memory.  Fills every chunk's `*_gpu`
        arrays (plus `source_active_gpu`), the clamped degrees `out_degree_gpu` / `in_degree_gpu`, `partition_offset`
        (the reference's partitioner unless given), `global_vertices`, `owned_vertices` and `owned_edges`; with
        dist=True also `mirror_index_gpu`, `owned_mirrors` and the whole-partition CSC `column_offset_gpu` /
        `row_indices_gpu`.  The host arrays (`column_offset`, `MirrorIndex`, ...) stay None.  The arrays are
        bit-identical to the host builder's (`generate_all`)."""
        import torch

        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        po = None if partition_offset is None else np.ascontiguousarray(partition_offset, dtype=np.uint32)
        with torch.cuda.device(dev):
            stream = _lib.stream(dev)
            h = _lib.load().nts_graph_build_from_file(os.fsencode(path), int(vertices), int(partitions),
                                                      int(partition_id), _ptr(po), int(block_edges),
                                                      _lib_flags(dist), stream)
            return PartitionedGraph._from_build(h, vertices, partitions, partition_id, dev, dist, stream)

    @staticmethod
    def from_device_edges(src, dst, vertices, partitions=1, partition_id=0, partition_offset=None,
                          out_degree=None, in_degree=None, dist=False):
        """Build the chunks of one rank from int32 / int64 edge tensors already on the GPU (src/dst of ALL edges, or
        - when the global degrees are given - at least of every edge whose destination this rank owns).  Degrees,
        given or computed from the edges, are clamped to >= 1.  Same kernels, outputs and attributes as
        `from_edge_file`; partition_offset is required for partitions > 1."""
        import torch

        if partition_offset is None and int(partitions) != 1:
            raise ValueError("partition_offset is required for partitions > 1")
        if src.dtype != dst.dtype or src.dtype not in (torch.int32, torch.int64):
            raise _lib.NtsError("src / dst must both be int32 or both int64 (got %s, %s)" % (src.dtype, dst.dtype))
        if (out_degree is None) != (in_degree is None):
            raise _lib.NtsError("give both degree tensors or neither")
        dev = src.device
        src, dst = src.contiguous(), dst.contiguous()
        if out_degree is not None:
            out_degree = out_degree.to(device=dev, dtype=src.dtype).contiguous()
            in_degree = in_degree.to(device=dev, dtype=src.dtype).contiguous()
        po = None if partition_offset is None else np.ascontiguousarray(partition_offset, dtype=np.uint32)
        dtype = 0 if src.dtype == torch.int32 else 1   # NTS_INDEX_I32 / NTS_INDEX_I64
        with torch.cuda.device(dev):
            stream = _lib.stream(dev)
            h = _lib.load().nts_graph_build_from_device(
                src.data_ptr() or None, dst.data_ptr() or None, dtype, int(src.numel()), int(vertices),
                int(partitions), int(partition_id), _ptr(po),
                None if out_degree is None else out_degree.data_ptr(),
                None if in_degree is None else in_degree.data_ptr(), _lib_flags(dist), stream)
            return PartitionedGraph._from_build(h, vertices, partitions, partition_id, dev, dist, stream)

    @staticmethod
    def _from_build(h, vertices, partitions, partition_id, dev, dist, stream):
        """Copy the arrays of an nts_graph_build handle into torch tensors (the caching allocator owns them), then
        destroy the handle.  Edge arrays get the 8-element tail slack of CSCSegment.copy_graph_to_device."""
        import torch

        L = _lib.load()
        if not h:
            _lib.check(-1, "nts_graph_build")
        try:
            V, P, p = int(vertices), int(partitions), int(partition_id)
            po = np.zeros(P + 1, dtype=np.uint32)
            counts = np.zeros(P, dtype=np.uint64)
            mirrors = np.zeros(1, dtype=np.uint32)
            scratch = np.zeros(1, dtype=np.uint64)
            secs = np.zeros(4, dtype=np.float64)
            _lib.call("nts_graph_build_info", h, _ptr(po), _ptr(counts), _ptr(mirrors), _ptr(scratch), _ptr(secs))
            pg = PartitionedGraph(None, P, p, po)
            pg.global_vertices = V
            pg.device = dev
            pg.build_stats = {"scratch_peak_bytes": int(scratch[0]),
                              "seconds": dict(zip(("degrees", "owned_edges", "chunks", "dist"), secs.tolist()))}

            def vec(n, dtype=torch.int32):
                return torch.empty(n, dtype=dtype, device=dev)

            def edges(n, dtype=torch.int32):
                return torch.empty(n + 8, dtype=dtype, device=dev)[:n]   # tail slack for 16-byte bulk copies

            def ptr(t):
                return t.data_ptr() if t.numel() else None

            v0, v1 = int(po[p]), int(po[p + 1])
            for i in range(P):
                s0, s1, Ei = int(po[i]), int(po[i + 1]), int(counts[i])
                c = CSCSegment()
                c.edge_size = Ei
                c.batch_size_forward, c.batch_size_backward = v1 - v0, s1 - s0
                c.src_range, c.dst_range = (s0, s1), (v0, v1)
                c.column_offset_gpu, c.row_offset_gpu = vec(v1 - v0 + 1), vec(s1 - s0 + 1)
                c.row_indices_gpu, c.column_indices_gpu = edges(Ei), edges(Ei)
                c.edge_weight_forward_gpu = edges(Ei, torch.float32)
                c.edge_weight_backward_gpu = edges(Ei, torch.float32)
                c.source_active_gpu = vec(s1 - s0, torch.uint8)
                _lib.call("nts_graph_build_export_chunk", h, i, ptr(c.column_offset_gpu), ptr(c.row_indices_gpu),
                          ptr(c.edge_weight_forward_gpu), ptr(c.row_offset_gpu), ptr(c.column_indices_gpu),
                          ptr(c.edge_weight_backward_gpu), ptr(c.source_active_gpu), stream)
                pg.graph_chunks.append(c)
            pg.owned_edges = int(counts.sum())
            pg.out_degree_gpu, pg.in_degree_gpu = vec(V), vec(V)
            _lib.call("nts_graph_build_export_degrees", h, ptr(pg.out_degree_gpu), ptr(pg.in_degree_gpu), stream)
            if dist:
                pg.owned_mirrors = int(mirrors[0])
                pg.mirror_index_gpu = vec(V + 1)
                pg.column_offset_gpu = vec(v1 - v0 + 1)
                pg.row_indices_gpu = edges(pg.owned_edges)
                _lib.call("nts_graph_build_export_dist", h, ptr(pg.mirror_index_gpu), ptr(pg.column_offset_gpu),
                          ptr(pg.row_indices_gpu), stream)
            return pg
        finally:
            L.nts_graph_build_destroy(h)   # cudaFree waits for the export copies


def _lib_flags(dist):
    return 1 if dist else 0   # NTS_GRAPH_BUILD_DIST
