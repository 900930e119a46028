"""Neighbour sampling for mini-batch training: the reference's `Sampler` / `SampledSubgraph` (core/ntsSampler.hpp,
core/FullyRepGraph.hpp) on the GPU (K8, `nts_sampler` of include/nts_b200.h).

`NeighborSampler(pg, fanout, max_seeds)` samples the single-partition graph `pg` hop by hop from a list of seed
vertices: hop 0's destinations are the seeds, hop h keeps min(indeg, fanout[h]) edge slots of every destination (a
uniform subset by Floyd's algorithm on a counter hash of (seed, step, hop, destination, j)), and hop h+1's
destinations are hop h's distinct sources, ascending by global id.  A sample is a pure function of (graph, seed, step)
and the seeds: it does not depend on launch configuration, batch composition or the position of a vertex in the batch.

`NeighborSampler(..., include_dst=True)` (NTS_SAMPLER_INCLUDE_DST) keeps the same edges but makes every hop's sources
include its destinations, and records each destination's position among them in `SampledBlock.dst_pos`: the block
layout of a layer whose destinations read their own previous-layer rows (a GAT layer's destination scores).

`NeighborSampler(topology.ShardedTopology, ...)` samples the same way over a CSC sharded by destination ranges over the
ranks of one node (nts_sampler_create_sharded): each destination's in-edges are read from its owner's shard, local or
peer memory, and the blocks are those of the single-partition graph, bit for bit.

`SampledSubgraph` holds the blocks of one sample as `SampledBlock`s (device tensors); `ops.MiniBatchFuseOp` and
`ops.MiniBatchGATOp` aggregate over them."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_FANOUT = 64
MAX_HOPS = 8


class SampledBlock:
    """One hop of a sample (the reference's sampled_sgs[hop]).

    dst [n_dst] global destination ids; column_offset [n_dst+1]; row_indices [n_edges] local source ids (into src);
    weight [n_edges]; src [n_src] global source ids; row_offset [n_src+1], column_indices [n_edges] (local destinations)
    and weight_backward [n_edges]: the transposed block.  row_global [n_edges] (global source ids) may be None.
    dst_pos [n_dst] (local source index of every destination, src[dst_pos] == dst) is None unless the sources
    include the destinations (NeighborSampler(..., include_dst=True)).
    Index arrays are int32 tensors holding uint32 values."""

    def __init__(self, dst, column_offset, row_indices, weight, src, row_offset=None, column_indices=None,
                 weight_backward=None, row_global=None, dst_pos=None):
        self.dst, self.column_offset, self.row_indices, self.weight = dst, column_offset, row_indices, weight
        self.src, self.row_global, self.dst_pos = src, row_global, dst_pos
        self.n_dst, self.n_src, self.n_edges = int(dst.numel()), int(src.numel()), int(row_indices.numel())
        if row_offset is None:
            row_offset, column_indices, weight_backward = transpose(column_offset, row_indices, weight, self.n_dst,
                                                                    self.n_src)
        self.row_offset, self.column_indices, self.weight_backward = row_offset, column_indices, weight_backward

    def to_numpy(self):
        """Host copies of every array (uint32 index arrays, float32 weights)."""
        out = {}
        for name in ("dst", "column_offset", "row_indices", "row_global", "weight", "src", "row_offset",
                     "column_indices", "weight_backward", "dst_pos"):
            t = getattr(self, name)
            if t is not None:
                a = t.cpu().numpy()
                out[name] = a.view(np.uint32) if a.dtype == np.int32 else a
        return out

    def clone(self):
        c = object.__new__(SampledBlock)
        c.__dict__.update({k: (v.clone() if torch.is_tensor(v) else v) for k, v in self.__dict__.items()})
        return c


class SampledSubgraph:
    """The blocks of one sample, hop 0 (the seeds' block) first.  `blocks[-1]` is the deepest hop: its row_global
    lets the first layer gather straight from the whole feature table (MiniBatchFuseOp(..., table=True))."""

    def __init__(self, blocks, owner=None, vertices=None):
        self.blocks = list(blocks)
        self.vertices = None if vertices is None else int(vertices)   # V of the sampled graph (table gathers)
        self._owner = owner           # keeps a sampler's memory alive while its views are in use

    @property
    def hops(self):
        return len(self.blocks)

    def seeds(self):
        return self.blocks[0].dst

    def clone(self):
        """A copy that the next sample of the same sampler does not overwrite."""
        return SampledSubgraph([b.clone() for b in self.blocks], vertices=self.vertices)

    @staticmethod
    def from_blocks(blocks, vertices=None):
        """From dicts of device tensors with keys dst, column_offset, row_indices (local), weight, src (sources in any
        order) and optionally row_global and dst_pos; the transposed blocks are built on the device
        (nts_sample_transpose).  `vertices` (the graph's V) is needed for table gathers."""
        return SampledSubgraph([SampledBlock(b["dst"], b["column_offset"], b["row_indices"], b["weight"], b["src"],
                                             row_global=b.get("row_global"), dst_pos=b.get("dst_pos"))
                                for b in blocks], vertices=vertices)


def transpose(column_offset, row_indices, weight, n_dst, n_src):
    """(row_offset [n_src+1], column_indices, weight_backward) of a block with local sources in [0, n_src)."""
    dev = row_indices.device
    n_edges = int(row_indices.numel())
    row_offset = torch.empty(n_src + 1, dtype=torch.int32, device=dev)
    column_indices = torch.empty(n_edges, dtype=torch.int32, device=dev)
    weight_backward = torch.empty(n_edges, dtype=torch.float32, device=dev)
    for t in (column_offset, row_indices, weight):
        if not t.is_cuda or not t.is_contiguous():
            raise _lib.NtsError("block arrays must be contiguous CUDA tensors")
    _lib.call("nts_sample_transpose", column_offset.data_ptr(), row_indices.data_ptr(), weight.data_ptr(),
              int(n_dst), int(n_src), n_edges, row_offset.data_ptr(), column_indices.data_ptr(),
              weight_backward.data_ptr(), _lib.stream())
    return row_offset, column_indices, weight_backward


def check_fanout(fanout):
    fanout = [int(k) for k in fanout]
    if not 1 <= len(fanout) <= MAX_HOPS:
        raise _lib.NtsError("fanout needs 1..%d hops, got %d" % (MAX_HOPS, len(fanout)))
    for k in fanout:
        if not 1 <= k <= MAX_FANOUT:
            raise _lib.NtsError("fanout %d is outside 1..%d" % (k, MAX_FANOUT))
    return fanout


class NeighborSampler:
    """K8 on the CSC of a single-partition graph (chunk 0's column_offset_gpu / row_indices_gpu /
    edge_weight_forward_gpu), or on a topology.ShardedTopology (the same blocks; the sampler keeps a reference to the
    topology).  Device scratch for max_seeds seeds is allocated once, here.  `sample()` synchronises the stream once
    per hop; the blocks it returns are views that the next `sample()` overwrites (clone() them to keep them).

    include_dst=True: every hop's sources include its destinations and each block carries dst_pos (module docstring);
    the edges are those of the default mode, bit for bit."""

    SAMPLER_INCLUDE_DST = 1   # NTS_SAMPLER_INCLUDE_DST of include/nts_b200.h

    def __init__(self, partitioned_graph, fanout, max_seeds, include_dst=False):
        from .topology import ShardedTopology
        pg = partitioned_graph
        sharded = isinstance(pg, ShardedTopology)
        if not sharded and pg.partitions != 1:
            raise _lib.NtsError("NeighborSampler needs a single-partition graph (partitions == 1) or a "
                                "ShardedTopology, got %d partitions" % pg.partitions)
        self.fanout = check_fanout(fanout)
        self.max_seeds = int(max_seeds)
        self.include_dst = bool(include_dst)
        L = _lib.load()
        ks = (C.c_int * len(self.fanout))(*self.fanout)
        flags = self.SAMPLER_INCLUDE_DST if self.include_dst else 0
        if sharded:
            if pg._buf is None:
                raise _lib.NtsError("the topology is closed")
            self.V, self.device, self._graph = pg.vertices, pg.device, pg
            n = len(pg.offsets) - 1
            cols, rows, ws = ((C.c_void_p * n)(*a) for a in pg.shard_arrays)
            offs = (C.c_uint32 * (n + 1))(*[int(o) for o in pg.offsets])
            self.handle = _lib.checked(L.nts_sampler_create_sharded(cols, rows, ws, offs, n, self.max_seeds,
                                                                    len(self.fanout), ks, flags, _lib.stream()),
                                       "nts_sampler_create_sharded")
        else:
            c = pg.graph_chunks[0]
            if c.column_offset_gpu is None:
                raise _lib.NtsError("the graph has no device arrays (generate_all(device=...))")
            self.V = int(pg.global_vertices)
            self.device = c.column_offset_gpu.device
            self._graph = (c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu)
            self.handle = _lib.checked(L.nts_sampler_create_ex(c.column_offset_gpu.data_ptr(),
                                                               c.row_indices_gpu.data_ptr(),
                                                               c.edge_weight_forward_gpu.data_ptr(), self.V,
                                                               int(c.edge_size), self.max_seeds, len(self.fanout), ks,
                                                               flags, _lib.stream()),
                                       "nts_sampler_create_ex")

    def bytes(self):
        return int(_lib.load().nts_sampler_bytes(self.handle))

    def _seeds(self, seeds):
        """Seeds as a contiguous int32 device tensor; ids are checked against V before any device work when they
        are given on the host (numpy, list, CPU tensor)."""
        t = _lib.device_ids(seeds, self.V, self.device, "seeds", "seed vertex ids")
        if t.numel() > self.max_seeds:
            raise _lib.NtsError("%d seeds, the sampler was created for at most %d" % (t.numel(), self.max_seeds))
        return t

    def sample(self, seeds, seed, step):
        """The SampledSubgraph of `seeds` for (seed, step)."""
        s = self._seeds(seeds)
        _lib.call("nts_sampler_sample", self.handle, s.data_ptr() if s.numel() else None, int(s.numel()),
                  int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF, _lib.stream())
        return SampledSubgraph([self._view(h) for h in range(len(self.fanout))], owner=self, vertices=self.V)

    def _view(self, hop):
        v = _lib.SampleHopView()
        _lib.call("nts_sampler_hop_view", self.handle, int(hop), C.byref(v))

        def arr(ptr, n, dtype=torch.int32):
            return _lib.borrowed(ptr, n, dtype, self.device)

        nd, ns, ne = int(v.n_dst), int(v.n_src), int(v.n_edges)
        dst_pos = None
        if self.include_dst:
            p = C.c_void_p()
            _lib.call("nts_sampler_hop_dst_pos", self.handle, int(hop), C.byref(p))
            dst_pos = arr(p.value, nd)
        return SampledBlock(arr(v.dst, nd), arr(v.column_offset, nd + 1), arr(v.row_indices, ne),
                            arr(v.weight, ne, torch.float32), arr(v.src, ns), arr(v.row_offset, ns + 1),
                            arr(v.column_indices, ne), arr(v.weight_backward, ne, torch.float32), arr(v.row_global, ne),
                            dst_pos)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _lib.load().nts_sampler_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
