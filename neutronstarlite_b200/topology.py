"""A graph's weighted in-edge CSC sharded by destination ranges over the GPUs of one node, sampled from any rank.

`ShardedTopology(column_offset, row_indices, weight, offsets, group=None)` is collective over the process group: rank
r owns destinations [offsets[r], offsets[r+1]) (any non-decreasing split of [0, V), empty shards allowed) and keeps
their in-edges as a CSC with local column offsets [V_r + 1], global source ids [E_r] and edge weights [E_r], in the
slot order of the single-partition CSC.  The three arrays live in one device buffer of the rank's own, at 16-byte
aligned sections, so that one CUDA-IPC handle per rank maps a whole shard; each rank derives its peers' section
addresses from their all-gathered (V_r, E_r).  `sample.NeighborSampler(topology, ...)` samples over every rank's
shard (nts_sampler_create_sharded), and gives the blocks of the whole-graph sampler bit for bit.

The constructor checks each shard's CSC before any copy (local column offsets from 0 to E_r that never decrease, source
ids in [0, V)), so that no sampler read leaves a shard's arrays.  `ShardedTopology.split(...)` puts every shard of a
whole-graph CSC into this one process, to run and time the sharded sampler on one GPU.

`ShardedTopology.from_partitioned_graph(pg)` builds rank r's shard from its PartitionedGraph (partitions == world,
partition_id == rank): nts_merge_chunk_csc merges the P chunk CSCs per destination, chunk 0 first, which is the slot
order of the single-partition CSC.  The PartitionedGraph may be dropped afterwards.

Scope is one node: at most 32 ranks, as for feature_table.ShardedFeatureTable, whose buffer lifecycle (PeerShards)
this class shares: close() is collective; without it a shard is freed at garbage collection only at world 1."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .feature_table import MAX_SHARDS, PeerShards, _group_rank_world


def _align16(nbytes):
    return (int(nbytes) + 15) // 16 * 16


def _sections(n_dst, n_edges):
    """Byte offsets of (column_offset, row_indices, weight) in a shard buffer, and its size."""
    row = _align16(4 * (n_dst + 1))
    w = row + _align16(4 * n_edges)
    return (0, row, w), w + _align16(4 * n_edges)


def _check_tensors(col, row, w):
    for name, t, dt in (("column_offset", col, torch.int32), ("row_indices", row, torch.int32),
                        ("weight", w, torch.float32)):
        if not torch.is_tensor(t) or not t.is_cuda or t.dtype != dt or t.dim() != 1:
            raise _lib.NtsError("%s must be a 1-D %s CUDA tensor" % (name, dt))
    if col.numel() < 1 or row.numel() != w.numel() or row.device != col.device or w.device != col.device:
        raise _lib.NtsError("column_offset needs at least one entry, and row_indices / weight the same edge count on "
                            "its device (got %d, %d)" % (row.numel(), w.numel()))


def _check_csc(col, row, V):
    """NtsError unless (col, row) is a CSC the sampler can read without leaving its arrays: col[0] == 0, col never
    decreases, col[-1] == row.numel(), and every source id is in [0, V).  Values are uint32 held in int32; one
    device-to-host copy of four scalars."""
    c = col.long() & 0xFFFFFFFF
    r = row.long() & 0xFFFFFFFF
    zero = torch.zeros((), dtype=torch.int64, device=col.device)
    stats = torch.stack([c[0], c[-1], (c[1:] < c[:-1]).sum() if c.numel() > 1 else zero,
                         r.max() if r.numel() else zero]).tolist()
    first, last, falls, top = stats
    if first != 0 or last != row.numel() or falls:
        raise _lib.NtsError("column_offset must be local offsets: start at 0, never decrease and end at the edge "
                            "count %d (got first %d, last %d, %d decreases)" % (row.numel(), first, last, falls))
    if row.numel() and top >= V:
        raise _lib.NtsError("row_indices holds source id %d, the graph has %d vertices" % (top, V))


class ShardedTopology(PeerShards):
    """See the module docstring.  Attributes: vertices (V), offsets ([n_shards+1] numpy), rank, world, group, device,
    local_edges (the edges this process holds), local_bytes (this process's shard buffer), shard_arrays (host lists of
    every shard's column offset / row / weight addresses in this process).  n_shards is world, except for split()."""

    def __init__(self, column_offset, row_indices, weight, offsets, group=None):
        """Collective: this rank's shard from device tensors - column_offset int32 [V_r + 1] (local offsets),
        row_indices int32 [E_r] (global source ids) and weight float32 [E_r], in the single-partition CSC's slot
        order.  The arrays are checked (_check_csc) and copied; a malformed shard raises NtsError on its rank."""
        col, row, w = column_offset, row_indices, weight
        _check_tensors(col, row, w)
        off = np.asarray(offsets, dtype=np.int64).reshape(-1)
        if off.size >= 1 and 0 < off[-1] < 2 ** 31:
            _check_csc(col, row, int(off[-1]))      # otherwise _build refuses the offsets

        def fill(dst):
            for p, t in zip(dst[0], (col, row, w)):
                _lib.borrowed(p, t.numel(), t.dtype, self.device).copy_(t)

        self._build(off, group, col.device, [(col.numel() - 1, row.numel())], fill)

    @classmethod
    def split(cls, column_offset, row_indices, weight, offsets):
        """Every shard in this process: the whole graph's CSC (column_offset [V+1], row_indices, weight) split at
        `offsets` ([n_shards+1], 1 <= n_shards <= 32, empty shards allowed), each shard with local column offsets in
        its own sections of one buffer.  What the sampler reads from n ranks' shards, on one GPU and without a process
        group (rank 0, world 1); for tests and measurements of the sharded sampler.  The CSC is checked as in the
        constructor."""
        col, row, w = column_offset, row_indices, weight
        _check_tensors(col, row, w)
        off = np.asarray(offsets, dtype=np.int64).reshape(-1)
        if not 2 <= off.size <= MAX_SHARDS + 1 or off[0] != 0 or (np.diff(off) < 0).any() or \
                not 0 < off[-1] < 2 ** 31 or col.numel() != off[-1] + 1:
            raise _lib.NtsError("offsets must be 2..%d non-decreasing vertex ids from 0 to V = column_offset.numel() "
                                "- 1 = %d, got %s" % (MAX_SHARDS + 1, col.numel() - 1, off.tolist()))
        _check_csc(col, row, int(off[-1]))
        c = col.long() & 0xFFFFFFFF
        bounds = [int(e) for e in c[torch.from_numpy(off).to(col.device)].tolist()]
        shards = [(int(off[o + 1] - off[o]), bounds[o + 1] - bounds[o]) for o in range(off.size - 1)]

        def fill(dst):
            for o, ((p_col, p_row, p_w), (n_dst, _)) in enumerate(zip(dst, shards)):
                lo, e0, e1 = int(off[o]), bounds[o], bounds[o + 1]
                local = (c[lo:lo + n_dst + 1] - e0).to(torch.int32)
                for p, t in ((p_col, local), (p_row, row[e0:e1]), (p_w, w[e0:e1])):
                    _lib.borrowed(p, t.numel(), t.dtype, self.device).copy_(t)

        self = cls.__new__(cls)
        self._build(off, None, col.device, shards, fill, split=True)
        return self

    @classmethod
    def from_partitioned_graph(cls, pg, group=None):
        """Rank r's shard from its PartitionedGraph `pg` (any builder, with device chunk arrays): collective."""
        rank, world = _group_rank_world(group)
        if pg.partitions != world or pg.partition_id != rank:
            raise _lib.NtsError("rank %d of %d needs partition %d of a %d-partition graph, got partition %d of %d"
                                % (rank, world, rank, world, pg.partition_id, pg.partitions))
        chunks = pg.graph_chunks
        if not chunks or any(c.column_offset_gpu is None for c in chunks):
            raise _lib.NtsError("the graph has no device chunk arrays")
        n_dst = int(pg.owned_vertices)
        n_edges = sum(int(c.edge_size) for c in chunks)
        P = len(chunks)

        def ptrs(name):
            return (C.c_void_p * P)(*[getattr(c, name).data_ptr() if getattr(c, name).numel() else None
                                      for c in chunks])

        def fill(dst):
            (p_col, p_row, p_w), = dst
            _lib.call("nts_merge_chunk_csc", ptrs("column_offset_gpu"), ptrs("row_indices_gpu"),
                      ptrs("edge_weight_forward_gpu"), P, n_dst, n_edges, p_col, p_row if n_edges else None,
                      p_w if n_edges else None, _lib.stream())

        self = cls.__new__(cls)
        self._build(pg.partition_offset, group, chunks[0].column_offset_gpu.device, [(n_dst, n_edges)], fill)
        return self

    def _build(self, off, group, device, shards, fill, split=False):
        """Allocate this process's buffer for `shards` ([(n_dst, n_edges)]: this rank's one shard, or every shard with
        split=True), fill(section addresses per shard) it, and share it with the group's other ranks."""
        self.group = group
        self.rank, self.world = _group_rank_world(group)
        if split:
            self.rank, self.world = 0, 1
        if self.world > MAX_SHARDS:
            raise _lib.NtsError("a sharded topology spans at most %d ranks, the group has %d"
                                % (MAX_SHARDS, self.world))
        off = np.asarray(off, dtype=np.int64).reshape(-1)
        n = len(shards) if split else self.world
        if off.size != n + 1 or off[0] != 0 or (np.diff(off) < 0).any() or not 0 < off[-1] < 2 ** 31:
            raise _lib.NtsError("offsets must be %d non-decreasing vertex ids from 0 to V (1 <= V < 2^31), got %s"
                                % (n + 1, off.tolist()))
        if not split:
            lo, hi = int(off[self.rank]), int(off[self.rank + 1])
            if shards[0][0] != hi - lo:
                raise _lib.NtsError("rank %d owns destinations [%d, %d) but its column_offset covers %d"
                                    % (self.rank, lo, hi, shards[0][0]))
        if any(e >= 2 ** 32 for _, e in shards):
            raise _lib.NtsError("a shard holds fewer than 2^32 edges, got %s" % [e for _, e in shards])
        self.offsets, self.vertices, self.device = off, int(off[-1]), torch.device(device)
        self.local_edges = sum(int(e) for _, e in shards)
        starts, total = [], 0
        for v_r, e_r in shards:
            starts.append(total)
            total += _sections(v_r, e_r)[1]
        self.local_bytes = total
        with torch.cuda.device(self.device):
            self._alloc(total)
            try:
                fill([[self._buf + b + s for s in _sections(v_r, e_r)[0]] for b, (v_r, e_r) in zip(starts, shards)])
                if split:
                    secs = [[self._buf + b + s for s in _sections(v_r, e_r)[0]]
                            for b, (v_r, e_r) in zip(starts, shards)]
                else:
                    ptrs, counts = self._share(shards[0])
                    for r, (v_r, _) in enumerate(counts):
                        if v_r != int(off[r + 1] - off[r]):
                            raise _lib.NtsError("rank %d holds %d destinations, the offsets give it %d"
                                                % (r, v_r, int(off[r + 1] - off[r])))
                    secs = [[p + s for s in _sections(v_r, e_r)[0]] for p, (v_r, e_r) in zip(ptrs, counts)]
            except Exception:
                self._release()
                raise
        # host lists of every shard's section addresses in this process (nts_sampler_create_sharded's arguments)
        self.shard_arrays = tuple([s[i] for s in secs] for i in range(3))
