"""A [V, F] feature table sharded by row ranges over the GPUs of one node, read by global row id from any rank.

`ShardedFeatureTable(local_rows, offsets, group, dtype=torch.float32)` is collective over the process group: rank r
owns rows [offsets[r], offsets[r+1]) (any non-decreasing split of [0, V), empty shards allowed; the callers' default is
graph.partition_offsets_from_out_degree, the reference's partitioner) and keeps them in one device buffer of its own
at a pitch of 4*ceil(F/4) floats.  The ranks exchange CUDA-IPC handles of these buffers once, so that every rank maps
every other rank's shard (peer memory, reached over NVLink between GPUs), and `gather(ids)` reads the rows of any ids
with one launch of nts_gather_rows_sharded (include/nts_b200.h).  A torch caching-allocator tensor cannot be exported
as it is (an IPC handle names the allocation's base, not the sub-block), hence the table's own buffer.

dtype=torch.bfloat16 stores the rows rounded to BF16 (nts_rows_to_bf16, round to nearest even) at a pitch of
8*ceil(F/8) values with zero pad columns: half the memory, and half the bytes per gathered row, local or remote.  Its
gathers run nts_gather_rows_sharded_bf16 and return BF16 rows, or the same rows widened to float32 on request.

`ShardedEmbedding` is the learnable twin: FP32 rows trained by row-sparse Adam (K11, nts_embedding_step), the ranks
sending gradient rows to the rows' owners through outboxes mapped over the same CUDA IPC.

Scope is one node: at most 32 ranks in one CUDA-IPC domain, as for the exchange engine (exchange.py).  With one rank
(or no process group) the table is a single shard and `gather` is a local gather."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .adam import AdamSchedule

MAX_SHARDS = 32


def _group_rank_world(group):
    if not dist.is_initialized():
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


def gat_shape_error(F, heads, dtype=torch.float32):
    """Why K10 (ShardedFeatureTable.gat_aggregate) refuses rows of width F in `heads` heads of dtype, or None: heads
    must divide 32 (the statistics' lanes are (edge, head) pairs) and F, and with heads > 1 a head must be a whole
    number of 16-byte loads (4 FP32 or 8 BF16 values)."""
    if heads < 1 or 32 % heads:
        return "%d heads: the head count must divide 32" % heads
    if F % heads:
        return "width %d is not a multiple of %d heads" % (F, heads)
    vec = 8 if dtype == torch.bfloat16 else 4
    if heads > 1 and (F // heads) % vec:
        return "%d heads of width %d: with more than one head, a head must be a multiple of %d %s values" % (
            heads, F // heads, vec, "BF16" if vec == 8 else "FP32")
    return None


class PeerShards:
    """One device buffer per rank of a process group (nts_malloc_device: a CUDA-IPC handle names the whole
    allocation), mapped by every other rank.  The lifecycle ShardedFeatureTable and topology.ShardedTopology share:
    `_alloc` this rank's buffer, fill it, `_share` it (one handle exchange, every peer buffer opened), and `close()`.
    Subclasses set group, rank and world first."""

    _buf = None
    _peers = ()

    def _alloc(self, nbytes):
        L = _lib.load()
        self._peers = []
        self._buf = _lib.checked(L.nts_malloc_device(max(int(nbytes), 16)), "nts_malloc_device")

    def _share(self, meta):
        """Collective: (ptrs, metas) - every rank's buffer address in this process, this rank's own first-hand, and
        every rank's `meta` (any picklable value).  Call once the buffer is filled on the current stream."""
        if self.world == 1:
            return [self._buf], [meta]
        # the fill is complete before any peer can map the buffer: every rank passes this point first
        torch.cuda.current_stream(self.device).synchronize()
        L = _lib.load()
        h = C.create_string_buffer(64)
        _lib.call("nts_ipc_get_handle", self._buf, h)
        info = [None] * self.world
        dist.all_gather_object(info, (bytes(h.raw), meta), group=self.group)
        ptrs = [self._buf] * self.world
        for j, (hj, _) in enumerate(info):
            if j == self.rank:
                continue
            p = _lib.checked(L.nts_ipc_open_handle(hj), "nts_ipc_open_handle")
            self._peers.append(p)
            ptrs[j] = p
        return ptrs, [m for _, m in info]

    def close(self):
        """Collective: synchronise this device, a barrier (no rank is still reading a peer's shard), then close the
        peer mappings and free this rank's buffer."""
        if self._buf is None:
            return
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        self._release()

    def _release(self):
        L = _lib.load()
        for p in self._peers:
            L.nts_ipc_close_handle(p)
        self._peers = []
        if self._buf:
            L.nts_free_device(self._buf)
        self._buf = None

    def __del__(self):
        # without close() a peer may still read this rank's shard: free it only when there is no peer
        try:
            if getattr(self, "_buf", None) and self.world == 1:
                self._release()
        except Exception:
            pass


class ShardedFeatureTable(PeerShards):
    """See the module docstring.  Attributes: rows (V), F, dtype, pitch (in elements of dtype), local_bytes (this
    rank's shard buffer), offsets ([world+1] numpy), rank, world, group, device."""

    def __init__(self, local_rows, offsets, group=None, dtype=torch.float32):
        self.group = group
        self.rank, self.world = _group_rank_world(group)
        if self.world > MAX_SHARDS:
            raise _lib.NtsError("a sharded feature table spans at most %d ranks, the group has %d"
                                % (MAX_SHARDS, self.world))
        if dtype not in (torch.float32, torch.bfloat16):
            raise _lib.NtsError("a feature table stores torch.float32 or torch.bfloat16 rows, not %s" % (dtype,))
        off = np.asarray(offsets, dtype=np.int64).reshape(-1)
        if off.size != self.world + 1 or off[0] != 0 or (np.diff(off) < 0).any() or off[-1] >= 2 ** 32:
            raise _lib.NtsError("offsets must be %d non-decreasing row ids starting at 0, got %s"
                                % (self.world + 1, off.tolist()))
        x = local_rows.detach()
        if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 2:
            raise _lib.NtsError("local_rows must be a 2-D float32 CUDA tensor")
        lo, hi = int(off[self.rank]), int(off[self.rank + 1])
        if x.shape[0] != hi - lo:
            raise _lib.NtsError("rank %d owns rows [%d, %d) but local_rows has %d rows" % (self.rank, lo, hi, x.shape[0]))
        self.offsets, self.rows, self.F, self.dtype = off, int(off[-1]), int(x.shape[1]), dtype
        bf16 = dtype == torch.bfloat16
        self.pitch = (self.F + 7) // 8 * 8 if bf16 else (self.F + 3) // 4 * 4
        self.device = x.device
        n = (hi - lo) * self.pitch
        self.local_bytes = n * (2 if bf16 else 4)
        self._alloc(self.local_bytes)
        try:
            if n and bf16:
                x = x.contiguous()
                _lib.call("nts_rows_to_bf16", x.data_ptr(), 0, self.F, self._buf, hi - lo, self.F, self.pitch,
                          _lib.stream())
            elif n:
                mine = _lib.borrowed(self._buf, n, torch.float32, self.device).view(hi - lo, self.pitch)
                mine[:, self.F:].zero_()
                mine[:, :self.F].copy_(x)
            ptrs, info = self._share((self.F, str(dtype)))
            widths = sorted(set(f for f, _ in info))
            if len(widths) != 1:
                raise _lib.NtsError("the ranks' local_rows have different widths: %s" % widths)
            dtypes = sorted(set(d for _, d in info))
            if len(dtypes) != 1:
                raise _lib.NtsError("the ranks' tables have different dtypes: %s" % dtypes)
            self._shards = torch.tensor(ptrs, dtype=torch.int64).to(self.device)
            self._offsets = torch.from_numpy(off.astype(np.uint32).view(np.int32)).to(self.device)
        except Exception:
            self._release()
            raise

    def gather(self, ids, dtype=None):
        """Rows of the global ids `ids` (any integer tensor, numpy array or list; any order, repeats allowed) as an
        [n, F] tensor on this rank's device, of the table's dtype by default.  A BF16 table returns a [n, F] view of
        [n, pitch] BF16 rows, or with dtype=torch.float32 the rows widened exactly; a float32 table refuses a BF16
        output.  Ids outside [0, V) and a refused dtype raise NtsError before any device work."""
        self._out_dtype(dtype)
        t = _lib.device_ids(ids, self.rows, self.device, "ids", "row ids")
        return self._gather(t, dtype)

    def aggregate(self, out, column_offset, row_indices, weight, edge_begin, edge_end):
        """out[r, :] += sum over the edges e in [column_offset[r], column_offset[r+1]) of weight[e] * row
        row_indices[e] of the table (nts_segment_gather_sum_sharded), for r < out.shape[0]: the gather-sum of a CSC
        slice whose sources are read by global id from every rank's shard, local or peer memory.  BF16 rows are widened
        exactly and summed in FP32.

        out: float32 CUDA [n_rows, F] contiguous (zero it for a plain sum).  column_offset: int32 CUDA, at least n_rows
        + 1 absolute edge positions from edge_begin to edge_end (a slice of a whole-graph CSC's offsets, or a shard's
        local offsets from 0).  row_indices (int32, global ids in [0, V)) and weight (float32, or None for 1) are
        indexed by absolute edge position.  Asynchronous on the current stream.  A closed table and operands of the
        wrong kind raise NtsError before any device work."""
        if self._buf is None:
            raise _lib.NtsError("the feature table is closed")
        if not self._check_csc(out, column_offset, row_indices, weight, edge_begin, edge_end):
            return out
        n_rows, eb, ee = int(out.shape[0]), int(edge_begin), int(edge_end)
        _lib.call("nts_segment_gather_sum_sharded", out.data_ptr(), self._shards.data_ptr(),
                  1 if self.dtype == torch.bfloat16 else 0, self._offsets.data_ptr(), self.world, self.pitch,
                  None if weight is None else weight.data_ptr(), row_indices.data_ptr(), column_offset.data_ptr(),
                  n_rows, eb, ee, self.F, _lib.stream())
        return out

    def _check_csc(self, out, column_offset, row_indices, weight, edge_begin, edge_end):
        """NtsError for operands of aggregate() / gat_aggregate() of the wrong kind; False when there is nothing to
        add (no rows or no edges)."""
        for name, t, dt in (("out", out, torch.float32), ("column_offset", column_offset, torch.int32),
                            ("row_indices", row_indices, torch.int32), ("weight", weight, torch.float32)):
            if t is None and name == "weight":
                continue
            if not torch.is_tensor(t) or not t.is_cuda or t.dtype != dt or t.device != self.device \
                    or not t.is_contiguous():
                raise _lib.NtsError("%s must be a contiguous %s tensor on %s" % (name, dt, self.device))
        n_rows = int(out.shape[0]) if out.dim() == 2 else -1
        if n_rows < 0 or out.shape[1] != self.F:
            raise _lib.NtsError("out must be [n_rows, %d], got %s" % (self.F, tuple(out.shape)))
        eb, ee = int(edge_begin), int(edge_end)
        if column_offset.numel() < n_rows + 1 or not 0 <= eb <= ee <= row_indices.numel() or \
                (weight is not None and weight.numel() < ee):
            raise _lib.NtsError("column_offset needs %d entries and [edge_begin, edge_end) = [%d, %d) must lie in the "
                                "%d edges of row_indices and weight" % (n_rows + 1, eb, ee, row_indices.numel()))
        return n_rows > 0 and eb < ee

    def gat_aggregate(self, out, scores, dst_score, column_offset, row_indices, edge_begin, edge_end, heads,
                      negative_slope=0.2):
        """Full-neighbour GAT attention over the table (K10: nts_gat_softmax_stats_sharded, then
        nts_gat_aggregate_sharded), for the destinations r < out.shape[0] of a CSC slice given as for aggregate():

            logit(e, h) = leaky_relu(s[src(e), h] + dst_score[r, h], negative_slope)
            out[r, h*D:(h+1)*D] += sum_e softmax_e(logit(., h)) * row src(e)[h*D:(h+1)*D]      D = F / heads

        over the edges e in [column_offset[r], column_offset[r+1]).  `scores` is a float32 ShardedFeatureTable of [V,
        heads] source scores over the same group and offsets: a source's row and scores are read by global id, local
        or peer memory, with one shard search per edge.  dst_score: float32 CUDA [n_rows, heads] contiguous.  BF16 rows
        are widened exactly and summed in FP32; scores and statistics are FP32.  Allocates the [n_rows, heads]
        statistics and runs both entries asynchronously on the current stream.  A closed table, a score table of
        another kind, heads that do not divide 32 or split a 16-byte load (gat_shape_error), and the operand errors of
        aggregate() raise NtsError before any device work."""
        heads = int(heads)
        if not isinstance(scores, ShardedFeatureTable) or scores.dtype != torch.float32 or scores.F != heads:
            raise _lib.NtsError("scores must be a float32 ShardedFeatureTable of %d columns" % heads)
        if self._buf is None or scores._buf is None:
            raise _lib.NtsError("the feature table is closed")
        why = gat_shape_error(self.F, heads, self.dtype)
        if why is not None:
            raise _lib.NtsError(why)
        if scores.world != self.world or scores.rank != self.rank or scores.device != self.device or \
                not np.array_equal(scores.offsets, self.offsets):
            raise _lib.NtsError("scores must span the same ranks and offsets as the table")
        n_rows = int(out.shape[0]) if torch.is_tensor(out) and out.dim() == 2 else -1
        if not torch.is_tensor(dst_score) or dst_score.dim() != 2 or tuple(dst_score.shape) != (n_rows, heads) or \
                not dst_score.is_cuda or dst_score.dtype != torch.float32 or dst_score.device != self.device or \
                not dst_score.is_contiguous():
            raise _lib.NtsError("dst_score must be a contiguous float32 [%d, %d] tensor on %s"
                                % (max(n_rows, 0), heads, self.device))
        if not self._check_csc(out, column_offset, row_indices, None, edge_begin, edge_end):
            return out
        eb, ee = int(edge_begin), int(edge_end)
        seg = torch.empty((2, n_rows, heads), dtype=torch.float32, device=self.device)
        st = _lib.stream()
        _lib.call("nts_gat_softmax_stats_sharded", seg[0].data_ptr(), seg[1].data_ptr(), scores._shards.data_ptr(),
                  self._offsets.data_ptr(), self.world, scores.pitch, dst_score.data_ptr(), row_indices.data_ptr(),
                  column_offset.data_ptr(), n_rows, eb, ee, heads, float(negative_slope), st)
        _lib.call("nts_gat_aggregate_sharded", out.data_ptr(), self._shards.data_ptr(),
                  1 if self.dtype == torch.bfloat16 else 0, self._offsets.data_ptr(), self.world, self.pitch,
                  scores._shards.data_ptr(), scores.pitch, dst_score.data_ptr(), seg[0].data_ptr(),
                  seg[1].data_ptr(), row_indices.data_ptr(), column_offset.data_ptr(), n_rows, eb, ee, self.F, heads,
                  float(negative_slope), st)
        return out

    def _out_dtype(self, dtype):
        dtype = self.dtype if dtype is None else dtype
        if dtype not in (torch.float32, torch.bfloat16) or (dtype == torch.bfloat16 and self.dtype == torch.float32):
            raise _lib.NtsError("a %s table gathers %s rows, not %s"
                                % (self.dtype, "float32" if self.dtype == torch.float32 else "bfloat16 or float32",
                                   dtype))
        return dtype

    def _gather(self, ids, dtype=None):
        """gather() without the range check, for ids known to be in [0, V): a contiguous int32 device tensor holding
        uint32 values (a sampled block's src)."""
        if self._buf is None:
            raise _lib.NtsError("the feature table is closed")
        dtype = self._out_dtype(dtype)
        n = int(ids.numel())
        idp = ids.data_ptr() if n else None
        if self.dtype == torch.float32:
            out = torch.empty((n, self.F), dtype=torch.float32, device=self.device)
            _lib.call("nts_gather_rows_sharded", out.data_ptr(), self._shards.data_ptr(), self._offsets.data_ptr(),
                      self.world, self.pitch, idp, n, self.F, _lib.stream())
            return out
        ld = self.pitch if dtype == torch.bfloat16 else self.F
        out = torch.empty((n, ld), dtype=dtype, device=self.device)
        _lib.call("nts_gather_rows_sharded_bf16", out.data_ptr(), 1 if dtype == torch.bfloat16 else 0, ld,
                  self._shards.data_ptr(), self._offsets.data_ptr(), self.world, self.pitch, idp, n, self.F,
                  _lib.stream())
        return out[:, :self.F]


class _Outbox(PeerShards):
    """A ShardedEmbedding's outbox: one buffer per rank, mapped by every peer (nts_embedding_step's layout)."""

    def __init__(self, owner, nbytes):
        self.group, self.rank, self.world, self.device = owner.group, owner.rank, owner.world, owner.device
        self._alloc(nbytes)


class ShardedEmbedding(ShardedFeatureTable, AdamSchedule):
    """A learnable float32 [V, F] table sharded like ShardedFeatureTable, trained by row-sparse Adam (K11,
    nts_embedding_step): `step(ids, grad)` sends the gradient rows of some global ids, and the owner of each row sums
    what every rank sent for it, in ascending rank order, and applies Parameter's update to the row and its Adam
    moments.  The update is lazy, as in torch.optim.SparseAdam: a step's touched rows get the step-wide alpha, beta1
    and beta2 of the schedule (adam.AdamSchedule, one next() per step, the models' defaults: Adam(0.9, 0.999, 1e-9)
    with learn_rate, weight_decay and the decay of set_decay(decay_rate, decay_epoch)); untouched rows and their
    moments keep their bits.  gather, aggregate, gat_aggregate and close work as for the base class, so they read the
    learned rows.

    The constructor is collective, like the base class's.  Besides the shard, each rank keeps the moments M and V of
    its own rows ([hi - lo, pitch] float32, zero at first), K11's scratch (a uint32 mask and position per owned row and
    rank, and a touched-row list), and an outbox of `capacity` (default V) ids and gradient rows at the shard's pitch,
    exported over CUDA IPC once: every rank maps every peer's outbox at construction, not per step.  dtype must be
    torch.float32 (BF16 storage would round every update away)."""

    def __init__(self, local_rows, offsets, group=None, dtype=torch.float32, capacity=None, learn_rate=0.01,
                 weight_decay=0.0001, decay_rate=0.97, decay_epoch=100):
        if dtype != torch.float32:
            raise _lib.NtsError("a learnable embedding stores torch.float32 rows, not %s" % (dtype,))
        self._outbox = None
        super().__init__(local_rows, offsets, group, dtype)
        try:
            self.capacity = self.rows if capacity is None else int(capacity)
            if not 0 <= self.capacity < 2 ** 32:
                raise _lib.NtsError("capacity must be in [0, 2^32), got %d" % self.capacity)
            lo, hi = (int(o) for o in self.offsets[self.rank:self.rank + 2])
            f32, i32 = dict(dtype=torch.float32, device=self.device), dict(dtype=torch.int32, device=self.device)
            self.M = torch.zeros((hi - lo, self.pitch), **f32)
            self.V = torch.zeros((hi - lo, self.pitch), **f32)
            self._mask = torch.zeros(hi - lo, **i32)
            self._positions = torch.empty((hi - lo) * self.world, **i32)
            self._touched = torch.empty(1 + hi - lo, **i32)
            rows_at = 16 + 16 * ((self.capacity + 3) // 4)
            nbytes = rows_at + 4 * self.capacity * self.pitch
            self._outbox = _Outbox(self, nbytes)
            box = self._outbox._buf
            whole = _lib.borrowed(box, nbytes // 4, torch.float32, self.device)
            whole.zero_()      # the gradient rows' pad columns stay zero
            self._count = _lib.borrowed(box, 1, torch.int32, self.device)
            self._ids = _lib.borrowed(box + 16, self.capacity, torch.int32, self.device)
            self._grad_rows = whole[rows_at // 4:].view(self.capacity, self.pitch)
            ptrs, _ = self._outbox._share(None)
            self._outboxes = torch.tensor(ptrs, dtype=torch.int64).to(self.device)
        except Exception:
            if self._outbox is not None:
                self._outbox._release()
            self._release()
            raise
        self._init_schedule(learn_rate, 0.9, 0.999, 1e-9, weight_decay)
        self.set_decay(decay_rate, decay_epoch)

    def step(self, ids, grad):
        """Collective: one Adam step of the rows `ids` with gradient rows `grad`, on every rank once per round (a rank
        with nothing to send passes empty ids and a [0, F] grad).  ids: int32 CUDA tensor of global ids, strictly
        ascending, in [0, V), at most `capacity` of them; grad: float32 CUDA [len(ids), F].  A row several ranks send
        gets the sum of their rows in ascending rank order.  Ids or grad of the wrong kind and a closed table raise
        NtsError before any device work (the order and range checks read the ids back to the host).

        The step writes this rank's outbox, fences, runs K11 on this rank's rows, and fences again; a fence is a
        synchronise of this rank's current stream and then a barrier of the group.  The two fences are enough: every
        rank's outbox is complete before the first fence's barrier, so no owner starts K11 before every outbox it
        reads is written; every rank's earlier gathers of peer rows, issued on the same stream, also ended before that
        barrier, so no owner updates a row a peer is still reading.  K11 has ended on every rank before the second
        fence's barrier, so no rank's next gather reads a row mid-update and no rank overwrites its outbox (at its next
        step) while an owner still reads it.  Between the fences a rank runs only K11, which reads the outboxes and
        writes its own shard, moments and scratch.  With one rank, stream order alone does all this."""
        self._check_open()
        if not torch.is_tensor(ids) or not ids.is_cuda or ids.dtype != torch.int32 or ids.dim() != 1 or \
                ids.device != self.device:
            raise _lib.NtsError("ids must be a 1-D int32 tensor on %s" % self.device)
        n = int(ids.numel())
        if not torch.is_tensor(grad) or not grad.is_cuda or grad.dtype != torch.float32 or grad.device != self.device \
                or tuple(grad.shape) != (n, self.F):
            raise _lib.NtsError("grad must be a float32 [%d, %d] tensor on %s" % (n, self.F, self.device))
        self._check_capacity(n)
        if n:
            u = ids.long() & 0xFFFFFFFF
            unsorted, out_of_range = torch.stack([(u[1:] <= u[:-1]).any(), u[-1] >= self.rows]).tolist()
            if unsorted:
                raise _lib.NtsError("ids must be strictly ascending (distinct, sorted)")
            if out_of_range:
                raise _lib.NtsError("ids must be in [0, %d)" % self.rows)
        self._step(ids, grad)

    def _step(self, ids, grad):
        """step() without the order and range checks, for ids known to be distinct, ascending and in [0, V): a
        contiguous int32 device tensor holding uint32 values (a sampled block's src).  A closed table and more than
        `capacity` ids still raise NtsError before any device work."""
        self._check_open()
        n = int(ids.numel())
        self._check_capacity(n)
        self._count.fill_(n)
        if n:
            self._ids[:n].copy_(ids)
            self._grad_rows[:n, :self.F].copy_(grad)
        self._fence()
        lo, hi = (int(o) for o in self.offsets[self.rank:self.rank + 2])
        _lib.call("nts_embedding_step", self._buf, self.M.data_ptr(), self.V.data_ptr(), self._mask.data_ptr(),
                  self._positions.data_ptr(), self._touched.data_ptr(), self._outboxes.data_ptr(), self.world,
                  self.capacity, lo, hi, self.pitch, self.F, float(self.weight_decay), float(self.beta1),
                  float(self.beta2), float(self.alpha), float(self.epsilon), _lib.stream())
        self._fence()
        self.next()

    def _check_open(self):
        if self._buf is None:
            raise _lib.NtsError("the feature table is closed")

    def _check_capacity(self, n):
        if n > self.capacity:
            raise _lib.NtsError("%d rows in one step, the outbox holds %d (capacity)" % (n, self.capacity))

    def _fence(self):
        if self.world > 1:
            torch.cuda.current_stream(self.device).synchronize()
            dist.barrier(group=self.group)

    def close(self):
        """Collective: closes the outboxes, then the table (PeerShards.close)."""
        if self._outbox is not None:
            self._outbox.close()
            self._outbox = None
        super().close()
