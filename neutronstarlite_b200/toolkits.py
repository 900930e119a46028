"""Callers of the hot path, mirrored from the reference so the path can be driven and timed end to end:

  * `Parameter`  <-> core/NtsScheduler.hpp:639-791 (weight, L2-regularised Adam with the reference's bias-correction
                     folded into alpha by `next()`, gradient SUM-allreduce - NCCL instead of MPI on host copies)
  * `GCNImpl`    <-> toolkits/GCN.hpp (2-layer GCN: aggregate -> X.W -> relu / log_softmax, nll loss on the train
                     mask, tape backward, Adam); the single-GPU op of toolkits/GCN_EAGER_single.hpp when P = 1.
  * `GCNEagerImpl` <-> toolkits/GCN_EAGER_single.hpp / GCN_EAGER.hpp order (X.W first, aggregate the narrow result).
  * `GATImpl`    <-> the flow of toolkits/GAT_CPU_DIST_OPTM.hpp on the fused multi-head aggregation (K7).
  * `GCNSampleImpl` <-> toolkits/GCN_CPU_SAMPLE.hpp (neighbour-sampled mini-batch GCN) on the K8 sampler and
                     ops.MiniBatchFuseOp, on one GPU or data-parallel over a feature_table.ShardedFeatureTable,
                     with the topology whole on every rank or sharded (topology.ShardedTopology).
  * `GATSampleImpl` <-> GATImpl's layers on GCNSampleImpl's batch loop: neighbour-sampled mini-batch GAT on the K8
                     sampler (destination-inclusive blocks) and K7 through ops.MiniBatchGATOp, on one GPU or
                     data-parallel like GCNSampleImpl.

Dense NN work (mm, relu, log_softmax, nll_loss, Adam element-wise) stays on torch/cuBLAS exactly as in the
reference (libtorch); the aggregation goes through libnts_b200."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.distributed as dist

from .adam import AdamSchedule
from .context import NtsContext
from . import _lib, ops


class Parameter(AdamSchedule):
    def __init__(self, w, h, alpha, beta1, beta2, epsilon, weight_decay, device=None, generator=None):
        scale = math.sqrt(6.0 / (w + h))
        W = (2 * scale) * torch.rand((w, h), dtype=torch.float32, generator=generator) - scale
        self.W = W.to(device).requires_grad_(True)
        self.M = torch.zeros((w, h), dtype=torch.float32, device=device)
        self.V = torch.zeros((w, h), dtype=torch.float32, device=device)
        self.W_gradient = None
        self._init_schedule(alpha, beta1, beta2, epsilon, weight_decay)

    def init_parameter(self):
        """Network_simple::broadcast from rank 0 (comm/network.h:205-211)."""
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(self.W.data, src=0)

    def all_reduce_to_gradient(self, grad):
        """SUM (not mean) over ranks, NtsScheduler.hpp:719-722 -> comm/network.h:198-203."""
        self.W_gradient = grad.detach().clone().contiguous()
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.W_gradient, op=dist.ReduceOp.SUM)

    def forward(self, x):
        return x.mm(self.W)

    def learn_with_decay_Adam(self):
        """learnC2G_with_decay_Adam, NtsScheduler.hpp:774-781.  On the GPU: ONE fused kernel (nts_adam_update)
        instead of the reference's six element-wise libtorch ops; the torch expression below is the host mirror
        used by the CPU tests (same arithmetic, pinned to the reference's golden vectors in tests/test_adam.py)."""
        with torch.no_grad():
            if self.W.is_cuda:
                _lib.call("nts_adam_update", self.W.data_ptr(), self.M.data_ptr(), self.V.data_ptr(),
                          self.W_gradient.data_ptr(), self.W.numel(), float(self.weight_decay), float(self.beta1),
                          float(self.beta2), float(self.alpha), float(self.epsilon), _lib.stream())
                return
            one = np.float32(1)
            W_g = self.W * float(self.weight_decay) + self.W_gradient
            self.M = float(self.beta1) * self.M + float(one - self.beta1) * W_g
            self.V = float(self.beta2) * self.V + float(one - self.beta2) * W_g * W_g
            self.W -= float(self.alpha) * self.M / (torch.sqrt(self.V) + float(self.epsilon))

    def zero_grad(self):
        self.W.grad = None


def _parameters(shapes, seed, device, learn_rate, weight_decay, decay=None):
    """One Parameter per (w, h) of `shapes`, in order: the generator seeded with `seed` draws them and rank 0's values
    are broadcast in that order.  decay = (decay_rate, decay_epoch) for Parameter.set_decay; None keeps Adam's
    defaults (no decay)."""
    gen = torch.Generator().manual_seed(seed)
    params = []
    for w, h in shapes:
        p = Parameter(w, h, learn_rate, 0.9, 0.999, 1e-9, weight_decay, device=device, generator=gen)
        p.init_parameter()
        if decay is not None:
            p.set_decay(*decay)
        params.append(p)
    return params


def _update(params, zero_fill_missing):
    """all_reduce_to_gradient, Adam and next() for every parameter.  A parameter without a gradient is skipped, or with
    zero_fill_missing reduced and stepped as zeros (data-parallel rounds: the collectives are then the same on every
    rank)."""
    for p in params:
        g = p.W.grad
        if g is None:
            if not zero_fill_missing:
                continue
            g = torch.zeros_like(p.W)
        p.all_reduce_to_gradient(g)
        p.learn_with_decay_Adam()
        p.next()


class _FullGraph:
    """The loss and update of the full-graph models."""

    def Loss(self):
        """GCN.hpp:198-207: nll_loss over the local train rows (mean)."""
        a = self.X[-1]
        self.loss = torch.nn.functional.nll_loss(a.index_select(0, self.train_rows),
                                                 self.L_GT.index_select(0, self.train_rows))
        self.ctx.appendNNOp(a, self.loss)

    def Update(self):
        """GCN.hpp:209-215."""
        _update(self.params(), False)


class GCNImpl(_FullGraph):
    """toolkits/GCN.hpp:33-354.  `layers` = LAYERS of the cfg, e.g. [602, 128, 41].

    gather_dtype=torch.bfloat16: every aggregation gathers its operand as BF16 rows with FP32 accumulation (the
    operator's option), and the input features, which the first aggregation reads directly, are stored as bfloat16
    (half the memory of the largest tensor).  Activations, weights and gradients stay float32.

    With FP32 gathers on the single-GPU op, input features on the GPU whose width is not a multiple of 4 are stored
    once as a [V, 4*ceil(F/4)] tensor viewed as X[0] = [:, :F] (a copy: the caller's tensor is left as it is)."""

    _input_is_gathered = True   # X[0] is the first aggregation's operand (stored as bfloat16 under BF16 gathers)

    def __init__(self, partitioned_graph, layers, features, labels, mask, learn_rate=0.01, weight_decay=0.0001,
                 decay_rate=0.97, decay_epoch=100, drop_rate=0.5, op_class=None, op_kwargs=None, seed=0,
                 gather_dtype=None):
        self.pg = partitioned_graph
        self.layers = list(layers)
        self.device = features.device
        self.drop_rate = drop_rate
        self.ctx = NtsContext()
        self.P = _parameters(zip(self.layers, self.layers[1:]), seed, self.device, learn_rate, weight_decay,
                             (decay_rate, decay_epoch))
        self.L_GT = labels.to(self.device)
        self.MASK = mask.to(self.device)
        self.train_rows = (self.MASK == 0).nonzero().view(-1)
        self.X = [None] * len(self.layers)
        self.gather_dtype = ops._check_gather_dtype(gather_dtype)
        if op_class is None:
            op_class = ops.ForwardSingleGPUfuseOp if partitioned_graph.partitions == 1 else ops.ForwardGPUfuseOp
        self.op_class = op_class
        # the single-GPU op takes row-pitched inputs: X[0] is stored once with its rows padded to 16 bytes, so that
        # the first aggregation gathers it in place every epoch instead of copying it into padded rows
        self._pitched_input = (self._input_is_gathered and self.gather_dtype is None and
                               isinstance(op_class, type) and issubclass(op_class, ops.ForwardSingleGPUfuseOp))
        if self.gather_dtype is not None and self._input_is_gathered:
            features = features.detach().to(self.gather_dtype)
        elif self._pitched_input and features.is_cuda and features.dim() == 2 and features.shape[1] % 4:
            F = features.shape[1]
            padded = torch.zeros((features.shape[0], (F + 3) // 4 * 4), dtype=features.dtype, device=features.device)
            padded[:, :F].copy_(features.detach())
            features = padded[:, :F]
        self.X[0] = features.requires_grad_(True)
        self.op_kwargs = dict(op_kwargs or {})
        if self.gather_dtype is not None:
            self.op_kwargs["gather_dtype"] = self.gather_dtype
        self.loss = None
        self.epoch = 0

    def params(self):
        return self.P

    def vertexForward(self, a, x, layer):
        """GCN.hpp:183-196."""
        if layer < len(self.layers) - 2:
            return torch.relu(self.P[layer].forward(a))
        return self.P[layer].forward(a).log_softmax(1)

    def Forward(self):
        """GCN.hpp:217-235."""
        for i in range(len(self.layers) - 1):
            x_i = self.X[i]
            if i != 0 and self.drop_rate > 0:
                # the reference drops in place (GCN.hpp:221-223); out of place + chaining onto the NN segment
                # keeps torch's autograd version check happy and is numerically the same operation
                dropped = torch.nn.functional.dropout(x_i, self.drop_rate, training=True)
                self.ctx.appendNNOp(x_i, dropped)
                x_i = dropped
            if not (self._pitched_input and ops.row_pitched(x_i)):
                x_i = x_i.contiguous()
            y_i = self.ctx.runGraphOp(self.op_class, self.pg, None, x_i, **self.op_kwargs)
            self.X[i + 1] = self.ctx.runVertexForward(lambda n, v, _l=i: self.vertexForward(n, v, _l), y_i, x_i)

    def Test(self, s):
        """GCN.hpp:150-181: accuracy over mask == s, summed over ranks."""
        sel = self.MASK == s
        correct = (self.X[-1].argmax(1) == self.L_GT)[sel].sum()
        total = sel.sum()
        pair = torch.stack([correct, total]).to(torch.int64)
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(pair)
        return pair

    def run_epoch(self, test=False):
        """One iteration of GCN.hpp:244-262."""
        if self.epoch != 0:
            for p in self.P:
                p.zero_grad()
        self.Forward()
        acc = [self.Test(s) for s in (0, 1, 2)] if test else None
        self.Loss()
        self.ctx.self_backward(True)
        self.Update()
        self.epoch += 1
        return self.loss, acc


class GCNEagerImpl(GCNImpl):
    """Transform-then-aggregate GCN: toolkits/GCN_EAGER_single.hpp:184-232 (P = 1) and toolkits/GCN_EAGER.hpp (P > 1).
    Each layer runs the weight GEMM first and aggregates the NARROW result (widths LAYERS[1:], e.g. 128 and 41
    instead of 602 and 128 - 4.7x fewer gathered bytes on config B), then `log_softmax` + `nll_loss` on the last
    aggregate.  The tape is [NNOP, GRAPHOP, NNOP, GRAPHOP, NNOP(loss)], so every aggregation has a backward
    (L forward + L backward calls per epoch).  Under gather_dtype the input features stay float32: they feed the
    first weight GEMM, not an aggregation."""

    _input_is_gathered = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        # the input features are the input of the first NN op here; nobody reads their gradient, so do not make
        # autograd compute dX0 = dY0 W0^T (a [V, LAYERS[0]] tensor) every epoch
        self.X[0] = self.X[0].detach()

    def vertexForward(self, a, x, layer):
        """GCN_EAGER_single.hpp:201-212: layer 0 = W0 x; deeper layers = W_l relu(dropout(a))."""
        if layer == 0:
            return self.P[layer].forward(a)
        if self.drop_rate > 0:
            a = torch.nn.functional.dropout(a, self.drop_rate, training=True)
        return self.P[layer].forward(torch.relu(a))

    def Forward(self):
        """GCN_EAGER_single.hpp:214-227."""
        for i in range(len(self.layers) - 1):
            y_i = self.ctx.runVertexForward(lambda n, v, _l=i: self.vertexForward(n, v, _l), self.X[i], self.X[i])
            self.X[i + 1] = self.ctx.runGraphOp(self.op_class, self.pg, None, y_i.contiguous(), **self.op_kwargs)

    def Loss(self):
        """GCN_EAGER_single.hpp:185-194."""
        a = self.X[-1].log_softmax(1)
        self.loss = torch.nn.functional.nll_loss(a.index_select(0, self.train_rows),
                                                 self.L_GT.index_select(0, self.train_rows))
        self.ctx.appendNNOp(self.X[-1], self.loss)


def _minibatch_op(sampled_subgraph, active, hop, table=False, gather_dtype=None):
    return ops.MiniBatchFuseOp(sampled_subgraph, hop, table=table, gather_dtype=gather_dtype)


class _SampledRounds:
    """The batch loop shared by GCNSampleImpl and GATSampleImpl, on one GPU or data-parallel over the ranks of a
    feature_table.ShardedFeatureTable.

    A pass cuts the ascending ids of one mask value into batches of batch_size.  Batch b of a pass samples with step
    base + b, and base advances by the pass's batch count on every rank, so at world 1 the steps are those of a run
    with a tensor.  With a table over N ranks the pass runs in rounds: round t runs batch t*N + r on rank r.  Every
    training round ends in one Adam step per parameter on every rank, after Parameter.all_reduce_to_gradient has
    SUM-reduced the gradients over the ranks in the same parameter order everywhere (the reference's semantics: the
    effective step grows with N).  A rank without a batch in the last round contributes zero gradients and still joins
    every collective.  Mean loss and accuracies are reduced over the ranks at the end of a pass, so every rank returns
    the same numbers.  Labels and mask are whole-graph on every rank.  The topology is either the whole graph as a
    single partition on every rank (the reference's FullyRepGraph), or a topology.ShardedTopology, of which each rank
    keeps only its own destinations' in-edges; the blocks, and so rounds, steps and collectives, are the same either
    way.  A topology sharded over N > 1 ranks needs a ShardedFeatureTable over the same ranks (its offsets may
    differ)."""

    def _init_rounds(self, partitioned_graph, layers, features, labels, mask, fanout, batch_size, sample_seed,
                     gather_dtype, include_dst, log_softmax_in_loss, retain_tape):
        """The set-up both models share.  What differs is passed in: include_dst for the sampler, log_softmax_in_loss
        (Forward returns logits, not log-probabilities) and retain_tape (self_backward's retain_graph)."""
        self.layers = list(layers)
        self.gather_dtype = ops._check_gather_dtype(gather_dtype)
        if len(fanout) != len(self.layers) - 1:
            raise _lib.NtsError("fanout needs one entry per layer (%d), got %d" % (len(self.layers) - 1, len(fanout)))
        self.batch_size = int(batch_size)
        if self.batch_size < 1:
            raise _lib.NtsError("batch_size must be >= 1")
        from .sample import NeighborSampler
        self.sampler = NeighborSampler(partitioned_graph, fanout, self.batch_size, include_dst=include_dst)
        self._init_features(features, self.sampler.V, partitioned_graph)
        self.sample_seed = int(sample_seed)
        self.step = 0
        self.ctx = NtsContext()
        self.L_GT = labels.to(self.device)
        mask = torch.as_tensor(mask).cpu()
        self.nids = [(mask == s).nonzero().view(-1) for s in (0, 1, 2)]    # train / val / test ids, ascending
        self.subgraph = None
        self.loss = None
        self.epoch = 0
        self._log_softmax_in_loss, self._retain_tape = log_softmax_in_loss, retain_tape

    def _init_features(self, features, vertices, topology):
        from .feature_table import ShardedFeatureTable
        from .topology import ShardedTopology
        if isinstance(topology, ShardedTopology) and topology.world > 1 and not (
                isinstance(features, ShardedFeatureTable) and features.world == topology.world
                and features.rank == topology.rank):
            raise _lib.NtsError("a topology sharded over %d ranks needs a ShardedFeatureTable over the same ranks"
                                % topology.world)
        if not isinstance(features, ShardedFeatureTable):
            self.table, self.rank, self.world = None, 0, 1
            self.features = ops._check_input(features.detach(), "features")
            self.device = features.device
            return
        if features.rows != vertices:
            raise _lib.NtsError("the feature table has %d rows, the graph has %d vertices" % (features.rows, vertices))
        if features.world != (dist.get_world_size() if dist.is_initialized() else 1):
            # Parameter reduces gradients over the default group
            raise _lib.NtsError("the feature table's group must span every rank of the default process group")
        self.table, self.features, self.device = features, None, features.device
        self.rank, self.world = features.rank, features.world

    @property
    def _learnable(self):
        from .feature_table import ShardedEmbedding
        return isinstance(self.table, ShardedEmbedding)

    def _input_rows(self, src, dtype=torch.float32, training=False):
        """Features of the sampled sources `src` (global ids of a block, from the sampler: in range), as float32 rows,
        or from a BF16 table with dtype=torch.bfloat16 as BF16 rows ([n, F] view of pitched rows).  Training on a
        ShardedEmbedding, the rows are a leaf that requires a gradient, kept with src for Update's embedding step."""
        if self.table is None:
            return self.features.index_select(0, src.long())
        x = self.table._gather(src, dtype)
        if training and self._learnable:
            x.requires_grad_(True)
            self._embedding_rows = (src, x)
        return x

    def _batches(self, ids):
        """The seeds this rank runs in each round of a pass over `ids` (None in a round without a batch for it); sets
        the step of every batch and leaves self.step at the next pass's base."""
        bs = self.batch_size
        n_batches = -(-ids.numel() // bs)
        base = self.step
        for t in range(-(-n_batches // self.world)):
            b = t * self.world + self.rank
            if b < n_batches:
                self.step = base + b
                yield ids[b * bs:(b + 1) * bs]
            else:
                yield None
        self.step = base + n_batches

    def _totals(self, *values):
        """The values (scalars or one-element tensors) summed over the ranks, as floats."""
        if self.world == 1:
            return [float(v) for v in values]
        dev = self.device if dist.get_backend(self.table.group) == "nccl" else torch.device("cpu")
        t = torch.tensor([float(v) for v in values], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.table.group)
        return t.tolist()

    def Update(self):
        """all_reduce_to_gradient, Adam and next() for every parameter.  At world 1 a parameter without a gradient is
        skipped; data-parallel, every rank reduces and steps every parameter (a missing gradient counts as zeros), so
        that the collectives are the same on every rank.  Then, on a ShardedEmbedding, one collective embedding step on
        every rank: the gradient rows of this round's deepest-hop sources, or an empty contribution from a rank without
        a batch."""
        _update(self.params(), self.world > 1)
        if self._learnable:
            rows, self._embedding_rows = getattr(self, "_embedding_rows", None), None
            if rows is not None and rows[1].grad is not None:
                self.table._step(rows[0], rows[1].grad)
            else:
                self.table._step(torch.empty(0, dtype=torch.int32, device=self.device),
                                 torch.empty((0, self.table.F), dtype=torch.float32, device=self.device))

    def Loss(self, out, seeds_dev):
        """GCN_CPU_SAMPLE.hpp:187-195: nll_loss over the batch's seeds, after log_softmax where Forward returns
        logits."""
        self.loss = torch.nn.functional.nll_loss(out.log_softmax(1) if self._log_softmax_in_loss else out,
                                                 self.L_GT.index_select(0, seeds_dev))
        self.ctx.appendNNOp(out, self.loss)
        return self.loss

    def train_step(self, seeds):
        """One batch: zero the gradients, sample, forward, loss, tape backward, Adam.  Returns (loss, correct)."""
        for p in self.params():
            p.zero_grad()
        self.ctx.train()
        out = self.Forward(seeds, True)
        seeds_dev = self.subgraph.seeds().long()
        loss = self.Loss(out, seeds_dev)
        correct = (out.argmax(1) == self.L_GT.index_select(0, seeds_dev)).sum()
        self.ctx.self_backward(self._retain_tape)
        self.Update()
        return loss.detach(), correct

    def evaluate(self, s):
        """Accuracy over mask == s from sampled forwards (no dropout, no update)."""
        self.ctx.eval()
        correct = torch.zeros((), dtype=torch.int64, device=self.device)
        ids = self.nids[s]
        with torch.no_grad():
            for seeds in self._batches(ids):
                if seeds is not None:
                    out = self.Forward(seeds, False)
                    correct += (out.argmax(1) == self.L_GT.index_select(0, self.subgraph.seeds().long())).sum()
        self.ctx.train()
        return self._totals(correct)[0] / max(ids.numel(), 1)

    def _own_csc(self):
        """(lo, hi, own_offsets, group, parts): this rank's destinations [lo, hi), the ownership offsets and process
        group the per-layer tables are built on, and the in-edge CSC pieces that cover [lo, hi) in order, as (rows,
        column offsets [n + 1] int32, row_indices, weight, edge_begin, edge_end), `rows` the piece's slice of [lo, hi)
        counted from lo - a ShardedTopology's shards held in this process (all of them after split()), or the slice
        [lo, hi) of the replicated single-partition CSC."""
        from .topology import ShardedTopology
        topo = self.sampler._graph
        group = None if self.table is None else self.table.group
        if isinstance(topo, ShardedTopology):
            if topo._buf is None:
                raise _lib.NtsError("the topology is closed")
            off = [int(o) for o in topo.offsets]
            mine = range(len(off) - 1) if topo.world == 1 else [topo.rank]
            lo, hi = off[mine[0]], off[mine[-1] + 1]
            parts = []
            for o in mine:
                col = _lib.borrowed(topo.shard_arrays[0][o], off[o + 1] - off[o] + 1, torch.int32, self.device)
                n_edges = int(col[-1])
                parts.append((slice(off[o] - lo, off[o + 1] - lo), col,
                              _lib.borrowed(topo.shard_arrays[1][o], n_edges, torch.int32, self.device),
                              _lib.borrowed(topo.shard_arrays[2][o], n_edges, torch.float32, self.device), 0, n_edges))
            return lo, hi, (off if topo.world > 1 else [0, off[-1]]), group, parts
        c_col, c_row, c_w = topo
        own = [0, self.sampler.V] if self.table is None else [int(o) for o in self.table.offsets]
        lo, hi = own[self.rank], own[self.rank + 1]
        col = c_col[lo:hi + 1]
        eb, ee = (int(e) & 0xFFFFFFFF for e in col[[0, -1]].tolist())
        return lo, hi, own, group, [(slice(0, hi - lo), col, c_row, c_w, eb, ee)]

    def evaluate_full(self, s):
        """Accuracy over mask == s from the model's infer(): each rank counts its own rows and the counts are summed
        over the ranks, so every rank returns the same number."""
        lo, out = self.infer()
        ids = self.nids[s].to(self.device)
        mine = ids[(ids >= lo) & (ids < lo + out.shape[0])]
        correct = (out.index_select(0, mine - lo).argmax(1) == self.L_GT.index_select(0, mine)).sum()
        return self._totals(correct)[0] / max(ids.numel(), 1)

    def run_epoch(self, test=True):
        """One pass over the train batches (one Adam step per round) and, with test=True, sampled validation and test
        forwards.  Returns (mean train loss, [train, val, test] accuracy) - val / test are None with test=False."""
        ids = self.nids[0]
        losses, correct = [], torch.zeros((), dtype=torch.int64, device=self.device)
        for seeds in self._batches(ids):
            if seeds is None:
                for p in self.params():
                    p.zero_grad()
                self.Update()
                continue
            loss, c = self.train_step(seeds)
            losses.append(loss)
            correct += c
        if self.world == 1:
            mean_loss = float(torch.stack(losses).mean()) if losses else float("nan")
            total = float(correct)
        else:
            n_batches = -(-ids.numel() // self.batch_size)
            loss_sum, total = self._totals(torch.stack(losses).double().sum() if losses else 0.0, correct)
            mean_loss = loss_sum / n_batches if n_batches else float("nan")
        acc = [total / max(ids.numel(), 1)]
        acc += [self.evaluate(1), self.evaluate(2)] if test else [None, None]
        self.epoch += 1
        return mean_loss, acc


class GCNSampleImpl(_SampledRounds):
    """Neighbour-sampled mini-batch GCN: toolkits/GCN_CPU_SAMPLE.hpp:150-289 (ALGORITHM:GCNSAMPLESINGLE) on the GPU.
    The train vertices (mask == 0), in id order, are cut into batches of `batch_size` seeds; each batch is sampled
    (sample.NeighborSampler, hop h with fanout[h]) and runs an L-layer GCN over hops L-1 .. 0 (layer l aggregates hop
    L-1-l with ops.MiniBatchFuseOp, then X.W, relu on hidden layers), log_softmax + nll_loss on the seeds, tape
    backward and one Adam step.  The first layer gathers straight from the [V, F] feature table.

    Deliberate differences from the reference (DESIGN.md §8): gradients are zeroed per batch (the reference zeroes once
    per epoch); validation and test forwards never step Adam; dropout applies only while training; the sampler is
    Floyd's algorithm on a counter hash, with sources ascending by global id.  Step t of a run samples with
    (seed, t): two runs with the same seeds sample the same blocks, bit for bit.  Losses and weights agree bit for bit
    only while no aggregation row is cut into three or more pieces by K1's edge quanta (rows longer than the quantum,
    at least 32 edges on small blocks); such rows sum in scheduling order and may differ in the last bits between
    runs (DESIGN.md §3 K8).

    features: the [V, F] tensor, or a feature_table.ShardedFeatureTable (float32 or bfloat16) for data-parallel rounds
    over its ranks (_SampledRounds); the first layer then gathers the deepest hop's distinct sources from the table
    once (nts_gather_rows_sharded, _bf16) and aggregates them on local ids with K1.  `partitioned_graph` is the whole
    graph as a single partition on every rank, or a topology.ShardedTopology (each rank keeps its own destinations'
    in-edges; the same blocks), which over N > 1 ranks needs a ShardedFeatureTable over the same ranks.

    gather_dtype=torch.bfloat16: every aggregation gathers BF16 rows with FP32 accumulation (ops.MiniBatchFuseOp's
    option, nts_segment_gather_sum_bf16); activations, weights and gradients stay float32.  Tensor features are then
    stored once as pitched BF16 rows [V, 8*ceil(F/8)] (the caller's tensor is left alone), which the first layer reads
    by global id; a BF16 table hands its rows over as BF16, a float32 table's gathered rows are rounded once.  With
    FP32 gathers a BF16 table's rows are widened exactly.  The reproducibility condition above holds as it is.

    features may be a feature_table.ShardedEmbedding: its gathered rows are then a leaf of the step, the tape also
    back-propagates the first aggregation (MiniBatchFuseOp on the deepest hop), and Update() sends the rows' gradient
    to the table (ShardedEmbedding._step) after the parameters' Adam, on every rank in every round.  Under BF16 gathers
    the rows are rounded by the operator as for a float32 table; their gradient stays float32."""

    def __init__(self, partitioned_graph, layers, features, labels, mask, fanout, batch_size, learn_rate=0.01,
                 weight_decay=0.0001, decay_rate=0.97, decay_epoch=100, drop_rate=0.5, seed=0, sample_seed=0,
                 gather_dtype=None):
        self._init_rounds(partitioned_graph, layers, features, labels, mask, fanout, batch_size, sample_seed,
                          gather_dtype, include_dst=False, log_softmax_in_loss=True, retain_tape=False)
        self.features16 = None
        if self.gather_dtype is not None and self.table is None:
            self.features16 = ops._bf16_rows(self.features, "minibatch_bf16_round")[:, :self.features.shape[1]]
        self.drop_rate = drop_rate
        self.P = _parameters(zip(self.layers, self.layers[1:]), seed, self.device, learn_rate, weight_decay,
                             (decay_rate, decay_epoch))

    def params(self):
        return self.P

    def Forward(self, seeds, training):
        """Sample the batch and run the layers; returns the last layer's [n_seeds, classes] output."""
        self.subgraph = sg = self.sampler.sample(seeds, self.sample_seed, self.step)
        self.step += 1
        L = len(self.layers) - 1
        if self.table is None:
            x = self.features if self.features16 is None else self.features16
        else:
            bf16 = self.gather_dtype is not None and self.table.dtype == torch.bfloat16
            x = self._input_rows(sg.blocks[L - 1].src, torch.bfloat16 if bf16 else torch.float32, training)
            if x.requires_grad:
                # a learnable table's rows: recorded as an NN entry ahead of the first aggregation, so that the tape
                # back-propagates that aggregation too (self_backward stops at a lone first graph op) and the rows'
                # gradient lands in x.grad
                self.ctx.appendNNOp(x, x)
        for l in range(L):
            hop = L - 1 - l
            if l != 0 and training and self.drop_rate > 0:
                dropped = torch.nn.functional.dropout(x, self.drop_rate, training=True)
                self.ctx.appendNNOp(x, dropped)
                x = dropped
            # the first layer's rows are contiguous float32 or pitched BF16 rows, which contiguous() would unpitch
            y = self.ctx.runGraphOp(_minibatch_op, sg, None, x if l == 0 else x.contiguous(), hop=hop,
                                    table=l == 0 and self.table is None, gather_dtype=self.gather_dtype)
            if l == L - 1:
                x = self.ctx.runVertexForward(lambda n, _l=l: self.P[_l].forward(n), y)
            else:
                x = self.ctx.runVertexForward(lambda n, _l=l: torch.relu(self.P[_l].forward(n)), y)
        return x

    @torch.no_grad()
    def infer(self):
        """Full-neighbour inference: collective over the ranks of the model's table.  Returns (lo, out), out the last
        layer's [hi - lo, classes] float32 outputs (before log_softmax, as Forward returns them) for the destinations
        [lo, hi) this rank owns: a ShardedTopology's, else the table's offsets, else [0, V).

        Layer l aggregates with the expectation of the sampled aggregation of its hop h = L-1-l, which keeps
        min(indeg(v), k_h) uniform in-edge slots of v:  X_{l+1} = relu(s ⊙ A (X_l W_l)), s_v = min(1, k_h / indeg(v))
        (1 when indeg(v) = 0), no relu on the last layer, no dropout.  With every fanout >= the largest in-degree it is
        the full-graph GCN.  A layer that narrows (F_out < F_in) computes H = X_own W_l on this rank first and
        aggregates H, otherwise it aggregates X and applies W_l after (GCN here has no bias: A(XW) = (AX)W).  The
        aggregated rows are read by global id from a ShardedFeatureTable (nts_segment_gather_sum_sharded): the
        features table itself for a widening first layer, otherwise one built for the layer from this rank's rows,
        storing float32 or, with gather_dtype=torch.bfloat16, BF16 rows.  Building such a table is the point after
        which every rank's rows are readable by its peers, and its close() the point after which no peer reads them
        any more; both are collective, and every table is closed before infer returns.  A rank without destinations
        joins every collective.  Neither the sampler, the step counter, the tape nor any gradient is touched."""
        from .feature_table import ShardedFeatureTable
        lo, hi, own, group, parts = self._own_csc()
        dtype = self.gather_dtype or torch.float32
        L = len(self.layers) - 1
        x = None
        for l in range(L):
            k = self.sampler.fanout[L - 1 - l]
            W = self.P[l].W.detach()
            narrows = self.layers[l + 1] < self.layers[l]
            if l == 0 and (narrows or self.table is None):
                x = self.features[lo:hi] if self.table is None else \
                    self.table.gather(np.arange(lo, hi), torch.float32)
            if narrows:
                src = ShardedFeatureTable(x.mm(W), own, group, dtype=dtype)
            elif l == 0 and self.table is not None:
                src = self.table
            else:
                src = ShardedFeatureTable(x.contiguous(), own, group, dtype=dtype)
            y = torch.zeros((hi - lo, src.F), dtype=torch.float32, device=self.device)
            scale = []
            for r, col, rows, w, eb, ee in parts:
                src.aggregate(y[r], col, rows, w, eb, ee)
                c = col.long() & 0xFFFFFFFF
                deg = (c[1:] - c[:-1]).double()
                scale.append(torch.where(deg > k, k / deg.clamp_min(1), torch.ones_like(deg)))
            if src is not self.table:
                src.close()
            y.mul_(torch.cat(scale).float().unsqueeze(1))
            if not narrows:
                y = y.mm(W)
            x = torch.relu(y) if l < L - 1 else y
        return lo, x


class GATImpl(_FullGraph):
    """Multi-head GAT on the fused aggregation path - the flow of toolkits/GAT_CPU_DIST_OPTM.hpp:196-241 (per-vertex
    attention scores -> [E, H] edge logits -> edge softmax -> DistAggregateDstFuseWeight) on the GPU operators, with
    H heads (the reference has one).  `layers` are total widths, e.g. [602, 64, 64, 41] with heads=8 gives hidden
    layers of 8 heads x 8 and a single-head output layer (config D of BASELINE.json).  Never materialises an [E, F]
    message; the only edge-sized tensors are [E, H].

    gather_dtype=torch.bfloat16 (needs fused_kernel=True and two_pass_backward=True): every fused layer gathers BF16
    mirror and gradient rows with FP32 accumulation (ops.DistGPUFusedGATOp's option).  The input features stay float32
    (they feed the first GEMM), and so do the mirror fetch, activations, weights and gradients.  A layer shape that
    either BF16 entry refuses (ops.gat_bf16_shape_error: e.g. 8 heads x 24) raises NtsError at construction."""

    def __init__(self, partitioned_graph, layers, features, labels, mask, heads=8, learn_rate=0.01,
                 weight_decay=0.0001, exchange=None, seed=0, sum_fanout_grads=True, fused_kernel=False,
                 two_pass_backward=True, gather_dtype=None):
        self.pg = partitioned_graph
        self.fused_kernel = fused_kernel  # True: K7 (ops.DistGPUFusedGATOp), no edge-sized tensors at all
        self.two_pass_backward = two_pass_backward
        self.gather_dtype = ops._check_gather_dtype(gather_dtype)
        if self.gather_dtype is not None and not (fused_kernel and two_pass_backward):
            raise _lib.NtsError("GATImpl gather_dtype needs fused_kernel=True and two_pass_backward=True")
        self.layers = list(layers)
        self.device = features.device
        self.heads = _gat_heads(self.layers, heads, self.gather_dtype)
        self.ctx = NtsContext(sum_fanout_grads=sum_fanout_grads)
        # GATImpl's Adam keeps its defaults: no learning-rate decay
        self.P, self.al, self.ar = _gat_parameters(self.layers, self.heads, seed, self.device, learn_rate,
                                                   weight_decay)
        if exchange is None:
            from .exchange import GpuExchange
            exchange = GpuExchange(partitioned_graph)
        self.exchange = exchange
        self.L_GT = labels.to(self.device)
        self.MASK = mask.to(self.device)
        self.train_rows = (self.MASK == 0).nonzero().view(-1)
        self.X = [None] * len(self.layers)
        self.X[0] = features.requires_grad_(True)
        self.loss = None
        self.epoch = 0

    def params(self):
        return self.P + self.al + self.ar

    def Forward(self):
        ctx, pg = self.ctx, self.pg
        for i in range(len(self.layers) - 1):
            last = i == len(self.layers) - 2
            X_trans = ctx.runVertexForward(lambda x, _i=i: self.P[_i].forward(x), self.X[i])
            mirror = ctx.runGraphOp(ops.DistGPUGetDepNbrOp, pg, None, X_trans.contiguous(), exchange=self.exchange)
            src_att = ctx.runVertexForward(lambda m, _i=i: _head_scores(m, self.al[_i].W), mirror)
            dst_att = ctx.runVertexForward(lambda x, _i=i: _head_scores(x, self.ar[_i].W), X_trans)
            if self.fused_kernel:
                nbr = ctx.runGraphOpN(ops.DistGPUFusedGATOp, pg, None, [mirror, src_att, dst_att],
                                      two_pass_backward=self.two_pass_backward, gather_dtype=self.gather_dtype)
            else:
                e_src = ctx.runGraphOp(ops.DistGPUScatterSrc, pg, None, src_att)
                e_dst = ctx.runGraphOp(ops.DistGPUScatterDst, pg, None, dst_att)
                e_msg = e_src + e_dst  # (the reference concatenates the two [E,1] columns and sums them, :218-224)
                m = ctx.runEdgeForward(lambda t: torch.nn.functional.leaky_relu(t, 0.2), e_msg)
                a = ctx.runGraphOp(ops.DistGPUEdgeSoftMax, pg, None, m)
                nbr = ctx.runGraphOp(ops.DistGPUAggregateDstFuseWeight, pg, None, mirror, a)
            if last:
                self.X[i + 1] = ctx.runVertexForward(lambda t: t.log_softmax(1), nbr)
            else:
                self.X[i + 1] = ctx.runVertexForward(lambda t: torch.relu(t), nbr)

    def run_epoch(self):
        if self.epoch != 0:
            for p in self.params():
                p.zero_grad()
        self.Forward()
        self.Loss()
        self.ctx.self_backward(True)
        self.Update()
        self.epoch += 1
        return self.loss


def _gat_heads(layers, heads, gather_dtype):
    """The heads of each layer: `heads` on the hidden layers, one on the output layer.  NtsError, before any device
    work, for a width that is not a multiple of its heads, and with BF16 gathers for the first layer whose shape a BF16
    K7 entry refuses (the backward has no fallback, so such a layer would otherwise run a whole forward and fail at its
    first backward)."""
    heads = [heads] * (len(layers) - 2) + [1]
    for i, H in enumerate(heads):
        if layers[i + 1] % H:
            raise _lib.NtsError("layer width %d is not a multiple of %d heads" % (layers[i + 1], H))
    if gather_dtype is not None:
        for i, H in enumerate(heads):
            why = ops.gat_bf16_shape_error(layers[i + 1], H)
            if why is not None:
                raise _lib.NtsError("layer %d (width %d, %d heads) cannot gather BF16 rows: %s"
                                    % (i, layers[i + 1], H, why))
    return heads


def _gat_parameters(layers, heads, seed, device, learn_rate, weight_decay, decay=None):
    """(P, al, ar): per layer the weight [in, H*D] and the source and destination attention vectors [H, D], drawn in
    the order W_l, al_l, ar_l, layer by layer."""
    shapes = []
    for i, H in enumerate(heads):
        shapes += [(layers[i], layers[i + 1]), (H, layers[i + 1] // H), (H, layers[i + 1] // H)]
    params = _parameters(shapes, seed, device, learn_rate, weight_decay, decay)
    return params[0::3], params[1::3], params[2::3]


def _head_scores(t, a):
    """Per-head scores <t[v, h], a[h]> of rows t [n, H*D] and attention vectors a [H, D], as a contiguous [n, H]."""
    return (t.view(-1, *a.shape) * a).sum(-1).contiguous()


def _minibatch_gat_op(sampled_subgraph, active, hop, gather_dtype=None):
    return ops.MiniBatchGATOp(sampled_subgraph, hop, gather_dtype=gather_dtype)


class GATSampleImpl(_SampledRounds):
    """Neighbour-sampled mini-batch multi-head GAT: GATImpl's layers on GCNSampleImpl's batch loop.  The train vertices
    (mask == 0), in id order, are cut into batches of `batch_size` seeds; each batch is sampled with
    NeighborSampler(..., include_dst=True), so that every hop's sources include its destinations, and runs the L layers
    over hops L-1 .. 0.  Layer l on hop h = L-1-l takes x [n_src, in] (the features of the hop's sources for l = 0,
    else the previous layer's output, whose rows are exactly this hop's sources), x_trans = x W_l, per-head scores
    src = <x_trans, al_l> and dst = <x_trans[dst_pos], ar_l>, and ops.MiniBatchGATOp (K7 on the block), then relu, or
    log_softmax on the last layer; nll_loss on the seeds, tape backward, one Adam step per parameter.  `layers` are
    total widths and the heads split as in GATImpl (hidden layers of `heads` heads, a single-head output layer);
    len(fanout) == len(layers) - 1.  No dropout, as in GATImpl.  gather_dtype=torch.bfloat16: K7 gathers BF16 rows
    with FP32 accumulation (ops.MiniBatchGATOp's option; hidden head widths must then be multiples of 8, and a layer
    shape that either BF16 entry refuses raises NtsError at construction, as in GATImpl).

    Reproducibility: step t of a run samples with (sample_seed, t), and a block is a pure function of (graph,
    sample_seed, t, seeds), so two runs see the same blocks bit for bit.  K7 splits the edges into quanta and finishes
    a row cut by a quantum boundary with atomic adds onto a zeroed row; two pieces give the same bits in either order,
    three or more may not.  The forward's quantum is a power of two of at least 32 edges (exactly 32 on small blocks:
    it shrinks until the grid fills the GPU), the statistics' is 512 and both backward passes' 256.  So losses and
    weights are bit-identical between runs while every fanout is at most 33 (a destination row of at most 33 edges
    spans at most two forward quanta), no source has more than 257 out-edges in a block (the backward's source-major
    pass), and no layer has a fallback shape of the backward (heads > 1 with a non-power-of-two head width in 4-float
    vectors, or rows wider than 128 vectors), which adds per edge with atomics.  Beyond these limits, rows may differ
    in the last bits between runs: fanouts of 34 to 64, hub sources of a large block (config B's deeper hops), fallback
    shapes.  On one H100, two Cora runs (1433-64-7, 8 heads, fanout 10-10, batch 64; the largest source has 17
    out-edges in a block) gave bit-identical losses and weights over three epochs with FP32 and with BF16 gathers
    (DESIGN.md §3 K8).

    features: the [V, F] tensor, or a feature_table.ShardedFeatureTable for data-parallel rounds over its ranks
    (_SampledRounds); the first layer then reads its sources' rows from the table (nts_gather_rows_sharded).  A
    bfloat16 table's rows are widened exactly to float32 (nts_gather_rows_sharded_bf16), since they feed x W.
    `partitioned_graph` is the whole graph as a single partition on every rank, or a topology.ShardedTopology as in
    GCNSampleImpl.  A feature_table.ShardedEmbedding is trained as in GCNSampleImpl (its rows' gradient reaches them
    through x W)."""

    def __init__(self, partitioned_graph, layers, features, labels, mask, fanout, batch_size, heads=8,
                 learn_rate=0.01, weight_decay=0.0001, decay_rate=0.97, decay_epoch=100, seed=0, sample_seed=0,
                 gather_dtype=None):
        self.heads = _gat_heads(list(layers), heads, ops._check_gather_dtype(gather_dtype))
        # Forward returns log-probabilities; the three NN segments of a layer share x_trans's autograd graph, so the
        # tape's backward keeps it until the last of them has run
        self._init_rounds(partitioned_graph, layers, features, labels, mask, fanout, batch_size, sample_seed,
                          gather_dtype, include_dst=True, log_softmax_in_loss=False, retain_tape=True)
        self.P, self.al, self.ar = _gat_parameters(self.layers, self.heads, seed, self.device, learn_rate,
                                                   weight_decay, (decay_rate, decay_epoch))

    def params(self):
        return self.P + self.al + self.ar

    def Forward(self, seeds, training=True):
        """Sample the batch and run the layers; returns the last layer's [n_seeds, classes] log-probabilities (the
        same with training=False: there is no dropout)."""
        self.subgraph = sg = self.sampler.sample(seeds, self.sample_seed, self.step)
        self.step += 1
        ctx = self.ctx
        L = len(self.layers) - 1
        x = None
        for l in range(L):
            hop = L - 1 - l
            b = sg.blocks[hop]
            if l == 0:
                x = self._input_rows(b.src, training=training)
            x_trans = ctx.runVertexForward(lambda t, _l=l: self.P[_l].forward(t), x)
            # the destination score reads the destinations' own rows; it is recorded before the source score, whose
            # input x_trans would otherwise chain onto x_trans's own tape entry (NtsContext.appendNNOp) and leave
            # d_x_trans without a producer to go to
            x_dst = x_trans.index_select(0, b.dst_pos.long())
            dst_att = ctx.runVertexForward(lambda t, _l=l: _head_scores(t, self.ar[_l].W), x_dst)
            src_att = ctx.runVertexForward(lambda t, _l=l: _head_scores(t, self.al[_l].W), x_trans)
            nbr = ctx.runGraphOpN(_minibatch_gat_op, sg, None, [x_trans, src_att, dst_att], hop=hop,
                                  gather_dtype=self.gather_dtype)
            if l == L - 1:
                x = ctx.runVertexForward(lambda t: t.log_softmax(1), nbr)
            else:
                x = ctx.runVertexForward(lambda t: torch.relu(t), nbr)
        return x

    @torch.no_grad()
    def infer(self):
        """Full-neighbour inference: collective over the ranks of the model's table.  Returns (lo, out), out the last
        layer's [hi - lo, classes] float32 log-probabilities (as Forward returns them) for the destinations [lo, hi)
        this rank owns: a ShardedTopology's, else the table's offsets, else [0, V).

        Layer l attends over every in-edge slot of each destination (a multi-edge counts once per slot, as the sampler
        counts it; edge weights are ignored, as in MiniBatchGATOp):  T = X_own W_l, s = <T, al_l>, d = <T, ar_l> per
        head, a[e, h] = softmax over the in-edge slots e of v of leaky_relu(s[src(e), h] + d[v, h], 0.2), Y[v, h] =
        sum_e a[e, h] T[src(e), h] (zero at in-degree 0), X_{l+1} = relu(Y), or log_softmax(Y) on the last layer; no
        dropout.  With every fanout >= the largest in-degree the sampled layer keeps every slot, so this is exactly
        Forward over all vertices and the full-graph GATImpl.  Unlike GCNSampleImpl.infer, there is no expectation to
        scale by: the sampled layer renormalises its softmax over the kept slots, a ratio estimator of this full
        softmax with no closed-form mean, and the full softmax is what it tends to as the fanouts grow.

        Every layer builds two ShardedFeatureTables from this rank's rows, T (float32, or BF16 with
        gather_dtype=torch.bfloat16; scores always come from the float32 T) and the float32 scores s, and aggregates
        each in-edge piece of [lo, hi) with ShardedFeatureTable.gat_aggregate (K10).  Building the tables is the point
        after which every rank's rows are readable by its peers, and their close() the point after which no peer
        reads them any more; both are collective.  A rank without destinations joins every collective.  A layer shape
        K10 refuses (feature_table.gat_shape_error) raises NtsError before the first collective, on every rank alike.
        Neither the sampler, the step counter, the tape nor any gradient is touched."""
        from .feature_table import ShardedFeatureTable, gat_shape_error
        dtype = self.gather_dtype or torch.float32
        for l, H in enumerate(self.heads):
            why = gat_shape_error(self.layers[l + 1], H, dtype)
            if why is not None:
                raise _lib.NtsError("layer %d cannot run full-neighbour inference: %s" % (l, why))
        lo, hi, own, group, parts = self._own_csc()
        x = self.features[lo:hi] if self.table is None else self.table.gather(np.arange(lo, hi), torch.float32)
        L = len(self.layers) - 1
        for l in range(L):
            H = self.heads[l]
            t = x.mm(self.P[l].W.detach())
            s = _head_scores(t, self.al[l].W.detach())
            d = _head_scores(t, self.ar[l].W.detach())
            rows = ShardedFeatureTable(t, own, group, dtype=dtype)
            scores = ShardedFeatureTable(s, own, group)
            y = torch.zeros((hi - lo, self.layers[l + 1]), dtype=torch.float32, device=self.device)
            for r, col, ids, _, eb, ee in parts:
                rows.gat_aggregate(y[r], scores, d[r], col, ids, eb, ee, H)
            rows.close()
            scores.close()
            x = torch.relu(y) if l < L - 1 else y.log_softmax(1)
        return lo, x

