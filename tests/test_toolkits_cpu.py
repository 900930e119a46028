"""Host logic of the callers (tape + toolkit mirrors) on CPU: the graph operators are replaced IN THE TEST by plain
torch index ops (same forward/backward contracts), so that `NtsContext` / `GCNImpl` / `GATImpl` can be checked against
torch autograd without a GPU.  The CUDA operators themselves are checked in tests/test_gpu_*.py."""
import numpy as np
import pytest
import torch

from neutronstarlite_b200 import ops
from neutronstarlite_b200.graph import HostGraph, PartitionedGraph


class FakePG:
    """whole-partition CSC as torch CPU tensors"""

    def __init__(self, V, E, seed):
        rng = np.random.default_rng(seed)
        e = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.uint32)
        e = np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1).astype(np.uint32)])
        pg = PartitionedGraph(HostGraph(e, V), 1, 0).generate_all(dist=True)
        self.pg = pg
        self.col = torch.from_numpy(pg.column_offset.astype(np.int64))
        self.src = torch.from_numpy(pg.row_indices.astype(np.int64))
        self.mi = torch.from_numpy(pg.MirrorIndex.astype(np.int64))
        self.dst = torch.repeat_interleave(torch.arange(V), self.col[1:] - self.col[:-1])
        self.slot = self.mi[self.src]
        self.M = pg.owned_mirrors
        self.V = V
        c = pg.graph_chunks[0]
        self.w = torch.from_numpy(c.edge_weight_forward)
        self.csc_src = torch.from_numpy(c.row_indices.astype(np.int64))
        self.active = torch.nonzero(self.mi[1:] != self.mi[:-1]).view(-1)


@pytest.fixture
def fake_ops(monkeypatch):
    G = FakePG(120, 900, 11)

    def nograd(fn):
        # the real operators run outside autograd and hand back fresh leaf tensors
        def wrapped(self, *a):
            with torch.no_grad():
                return fn(self, *[t.detach() if isinstance(t, torch.Tensor) else t for t in a]).detach()
        return wrapped

    def patch(cls, fwd, bwd, extra=None):
        monkeypatch.setattr(cls, "__init__", lambda self, pg, active=None, **kw: None)
        monkeypatch.setattr(cls, "forward", nograd(fwd))
        monkeypatch.setattr(cls, "backward", nograd(bwd))
        if extra:
            monkeypatch.setattr(cls, "get_additional_grad", extra)

    patch(ops.ForwardSingleGPUfuseOp,
          lambda self, x, x2=None: torch.zeros(G.V, x.shape[1]).index_add_(0, G.dst, x[G.csc_src] * G.w[:, None]),
          lambda self, g: torch.zeros(G.V, g.shape[1]).index_add_(0, G.csc_src, g[G.dst] * G.w[:, None]))
    patch(ops.DistGPUGetDepNbrOp,
          lambda self, x, x2=None: x[G.active].clone(),
          lambda self, g: torch.zeros(G.V, g.shape[1]).index_add_(0, G.active, g))
    patch(ops.DistGPUScatterSrc,
          lambda self, x, x2=None: x[G.slot].clone(),
          lambda self, g: torch.zeros(G.M, g.shape[1]).index_add_(0, G.slot, g))
    patch(ops.DistGPUScatterDst,
          lambda self, x, x2=None: x[G.dst].clone(),
          lambda self, g: torch.zeros(G.V, g.shape[1]).index_add_(0, G.dst, g))

    def sm_fwd(self, m, x2=None):
        H = m.shape[1]
        mx = torch.full((G.V, H), -float("inf")).scatter_reduce(0, G.dst[:, None].expand(-1, H), m, "amax")
        ex = torch.exp(m - mx[G.dst])
        den = torch.zeros(G.V, H).index_add_(0, G.dst, ex)
        self._a = ex / den[G.dst]
        return self._a.clone()

    def sm_bwd(self, g):
        a = self._a
        dot = torch.zeros(G.V, g.shape[1]).index_add_(0, G.dst, a * g)
        return a * g - a * dot[G.dst]
    patch(ops.DistGPUEdgeSoftMax, sm_fwd, sm_bwd)

    def fw_fwd(self, mirror, a):
        H = a.shape[1]
        D = mirror.shape[1] // H
        self._m, self._aw = mirror, a
        msg = mirror[G.slot].view(-1, H, D) * a[:, :, None]
        return torch.zeros(G.V, H, D).index_add_(0, G.dst, msg).reshape(G.V, H * D)

    def fw_bwd(self, g):
        H = self._aw.shape[1]
        D = g.shape[1] // H
        gd = g[G.dst].view(-1, H, D)
        self._dw = (self._m[G.slot].view(-1, H, D) * gd).sum(-1)
        return torch.zeros(G.M, H, D).index_add_(0, G.slot, gd * self._aw[:, :, None]).reshape(G.M, H * D)
    patch(ops.DistGPUAggregateDstFuseWeight, fw_fwd, fw_bwd, lambda self: self._dw)

    # K7 stand-in: same contract as ops.DistGPUFusedGATOp, gradients from a local autograd graph
    def fg_fwd(self, mirror, s, d):
        with torch.enable_grad():
            m_, s_, d_ = (t.detach().clone().requires_grad_(True) for t in (mirror, s, d))
            H = s.shape[1]
            D = mirror.shape[1] // H
            lg = torch.nn.functional.leaky_relu(s_[G.slot] + d_[G.dst], 0.2)
            mx = torch.full((G.V, H), -float("inf")).scatter_reduce(0, G.dst[:, None].expand(-1, H), lg.detach(), "amax")
            ex = torch.exp(lg - mx[G.dst])
            a = ex / torch.zeros(G.V, H).index_add_(0, G.dst, ex)[G.dst]
            out = torch.zeros(G.V, H, D).index_add_(0, G.dst, m_[G.slot].view(-1, H, D) * a[:, :, None]).reshape(G.V, H * D)
        self._g = (m_, s_, d_, out)
        return out.detach()

    def fg_bwd(self, g):
        m_, s_, d_, out = self._g
        return torch.autograd.grad(out, (m_, s_, d_), g.detach())
    monkeypatch.setattr(ops.DistGPUFusedGATOp, "__init__", lambda self, pg, active=None, **kw: None)
    monkeypatch.setattr(ops.DistGPUFusedGATOp, "forward", fg_fwd)
    monkeypatch.setattr(ops.DistGPUFusedGATOp, "backward", fg_bwd)
    return G


def _ref_gcn(G, layers, feats, labels, mask, Ws):
    agg = lambda x: torch.zeros(G.V, x.shape[1]).index_add_(0, G.dst, x[G.csc_src] * G.w[:, None])
    h = torch.relu(agg(feats) @ Ws[0])
    out = (agg(h) @ Ws[1]).log_softmax(1)
    tr = (mask == 0).nonzero().view(-1)
    return torch.nn.functional.nll_loss(out[tr], labels[tr])


def _ref_gat(G, layers, heads, feats, labels, mask, Ws, als, ars):
    x = feats
    for i in range(len(layers) - 1):
        H = heads[i]
        D = layers[i + 1] // H
        xt = (x @ Ws[i]).view(-1, H, D)
        m = torch.nn.functional.leaky_relu((xt * als[i]).sum(-1)[G.src] + (xt * ars[i]).sum(-1)[G.dst], 0.2)
        mx = torch.full((G.V, H), -float("inf")).scatter_reduce(0, G.dst[:, None].expand(-1, H), m, "amax")
        ex = torch.exp(m - mx[G.dst])
        a = ex / torch.zeros(G.V, H).index_add_(0, G.dst, ex)[G.dst]
        out = torch.zeros(G.V, H, D).index_add_(0, G.dst, xt[G.src] * a[:, :, None]).reshape(G.V, H * D)
        x = out.log_softmax(1) if i == len(layers) - 2 else torch.relu(out)
    tr = (mask == 0).nonzero().view(-1)
    return torch.nn.functional.nll_loss(x[tr], labels[tr])


def _data(V, F, C):
    gen = torch.Generator().manual_seed(0)
    feats = torch.rand((V, F), generator=gen) * 2 - 1
    labels = torch.randint(0, C, (V,), generator=gen)
    mask = torch.arange(V) % 3
    return feats, labels, mask


def test_gcn_tape_matches_autograd(fake_ops):
    from neutronstarlite_b200.toolkits import GCNImpl
    G = fake_ops
    layers = [19, 8, 4]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    model = GCNImpl(G.pg, layers, feats.clone(), labels, mask, drop_rate=0.0, op_class=ops.ForwardSingleGPUfuseOp)
    Ws = [p.W.detach().clone().requires_grad_(True) for p in model.P]
    ref = _ref_gcn(G, layers, feats, labels, mask, Ws)
    ref.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref)
    for p, W in zip(model.P, Ws):
        torch.testing.assert_close(p.W.grad, W.grad, rtol=1e-4, atol=1e-6)
    model.Update()
    loss2, _ = model.run_epoch()
    assert torch.isfinite(loss2)


def test_gcn_eager_tape_matches_autograd(fake_ops):
    """Transform-then-aggregate flow of GCN_EAGER_single.hpp: every aggregation is back-propagated."""
    from neutronstarlite_b200.toolkits import GCNEagerImpl
    G = fake_ops
    layers = [19, 8, 4]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    model = GCNEagerImpl(G.pg, layers, feats.clone(), labels, mask, drop_rate=0.0,
                         op_class=ops.ForwardSingleGPUfuseOp)
    Ws = [p.W.detach().clone().requires_grad_(True) for p in model.P]
    agg = lambda x: torch.zeros(G.V, x.shape[1]).index_add_(0, G.dst, x[G.csc_src] * G.w[:, None])
    out = agg(torch.relu(agg(feats @ Ws[0])) @ Ws[1]).log_softmax(1)
    tr = (mask == 0).nonzero().view(-1)
    ref = torch.nn.functional.nll_loss(out[tr], labels[tr])
    ref.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref)
    for p, W in zip(model.P, Ws):
        torch.testing.assert_close(p.W.grad, W.grad, rtol=1e-4, atol=1e-6)
    model.Update()
    loss2, _ = model.run_epoch()
    assert torch.isfinite(loss2)


@pytest.mark.parametrize("fused_kernel", [False, True])
@pytest.mark.parametrize("heads", [1, 4])
def test_gat_tape_matches_autograd(fake_ops, heads, fused_kernel):
    from neutronstarlite_b200.toolkits import GATImpl
    G = fake_ops
    layers = [13, 16, 8, 5]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    model = GATImpl(G.pg, layers, feats.clone(), labels, mask, heads=heads, exchange=object(), sum_fanout_grads=True,
                    fused_kernel=fused_kernel)
    clone = lambda ps: [p.W.detach().clone().requires_grad_(True) for p in ps]
    Ws, als, ars = clone(model.P), clone(model.al), clone(model.ar)
    ref = _ref_gat(G, layers, model.heads, feats, labels, mask, Ws, als, ars)
    ref.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref)
    for mine, r in zip(model.P + model.al + model.ar, Ws + als + ars):
        torch.testing.assert_close(mine.W.grad, r.grad, rtol=1e-4, atol=1e-6)


def test_reference_tape_drops_the_fanout_gradient(fake_ops):
    """Documented reference behaviour (ntsContext.hpp:289-291): without sum_fanout_grads the gradient that reaches the
    mirror matrix through the attention scores is overwritten by the aggregation's gradient."""
    from neutronstarlite_b200.toolkits import GATImpl
    G = fake_ops
    layers = [13, 8, 5]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    grads = []
    for flag in (False, True):
        model = GATImpl(G.pg, layers, feats.clone(), labels, mask, heads=2, exchange=object(), sum_fanout_grads=flag)
        model.Forward()
        model.Loss()
        model.ctx.self_backward(True)
        grads.append(model.P[0].W.grad.clone())
    assert not torch.allclose(grads[0], grads[1])


def test_gat_refuses_a_width_that_is_not_a_multiple_of_its_heads(fake_ops):
    """An NtsError, as GATSampleImpl raises it (not an assert, which python -O strips), before any device work."""
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.toolkits import GATImpl
    G = fake_ops
    layers = [13, 12, 5]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    with pytest.raises(_lib.NtsError, match="layer width 12 is not a multiple of 8 heads"):
        GATImpl(G.pg, layers, feats, labels, mask, heads=8, exchange=object())


@pytest.mark.parametrize("eager", [False, True])
def test_input_buffer_can_be_swapped_between_epochs(fake_ops, eager):
    """A host-fed trainer alternates two input buffers (bench.py's end-to-end leg): same losses as a resident input."""
    import time
    from neutronstarlite_b200.toolkits import GCNEagerImpl, GCNImpl
    G = fake_ops
    layers = [19, 8, 4]
    feats, labels, mask = _data(G.V, layers[0], layers[-1])
    cls = GCNEagerImpl if eager else GCNImpl
    a = cls(G.pg, layers, feats.clone(), labels, mask, drop_rate=0.0, op_class=ops.ForwardSingleGPUfuseOp)
    b = cls(G.pg, layers, feats.clone(), labels, mask, drop_rate=0.0, op_class=ops.ForwardSingleGPUfuseOp)
    bufs = [feats.clone(), feats.clone()]
    t0 = time.perf_counter()
    for k in range(4):
        b.X[0] = bufs[k & 1] if eager else bufs[k & 1].requires_grad_(True)
        la, _ = a.run_epoch()
        lb, _ = b.run_epoch()
        torch.testing.assert_close(la, lb)
    assert time.perf_counter() - t0 < 20


def test_slot_indices_and_slot_csr_on_reference_partitions(golden):
    """Setup-time index structures of the fused GAT layer (torch ops, device-agnostic) on the reference's own
    whole-partition CSC + MirrorIndex at P = 1, 2, 4, 8: the slot CSR must list exactly the CSC's edges, keyed by
    mirror slot, and every mirror slot must own at least one edge."""
    import types
    g = golden
    for r in range(g.P):
        pg = types.SimpleNamespace()
        pg.column_offset_gpu = torch.from_numpy(g.get(r, "whole_column_offset").astype(np.int32))
        pg.row_indices_gpu = torch.from_numpy(g.get(r, "whole_row_indices").astype(np.int32))
        pg.mirror_index_gpu = torch.from_numpy(g.get(r, "mirror_index").astype(np.int32))
        meta = g.get(r, "meta")
        pg.owned_vertices, pg.owned_edges, pg.owned_mirrors = int(meta[4]), int(meta[5]), int(meta[6])
        slots = ops.DistGPUFusedGATOp.slot_indices(pg)
        assert slots.dtype == torch.int32 and slots.numel() == pg.owned_edges
        if pg.owned_edges == 0:
            continue
        assert int(slots.max()) < pg.owned_mirrors and int(slots.min()) >= 0
        off, dst = ops.DistGPUFusedGATOp.slot_csr(pg)
        off, dst = off.long(), dst.long()
        assert off.numel() == pg.owned_mirrors + 1 and int(off[0]) == 0 and int(off[-1]) == pg.owned_edges
        assert bool((off[1:] > off[:-1]).all()), "a mirror slot without edges"
        col = pg.column_offset_gpu.long()
        csc_dst = torch.repeat_interleave(torch.arange(pg.owned_vertices), col[1:] - col[:-1])
        csc_pairs = torch.sort(slots.long() * pg.owned_vertices + csc_dst).values
        csr_slot = torch.repeat_interleave(torch.arange(pg.owned_mirrors), off[1:] - off[:-1])
        csr_pairs = torch.sort(csr_slot * pg.owned_vertices + dst).values
        assert torch.equal(csc_pairs, csr_pairs)
