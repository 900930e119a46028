"""Sampled mini-batch GAT on the GPU: ops.MiniBatchGATOp (K7 on a destination-inclusive sampled block) against float64
torch autograd of the same block, FP32 and BF16 gathers, one GATSampleImpl step against a float64 restatement of that
step, repeatability, and Cora accuracy against full-graph GATImpl."""
import numpy as np
import pytest

from test_gat_bf16 import layer_reference
from test_gather_plan_bf16 import cora_tables, row_close
from test_sample_gpu import cora_edges, dev, graph, zipf_hub_edges

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
# (H, D): single head at 8 and 64, 8 heads at 8 and 64, and config D's 41-wide single-head output layer
SHAPES = [(1, 8), (1, 64), (8, 8), (8, 64), (1, 41)]

_cache = {}


def hub_block():
    """Hop 0 of a destination-inclusive sample of the Zipf graph at fanout 64: hub destinations with 64 kept edges,
    repeated (destination, source) pairs from the graph's multi-edges, destinations that are their own sources."""
    if "hub" not in _cache:
        from neutronstarlite_b200.sample import NeighborSampler
        edges, V = zipf_hub_edges()
        pg = graph(edges, V)
        seeds = np.concatenate([[5, 77], np.arange(1000, 1510)])
        sg = NeighborSampler(pg, [64, 10], len(seeds), include_dst=True).sample(seeds, 3, 1).clone()
        b = sg.blocks[0].to_numpy()
        deg = np.diff(b["column_offset"].astype(np.int64))
        assert deg.max() == 64
        pairs = np.stack([np.repeat(np.arange(deg.size), deg), b["row_indices"].astype(np.int64)], 1)
        assert np.unique(pairs, axis=0).shape[0] < pairs.shape[0]        # multi-edges survive sampling
        _cache["hub"] = (sg, b)
    return _cache["hub"]


def operands(b, H, D, seed):
    d = dev()
    gen = torch.Generator().manual_seed(seed)
    n_src, n_dst, F = b["src"].size, b["dst"].size, H * D
    x = (torch.rand((n_src, F), generator=gen) * 2 - 1).to(d)
    s = (torch.rand((n_src, H), generator=gen) * 4 - 2).to(d)
    dsc = (torch.rand((n_dst, H), generator=gen) * 4 - 2).to(d)
    g = (torch.rand((n_dst, F), generator=gen) * 2 - 1).to(d)
    return x, s, dsc, g


def floor_close(actual, desired, rtol, floor=1e-2):
    """row_close with each row's scale floored at `floor` of the largest |desired| (score gradients are sums of
    terms of both signs; the FP32 rounding scales with the terms, not with their sum)."""
    a, r = actual.cpu().numpy(), desired.cpu().numpy()
    scale = np.maximum(np.abs(r).max(axis=1, keepdims=True), floor * np.abs(r).max())
    row_close(a, r, rtol=rtol, scale=scale)


@pytest.mark.parametrize("H,D", SHAPES)
def test_minibatch_gat_op_matches_float64_autograd(H, D):
    from neutronstarlite_b200 import ops
    sg, b = hub_block()
    x, s, dsc, g = operands(b, H, D, seed=H * 100 + D)
    op = ops.MiniBatchGATOp(sg, 0)
    out = op.forward(x, s, dsc)
    dx, ds, dd = op.backward(g)
    torch.cuda.synchronize()
    out_ref, dx_ref, ds_ref, dd_ref, out_mag, dx_mag = layer_reference(b["column_offset"], b["row_indices"], x, s,
                                                                       dsc, g, H)
    row_close(out.cpu().numpy(), out_ref.cpu().numpy(), rtol=1e-4, scale=out_mag.cpu().numpy())
    row_close(dx.cpu().numpy(), dx_ref.cpu().numpy(), rtol=1e-4, scale=dx_mag.cpu().numpy())
    floor_close(ds, ds_ref, 1e-4)
    floor_close(dd, dd_ref, 1e-4)


@pytest.mark.parametrize("H,D,dtype", [(8, 8, None), (1, 41, None), (8, 8, BF16), (1, 41, BF16)])
def test_minibatch_gat_op_is_bit_stable_at_fanout_33(H, D, dtype):
    """The documented limit of GATSampleImpl's reproducibility: with destination rows of at most 33 edges (at most two
    pieces of the forward's 32-edge quantum on small inputs) and sources of at most 257 out-edges (two pieces of the
    backward's 256-edge quantum), every output of K7 is the same bit for bit from call to call."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.sample import NeighborSampler
    pg = graph(cora_edges(), 2708)
    col = pg.graph_chunks[0].column_offset.astype(np.int64)
    indeg = np.diff(col)
    seeds = np.concatenate([np.nonzero(indeg >= 33)[0], np.arange(0, 2708, 5)])
    seeds = np.unique(seeds)
    sg = NeighborSampler(pg, [33], len(seeds), include_dst=True).sample(seeds, 2, 4).clone()
    b = sg.blocks[0].to_numpy()
    deg = np.diff(b["column_offset"].astype(np.int64))
    start = b["column_offset"][:-1].astype(np.int64)
    assert deg.max() == 33 and ((deg == 33) & (start % 32 != 0)).sum() >= 5     # rows really cut by a boundary
    assert np.diff(b["row_offset"].astype(np.int64)).max() <= 257
    x, s, dsc, g = operands(b, H, D, seed=7)
    runs = []
    for _ in range(3):
        op = ops.MiniBatchGATOp(sg, 0, gather_dtype=dtype)
        runs.append((op.forward(x, s, dsc),) + tuple(op.backward(g)))
    for r in runs[1:]:
        for a, c in zip(runs[0], r):
            assert torch.equal(a, c)


@pytest.mark.parametrize("H,D", [(1, 8), (1, 64), (8, 8), (8, 64), (1, 41), (2, 16)])
def test_minibatch_gat_op_bf16_matches_float64_at_rounded_operands(H, D):
    from neutronstarlite_b200 import ops
    sg, b = hub_block()
    x, s, dsc, g = operands(b, H, D, seed=H * 10 + D)
    op = ops.MiniBatchGATOp(sg, 0, gather_dtype=BF16)
    out = op.forward(x, s, dsc)
    dx, ds, dd = op.backward(g)
    torch.cuda.synchronize()
    xt, gt = x.to(BF16).float(), g.to(BF16).float()
    out_ref, dx_ref, ds_ref, dd_ref, out_mag, dx_mag = layer_reference(b["column_offset"], b["row_indices"], xt, s,
                                                                       dsc, gt, H)
    row_close(out.cpu().numpy(), out_ref.cpu().numpy(), scale=out_mag.cpu().numpy())
    row_close(dx.cpu().numpy(), dx_ref.cpu().numpy(), scale=dx_mag.cpu().numpy())
    torch.testing.assert_close(ds, ds_ref.float(), rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(dd, dd_ref.float(), rtol=1e-3, atol=2e-5)


def test_minibatch_gat_op_refuses_bad_blocks_and_shapes():
    from neutronstarlite_b200 import _lib, ops
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    pg = graph(cora_edges(), 2708)
    plain = NeighborSampler(pg, [5], 64).sample(np.arange(20), 0, 0)
    with pytest.raises(_lib.NtsError, match="dst_pos"):
        ops.MiniBatchGATOp(plain, 0)
    sg = NeighborSampler(pg, [5], 64, include_dst=True).sample(np.arange(20), 0, 0)
    b = sg.blocks[0]
    op = ops.MiniBatchGATOp(sg, 0)
    x, s, dsc = torch.rand((b.n_src, 16), device=d), torch.rand((b.n_src, 2), device=d), torch.rand((20, 2), device=d)
    for args in ((x[:-1], s[:-1], dsc), (x, s, dsc[:-1]), (x, s[:-1], dsc)):
        with pytest.raises(_lib.NtsError):
            op.forward(*args)
    op.forward(x, s, dsc)
    with pytest.raises(_lib.NtsError):
        op.backward(torch.rand((19, 16), device=d))
    # BF16 with heads > 1 and D % 8 != 0: the full-graph op's refusal, word for word
    from test_gat_bf16 import hub_layer_graph
    fpg, _, _ = hub_layer_graph(3, 5)
    with pytest.raises(_lib.NtsError) as full:
        ops.DistGPUFusedGATOp(fpg, gather_dtype=BF16).forward(
            torch.rand((fpg.owned_mirrors, 15), device=d), torch.rand((fpg.owned_mirrors, 3), device=d),
            torch.rand((fpg.owned_vertices, 3), device=d))
    with pytest.raises(_lib.NtsError) as mine:
        ops.MiniBatchGATOp(sg, 0, gather_dtype=BF16).forward(torch.rand((b.n_src, 15), device=d),
                                                             torch.rand((b.n_src, 3), device=d),
                                                             torch.rand((20, 3), device=d))
    assert str(mine.value) == str(full.value)
    # a block without edges launches nothing, and still refuses that shape in the same words
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    lone = PartitionedGraph(HostGraph(np.array([[1, 0]], dtype=np.uint32), 3), 1, 0).generate_all(device=d)
    sg0 = NeighborSampler(lone, [5], 4, include_dst=True).sample(np.array([2]), 0, 0)
    assert sg0.blocks[0].n_edges == 0
    with pytest.raises(_lib.NtsError) as empty:
        ops.MiniBatchGATOp(sg0, 0, gather_dtype=BF16).forward(torch.rand((1, 15), device=d),
                                                              torch.rand((1, 3), device=d), torch.rand((1, 3), device=d))
    assert str(empty.value) == ops.BF16_HEAD_WIDTH_ERROR and ops.BF16_HEAD_WIDTH_ERROR in str(full.value)
    assert torch.equal(ops.MiniBatchGATOp(sg0, 0, gather_dtype=BF16).forward(
        torch.ones((1, 16), device=d), torch.ones((1, 2), device=d), torch.ones((1, 2), device=d)),
        torch.zeros((1, 16), device=d))


def float64_step(blocks, feats, labels, params, heads, layers, slope=0.2):
    """One GATSampleImpl step restated in float64 torch autograd on host copies of its blocks: edge-list softmax with
    max subtraction.  Returns the loss and the gradients of (W, al, ar) of every layer."""
    dv = feats.device
    dd = torch.float64
    leaves = [p.detach().to(dd).requires_grad_(True) for p in params]
    L = len(layers) - 1
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dv)
    x = None
    for l in range(L):
        b = blocks[L - 1 - l]
        W, al, ar = leaves[l], leaves[L + l], leaves[2 * L + l]
        H = heads[l]
        D = layers[l + 1] // H
        if l == 0:
            x = feats.to(dd)[t(b["src"])]
        xt = x @ W
        s = (xt.view(-1, H, D) * al).sum(-1)
        dsc = (xt[t(b["dst_pos"])].view(-1, H, D) * ar).sum(-1)
        n_dst = b["dst"].size
        dst = torch.repeat_interleave(torch.arange(n_dst, device=dv), t(np.diff(b["column_offset"].astype(np.int64))))
        src = t(b["row_indices"])
        logit = torch.nn.functional.leaky_relu(s[src] + dsc[dst], slope)
        mx = torch.full((n_dst, H), -float("inf"), dtype=dd, device=dv).scatter_reduce(
            0, dst[:, None].expand(-1, H), logit.detach(), "amax")
        ex = torch.exp(logit - mx[dst])
        a = ex / torch.zeros((n_dst, H), dtype=dd, device=dv).index_add(0, dst, ex)[dst]
        out = torch.zeros((n_dst, H, D), dtype=dd, device=dv).index_add(
            0, dst, xt[src].view(-1, H, D) * a[:, :, None]).reshape(n_dst, H * D)
        x = out.log_softmax(1) if l == L - 1 else torch.relu(out)
    loss = torch.nn.functional.nll_loss(x, labels[t(blocks[0]["dst"])])
    loss.backward()
    return loss.detach(), [p.grad for p in leaves]


def small_model(layers, heads, fanout, batch, **kw):
    from neutronstarlite_b200.toolkits import GATSampleImpl
    d = dev()
    edges, V = zipf_hub_edges(V=5000, E=60000)
    pg = graph(edges, V)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = torch.arange(V) % 3
    return GATSampleImpl(pg, layers, feats, labels, mask, fanout=fanout, batch_size=batch, heads=heads, **kw), \
        feats, labels


def test_training_step_matches_float64_torch():
    layers, heads = [37, 32, 5], 4
    model, feats, labels = small_model(layers, heads, [8, 12], 128)
    ids = model.nids[0]
    for step in range(2):
        params = [p.W.detach().clone() for p in model.params()]
        loss, _ = model.train_step(ids[step * 128:(step + 1) * 128])
        blocks = [b.to_numpy() for b in model.subgraph.blocks]
        ref_loss, ref_grads = float64_step(blocks, feats, labels, params, model.heads, layers)
        torch.testing.assert_close(loss.double(), ref_loss, rtol=1e-5, atol=0)
        for p, g in zip(model.params(), ref_grads):
            scale = float(g.abs().max())
            torch.testing.assert_close(p.W_gradient.double(), g, rtol=1e-5, atol=1e-5 * scale)


def test_two_runs_with_the_same_seeds_sample_the_same_blocks_and_agree():
    runs = []
    for _ in range(2):
        model, _, _ = small_model([37, 16, 5], 2, [10, 10], 256)
        loss, acc = model.run_epoch(test=False)
        runs.append((loss, [b.to_numpy() for b in model.subgraph.blocks], [p.W.detach().clone() for p in model.P]))
    for a, b in zip(runs[0][1], runs[1][1]):
        for k in a:
            assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
    assert abs(runs[0][0] - runs[1][0]) <= 1e-5 * abs(runs[0][0])
    for a, b in zip(runs[0][2], runs[1][2]):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-6)


def test_sampled_gat_reaches_full_graph_gat_accuracy_on_cora():
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl, GATSampleImpl
    d = dev()
    feats, labels, masks = cora_tables()
    layers = [1433, 64, 7]
    pg = graph(cora_edges(), 2708)
    torch.manual_seed(0)
    m = GATSampleImpl(pg, layers, torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                      torch.from_numpy(masks), fanout=[10, 10], batch_size=64, heads=8, seed=0, sample_seed=0)
    for _ in range(20):
        loss, _ = m.run_epoch(test=False)
    sampled = m.evaluate(2)
    fpg = PartitionedGraph(HostGraph(cora_edges(), 2708), 1, 0).generate_all(device=d, dist=True)
    torch.manual_seed(0)
    full = GATImpl(fpg, layers, torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                   torch.from_numpy(masks).to(d), heads=8, seed=0, fused_kernel=True)
    for _ in range(20):
        full.run_epoch()
    full.Forward()                          # the forward after 20 updates
    test = torch.from_numpy(masks).to(d) == 2
    full_acc = float((full.X[-1].argmax(1) == full.L_GT)[test].float().mean())
    assert np.isfinite(loss)
    assert sampled >= full_acc - 0.05, (sampled, full_acc)
