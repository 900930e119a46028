"""The neighbour sampler (K8), MiniBatchFuseOp and GCNSampleImpl on the GPU: blocks bit-exact against the numpy
restatement (tests/sample_oracle.py), the operator against float64 torch, a training step against a float64 torch
restatement of the same step, determinism, accuracy on Cora, and the argument errors."""
import numpy as np
import pytest

import golden_store
import sample_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

KEYS = ("dst", "column_offset", "row_indices", "row_global", "weight", "src", "row_offset", "column_indices",
        "weight_backward")


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def cora_edges(self_loops=True):
    e = golden_store.load("cora_self_P1_F8")["edges"]
    return e if self_loops else e[e[:, 0] != e[:, 1]]


def zipf_hub_edges(V=60000, E=400000, seed=1):
    """Power-law sources, two hub destinations with 20 000 and 12 000 in-edges (multi-edges included)."""
    rng = np.random.default_rng(seed)
    src = np.minimum(rng.zipf(1.6, E) - 1, V - 1)
    dst = rng.integers(0, V, E)
    dst[:20000] = 5
    dst[20000:32000] = 77
    return np.stack([src, dst], 1).astype(np.uint32), V


def graph(edges, V):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    return PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev())


def check_against_oracle(pg, seeds, fanout, seed, step):
    from neutronstarlite_b200.sample import NeighborSampler
    c = pg.graph_chunks[0]
    s = NeighborSampler(pg, fanout, max(len(seeds), 1))
    sg = s.sample(seeds, seed, step)
    ref = so.sample(c.column_offset, c.row_indices, c.edge_weight_forward, seeds, fanout, seed, step)
    assert sg.hops == len(fanout)
    for h, (b, r) in enumerate(zip(sg.blocks, ref)):
        got = b.to_numpy()
        for k in KEYS:
            assert got[k].dtype == r[k].dtype, (h, k)
            assert np.array_equal(got[k].view(np.uint32), r[k].view(np.uint32)), "hop %d %s differs" % (h, k)
    return ref


CORA_CASES = [([1, 1], 0, 0), ([64, 64], 1, 3), ([5, 10], 2, 7), ([25, 10, 3], 3, 1), ([64, 2, 64], 4, 12)]


@pytest.mark.parametrize("self_loops", [True, False])
@pytest.mark.parametrize("fanout,seed,step", CORA_CASES)
def test_sampler_matches_numpy_on_cora(self_loops, fanout, seed, step):
    edges = cora_edges(self_loops)
    if not self_loops:
        edges = edges[edges[:, 1] >= 10]         # vertices 0..9 keep no in-edge: zero-in-degree destinations
    pg = graph(edges, 2708)
    rng = np.random.default_rng(seed)
    seeds = np.concatenate([np.arange(12), rng.choice(np.arange(12, 2708), 300, replace=False)])
    ref = check_against_oracle(pg, seeds, fanout, seed, step)
    if not self_loops:
        assert (np.diff(ref[0]["column_offset"].astype(np.int64))[:10] == 0).all()


@pytest.mark.parametrize("fanout,seed,step", [([1, 1], 0, 0), ([64, 64], 5, 2), ([25, 10], 6, 9),
                                              ([10, 5, 3], 7, 4)])
def test_sampler_matches_numpy_on_a_zipf_graph_with_hubs(fanout, seed, step):
    edges, V = zipf_hub_edges()
    pg = graph(edges, V)
    assert int(np.diff(pg.graph_chunks[0].column_offset.astype(np.int64)).max()) > 10 ** 4
    rng = np.random.default_rng(seed)
    seeds = np.concatenate([[5, 77, 0, 1], rng.choice(np.arange(100, V), 1020, replace=False)])
    check_against_oracle(pg, seeds, fanout, seed, step)


def test_empty_seed_list_gives_empty_blocks():
    pg = graph(cora_edges(), 2708)
    ref = check_against_oracle(pg, np.zeros(0, dtype=np.int64), [5, 10], 0, 0)
    assert all(r["row_indices"].size == 0 for r in ref)


def dense_agg(col, idx, w, x):
    """float64 Y[d] = sum_e w_e x[idx_e] with torch index_add_ (col, idx, w as device tensors)."""
    n = col.numel() - 1
    e_dst = torch.repeat_interleave(torch.arange(n, device=x.device), (col[1:] - col[:-1]).long())
    out = torch.zeros((n, x.shape[1]), dtype=torch.float64, device=x.device)
    out.index_add_(0, e_dst, x.double()[idx.long()] * w.double()[:, None])
    return out


def test_minibatch_op_against_float64_and_the_table_gather():
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.sample import NeighborSampler, SampledSubgraph
    d = dev()
    edges, V = zipf_hub_edges()
    pg = graph(edges, V)
    sg = NeighborSampler(pg, [25, 10], 1024).sample(np.arange(1000, 2024), 3, 0).clone()
    gen = torch.Generator().manual_seed(0)
    table = (torch.rand((V, 37), generator=gen) * 2 - 1).to(d)
    deep, top = sg.blocks[1], sg.blocks[0]
    x_src = table[deep.src.long()].contiguous()
    y_table = ops.MiniBatchFuseOp(sg, 1, table=True).forward(table)
    y_local = ops.MiniBatchFuseOp(sg, 1).forward(x_src)
    assert torch.equal(y_table, y_local)
    torch.testing.assert_close(y_local.double(), dense_agg(deep.column_offset, deep.row_indices, deep.weight, x_src),
                               rtol=1e-5, atol=1e-6)
    x = (torch.rand((top.n_src, 64), generator=gen) * 2 - 1).to(d)
    g = (torch.rand((top.n_dst, 64), generator=gen) * 2 - 1).to(d)
    op = ops.MiniBatchFuseOp(sg, 0)
    y, dx = op.forward(x), op.backward(g)
    torch.testing.assert_close(y.double(), dense_agg(top.column_offset, top.row_indices, top.weight, x),
                               rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(dx.double(), dense_agg(top.row_offset, top.column_indices, top.weight_backward, g),
                               rtol=1e-5, atol=1e-6)
    # the same block with its sources in another order (as the reference stores them, by first appearance): the
    # transposed block is rebuilt on the device and the results move with the sources (the forward bit for bit; the
    # backward's rows sit at other edge positions, where K1 may cut them into differently summed pieces)
    perm = torch.randperm(top.n_src, generator=gen).to(d)
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(top.n_src, device=d)
    other = SampledSubgraph.from_blocks([{"dst": top.dst, "column_offset": top.column_offset,
                                          "row_indices": inv[top.row_indices.long()].int().contiguous(),
                                          "weight": top.weight, "src": top.src[perm].contiguous()}])
    op2 = ops.MiniBatchFuseOp(other, 0)
    assert torch.equal(op2.forward(x[perm].contiguous()), y)
    torch.testing.assert_close(op2.backward(g)[inv], dx, rtol=1e-5, atol=1e-6)
    a, b, p = top.to_numpy(), other.blocks[0].to_numpy(), perm.cpu().numpy()
    assert np.array_equal(np.diff(b["row_offset"]), np.diff(a["row_offset"])[p])
    for k in ("column_indices", "weight_backward"):    # edges of a source in edge order, sources in the new order
        seg = [a[k][a["row_offset"][q]:a["row_offset"][q + 1]] for q in p]
        assert np.array_equal(b[k], np.concatenate(seg))
    with pytest.raises(Exception):
        ops.MiniBatchFuseOp(sg, 1, table=True).backward(y_table)


def float64_step(blocks, table, labels, Ws):
    """One GCNSampleImpl step restated in float64 torch on host copies of its blocks: loss and weight gradients."""
    Wd = [W.detach().double().requires_grad_(True) for W in Ws]
    L = len(Wd)
    h = table.double()
    for l in range(L):
        b = blocks[L - 1 - l]
        idx = b["row_global"] if l == 0 else b["row_indices"]
        t = {k: torch.from_numpy(v.astype(np.int64) if v.dtype == np.uint32 else v).to(table.device)
             for k, v in b.items()}
        n = t["column_offset"].numel() - 1
        e_dst = torch.repeat_interleave(torch.arange(n, device=h.device), t["column_offset"].diff())
        y = torch.zeros((n, h.shape[1]), dtype=torch.float64, device=h.device)
        y = y.index_add(0, e_dst, h[torch.from_numpy(idx.astype(np.int64)).to(h.device)] * t["weight"].double()[:, None])
        h = y @ Wd[l]
        if l < L - 1:
            h = torch.relu(h)
    seeds = torch.from_numpy(blocks[0]["dst"].astype(np.int64)).to(h.device)
    loss = torch.nn.functional.nll_loss(h.log_softmax(1), labels[seeds])
    loss.backward()
    return loss.detach(), [W.grad for W in Wd]


def test_training_step_matches_float64_torch_for_three_steps():
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    edges, V = zipf_hub_edges(V=5000, E=60000)
    pg = graph(edges, V)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, 37), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, 5, (V,), generator=gen).to(d)
    mask = torch.arange(V) % 3
    model = GCNSampleImpl(pg, [37, 16, 5], feats, labels, mask, fanout=[8, 12], batch_size=128, drop_rate=0.0)
    ids = model.nids[0]
    for step in range(3):
        Ws = [p.W.detach().clone() for p in model.P]
        loss, _ = model.train_step(ids[step * 128:(step + 1) * 128])
        blocks = [b.to_numpy() for b in model.subgraph.blocks]
        ref_loss, ref_grads = float64_step(blocks, feats, labels, Ws)
        torch.testing.assert_close(loss.double(), ref_loss, rtol=1e-5, atol=0)
        for p, g in zip(model.P, ref_grads):
            scale = float(g.abs().max())
            torch.testing.assert_close(p.W_gradient.double(), g, rtol=1e-5, atol=1e-5 * scale)


def cora_model(pg, fanout=(5, 10), batch=64, drop_rate=0.5, seed=0):
    from test_gather_plan_bf16 import cora_tables
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    feats, labels, masks = cora_tables()
    torch.manual_seed(seed)
    return GCNSampleImpl(pg, [1433, 128, 7], torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                         torch.from_numpy(masks), fanout=list(fanout), batch_size=batch, drop_rate=drop_rate,
                         seed=seed, sample_seed=seed)


def test_two_runs_with_the_same_seeds_are_bit_identical():
    pg = graph(cora_edges(), 2708)
    runs = []
    for _ in range(2):
        m = cora_model(pg)
        loss, acc = m.run_epoch(test=False)
        runs.append((loss, acc[0], [p.W.detach().clone() for p in m.P]))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    for a, b in zip(runs[0][2], runs[1][2]):
        assert torch.equal(a, b)


def test_sampled_training_reaches_full_graph_accuracy_on_cora():
    from test_gather_plan_bf16 import cora_tables
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    pg = graph(cora_edges(), 2708)
    m = cora_model(pg, drop_rate=0.0)
    for _ in range(20):
        loss, acc = m.run_epoch(test=False)
    sampled = m.evaluate(2)
    feats, labels, masks = cora_tables()
    torch.manual_seed(0)
    full = GCNImpl(pg, [1433, 128, 7], torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                   torch.from_numpy(masks).to(d), seed=0, drop_rate=0.0)
    for _ in range(20):
        full.run_epoch()
    _, a = full.run_epoch(test=True)        # accuracy of the forward after 20 updates
    correct, total = a[2].tolist()
    full_acc = correct / total
    assert np.isfinite(loss)
    assert sampled >= full_acc - 0.05, (sampled, full_acc)


def test_errors_are_raised_before_any_device_work():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.sample import NeighborSampler
    pg = graph(cora_edges(), 2708)
    s = NeighborSampler(pg, [5, 10], 64)
    two = PartitionedGraph(HostGraph(cora_edges(), 2708), 2, 0)
    torch.cuda.synchronize()
    L = _lib.load()
    n0 = L.nts_kernel_launch_count()
    with pytest.raises(_lib.NtsError):
        NeighborSampler(two, [5, 10], 64)
    for bad in ([0, 10], [5, 65]):
        with pytest.raises(_lib.NtsError):
            NeighborSampler(pg, bad, 64)
    with pytest.raises(_lib.NtsError):
        s.sample(np.array([3, 2708]), 0, 0)
    with pytest.raises(_lib.NtsError):
        s.sample(np.arange(65), 0, 0)
    assert L.nts_kernel_launch_count() == n0


def test_table_gather_and_device_seeds_are_range_checked():
    from neutronstarlite_b200 import _lib, ops
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    pg = graph(cora_edges(), 2708)
    s = NeighborSampler(pg, [5, 10], 64)
    # an int64 id of 2^32 + 3 would wrap to 3 if it were cast before the check
    for bad in (torch.tensor([1, (1 << 32) + 3], device=d), torch.tensor([-1, 2], device=d)):
        with pytest.raises(_lib.NtsError):
            s.sample(bad, 0, 0)
    sg = s.sample(torch.tensor([1, 3, 2707], device=d), 0, 0)
    assert sg.vertices == 2708
    op = ops.MiniBatchFuseOp(sg, 1, table=True)
    with pytest.raises(_lib.NtsError):
        op.forward(torch.zeros((2707, 8), device=d))        # a table shorter than V would be read out of bounds
    assert op.forward(torch.zeros((2708, 8), device=d)).shape == (sg.blocks[1].n_dst, 8)
