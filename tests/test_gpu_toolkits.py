"""End-to-end checks of the callers of the hot path on the GPU: the tape + operators must produce the same loss and
parameter gradients as a plain PyTorch fp32 autograd implementation of the same model (dense index ops)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def small_graph(V=300, E=3000, seed=3):
    rng = np.random.default_rng(seed)
    e = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.uint32)
    e = np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1).astype(np.uint32)])
    e[:200, 1] = 7  # hub
    return e


def torch_gcn_reference(pg, layers, feats, labels, mask, Ws):
    """2-layer GCN with torch sparse ops on the whole-partition CSC; mirrors toolkits/GCN.hpp incl. the tape's quirk
    that the first aggregation is not back-propagated (irrelevant for parameter gradients)."""
    c = pg.graph_chunks[0]
    col = c.column_offset_gpu.long()
    src = c.row_indices_gpu.long()
    w = c.edge_weight_forward_gpu
    dst = torch.repeat_interleave(torch.arange(col.numel() - 1, device=col.device), col[1:] - col[:-1])

    def agg(x):
        out = torch.zeros_like(x)
        out.index_add_(0, dst, x[src] * w[:, None])
        return out
    x = feats
    h = torch.relu(agg(x) @ Ws[0])
    out = (agg(h) @ Ws[1]).log_softmax(1)
    tr = (mask == 0).nonzero().view(-1)
    return torch.nn.functional.nll_loss(out[tr], labels[tr])


def test_gcn_epoch_matches_torch_autograd():
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    V = 300
    layers = [37, 16, 5]
    pg = PartitionedGraph(HostGraph(small_graph(V), V), 1, 0).generate_all(device=d, dist=True)
    gen = torch.Generator().manual_seed(0)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    model = GCNImpl(pg, layers, feats.clone(), labels, mask, drop_rate=0.0)
    Ws = [p.W.detach().clone().requires_grad_(True) for p in model.P]
    ref_loss = torch_gcn_reference(pg, layers, feats, labels, mask, Ws)
    ref_loss.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref_loss, rtol=1e-4, atol=1e-6)
    for p, W in zip(model.P, Ws):
        torch.testing.assert_close(p.W.grad, W.grad, rtol=1e-3, atol=1e-6)
    # a full step (Adam) runs and changes the weights
    before = model.P[0].W.detach().clone()
    model.Update()
    assert not torch.equal(before, model.P[0].W.detach())


def torch_gat_reference(pg, layers, heads, feats, labels, mask, Ws, als, ars):
    col = pg.column_offset_gpu.long()
    src = pg.row_indices_gpu.long()
    Vp = col.numel() - 1
    dst = torch.repeat_interleave(torch.arange(Vp, device=col.device), col[1:] - col[:-1])
    x = feats
    for i in range(len(layers) - 1):
        H = heads[i]
        D = layers[i + 1] // H
        xt = (x @ Ws[i]).view(-1, H, D)
        s_att = (xt * als[i]).sum(-1)
        d_att = (xt * ars[i]).sum(-1)
        m = torch.nn.functional.leaky_relu(s_att[src] + d_att[dst], 0.2)          # [E, H]
        mx = torch.full((Vp, H), -float("inf"), device=m.device).scatter_reduce(0, dst[:, None].expand(-1, H), m, "amax")
        ex = torch.exp(m - mx[dst])
        den = torch.zeros((Vp, H), device=m.device).index_add_(0, dst, ex)
        a = ex / den[dst]
        out = torch.zeros((Vp, H, D), device=m.device).index_add_(0, dst, xt[src] * a[:, :, None]).reshape(Vp, H * D)
        x = out.log_softmax(1) if i == len(layers) - 2 else torch.relu(out)
    tr = (mask == 0).nonzero().view(-1)
    return torch.nn.functional.nll_loss(x[tr], labels[tr])


@pytest.mark.parametrize("fused_kernel", [False, True])
@pytest.mark.parametrize("heads", [1, 4])
def test_gat_epoch_matches_torch_autograd(heads, fused_kernel):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    V = 300
    layers = [23, 16, 8, 5]
    pg = PartitionedGraph(HostGraph(small_graph(V, seed=5), V), 1, 0).generate_all(device=d, dist=True)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    model = GATImpl(pg, layers, feats.clone(), labels, mask, heads=heads, sum_fanout_grads=True,
                    fused_kernel=fused_kernel)
    clone = lambda ps: [p.W.detach().clone().requires_grad_(True) for p in ps]
    Ws, als, ars = clone(model.P), clone(model.al), clone(model.ar)
    ref_loss = torch_gat_reference(pg, layers, model.heads, feats, labels, mask, Ws, als, ars)
    ref_loss.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref_loss, rtol=1e-4, atol=1e-6)
    for mine, ref in zip(model.P + model.al + model.ar, Ws + als + ars):
        torch.testing.assert_close(mine.W.grad, ref.grad, rtol=2e-3, atol=2e-6)
    model.Update()


def test_bench_prints_the_contract_line_on_a_tiny_workload(tmp_path):
    """`bench.py` (our arm) end to end on the tiny workload: one JSON line with every key of the bench contract,
    kernels of libnts_b200 actually launched, roofline and e2e present, and the last timed step's outputs dumped."""
    import json
    import os
    import subprocess
    import sys
    dev()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--workload", "tiny", "--steps", "3",
                          "--warmup", "3", "--no-cpu-baseline", "--no-ref-gpu", "--dump-outputs", str(tmp_path)],
                         stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-1500:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "clocks"):
        assert key in line, key
    assert line["gpu_launches"] >= 9 and line["value"] > 0
    assert line["e2e"]["h2d_bytes_per_step"] > 0 and line["e2e"]["d2h_bytes_per_step"] > 0
    assert line["roofline"]["bound"] == "hbm" and line["roofline"]["achieved"] > 0
    import numpy as np
    out = np.load(tmp_path / "output.npy")
    loss = np.load(tmp_path / "loss.npy")
    assert out.shape == (20000, 41) and out.dtype == np.float32 and np.isfinite(out).all()
    assert loss.shape == (1,) and np.isfinite(loss).all() and loss[0] > 0
