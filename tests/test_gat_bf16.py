"""BF16 mirror gathers with FP32 accumulation for the fused GAT layer (K7: nts_gat_fused_aggregate_forward_bf16,
nts_gat_fused_aggregate_backward_two_pass_bf16, ops.DistGPUFusedGATOp / toolkits.GATImpl gather_dtype).

Precision contract: with m~ = bf16(mirror) and g~ = bf16(grad_out) (torch's rounding), the layer computes the FP32
layer's function and gradients at m~ and g~.  So every result is checked against float64 torch autograd of the layer
evaluated at the rounded operands, and the rounding itself value for value through an identity graph."""
import numpy as np
import pytest

from test_gather_plan_bf16 import cora_tables, row_close
from test_gpu_parity import random_csr

torch = pytest.importorskip("torch")

BF16 = torch.bfloat16
SHAPES = [(8, 8), (8, 64), (1, 64), (2, 16), (1, 41), (1, 200), (4, 32)]


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def up_u32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(dev())


def stub_graph(off, idx, mi):
    """A one-partition PartitionedGraph carrying only the whole-partition CSC and MirrorIndex that K7 reads."""
    from neutronstarlite_b200.graph import PartitionedGraph
    Vp = off.shape[0] - 1
    pg = PartitionedGraph(None, 1, 0, np.array([0, Vp], dtype=np.uint32))
    pg.owned_vertices, pg.owned_edges, pg.owned_mirrors = Vp, idx.shape[0], int(mi[-1])
    pg.column_offset_gpu, pg.row_indices_gpu, pg.mirror_index_gpu = up_u32(off), up_u32(idx), up_u32(mi)
    return pg


def hub_layer_graph(H, D):
    """The graph of test_gpu_parity.py::test_fully_fused_gat_layer_vs_operator_chain (hub segment included)."""
    Vp, Vg, E = 500, 1500, 30000
    off, idx, _ = random_csr(Vp, Vg, E, seed=H * 7 + D, hub_rows=1)
    used = np.unique(idx)
    mi = np.zeros(Vg + 1, dtype=np.uint32)
    mi[used + 1] = 1
    mi = np.cumsum(mi, dtype=np.uint32)
    return stub_graph(off, idx, mi), off, mi[idx]


def layer_reference(off, slot, mt, s, d, gt, H, slope=0.2):
    """float64 autograd of the K7 layer at the rounded operands: returns out and the gradients of (m~, s, d) for the
    upstream gradient g~, and the per-row magnitudes sum_e a |m~| and sum_e a |g~| that out and d_mirror are
    compared against (a hub row's terms cancel; its FP32 rounding scales with the terms, not with their sum)."""
    dd = torch.float64
    m64 = mt.to(dd).requires_grad_(True)
    s64 = s.to(dd).requires_grad_(True)
    d64 = d.to(dd).requires_grad_(True)
    dv = mt.device
    Vp = off.shape[0] - 1
    src = torch.from_numpy(slot.astype(np.int64)).to(dv)
    dst = torch.repeat_interleave(torch.arange(Vp, device=dv), torch.from_numpy(np.diff(off).astype(np.int64)).to(dv))
    logit = torch.nn.functional.leaky_relu(s64[src] + d64[dst], slope)
    mx = torch.full((Vp, H), -float("inf"), dtype=dd, device=dv).scatter_reduce(
        0, dst[:, None].expand(-1, H), logit.detach(), "amax")
    ex = torch.exp(logit - mx[dst])
    a = ex / torch.zeros((Vp, H), dtype=dd, device=dv).index_add(0, dst, ex)[dst]
    F = mt.shape[1]
    out = torch.zeros((Vp, H, F // H), dtype=dd, device=dv).index_add(
        0, dst, m64[src].view(-1, H, F // H) * a[:, :, None]).reshape(Vp, F)
    out.backward(gt.to(dd))
    with torch.no_grad():
        ae = a.detach()[:, :, None]
        out_mag = torch.zeros_like(out).view(Vp, H, -1).index_add(0, dst, m64.abs()[src].view(-1, H, F // H) * ae)
        dm_mag = torch.zeros_like(m64).view(-1, H, F // H).index_add(0, src, gt.to(dd).abs()[dst].view(-1, H, F // H)
                                                                      * ae)
    return out.detach(), m64.grad, s64.grad, d64.grad, out_mag.reshape(Vp, F), dm_mag.reshape(-1, F)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_bf16_gat_symbols_are_exported_and_reject_bad_layouts():
    """The new entry points exist, and layouts outside the BF16 rule are argument errors before any device work."""
    from neutronstarlite_b200 import _lib
    lib = _lib.load()
    for name in ("nts_rows_to_bf16", "nts_gat_fused_aggregate_forward_bf16",
                 "nts_gat_fused_aggregate_backward_two_pass_bf16"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    fwd = lib.nts_gat_fused_aggregate_forward_bf16
    bwd = lib.nts_gat_fused_aggregate_backward_two_pass_bf16
    # (H, F, ld): D % 8 != 0 with several heads, a stride that is not a whole number of chunks, a stride below F
    for H, F, ld in ((3, 15, 16), (16, 64, 64), (1, 41, 44), (1, 64, 56), (2, 32, 40)):
        assert fwd(*([None] * 9), 10, 100, F, ld, H, 0.2, None) != 0
        assert b"BF16" in lib.nts_last_error() or b"heads" in lib.nts_last_error()
        assert bwd(*([None] * 16), 10, 10, F, ld, H, 0.2, None) != 0
    # a shape the two passes do not cover (no fallback): 8 heads of 24 values
    assert bwd(*([None] * 16), 10, 10, 192, 192, 8, 0.2, None) != 0
    assert b"two-pass" in lib.nts_last_error()


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rows_to_bf16_is_torch_rounding_bit_for_bit():
    """nts_rows_to_bf16 equals x.to(torch.bfloat16) bit for bit (ties, overflow to inf, +-inf, subnormals, -0; a NaN
    stays a NaN), and writes zeros into the pad columns."""
    from neutronstarlite_b200 import _lib
    d = dev()
    specials = np.array([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.3895314e38, 3.4e38, -3.4e38,
                         np.inf, -np.inf, np.nan, 1e-40, -1e-40, 2 ** -133, 1.1754942e-38, 0.0, -0.0,
                         65504.0, 1.0 / 3.0, -2.71828], dtype=np.float32)
    rng = np.random.default_rng(4)
    for F in (41, 64, 7, 200, 8):
        V = 300
        X = (rng.standard_normal((V, F)) * 10.0 ** rng.integers(-30, 30, (V, F))).astype(np.float32)
        X.reshape(-1)[: specials.size * 5] = np.tile(specials, 5)
        hi = np.arange(256, dtype=np.uint32) + 0x3F00
        X[44:, 0] = ((hi[: V - 44] << 16) | 0x8000).view(np.float32)     # exact ties
        x = torch.from_numpy(X).to(d)
        ld = (F + 7) // 8 * 8
        r = torch.full((V, ld), -1.0, dtype=BF16, device=d)
        _lib.call("nts_rows_to_bf16", x.data_ptr(), 0, F, r.data_ptr(), V, F, ld, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        want = x.to(BF16).view(torch.int16).cpu().numpy()
        got = r[:, :F].contiguous().view(torch.int16).cpu().numpy()
        nan = np.isnan(X)
        assert np.array_equal(got[~nan], want[~nan])
        assert np.isnan(r[:, :F].float().cpu().numpy()[nan]).all()
        assert not r[:, F:].view(torch.int16).any()


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", SHAPES)
def test_bf16_fused_gat_layer_vs_float64_autograd_at_rounded_operands(H, D):
    from neutronstarlite_b200 import ops
    d = dev()
    pg, off, slot = hub_layer_graph(H, D)
    rng = np.random.default_rng(H * 1000 + D)
    M, F = pg.owned_mirrors, H * D
    mirror = torch.from_numpy(rng.uniform(-1, 1, (M, F)).astype(np.float32)).to(d)
    s = torch.from_numpy(rng.uniform(-2, 2, (M, H)).astype(np.float32)).to(d)
    dsc = torch.from_numpy(rng.uniform(-2, 2, (pg.owned_vertices, H)).astype(np.float32)).to(d)
    g = torch.from_numpy(rng.uniform(-1, 1, (pg.owned_vertices, F)).astype(np.float32)).to(d)
    op = ops.DistGPUFusedGATOp(pg, negative_slope=0.2, gather_dtype=BF16)
    out = op.forward(mirror, s, dsc)
    dm, ds, dd = op.backward(g)
    torch.cuda.synchronize()
    assert out.shape == (pg.owned_vertices, F) and dm.shape == (M, F)
    assert out.dtype == dm.dtype == ds.dtype == dd.dtype == torch.float32
    mt, gt = mirror.to(BF16).float(), g.to(BF16).float()
    out_ref, dm_ref, ds_ref, dd_ref, out_mag, dm_mag = layer_reference(off, slot, mt, s, dsc, gt, H)
    row_close(out.cpu().numpy(), out_ref.cpu().numpy(), scale=out_mag.cpu().numpy())
    row_close(dm.cpu().numpy(), dm_ref.cpu().numpy(), scale=dm_mag.cpu().numpy())
    torch.testing.assert_close(ds, ds_ref.float(), rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(dd, dd_ref.float(), rtol=1e-3, atol=2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [41, 64, 8])
def test_bf16_fused_gat_identity_graph_returns_the_rounded_mirror(F):
    """One in-edge per destination from its own slot: every attention weight is exactly 1, so out == m~ value for value
    (the FP32 accumulator starts at +0: -0 comes out as +0, which compares equal; NaN by class)."""
    from neutronstarlite_b200 import ops
    d = dev()
    V = 1000
    off = np.arange(V + 1, dtype=np.uint32)
    pg = stub_graph(off, np.arange(V, dtype=np.uint32), np.arange(V + 1, dtype=np.uint32))
    rng = np.random.default_rng(F)
    X = (rng.standard_normal((V, F)) * 10.0 ** rng.integers(-30, 30, (V, F))).astype(np.float32)
    X[:3, :3] = [[np.inf, -np.inf, np.nan], [1e-40, -0.0, 3.4e38], [1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 2 ** -133]]
    x = torch.from_numpy(X).to(d)
    s = torch.from_numpy(rng.uniform(-2, 2, (V, 1)).astype(np.float32)).to(d)
    out = ops.DistGPUFusedGATOp(pg, gather_dtype=BF16).forward(x, s, torch.zeros_like(s)).cpu().numpy()
    want = x.to(BF16).float().cpu().numpy()
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(out), nan)
    assert np.array_equal(out[~nan], want[~nan])


@pytest.mark.gpu
def test_bf16_fused_gat_rejections():
    from neutronstarlite_b200 import _lib, ops
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    for H, D in ((3, 5), (16, 4)):
        pg, _, _ = hub_layer_graph(H, D)
        M, F = pg.owned_mirrors, H * D
        op = ops.DistGPUFusedGATOp(pg, gather_dtype=BF16)
        with pytest.raises(_lib.NtsError):
            op.forward(torch.rand((M, F), device=d), torch.rand((M, H), device=d),
                       torch.rand((pg.owned_vertices, H), device=d))
    with pytest.raises(_lib.NtsError):
        ops.DistGPUFusedGATOp(pg, two_pass_backward=False, gather_dtype=BF16)
    with pytest.raises(_lib.NtsError):
        ops.DistGPUFusedGATOp(pg, gather_dtype=torch.float16)
    V = 50
    e = np.stack([np.arange(V), (np.arange(V) + 1) % V], 1).astype(np.uint32)
    gpg = PartitionedGraph(HostGraph(e, V), 1, 0).generate_all(device=d, dist=True)
    feats, labels, mask = torch.rand((V, 16), device=d), torch.zeros(V, dtype=torch.int64, device=d), \
        torch.zeros(V, dtype=torch.int64, device=d)
    for kw in ({"fused_kernel": False, "gather_dtype": BF16},
               {"fused_kernel": True, "two_pass_backward": False, "gather_dtype": BF16},
               {"fused_kernel": True, "gather_dtype": torch.float16},
               {"fused_kernel": True, "gather_dtype": torch.float32}):
        with pytest.raises(_lib.NtsError):
            GATImpl(gpg, [16, 16, 4], feats, labels, mask, heads=2, **kw)


def small_graph(V=300, E=3000, seed=5):
    rng = np.random.default_rng(seed)
    e = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.uint32)
    e = np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1).astype(np.uint32)])
    e[:200, 1] = 7  # hub
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("heads,layers", [(1, [23, 16, 8, 5]), (4, [23, 32, 32, 5])])
def test_gat_epoch_with_bf16_gathers_matches_torch_autograd(heads, layers):
    """Loss and every parameter gradient of one fused GATImpl(gather_dtype=bf16) epoch against a torch autograd model
    whose aggregation gathers bf16-rounded rows (forward: the transformed features; backward: the output gradient),
    at the tolerances of the FP32 toolkit test (tests/test_gpu_toolkits.py)."""
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    V = 300
    pg = PartitionedGraph(HostGraph(small_graph(V), V), 1, 0).generate_all(device=d, dist=True)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    model = GATImpl(pg, layers, feats.clone(), labels, mask, heads=heads, fused_kernel=True, gather_dtype=BF16)
    assert model.X[0].dtype == torch.float32
    clone = lambda ps: [p.W.detach().clone().requires_grad_(True) for p in ps]
    Ws, als, ars = clone(model.P), clone(model.al), clone(model.ar)
    col = pg.column_offset_gpu.long()
    src = pg.row_indices_gpu.long()
    dst = torch.repeat_interleave(torch.arange(V, device=d), col[1:] - col[:-1])

    class Agg(torch.autograd.Function):   # out = sum_e a * bf16(xt)[src];  d_xt = sum a * bf16(g), d_a = <bf16(xt), bf16(g)>
        @staticmethod
        def forward(ctx, xt, a):
            xr = xt.to(BF16).float()
            ctx.save_for_backward(xr, a)
            return torch.zeros_like(xt).index_add_(0, dst, xr[src] * a[:, :, None])

        @staticmethod
        def backward(ctx, go):
            xr, a = ctx.saved_tensors
            gr = go.to(BF16).float()
            return torch.zeros_like(xr).index_add_(0, src, gr[dst] * a[:, :, None]), (xr[src] * gr[dst]).sum(-1)

    x = feats
    for i in range(len(layers) - 1):
        H = model.heads[i]
        D = layers[i + 1] // H
        xt = (x @ Ws[i]).view(-1, H, D)
        m = torch.nn.functional.leaky_relu((xt * als[i]).sum(-1)[src] + (xt * ars[i]).sum(-1)[dst], 0.2)
        mx = torch.full((V, H), -float("inf"), device=d).scatter_reduce(0, dst[:, None].expand(-1, H), m, "amax")
        ex = torch.exp(m - mx[dst])
        a = ex / torch.zeros((V, H), device=d).index_add_(0, dst, ex)[dst]
        out = Agg.apply(xt, a).reshape(V, H * D)
        x = out.log_softmax(1) if i == len(layers) - 2 else torch.relu(out)
    tr = (mask == 0).nonzero().view(-1)
    ref_loss = torch.nn.functional.nll_loss(x[tr], labels[tr])
    ref_loss.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref_loss, rtol=1e-4, atol=1e-6)
    for mine, ref in zip(model.P + model.al + model.ar, Ws + als + ars):
        torch.testing.assert_close(mine.W.grad, ref.grad, rtol=2e-3, atol=2e-6)
    model.Update()


@pytest.mark.gpu
def test_cora_100_epochs_bf16_gat_accuracy_close_to_fp32():
    """100 epochs of the fused 8-head Cora GAT ([1433, 64, 7]) with the same seed in both arms: the final test accuracy
    of the BF16-gather run is within 0.02 of the FP32 run."""
    import golden_store
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    feats, labels, masks = cora_tables()
    V = feats.shape[0]
    pg = PartitionedGraph(HostGraph(golden_store.load("cora_self_P1_F8")["edges"], V), 1, 0).generate_all(
        device=d, dist=True)
    test_rows = torch.from_numpy(masks == 2).to(d)
    lab = torch.from_numpy(labels).to(d)
    acc = {}
    for arm in (None, BF16):
        torch.manual_seed(0)
        model = GATImpl(pg, [1433, 64, 7], torch.from_numpy(feats).to(d), lab, torch.from_numpy(masks).to(d),
                        heads=8, seed=0, fused_kernel=True, gather_dtype=arm)
        for _ in range(100):
            model.run_epoch()
        model.Forward()
        pred = model.X[-1].argmax(1)
        acc[arm] = float((pred == lab)[test_rows].float().mean())
    assert acc[None] > 0.3
    assert abs(acc[BF16] - acc[None]) <= 0.02, acc
