"""BF16 gathers with FP32 accumulation (nts_gather_plan_run_bf16_ex, csrc/nts_plan.cu) and the options above them.

Precision contract: out[r,:] += sum_e w(e) * float(bf16(x[src(e),:])), bf16() = round to nearest even exactly as
torch's x.to(torch.bfloat16); weights, accumulation and outputs FP32.  So every result is checked against the C oracle
of the reference's aggregation loop run on the bf16-ROUNDED operand, per row at 1e-4 (the FP32 rule), and the rounding
itself bit for bit through an identity graph."""
import gzip
import os

import numpy as np
import pytest

import golden_store
import oracle_c

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

WIDTHS = [602, 128, 100, 41, 7, 1, 1433, 64]


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def up_u32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(dev())


def rounded(x):
    """The operand the contract is stated on: bf16(x) widened back to FP32 (numpy, for the oracle)."""
    t = x if torch.is_tensor(x) else torch.from_numpy(x)
    return t.to(torch.bfloat16).float().cpu().numpy()


def row_close(actual, desired, rtol=1e-4, scale=None):
    """max |err| of every row <= rtol * scale of THAT row (default: max |desired| of the row)."""
    err = np.abs(actual.astype(np.float64) - desired.astype(np.float64)).max(axis=1)
    scale = np.abs(desired if scale is None else scale).max(axis=1).astype(np.float64)
    bad = np.nonzero(err > rtol * scale + 1e-30)[0]
    assert bad.size == 0, "rows %s: err %s vs scale %s" % (bad[:5], err[bad[:5]], scale[bad[:5]])


def agg_close(actual, off, idx, w, Xr, rtol=1e-4):
    """Against the oracle on the rounded operand Xr, per row relative to the row's sum of |w| * |x| (the dense hub
    blocks add a row's terms in another order than the edge loop; where they cancel only that magnitude is small)."""
    row_close(actual, oracle_c.segment_gather_sum(off, idx, w, Xr), rtol,
              scale=oracle_c.segment_gather_sum(off, idx, None if w is None else np.abs(w), np.abs(Xr)))


def csr(dst, src, n_rows, rng):
    order = np.lexsort((src, dst))
    dst, src = dst[order], src[order]
    off = np.zeros(n_rows + 1, dtype=np.uint32)
    np.add.at(off, dst + 1, 1)
    off = np.cumsum(off).astype(np.uint32)
    w = rng.uniform(0.1, 1.0, dst.shape[0]).astype(np.float32)
    return off, src.astype(np.uint32), w


def hub_graph(rng, n_rows=700, n_src=900, n_edges=40000):
    """Zipf endpoints (hub sources and hub destinations), repeated (dst, src) pairs, empty destination rows."""
    dst = np.minimum(rng.zipf(1.6, n_edges) - 1, n_rows - 1)
    src = np.minimum(rng.zipf(1.6, n_edges) - 1, n_src - 1)
    dst = rng.permutation(n_rows)[dst]
    src = rng.permutation(n_src)[src]
    dst = np.concatenate([dst, dst[:5000]])
    src = np.concatenate([src, src[:5000]])
    keep = dst % 9 != 4
    return csr(dst[keep], src[keep], n_rows, rng)


def make_plan(off, idx, w, base, n_src, slabs, hubs=(0, 0), slot_of=None):
    from neutronstarlite_b200 import ops
    return ops.GatherPlan(up_u32(off), up_u32(idx), None if w is None else torch.from_numpy(w).to(dev()), base,
                          off.shape[0] - 1, idx.shape[0], n_src, slabs,
                          slot_of=None if slot_of is None else up_u32(slot_of), hubs=hubs)


def run(plan, x, out=None):
    x = x if torch.is_tensor(x) else torch.from_numpy(x).to(dev())
    if out is None:
        out = torch.zeros((plan.n_rows, x.shape[1]), dtype=torch.float32, device=dev())
    plan.run(x, out, gather_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("in_dtype", ["float32", "bfloat16"])
@pytest.mark.parametrize("slabs", [1, 3, 16])
def test_bf16_plan_matches_oracle_on_rounded_input(slabs, in_dtype):
    rng = np.random.default_rng(100 + slabs)
    n_rows, n_src, base = 700, 900, 5000
    off, idx, w = hub_graph(rng, n_rows, n_src)
    plan = make_plan(off, idx + base, w, base, n_src, slabs)
    assert plan.slabs == slabs
    for F in WIDTHS:
        x = torch.from_numpy(rng.uniform(-1, 1, (n_src, F)).astype(np.float32)).to(dev())
        xin = x if in_dtype == "float32" else x.to(torch.bfloat16)
        got = run(plan, xin).cpu().numpy()
        row_close(got, oracle_c.segment_gather_sum(off, idx, w, rounded(x)))


@pytest.mark.parametrize("hubs", [(0, 0), (32, 0), (0, 32), (64, 64)])
@pytest.mark.parametrize("slabs", [1, 3])
def test_bf16_hub_blocks_match_oracle(slabs, hubs):
    rng = np.random.default_rng(200 + slabs + hubs[0] + 3 * hubs[1])
    n_rows, n_src = 700, 900
    off, idx, w = hub_graph(rng, n_rows, n_src)
    plan = make_plan(off, idx, w, 0, n_src, slabs, hubs)
    assert (plan.hub_cols, plan.hub_rows) == hubs
    for F in (602, 128, 41, 7):
        x = torch.from_numpy(rng.uniform(-1, 1, (n_src, F)).astype(np.float32)).to(dev())
        for xin in (x, x.to(torch.bfloat16)):
            agg_close(run(plan, xin).cpu().numpy(), off, idx, w, rounded(x))


def test_bf16_slot_table_unaligned_views_and_accumulation():
    """Indices through a slot table; bf16 and float32 input views whose base is not 16-byte aligned (re-strided into
    the workspace); output views that are 4- and 8-byte aligned; accumulation into a non-zero output."""
    rng = np.random.default_rng(77)
    n_rows, n_src = 300, 500
    off, idx, w = hub_graph(rng, n_rows, n_src, 20000)
    ids = rng.permutation(4000)[:n_src].astype(np.uint32)
    slot_of = np.zeros(4000, dtype=np.uint32)
    slot_of[ids] = np.arange(n_src, dtype=np.uint32)
    plan = make_plan(off, ids[idx], w, 0, n_src, 3, (32, 20), slot_of=slot_of)
    for F, shift, dtype in ((128, 1, torch.bfloat16), (602, 2, torch.float32), (64, 3, torch.bfloat16),
                            (41, 1, torch.float32)):
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        Xr = rounded(X)
        ref = oracle_c.segment_gather_sum(off, idx, w, Xr)
        mag = oracle_c.segment_gather_sum(off, idx, w, np.abs(Xr))
        flat = torch.zeros(n_src * F + 1, dtype=dtype, device=dev())
        flat[1:] = torch.from_numpy(X).to(dev()).reshape(-1).to(dtype)
        xv = flat[1:].view(n_src, F)
        assert xv.data_ptr() % 16 != 0
        oflat = torch.ones(n_rows * F + shift, dtype=torch.float32, device=dev())
        ov = oflat[shift:].view(n_rows, F)
        run(plan, xv, ov)
        run(plan, xv, ov)
        row_close(ov.cpu().numpy(), 1.0 + 2.0 * ref, rtol=2e-4, scale=1.0 + 2.0 * mag)
        assert float(oflat[:shift].sum()) == shift


def test_bf16_conversion_is_torch_rounding_exactly():
    """Identity graph (one edge of weight 1 per row): the output is bf16(x) widened, value for value, for rounding
    ties, values that round to inf, +-inf, NaN and subnormals.  (The FP32 accumulator starts at +0, so -0 comes out
    as +0, and a NaN as the canonical NaN: those two compare by value / by class.)"""
    from neutronstarlite_b200 import ops
    V = 1024
    specials = np.array([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.3895314e38, 3.4e38, -3.4e38,
                         np.inf, -np.inf, np.nan, 1e-40, -1e-40, 2 ** -133, 1.1754942e-38, 0.0, -0.0,
                         65504.0, 1.0 / 3.0, -2.71828], dtype=np.float32)
    rng = np.random.default_rng(1)
    for F in (602, 128, 8, 7, 1):
        X = (rng.standard_normal((V, F)) * 10.0 ** rng.integers(-30, 30, (V, F))).astype(np.float32)
        flat = X.reshape(-1)
        flat[: specials.size * 7] = np.tile(specials, 7)
        # exactly half-way between two bf16 values (odd and even lower neighbours), small and ordinary magnitudes
        hi = np.concatenate([np.arange(256), 0x3F00 + np.arange(256)]).astype(np.uint32)
        X[512:, -1] = ((hi << 16) | 0x8000).view(np.float32)
        off = np.arange(V + 1, dtype=np.uint32)
        plan = ops.GatherPlan(up_u32(off), up_u32(np.arange(V)), None, 0, V, V, V, 1)
        x = torch.from_numpy(X).to(dev())
        want = x.to(torch.bfloat16).float().cpu().numpy()
        for xin in (x, x.to(torch.bfloat16)):
            got = run(plan, xin).cpu().numpy()
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(got), nan)
            assert np.array_equal(got[~nan], want[~nan])


def test_tuned_bf16_plan_on_a_large_graph_and_sharing():
    """A tuned BF16 plan (timed as BF16 gathers) on a graph of more than 2^20 edges computes the contract; the FP32 and
    BF16 tuned plans of one chunk direction share their arrays exactly when their slab and hub counts agree."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    rng = np.random.default_rng(12)
    V, E = 40000, 1 << 21
    edges = np.stack([rng.zipf(1.4, E) % V, rng.integers(0, V, E)], 1).astype(np.uint32)
    pg = PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev())
    c = pg.graph_chunks[0]
    assert c.edge_size >= 1 << 20
    F = 128
    x = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).to(dev())
    y16 = ops.gather_by_dst_from_src(c, torch.zeros_like(x), x, gather_dtype=torch.bfloat16)
    y32 = ops.gather_by_dst_from_src(c, torch.zeros_like(x), x)
    torch.cuda.synchronize()
    p16 = c._gather_plan_for[("fwd", "F", F, "bf16")]
    p32 = c._gather_plan_for[("fwd", "F", F)]
    assert (p16 is p32) == (p16.key() == p32.key())
    assert c._gather_plans[("fwd",) + p16.key()] is p16
    agg_close(y16.cpu().numpy(), c.column_offset, c.row_indices, c.edge_weight_forward, rounded(x))
    row_close(y32.cpu().numpy(), oracle_c.segment_gather_sum(c.column_offset, c.row_indices, c.edge_weight_forward,
                                                             x.cpu().numpy()))


def test_fp32_and_bf16_plans_share_arrays_when_counts_match():
    """Forced counts: BF16 and FP32 plans of one chunk that settle on the same slab and hub counts are one object,
    those that do not keep their own arrays; both compute their contract."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    rng = np.random.default_rng(11)
    V, E = 3000, 200000
    edges = np.stack([rng.zipf(1.5, E) % V, rng.zipf(1.5, E) % V], 1).astype(np.uint32)
    pg = PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev())
    c = pg.graph_chunks[0]
    real = ops.GatherPlan
    picks = {(602, None): (64, 32), (602, "bf16"): (64, 32), (128, None): (0, 0), (128, "bf16"): (32, 0)}

    def forced(*a, tune_for=0, gather_dtype=None, **kw):
        return real(*a[:7], 2, hubs=picks[(tune_for, None if gather_dtype is None else "bf16")], **kw)
    ops.GatherPlan = forced
    ops.set_plan_mode("on", 0)
    try:
        res = {}
        for (F, t) in picks:
            x = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).to(dev())
            gd = torch.bfloat16 if t else None
            y = ops.gather_by_dst_from_src(c, torch.zeros_like(x), x, gather_dtype=gd)
            torch.cuda.synchronize()
            res[(F, t)] = (x, y.cpu().numpy())
    finally:
        ops.GatherPlan = real
        ops.set_plan_mode("auto", 0)
    tuned = c._gather_plan_for
    assert tuned[("fwd", "F", 602)] is tuned[("fwd", "F", 602, "bf16")]
    assert tuned[("fwd", "F", 128)] is not tuned[("fwd", "F", 128, "bf16")]
    for (F, t), (x, y) in res.items():
        xr = rounded(x) if t else x.cpu().numpy()
        agg_close(y, c.column_offset, c.row_indices, c.edge_weight_forward, xr)


# ---- operators and toolkits ---------------------------------------------------------------------------------------
def golden_pg(name):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    g = golden_store.load(name)
    edges = g["edges"]
    V = int(g["r0/partition_offset"][-1])
    return PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev(), dist=True), V


def dense_agg(c, x64, forward=True):
    """float64 torch aggregation on the chunk's CSC (forward: Y = A X, backward: dX = A^T dY)."""
    col = c.column_offset_gpu.long()
    src = c.row_indices_gpu.long()
    dst = torch.repeat_interleave(torch.arange(col.numel() - 1, device=col.device), col[1:] - col[:-1])
    w = c.edge_weight_forward_gpu.double() if forward else None
    if forward:
        return torch.zeros((c.batch_size_forward, x64.shape[1]), dtype=torch.float64,
                           device=x64.device).index_add_(0, dst, x64[src] * w[:, None])
    # backward weights live on the CSR; recompute from the CSR arrays
    ro = c.row_offset_gpu.long()
    ci = c.column_indices_gpu.long() - c.dst_range[0]
    s = torch.repeat_interleave(torch.arange(ro.numel() - 1, device=ro.device), ro[1:] - ro[:-1])
    wb = c.edge_weight_backward_gpu.double()
    return torch.zeros((c.batch_size_backward, x64.shape[1]), dtype=torch.float64,
                       device=x64.device).index_add_(0, s, x64[ci] * wb[:, None])


@pytest.mark.parametrize("case", ["cora_self_P1_F8", "synth9k_P1_F2"])
def test_single_gpu_op_bf16_forward_backward(case):
    from neutronstarlite_b200 import ops
    pg, V = golden_pg(case)
    c = pg.graph_chunks[0]
    rng = np.random.default_rng(5)
    for F in (602, 128, 41):
        x = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).to(dev())
        g = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).to(dev())
        op = ops.ForwardSingleGPUfuseOp(pg, None, gather_dtype=torch.bfloat16)
        for xin in (x, x.to(torch.bfloat16)):
            y = op.forward(xin)
            assert y.dtype == torch.float32
            ref = dense_agg(c, x.to(torch.bfloat16).double())
            row_close(y.cpu().numpy(), ref.cpu().numpy(),
                      scale=dense_agg(c, x.to(torch.bfloat16).double().abs()).cpu().numpy())
        dx = op.backward(g)
        assert dx.dtype == torch.float32
        ref = dense_agg(c, g.to(torch.bfloat16).double(), forward=False)
        row_close(dx.cpu().numpy(), ref.cpu().numpy(),
                  scale=dense_agg(c, g.to(torch.bfloat16).double().abs(), forward=False).cpu().numpy())


def test_bf16_options_reject_wrong_inputs():
    from neutronstarlite_b200 import _lib, ops
    pg, V = golden_pg("cora_self_P1_F8")
    with pytest.raises(_lib.NtsError):
        ops.ForwardSingleGPUfuseOp(pg, None, gather_dtype=torch.float16)
    with pytest.raises(_lib.NtsError):
        ops.ForwardSingleGPUfuseOp(pg, None, gather_dtype=torch.float32)
    op = ops.ForwardSingleGPUfuseOp(pg, None, gather_dtype=torch.bfloat16)
    x = torch.zeros((V, 16), device=dev())
    for bad in (x.half(), x.double(), x.cpu(), x.to(torch.bfloat16).cpu(), x.to(torch.bfloat16)[:, ::2],
                x[:, ::2], x[0]):
        with pytest.raises(_lib.NtsError):
            op.forward(bad)
    with pytest.raises(_lib.NtsError):
        op.backward(x.to(torch.bfloat16))               # backward takes float32 gradients
    with pytest.raises(_lib.NtsError):
        ops.ForwardSingleGPUfuseOp(pg).forward(x.to(torch.bfloat16))   # bf16 without the option, as before
    with pytest.raises(_lib.NtsError):
        ops.ForwardGPUfuseOp(pg, None, gather_dtype=torch.float16)


def test_gcn_epoch_with_bf16_gathers_matches_torch_autograd():
    """Loss and weight gradients of one GCNImpl(gather_dtype=bf16) epoch against a torch autograd model whose
    aggregation inputs are bf16-rounded (the construction of test_gpu_toolkits.py, drop_rate=0)."""
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    V, E = 300, 3000
    rng = np.random.default_rng(3)
    e = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.uint32)
    e = np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1).astype(np.uint32)])
    e[:200, 1] = 7
    layers = [37, 16, 5]
    pg = PartitionedGraph(HostGraph(e, V), 1, 0).generate_all(device=d, dist=True)
    gen = torch.Generator().manual_seed(0)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    model = GCNImpl(pg, layers, feats.clone(), labels, mask, drop_rate=0.0, gather_dtype=torch.bfloat16)
    assert model.X[0].dtype == torch.bfloat16
    Ws = [p.W.detach().clone().requires_grad_(True) for p in model.P]
    c = pg.graph_chunks[0]
    col = c.column_offset_gpu.long()
    src = c.row_indices_gpu.long()
    w = c.edge_weight_forward_gpu
    dst = torch.repeat_interleave(torch.arange(col.numel() - 1, device=d), col[1:] - col[:-1])

    class Agg(torch.autograd.Function):   # Y = A bf16(X); dX = A^T bf16(dY)
        @staticmethod
        def forward(ctx, x):
            xr = x.to(torch.bfloat16).float()
            return torch.zeros_like(x).index_add_(0, dst, xr[src] * w[:, None])

        @staticmethod
        def backward(ctx, gy):
            gr = gy.to(torch.bfloat16).float()
            return torch.zeros_like(gy).index_add_(0, src, gr[dst] * w[:, None])
    h = torch.relu(Agg.apply(feats) @ Ws[0])
    out = (Agg.apply(h) @ Ws[1]).log_softmax(1)
    tr = (mask == 0).nonzero().view(-1)
    ref_loss = torch.nn.functional.nll_loss(out[tr], labels[tr])
    ref_loss.backward()
    model.Forward()
    model.Loss()
    model.ctx.self_backward(True)
    torch.testing.assert_close(model.loss, ref_loss, rtol=1e-4, atol=1e-6)
    for p, W in zip(model.P, Ws):
        torch.testing.assert_close(p.W.grad, W.grad, rtol=1e-3, atol=1e-6)


def cora_tables():
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cora_tables")
    V, F = 2708, 1433
    feats = np.zeros((V, F), dtype=np.float32)
    labels = np.zeros(V, dtype=np.int64)
    masks = np.zeros(V, dtype=np.int64)
    names = {"train": 0, "eval": 1, "val": 1, "test": 2}
    with gzip.open(os.path.join(root, "cora.featuretable.gz"), "rt") as ff, \
            gzip.open(os.path.join(root, "cora.labeltable.gz"), "rt") as fl, \
            gzip.open(os.path.join(root, "cora.mask.gz"), "rt") as fm:
        for lf, ll, lm in zip(ff, fl, fm):
            tok = lf.split()
            if not tok:
                continue
            vid = int(tok[0])
            feats[vid] = np.array(tok[1:1 + F], dtype=np.float32)
            labels[vid] = int(ll.split()[1])
            masks[vid] = names.get(lm.split()[1], 3)
    return feats, labels, masks


def test_cora_100_epochs_bf16_accuracy_close_to_fp32():
    """100 epochs of the Cora GCN ([1433, 128, 7]) with the same seed in both arms: the final test accuracy of the
    BF16-gather run is within 0.02 of the FP32 run."""
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    feats, labels, masks = cora_tables()
    g = golden_store.load("cora_self_P1_F8")
    V = feats.shape[0]
    pg = PartitionedGraph(HostGraph(g["edges"], V), 1, 0).generate_all(device=d, dist=True)
    acc = {}
    for arm in (None, torch.bfloat16):
        torch.manual_seed(0)
        model = GCNImpl(pg, [1433, 128, 7], torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                        torch.from_numpy(masks).to(d), seed=0, gather_dtype=arm)
        for _ in range(100):
            _, a = model.run_epoch(test=True)
        correct, total = a[2].tolist()
        acc[arm] = correct / max(total, 1)
    assert acc[None] > 0.3
    assert abs(acc[torch.bfloat16] - acc[None]) <= 0.02, acc
