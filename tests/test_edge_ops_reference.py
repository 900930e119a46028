"""The unfused GAT chain (K5 row movers and segment kernels, K6 edge softmax, the fused-weight aggregation of
DistGPUAggregateDstFuseWeight) against float64 on the structured graph of test_gat_fp32_reference.py (empty rows,
segments of 4096 / 4097 / 20 011 edges, duplicates, a hub source, slots without out-edges), and the 64-edge-quantum
kernels on the Zipf graph past the grid-stride boundary.

Copies must be bit-exact.  Sums are compared per row against the float64 sum, scaled by the row's sum of magnitudes
(row_close); attention weights as |a - a64| <= 1e-4 a64 + 1e-7."""
import numpy as np
import pytest

from test_gat_fp32_reference import GRID, np64, structured, zipf_graph  # noqa: F401  (zipf_graph is a fixture)
from test_gather_plan_bf16 import row_close

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream().cuda_stream


def dst_of_edges(off):
    return torch.repeat_interleave(torch.arange(off.numel() - 1, device=off.device), torch.diff(off))


def seg_sum64(rows, vals, n):
    """float64 index_add of vals into n rows, and the same sum of |vals|."""
    v = vals.double()
    return (torch.zeros((n,) + v.shape[1:], dtype=torch.float64, device=v.device).index_add_(0, rows, v),
            torch.zeros((n,) + v.shape[1:], dtype=torch.float64, device=v.device).index_add_(0, rows, v.abs()))


def sum_close(got, rows, vals, n, init=None):
    want, mag = seg_sum64(rows, vals, n)
    if init is not None:
        want, mag = want + init.double(), mag + init.double().abs()
    row_close(np64(got), np64(want), scale=np64(mag))


def check_fuse_weight(pg, off, slot, H, D, seed):
    """DistGPUAggregateDstFuseWeight: out = sum a[e,h] m[slot], d_mirror = sum a g[dst], d_a = <m[slot], g[dst]>."""
    from neutronstarlite_b200 import ops
    d = off.device
    V, M, E, F = pg.owned_vertices, pg.owned_mirrors, pg.owned_edges, H * D
    gen = torch.Generator(device=d).manual_seed(seed)
    m = torch.rand((M, F), generator=gen, device=d) * 2 - 1
    a = torch.rand((E, H), generator=gen, device=d)
    g = torch.rand((V, F), generator=gen, device=d) * 2 - 1
    op = ops.DistGPUAggregateDstFuseWeight(pg)
    out = op.forward(m, a)
    dm = op.backward(g)
    da = op.get_additional_grad()
    torch.cuda.synchronize()
    dst = dst_of_edges(off)
    ms = m.double()[slot].view(E, H, D)
    gd = g.double()[dst].view(E, H, D)
    sum_close(out, dst, (ms * a.double()[:, :, None]).view(E, F), V)
    sum_close(dm, slot, (gd * a.double()[:, :, None]).view(E, F), M)
    err = (da.double() - (ms * gd).sum(-1)).abs()
    assert bool((err <= 1e-4 * (ms.abs() * gd.abs()).sum(-1) + 1e-30).all()), float(err.max())


# ---- K6 edge softmax -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [1, 3, 8, 32])
def test_edge_softmax_vs_float64(H):
    """Forward and backward at H columns on the structured graph: warp segments, and the whole-CTA path of the
    4097- and 20 011-edge segments with H > 1.  Constant logits in every third segment give a == fl(1/deg) exactly."""
    from neutronstarlite_b200 import ops
    d = dev()
    st = structured()
    pg = st.graph()
    off, _ = st.torch_csc(d)
    dst = dst_of_edges(off)
    gen = torch.Generator(device=d).manual_seed(H)
    x = torch.rand((st.E, H), generator=gen, device=d) * 8 - 4
    flat = dst % 3 == 0
    x[flat] = (dst[flat] % 5).float()[:, None].expand(-1, H)
    g = torch.rand((st.E, H), generator=gen, device=d) * 2 - 1
    op = ops.DistGPUEdgeSoftMax(pg)
    a = op.forward(x)
    gi = op.backward(g)
    torch.cuda.synchronize()
    assert torch.equal(op.IntermediateResult, a)
    x64 = x.double()
    mx = torch.full((st.Vp, H), -float("inf"), dtype=torch.float64, device=d).scatter_reduce(
        0, dst[:, None].expand(-1, H), x64, "amax")
    ex = torch.exp(x64 - mx[dst])
    a64 = ex / torch.zeros((st.Vp, H), dtype=torch.float64, device=d).index_add_(0, dst, ex)[dst]
    err = (a.double() - a64).abs()
    assert bool((err <= 1e-4 * a64 + 1e-7).all()), float((err / a64).max())
    deg = torch.diff(off)[dst].float()
    assert torch.equal(a[flat], (1.0 / deg[flat])[:, None].expand(-1, H))
    ag = a64 * g.double()
    dot = torch.zeros((st.Vp, H), dtype=torch.float64, device=d).index_add_(0, dst, ag)[dst]
    dot_mag = torch.zeros((st.Vp, H), dtype=torch.float64, device=d).index_add_(0, dst, ag.abs())[dst]
    err = (gi.double() - (ag - a64 * dot)).abs()
    assert bool((err <= 1e-4 * (ag.abs() + a64 * dot_mag) + 1e-12).all()), float(err.max())


# ---- K7 chain: fused-weight aggregation ---------------------------------------------------------------------------------
@pytest.mark.parametrize("H,D", [(H, D) for H, D, tiles, _ in GRID if tiles > 1])
def test_fuse_weight_aggregation_multi_tile_vs_float64(H, D):
    """Head mode 1 of the aggregation with 2-3 column tiles (head boundaries inside a tile) and
    fuse_weight_backward_kernel at the same widths."""
    d = dev()
    st = structured()
    off, slot = st.torch_csc(d)
    check_fuse_weight(st.graph(), off, slot, H, D, seed=H * 100 + D)


# ---- K5 row movers and segment kernels ---------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 3, 64, 129, 602])
def test_scatter_and_aggregate_operators_vs_float64(F):
    """ScatterSrc / ScatterDst forward and AggregateDst backward are copies (bit-exact); ScatterSrc backward (atomic
    scatter into mirror slots, duplicates included), ScatterDst backward and AggregateDst forward (segment sums, in
    column passes of 32 vectors at F > 128) against float64."""
    from neutronstarlite_b200 import ops
    d = dev()
    st = structured()
    pg = st.graph()
    off, slot = st.torch_csc(d)
    dst = dst_of_edges(off)
    gen = torch.Generator(device=d).manual_seed(F)
    m = torch.rand((st.M, F), generator=gen, device=d) * 2 - 1
    x = torch.rand((st.Vp, F), generator=gen, device=d) * 2 - 1
    msg = torch.rand((st.E, F), generator=gen, device=d) * 2 - 1
    src_op, dst_op, agg_op = ops.DistGPUScatterSrc(pg), ops.DistGPUScatterDst(pg), ops.DistGPUAggregateDst(pg)
    assert torch.equal(src_op.forward(m), m[slot])
    assert torch.equal(dst_op.forward(x), x[dst])
    assert torch.equal(agg_op.backward(x), x[dst])
    sum_close(src_op.backward(msg), slot, msg, st.M)
    sum_close(dst_op.backward(msg), dst, msg, st.Vp)
    sum_close(agg_op.forward(msg), dst, msg, st.Vp)


@pytest.mark.parametrize("F", [1, 3, 64, 602])
def test_scatter_grad_back_to_message_and_atomic_row_scatter(F):
    """nts_scatter_grad_back_to_message adds the destination row to every edge of its segment (one FP32 add per
    element, so bit-exact); nts_scatter_add_rows_atomic adds source rows into destination rows that repeat."""
    from neutronstarlite_b200 import _lib
    d = dev()
    st = structured()
    pg = st.graph()
    off, _ = st.torch_csc(d)
    gen = torch.Generator(device=d).manual_seed(F + 1)
    x = torch.rand((st.Vp, F), generator=gen, device=d) * 2 - 1
    msg0 = torch.rand((st.E, F), generator=gen, device=d) * 2 - 1
    msg = msg0.clone()
    _lib.call("nts_scatter_grad_back_to_message", x.data_ptr(), msg.data_ptr(), pg.row_indices_gpu.data_ptr(),
              pg.column_offset_gpu.data_ptr(), st.Vp, F, stream())
    torch.cuda.synchronize()
    assert torch.equal(msg, msg0 + x[dst_of_edges(off)])
    n_rows, n_dst = 50_000, 300
    rows = torch.randint(0, n_dst, (n_rows,), generator=gen, device=d)
    rows[: n_rows // 4] = 17                          # one row hit 12 500 times
    src = torch.rand((n_rows, F), generator=gen, device=d) * 2 - 1
    out0 = torch.rand((n_dst, F), generator=gen, device=d) * 2 - 1
    out = out0.clone()
    rows32 = rows.to(torch.int32)
    _lib.call("nts_scatter_add_rows_atomic", out.data_ptr(), src.data_ptr(), rows32.data_ptr(), n_rows, F, stream())
    torch.cuda.synchronize()
    sum_close(out, rows, src, n_dst, init=out0)


# ---- the 64-edge kernels past the grid-stride boundary ---------------------------------------------------------------
def test_chain_kernels_past_the_grid_stride_boundary(zipf_graph):
    """On > 10 M edges every warp of the 64-edge-quantum kernels (segment sum, segment broadcast, accumulating
    broadcast, fuse_weight_backward_kernel) strides past its first ~1 M edges."""
    from neutronstarlite_b200 import _lib, ops
    pg, off, slot = zipf_graph
    d = off.device
    F = 8
    dst = dst_of_edges(off)
    gen = torch.Generator(device=d).manual_seed(12)
    x = torch.rand((pg.owned_vertices, F), generator=gen, device=d) * 2 - 1
    msg = torch.rand((pg.owned_edges, F), generator=gen, device=d) * 2 - 1
    agg = ops.DistGPUAggregateDst(pg)
    sum_close(agg.forward(msg), dst, msg, pg.owned_vertices)
    acc = msg.clone()
    _lib.call("nts_scatter_grad_back_to_message", x.data_ptr(), acc.data_ptr(), pg.row_indices_gpu.data_ptr(),
              pg.column_offset_gpu.data_ptr(), pg.owned_vertices, F, stream())
    torch.cuda.synchronize()
    assert torch.equal(acc, msg + x[dst])
    del acc
    assert torch.equal(agg.backward(x), x[dst])
    del msg
    check_fuse_weight(pg, off, slot, 2, 4, seed=13)
