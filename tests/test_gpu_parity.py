"""Parity of the sm_90a kernels, called through the C ABI, against
  (1) the golden vectors of the UNMODIFIED reference CPU operators (tests/golden, P = 1, 2, 4, 8),
  (2) the C / numpy oracle on seeded random multigraphs (hubs, empty rows, duplicates; every vector-width class),
  (3) size-independent properties at larger sizes (exact in-degree counts, linearity).
Tolerance for float results: 1e-4 relative (BASELINE.json north_star), written as RTOL below; integer-valued
results (copies, counts) must be bit-exact."""
import numpy as np
import pytest

import nts_oracle as O
import oracle_c

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

RTOL = 1e-4
ATOL = 1e-5


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def up(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.view(dtype) if t.element_size() == torch.tensor([], dtype=dtype).element_size() else t.to(dtype)
    return t.to(dev())


def up_u32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(dev())


def close(actual, desired, rtol=RTOL, atol=ATOL):
    """Element-wise rtol plus, for 2-D results, a per-ROW check: the largest error of a row against the largest
    magnitude of THAT row (a global scale would let the hub rows hide errors in ordinary rows)."""
    actual, desired = np.asarray(actual), np.asarray(desired)
    if desired.ndim == 2 and desired.size:
        err = np.abs(actual.astype(np.float64) - desired.astype(np.float64)).max(axis=1)
        scale = np.abs(desired).max(axis=1).astype(np.float64)
        bad = np.nonzero(err > 10 * rtol * scale + atol)[0]
        assert bad.size == 0, "rows %s: err %s, row scale %s" % (bad[:4], err[bad[:4]], scale[bad[:4]])
    scale = max(1.0, float(np.abs(desired).max()) if desired.size else 1.0)
    np.testing.assert_allclose(actual, desired, rtol=rtol, atol=atol * scale)


def lib():
    from neutronstarlite_b200 import _lib
    return _lib


def stream():
    return torch.cuda.current_stream().cuda_stream


def gpu_segment_gather(offsets, indices, w, X, base, out=None, slots=None):
    L = lib()
    n_rows = offsets.shape[0] - 1
    d_off, d_idx = up_u32(offsets), up_u32(indices)
    d_w = None if w is None else up(w.astype(np.float32))
    d_x = up(X.astype(np.float32))
    d_out = torch.zeros((n_rows, X.shape[1]), dtype=torch.float32, device=dev()) if out is None else up(out)
    if slots is None:
        L.call("nts_segment_gather_sum", d_x.data_ptr(), d_out.data_ptr(), 0 if d_w is None else d_w.data_ptr(),
               d_idx.data_ptr(), d_off.data_ptr(), int(base), n_rows, int(indices.shape[0]), X.shape[1], stream())
    else:
        d_s = up_u32(slots)
        L.call("nts_segment_gather_sum_slots", d_x.data_ptr(), d_out.data_ptr(), 0 if d_w is None else d_w.data_ptr(),
               d_idx.data_ptr(), d_off.data_ptr(), d_s.data_ptr(), n_rows, int(indices.shape[0]), X.shape[1], stream())
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


# ------------------------------------------------------------------------------------------------------------
# (1) golden vectors of the reference
# ------------------------------------------------------------------------------------------------------------
def test_golden_gcn_forward_backward_per_rank(golden):
    """Each rank's chunks exactly as the reference built them (its own arrays), run chunk after chunk in the
    reference's ring order through nts_gather_by_dst_from_src / nts_gather_by_src_from_dst."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import CSCSegment
    g = golden
    po = g.partition_offset
    Xg = np.concatenate([g.mat(r, "X") for r in range(g.P)], axis=0)
    dX_acc = np.zeros((g.V, g.F), dtype=np.float32)
    for r in range(g.P):
        Vp = int(po[r + 1] - po[r])
        y = torch.zeros((Vp, g.F), dtype=torch.float32, device=dev())
        G = up(g.mat(r, "G"))
        for step in range(g.P):
            i = (r + step) % g.P
            t = "chunk%d_" % i
            c = CSCSegment()
            meta = g.get(r, t + "meta")
            c.edge_size, c.batch_size_forward, c.batch_size_backward = int(meta[0]), int(meta[1]), int(meta[2])
            c.src_range, c.dst_range = (int(meta[3]), int(meta[4])), (int(meta[5]), int(meta[6]))
            for name in ("column_offset", "row_indices", "row_offset", "column_indices"):
                setattr(c, name + "_gpu", up_u32(g.get(r, t + name)))
            c.edge_weight_forward_gpu = up(g.get(r, t + "edge_weight_forward"))
            c.edge_weight_backward_gpu = up(g.get(r, t + "edge_weight_backward"))
            xs = up(Xg[c.src_range[0]:c.src_range[1]])
            if xs.shape[0] and Vp:
                ops.gather_by_dst_from_src(c, y, xs)
            if c.batch_size_backward and Vp:
                part = torch.zeros((c.batch_size_backward, g.F), dtype=torch.float32, device=dev())
                ops.gather_by_src_from_dst(c, part, G)
                dX_acc[c.src_range[0]:c.src_range[1]] += part.cpu().numpy()
        close(y.cpu().numpy(), g.mat(r, "gcn_Y"))
    ref_dX = np.concatenate([g.mat(r, "gcn_dX") for r in range(g.P)], axis=0)
    close(dX_acc, ref_dX)


def test_golden_edge_ops(golden):
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import PartitionedGraph
    g = golden
    po = g.partition_offset
    for r in range(g.P):
        Vp, Ep, M = (int(x) for x in g.get(r, "meta")[4:7])
        if Vp == 0:
            continue
        pg = PartitionedGraph(None, g.P, r, po)
        pg.owned_vertices, pg.owned_edges, pg.owned_mirrors = Vp, Ep, M
        pg.column_offset_gpu = up_u32(g.get(r, "whole_column_offset"))
        pg.row_indices_gpu = up_u32(g.get(r, "whole_row_indices"))
        pg.mirror_index_gpu = up_u32(g.get(r, "mirror_index"))
        mirror = up(g.mat(r, "dep_mirror"))
        X = up(g.mat(r, "X"))
        G = up(g.mat(r, "G"))
        Ge = up(g.mat(r, "Ge"))
        # copies: bit-exact
        op = ops.DistGPUScatterSrc(pg)
        msg = op.forward(mirror).cpu().numpy()
        assert np.array_equal(msg, g.mat(r, "dep_mirror")[g.get(r, "mirror_index")[g.get(r, "whole_row_indices")]])
        if g.has(r, "scatter_src_msg"):
            assert np.array_equal(msg, g.mat(r, "scatter_src_msg"))
        close(op.backward(Ge).cpu().numpy(), g.mat(r, "scatter_src_dmirror"))
        op = ops.DistGPUScatterDst(pg)
        msg = op.forward(X).cpu().numpy()
        if g.has(r, "scatter_dst_msg"):
            assert np.array_equal(msg, g.mat(r, "scatter_dst_msg"))
        close(op.backward(Ge).cpu().numpy(), g.mat(r, "scatter_dst_dX"))
        op = ops.DistGPUAggregateDst(pg)
        close(op.forward(Ge).cpu().numpy(), g.mat(r, "aggregate_dst_Y"))
        dmsg = op.backward(G).cpu().numpy()
        if g.has(r, "aggregate_dst_dmsg"):
            assert np.array_equal(dmsg, g.mat(r, "aggregate_dst_dmsg"))
        # softmax: reference tolerance is 1e-7 on a constant input (test_getdepneighbor_gpu.hpp:316); we use 1e-5 abs
        op = ops.DistGPUEdgeSoftMax(pg)
        a = op.forward(up(g.mat(r, "softmax_in", 1)))
        np.testing.assert_allclose(a.cpu().numpy(), g.mat(r, "softmax_out", 1), rtol=RTOL, atol=1e-6)
        gin = op.backward(up(g.mat(r, "softmax_gout", 1)))
        np.testing.assert_allclose(gin.cpu().numpy(), g.mat(r, "softmax_gin", 1), rtol=RTOL, atol=1e-5)
        # fused aggregation
        op = ops.DistGPUAggregateDstFuseWeight(pg)
        att = up(g.mat(r, "softmax_out", 1))
        close(op.forward(mirror, att).cpu().numpy(), g.mat(r, "fuse_Y"))
        dm = op.backward(G).cpu().numpy()
        dw = op.get_additional_grad().cpu().numpy()
        close(dw, g.mat(r, "fuse_dweight", 1))
        # the reference adds the unweighted gradient once more (core/ntsDistCPUGraphOp.hpp:572) and races; compare
        # with the oracle restatement of the correct gradient instead
        co, ri, mi = g.get(r, "whole_column_offset"), g.get(r, "whole_row_indices"), g.get(r, "mirror_index")
        dm_o, dw_o = O.aggregate_dst_fuse_weight_backward(co, ri, mi, g.mat(r, "dep_mirror"),
                                                          g.mat(r, "softmax_out", 1), g.mat(r, "G"), M)
        close(dm, dm_o)
        close(dw, dw_o)


def test_golden_dep_neighbor_single_gpu(golden):
    """DistGPUGetDepNbrOp at P=1 (no communication): mirror rows and returned gradients vs the reference."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.exchange import GpuExchange
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    g = golden
    if g.P != 1:
        pytest.skip("single-partition case only (P>1 is covered by tests/test_multi_gpu.py)")
    pg = PartitionedGraph(HostGraph(g.edges, g.V), 1, 0).generate_all(device=dev(), dist=True)
    op = ops.DistGPUGetDepNbrOp(pg, None, exchange=GpuExchange(pg))
    mirror = op.forward(up(g.mat(0, "X")))
    assert np.array_equal(mirror.cpu().numpy(), g.mat(0, "dep_mirror"))
    dx = op.backward(up(g.mat(0, "dep_Gm")))
    close(dx.cpu().numpy(), g.mat(0, "dep_dX"))


# ------------------------------------------------------------------------------------------------------------
# (2) seeded random multigraphs against the C oracle
# ------------------------------------------------------------------------------------------------------------
def random_csr(n_rows, n_src, n_edges, seed, hub_rows=2, empty_every=7):
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, n_rows, n_edges)
    rows[rows % empty_every == 3] = (rows[rows % empty_every == 3] + 1) % n_rows  # leave some rows empty
    for h in range(hub_rows):
        rows[rng.integers(0, n_edges, n_edges // 6)] = (h * 31 + 5) % n_rows      # hubs cut by many quanta
    rows.sort()
    idx = rng.integers(0, n_src, n_edges).astype(np.uint32)
    off = np.zeros(n_rows + 1, dtype=np.uint32)
    np.cumsum(np.bincount(rows, minlength=n_rows), out=off[1:])
    w = rng.uniform(-1, 1, n_edges).astype(np.float32)
    return off, idx, w


@pytest.mark.parametrize("F", [1, 2, 7, 41, 47, 64, 100, 128, 172, 256, 602, 1433])
@pytest.mark.parametrize("variant", [1, 2])
def test_random_graph_vs_c_oracle(F, variant):
    """Every vector-width / chunk-count class of the kernel, both index-staging variants, accumulate-into-output
    semantics and a non-zero index base (global source ids of a remote partition)."""
    L = lib()
    off, idx, w = random_csr(1500, 1100, 40000, seed=F * 13 + variant)
    rng = np.random.default_rng(F)
    X = rng.uniform(-1, 1, (1100, F)).astype(np.float32)
    init = rng.uniform(-1, 1, (1500, F)).astype(np.float32)  # kernels ACCUMULATE into the output
    base = 4096
    try:
        L.call("nts_aggregate_set_variant", variant, 0)
        got0 = gpu_segment_gather(off, idx, w, X, 0, out=init)
        got1 = gpu_segment_gather(off, idx + base, w, X, base, out=init)
    finally:
        L.call("nts_aggregate_set_variant", 0, 0)
    ref = oracle_c.segment_gather_sum(off, idx, w, X, base=0, out=init.copy())
    close(got0, ref)
    close(got1, ref)


@pytest.mark.parametrize("Q", [32, 64, 512])
def test_quantum_sizes_and_unweighted(Q):
    L = lib()
    off, idx, w = random_csr(700, 900, 30000, seed=Q)
    X = np.random.default_rng(Q).uniform(-1, 1, (900, 96)).astype(np.float32)
    try:
        for variant in (1, 2):
            L.call("nts_aggregate_set_variant", variant, Q)
            close(gpu_segment_gather(off, idx, None, X, 0), oracle_c.segment_gather_sum(off, idx, None, X))
            close(gpu_segment_gather(off, idx, w, X, 0), oracle_c.segment_gather_sum(off, idx, w, X))
    finally:
        L.call("nts_aggregate_set_variant", 0, 0)


def test_slot_table_variant():
    off, idx, w = random_csr(300, 5000, 9000, seed=5)
    rng = np.random.default_rng(9)
    used = np.unique(idx)
    slot_of = np.zeros(5000, dtype=np.uint32)
    slot_of[used] = rng.permutation(used.shape[0]).astype(np.uint32)
    Xc = rng.uniform(-1, 1, (used.shape[0], 64)).astype(np.float32)
    ref = oracle_c.segment_gather_sum(off, slot_of[idx], w, Xc)
    close(gpu_segment_gather(off, idx, w, Xc, 0, slots=slot_of), ref)


def test_empty_and_degenerate_inputs():
    L = lib()
    # no edges at all: the output must be untouched
    off = np.zeros(11, dtype=np.uint32)
    out = gpu_segment_gather(off, np.zeros(0, dtype=np.uint32), None, np.ones((4, 8), np.float32), 0,
                             out=np.full((10, 8), 3.0, np.float32))
    assert (out == 3.0).all()
    # one row owning every edge (a pure hub), one edge, leading/trailing empty rows
    rng = np.random.default_rng(1)
    idx = rng.integers(0, 50, 5000).astype(np.uint32)
    w = rng.uniform(-1, 1, 5000).astype(np.float32)
    X = rng.uniform(-1, 1, (50, 602)).astype(np.float32)
    off = np.array([0, 0, 0, 5000, 5000], dtype=np.uint32)
    close(gpu_segment_gather(off, idx, w, X, 0), oracle_c.segment_gather_sum(off, idx, w, X))
    off = np.array([0, 0, 1, 1], dtype=np.uint32)
    close(gpu_segment_gather(off, idx[:1], w[:1], X, 0), oracle_c.segment_gather_sum(off, idx[:1], w[:1], X))


def test_gather_scatter_rows_and_records():
    L = lib()
    rng = np.random.default_rng(3)
    src = rng.uniform(-1, 1, (500, 602)).astype(np.float32)
    rows = rng.permutation(500)[:200].astype(np.uint32)
    d_src, d_rows = up(src), up_u32(rows)
    d_dst = torch.zeros((200, 602), dtype=torch.float32, device=dev())
    L.call("nts_gather_rows", d_dst.data_ptr(), d_src.data_ptr(), d_rows.data_ptr(), 200, 602, stream())
    assert np.array_equal(d_dst.cpu().numpy(), src[rows])
    acc = rng.uniform(-1, 1, (500, 602)).astype(np.float32)
    d_acc = up(acc)
    L.call("nts_scatter_add_rows", d_acc.data_ptr(), d_dst.data_ptr(), d_rows.data_ptr(), 200, 602, stream())
    expect = acc.copy()
    expect[rows] += src[rows]
    assert np.array_equal(d_acc.cpu().numpy(), expect)
    # (vid,row) records through mapped pinned memory, the reference's message format
    F, n = 16, 300
    rec = np.zeros((n, F + 1), dtype=np.float32)
    vids = rng.permutation(1000)[:n].astype(np.uint32)
    rec[:, 0] = vids.view(np.float32)
    rec[:, 1:] = rng.uniform(-1, 1, (n, F)).astype(np.float32)
    hp = L.load().nts_malloc_pinned(rec.nbytes)
    import ctypes
    ctypes.memmove(hp, rec.ctypes.data, rec.nbytes)
    dp = L.load().nts_pinned_device_pointer(hp)
    mirror = torch.zeros((400, F), dtype=torch.float32, device=dev())
    L.call("nts_deserialize_records", mirror.data_ptr(), dp, n, F, 100, 500, stream())
    torch.cuda.synchronize()
    expect = np.zeros((400, F), dtype=np.float32)
    sel = (vids >= 100) & (vids < 500)
    expect[vids[sel] - 100] = rec[sel, 1:]
    assert np.array_equal(mirror.cpu().numpy(), expect)
    L.call("nts_aggregate_records", mirror.data_ptr(), dp, n, F, 100, 500, stream())
    torch.cuda.synchronize()
    assert np.array_equal(mirror.cpu().numpy(), expect * 2)
    L.load().nts_free_pinned(hp)


@pytest.mark.parametrize("H", [1, 2, 3, 8])
def test_edge_softmax_multi_column_with_hub(H):
    L = lib()
    rng = np.random.default_rng(H)
    deg = rng.integers(0, 40, 400)
    deg[7] = 20000  # block-cooperative path (> kHubDegree)
    off = np.zeros(401, dtype=np.uint32)
    np.cumsum(deg, out=off[1:])
    E = int(off[-1])
    m = (rng.standard_normal((E, H)) * 4).astype(np.float32)
    ref = oracle_c.edge_softmax(off, m)
    d_off, d_m = up_u32(off), up(m)
    d_a = torch.zeros_like(d_m)
    d_c = torch.zeros_like(d_m)
    L.call("nts_edge_softmax_forward", d_a.data_ptr(), d_m.data_ptr(), d_c.data_ptr(), 0, d_off.data_ptr(), 400, H, stream())
    np.testing.assert_allclose(d_a.cpu().numpy(), ref, rtol=RTOL, atol=1e-7)
    assert torch.equal(d_a, d_c)
    g = rng.standard_normal((E, H)).astype(np.float32)
    d_g = up(g)
    d_gi = torch.zeros_like(d_g)
    L.call("nts_edge_softmax_backward", d_gi.data_ptr(), d_g.data_ptr(), d_c.data_ptr(), 0, d_off.data_ptr(), 400, H, stream())
    np.testing.assert_allclose(d_gi.cpu().numpy(), O.edge_softmax_backward(off, ref, g), rtol=RTOL, atol=2e-5)


# ------------------------------------------------------------------------------------------------------------
# (3) size-independent properties on a larger graph
# ------------------------------------------------------------------------------------------------------------
def test_properties_at_scale():
    """2M edges, F=602 (the headline width): unweighted aggregation of all-ones counts in-degrees EXACTLY;
    the weighted op is linear; fwd and bwd are adjoint: <A x, g> == <x, A^T g>."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import PartitionedGraph
    d = dev()
    V, E, F = 20000, 2_000_000, 602
    gen = torch.Generator(device=d).manual_seed(0x5EED0001)
    w = 1.0 / torch.arange(1, V + 1, device=d, dtype=torch.float64)
    cdf = torch.cumsum(w / w.sum(), 0)
    perm = torch.randperm(V, generator=gen, device=d)
    src = perm[torch.searchsorted(cdf, torch.rand(E, generator=gen, device=d, dtype=torch.float64)).clamp_(max=V - 1)]
    dst = perm[torch.searchsorted(cdf, torch.rand(E, generator=gen, device=d, dtype=torch.float64)).clamp_(max=V - 1)]
    pg = PartitionedGraph.from_device_edges(src, dst, V)
    c = pg.graph_chunks[0]
    ones = torch.ones((V, F), device=d)
    y = torch.zeros((V, F), device=d)
    ops.gather_by_dst_from_src(c, y, ones, with_weight=False)
    indeg = torch.bincount(dst, minlength=V).to(torch.float32)
    assert torch.equal(y, indeg[:, None].expand(V, F))          # bit-exact integer counts (< 2^24)
    x1 = torch.rand((V, F), generator=gen, device=d) * 2 - 1
    x2 = torch.rand((V, F), generator=gen, device=d) * 2 - 1
    op = ops.ForwardSingleGPUfuseOp(pg)
    y1, y2, y12 = op.forward(x1), op.forward(x2), op.forward(x1 + 0.5 * x2)
    torch.testing.assert_close(y12, y1 + 0.5 * y2, rtol=RTOL, atol=1e-4)
    g = torch.rand((V, F), generator=gen, device=d) * 2 - 1
    lhs = (y1.double() * g.double()).sum()
    rhs = (x1.double() * op.backward(g).double()).sum()
    assert abs(lhs - rhs) <= 1e-6 * max(1.0, abs(lhs))
    # device-built chunk == host-built chunk (bit-exact arrays) on a slice small enough for the host path
    from neutronstarlite_b200.graph import HostGraph
    sub = 200_000
    e_np = torch.stack([src[:sub], dst[:sub]], 1).cpu().numpy().astype(np.uint32)
    hpg = PartitionedGraph(HostGraph(e_np, V), 1, 0).generate_all()
    dpg = PartitionedGraph.from_device_edges(src[:sub], dst[:sub], V)
    hc, dc = hpg.graph_chunks[0], dpg.graph_chunks[0]
    for name in ("column_offset", "row_indices", "row_offset", "column_indices"):
        assert np.array_equal(getattr(hc, name).view(np.int32), getattr(dc, name + "_gpu").cpu().numpy()), name
    for name in ("edge_weight_forward", "edge_weight_backward"):
        assert np.array_equal(getattr(hc, name).view(np.uint32),
                              getattr(dc, name + "_gpu").cpu().numpy().view(np.uint32)), name


@pytest.mark.parametrize("H,D", [(1, 24), (2, 16), (8, 64), (8, 8), (3, 5), (4, 2), (4, 1)])
def test_multi_head_fused_aggregation(H, D):
    """Fused GAT aggregation with [E, H] attention weights (config D of BASELINE.json uses 8 heads): head h scales
    columns [h*D, (h+1)*D).  Oracle: the single-head C loop applied per head; backward against the numpy restatement
    of DistAggregateDstFuseWeight::backward (core/ntsDistCPUGraphOp.hpp:548-589, without its extra add)."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import PartitionedGraph
    rng = np.random.default_rng(H * 100 + D)
    Vp, Vg, E = 600, 2000, 20000
    off, idx, _ = random_csr(Vp, Vg, E, seed=H + D)
    used = np.unique(idx)
    mi = np.zeros(Vg + 1, dtype=np.uint32)
    mi[used + 1] = 1
    mi = np.cumsum(mi, dtype=np.uint32)
    M = int(mi[-1])
    F = H * D
    mirror = rng.uniform(-1, 1, (M, F)).astype(np.float32)
    a = rng.uniform(0, 1, (E, H)).astype(np.float32)
    g = rng.uniform(-1, 1, (Vp, F)).astype(np.float32)
    pg = PartitionedGraph(None, 1, 0, np.array([0, Vp], dtype=np.uint32))
    pg.owned_vertices, pg.owned_edges, pg.owned_mirrors = Vp, E, M
    pg.column_offset_gpu, pg.row_indices_gpu, pg.mirror_index_gpu = up_u32(off), up_u32(idx), up_u32(mi)
    op = ops.DistGPUAggregateDstFuseWeight(pg)
    y = op.forward(up(mirror), up(a)).cpu().numpy()
    slot = mi[idx]
    ref = np.zeros((Vp, F), dtype=np.float32)
    for h in range(H):
        ref[:, h * D:(h + 1) * D] = oracle_c.segment_gather_sum(off, slot, a[:, h], mirror[:, h * D:(h + 1) * D])
    close(y, ref)
    dm = op.backward(up(g)).cpu().numpy()
    dw = op.get_additional_grad().cpu().numpy()
    dm_ref = np.zeros((M, F), dtype=np.float32)
    dw_ref = np.zeros((E, H), dtype=np.float32)
    for h in range(H):
        sl = slice(h * D, (h + 1) * D)
        dmh, dwh = O.aggregate_dst_fuse_weight_backward(off, idx, mi, mirror[:, sl], a[:, h:h + 1], g[:, sl], M)
        dm_ref[:, sl] = dmh
        dw_ref[:, h:h + 1] = dwh
    close(dm, dm_ref)
    close(dw, dw_ref)


def test_offsets_beyond_32_bits():
    """Rows whose element offset exceeds 2^32 (the reference kernels compute feature_size*batch_size in 32 bits,
    cuda/ntsCUDAFuseKernel.cuh:280,299, and wrap): 9.0 M source rows x 512 floats = 4.6e9 elements (18.4 GB)."""
    d = dev()
    free, _ = torch.cuda.mem_get_info()
    if free < 30e9:
        pytest.skip("needs ~20 GB of free device memory")
    V_src, F, n_rows = 9_000_000, 512, 257
    x = torch.zeros((V_src, F), dtype=torch.float32, device=d)
    rng = np.random.default_rng(11)
    # sources concentrated at both ends of the matrix, in particular beyond element 2^32 (row 8 388 608)
    picks = np.concatenate([rng.integers(0, 1000, 2000), rng.integers(V_src - 1000, V_src, 6000),
                            rng.integers(8_388_608, 8_389_608, 2000)]).astype(np.uint32)
    rng.shuffle(picks)
    uniq = np.unique(picks)
    vals = rng.uniform(-1, 1, (uniq.shape[0], F)).astype(np.float32)
    x[torch.from_numpy(uniq.astype(np.int64)).to(d)] = torch.from_numpy(vals).to(d)
    deg = rng.integers(0, 80, n_rows)
    deg[5] = 3000  # one long row
    off = np.zeros(n_rows + 1, dtype=np.uint32)
    np.cumsum(deg, out=off[1:])
    E = int(off[-1])
    idx = np.resize(picks, E).astype(np.uint32)
    w = rng.uniform(-1, 1, E).astype(np.float32)
    out = torch.zeros((n_rows, F), dtype=torch.float32, device=d)
    L = lib()
    d_off, d_idx, d_w = up_u32(off), up_u32(idx), up(w)
    L.call("nts_segment_gather_sum", x.data_ptr(), out.data_ptr(), d_w.data_ptr(), d_idx.data_ptr(), d_off.data_ptr(),
           0, n_rows, E, F, stream())
    torch.cuda.synchronize()
    # oracle on the compacted matrix
    pos = np.searchsorted(uniq, idx).astype(np.uint32)
    ref = oracle_c.segment_gather_sum(off, pos, w, vals)
    close(out.cpu().numpy(), ref)
    del x
    torch.cuda.empty_cache()


@pytest.mark.parametrize("two_pass", [True, False])
@pytest.mark.parametrize("H,D", [(8, 8), (8, 64), (1, 64), (3, 5), (2, 16), (1, 41), (16, 4), (1, 200), (4, 32)])
def test_fully_fused_gat_layer_vs_operator_chain(H, D, two_pass):
    """K7 (stats + attention-weighted aggregation + single-pass backward) against the chain of individually tested
    operators (scatter-src / scatter-dst / leaky-relu / edge-softmax / fused aggregation) on a graph with a hub
    segment longer than the block-cooperative threshold."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import PartitionedGraph
    rng = np.random.default_rng(H * 1000 + D)
    Vp, Vg, E = 500, 1500, 30000
    off, idx, _ = random_csr(Vp, Vg, E, seed=H * 7 + D, hub_rows=1)
    used = np.unique(idx)
    mi = np.zeros(Vg + 1, dtype=np.uint32)
    mi[used + 1] = 1
    mi = np.cumsum(mi, dtype=np.uint32)
    M = int(mi[-1])
    F = H * D
    pg = PartitionedGraph(None, 1, 0, np.array([0, Vp], dtype=np.uint32))
    pg.owned_vertices, pg.owned_edges, pg.owned_mirrors = Vp, E, M
    pg.column_offset_gpu, pg.row_indices_gpu, pg.mirror_index_gpu = up_u32(off), up_u32(idx), up_u32(mi)
    mirror = up(rng.uniform(-1, 1, (M, F)).astype(np.float32))
    s_att = up(rng.uniform(-2, 2, (M, H)).astype(np.float32))
    d_att = up(rng.uniform(-2, 2, (Vp, H)).astype(np.float32))
    g = up(rng.uniform(-1, 1, (Vp, F)).astype(np.float32))
    # operator chain
    sc_s, sc_d, sm, fw = ops.DistGPUScatterSrc(pg), ops.DistGPUScatterDst(pg), ops.DistGPUEdgeSoftMax(pg), \
        ops.DistGPUAggregateDstFuseWeight(pg)
    pre = sc_s.forward(s_att) + sc_d.forward(d_att)
    logit = torch.nn.functional.leaky_relu(pre, 0.2)
    a = sm.forward(logit)
    out_ref = fw.forward(mirror, a)
    dm_ref = fw.backward(g)
    d_logit = sm.backward(fw.get_additional_grad())
    d_pre = d_logit * torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, 0.2))
    ds_ref = sc_s.backward(d_pre.contiguous())
    dd_ref = sc_d.backward(d_pre.contiguous())
    # K7
    fused = ops.DistGPUFusedGATOp(pg, negative_slope=0.2, two_pass_backward=two_pass)
    out = fused.forward(mirror, s_att, d_att)
    dm, ds, dd = fused.backward(g)
    torch.cuda.synchronize()
    torch.testing.assert_close(out, out_ref, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dm, dm_ref, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(ds, ds_ref, rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(dd, dd_ref, rtol=1e-3, atol=2e-5)


def test_full_size_reddit_shaped_graph():
    """Config B of BASELINE.json at FULL size (232 965 V, 114.8 M edges, F = 602 / 128): exact in-degree counts,
    adjointness of forward / backward, and an independent float64 PyTorch reference (index_add over the edge list) on
    an 8-column slice - the hub destination sums 8.9 M edges, so this also pins accuracy where fp32 order matters."""
    from neutronstarlite_b200 import ops, synth
    from neutronstarlite_b200.graph import PartitionedGraph
    d = dev()
    free, _ = torch.cuda.mem_get_info()
    if free < 40e9:
        pytest.skip("needs ~25 GB of free device memory")
    V, E_rand, layers = synth.WORKLOADS["reddit"]
    src, dst = synth.zipf_edges(V, E_rand, d)
    pg = PartitionedGraph.from_device_edges(src, dst, V)
    c = pg.graph_chunks[0]
    assert c.edge_size == E_rand + V
    indeg = torch.bincount(dst, minlength=V)
    assert int(indeg.max()) < (1 << 24)
    del src, dst
    F = layers[0]
    ones = torch.ones((V, F), device=d)
    y = torch.zeros((V, F), device=d)
    ops.gather_by_dst_from_src(c, y, ones, with_weight=False)
    assert torch.equal(y[:, 0], indeg.to(torch.float32)) and torch.equal(y[:, F - 1], indeg.to(torch.float32))
    del ones
    gen = torch.Generator(device=d).manual_seed(3)
    x = torch.rand((V, F), generator=gen, device=d) * 2 - 1
    y.zero_()
    ops.gather_by_dst_from_src(c, y, x)
    # float64 reference on 8 columns straight from the CSC arrays
    col = c.column_offset_gpu.long()
    dst_of_edge = torch.repeat_interleave(torch.arange(V, device=d), col[1:] - col[:-1])
    srcs = c.row_indices_gpu.long()
    ref = torch.zeros((V, 8), dtype=torch.float64, device=d)
    ref.index_add_(0, dst_of_edge, x[srcs, :8].double() * c.edge_weight_forward_gpu.double()[:, None])
    # per-ROW relative error: the hub row (8.9 M summands) must not set the scale for everybody else
    row_err = (y[:, :8].double() - ref).abs().amax(dim=1) / ref.abs().amax(dim=1).clamp(min=1e-30)
    assert float(row_err.max()) < 1e-4, (float(row_err.max()), int(row_err.argmax()))
    del ref, dst_of_edge, srcs
    # adjointness at the second width: <A x, g> == <x, A^T g>
    F2 = layers[1]
    x2 = torch.rand((V, F2), generator=gen, device=d) * 2 - 1
    g2 = torch.rand((V, F2), generator=gen, device=d) * 2 - 1
    op = ops.ForwardSingleGPUfuseOp(pg)
    lhs = (op.forward(x2).double() * g2.double()).sum()
    rhs = (x2.double() * op.backward(g2).double()).sum()
    assert abs(float(lhs - rhs)) <= 1e-6 * max(1.0, abs(float(lhs)))
