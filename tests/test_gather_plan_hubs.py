"""nts_gather_plan with dense hub blocks (nts_gather_plan_create_hybrid, csrc/nts_plan.cu): the hub-column block
[rows x hub cols], the hub-row block [hub rows x gathered rows] and the slab-bucketed residual together against the C
oracle of the reference's aggregation loop, per ROW relative to that row's magnitude (1e-4, north_star), integer
artefacts (every edge counted once) exactly through the all-ones product."""
import numpy as np
import pytest

import oracle_c

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HUBS = [0, 1, 17, 64, 5000]     # 5000: more than the rows of either side (clamped)
WIDTHS = [602, 128, 100, 41, 7, 1, 1433, 64]


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def up_u32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(dev())


def row_close(actual, desired, rtol=1e-4, scale=None):
    """max |err| of every row <= rtol * scale of THAT row (default: max |desired| of the row)."""
    err = np.abs(actual.astype(np.float64) - desired.astype(np.float64)).max(axis=1)
    scale = np.abs(desired if scale is None else scale).max(axis=1).astype(np.float64)
    bad = np.nonzero(err > rtol * scale + 1e-30)[0]
    assert bad.size == 0, "rows %s: err %s vs scale %s" % (bad[:5], err[bad[:5]], scale[bad[:5]])


def agg_close(actual, off, idx, w, X, rtol=1e-4):
    """Against the oracle, per row relative to the row's sum of |w| * |x|: the dense blocks add a hub row's thousands of
    signed terms in another order than the oracle's edge loop (cell weights first, split K), so where those terms
    cancel, the error is only small next to their magnitude, not next to the nearly zero result."""
    row_close(actual, oracle_c.segment_gather_sum(off, idx, w, X), rtol,
              scale=oracle_c.segment_gather_sum(off, idx, None if w is None else np.abs(w), np.abs(X)))


def csr(dst, src, n_rows, rng):
    order = np.lexsort((src, dst))
    dst, src = dst[order], src[order]
    off = np.zeros(n_rows + 1, dtype=np.uint32)
    np.add.at(off, dst + 1, 1)
    off = np.cumsum(off).astype(np.uint32)
    w = rng.uniform(0.1, 1.0, dst.shape[0]).astype(np.float32)
    return off, src.astype(np.uint32), w


def hub_graph(rng, n_rows=700, n_src=900, n_edges=40000):
    """Power-law-ish multigraph: Zipf endpoints (hub sources and hub destinations), repeated (dst, src) pairs, empty
    destination rows."""
    dst = np.minimum(rng.zipf(1.6, n_edges) - 1, n_rows - 1)
    src = np.minimum(rng.zipf(1.6, n_edges) - 1, n_src - 1)
    dst = rng.permutation(n_rows)[dst]
    src = rng.permutation(n_src)[src]
    dst = np.concatenate([dst, dst[:5000]])                  # multi-edges
    src = np.concatenate([src, src[:5000]])
    keep = dst % 9 != 4                                      # some destinations without edges
    return csr(dst[keep], src[keep], n_rows, rng)


def make_plan(off, idx, w, base, n_src, slabs, hubs, slot_of=None):
    from neutronstarlite_b200 import ops
    return ops.GatherPlan(up_u32(off), up_u32(idx), None if w is None else torch.from_numpy(w).to(dev()), base,
                          off.shape[0] - 1, idx.shape[0], n_src, slabs, slot_of=None if slot_of is None else
                          up_u32(slot_of), hubs=hubs)


def run(plan, X, out=None):
    x = X if torch.is_tensor(X) else torch.from_numpy(X).to(dev())
    if out is None:
        out = torch.zeros((plan.n_rows, x.shape[1]), dtype=torch.float32, device=dev())
    plan.run(x, out)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("hub_rows", HUBS)
@pytest.mark.parametrize("hub_cols", HUBS)
@pytest.mark.parametrize("slabs", [1, 3])
def test_hybrid_plan_matches_oracle(slabs, hub_cols, hub_rows):
    rng = np.random.default_rng(3000 + slabs * 100 + hub_cols + 7 * hub_rows)
    n_rows, n_src = 700, 900
    off, idx, w = hub_graph(rng, n_rows, n_src)
    base = 5000
    plan = make_plan(off, idx + base, w, base, n_src, slabs, (hub_cols, hub_rows))
    assert plan.slabs == slabs
    assert (plan.hub_cols, plan.hub_rows) == (min(hub_cols, n_src), min(hub_rows, n_rows))
    for F in WIDTHS:
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        agg_close(run(plan, X).cpu().numpy(), off, idx, w, X)
    # every edge counted exactly once: all-ones input, unit weights -> in-degree counts
    ones = make_plan(off, idx + base, None, base, n_src, slabs, (hub_cols, hub_rows))
    cnt = run(ones, np.ones((n_src, 4), dtype=np.float32)).cpu().numpy()
    assert np.array_equal(cnt[:, 0], np.diff(off.astype(np.int64)).astype(np.float32))


def test_all_hub_plan_and_share_keys():
    """A plan without hubs keeps the plain share key; one whose hub columns are every gathered row (no residual edge
    left for the slab launches) matches the oracle and reports its hub counts in the key."""
    rng = np.random.default_rng(41)
    off, idx, w = hub_graph(rng, 300, 400, 20000)
    assert make_plan(off, idx, w, 0, 400, 2, (0, 0)).key() == (2,)
    p = make_plan(off, idx, w, 0, 400, 2, (400, 0))            # every gathered row is a hub: no residual edges
    X = rng.uniform(-1, 1, (400, 33)).astype(np.float32)
    agg_close(run(p, X).cpu().numpy(), off, idx, w, X)
    assert p.key() == (2, 400, 0)


def test_hybrid_plan_slot_table_unaligned_views_and_accumulation():
    """Indices through a slot table, an input view whose base is only 4-byte aligned (padded workspace), output views
    that are 4- and 8-byte aligned (scalar and 2-wide stores of the dense epilogues), accumulation into a non-zero
    output."""
    rng = np.random.default_rng(77)
    n_rows, n_src = 300, 500
    off, idx, w = hub_graph(rng, n_rows, n_src, 20000)
    ids = rng.permutation(4000)[:n_src].astype(np.uint32)
    slot_of = np.zeros(4000, dtype=np.uint32)
    slot_of[ids] = np.arange(n_src, dtype=np.uint32)
    plan = make_plan(off, ids[idx], w, 0, n_src, 3, (32, 20), slot_of=slot_of)
    for F, shift in ((128, 1), (602, 2), (64, 2), (41, 1)):
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        ref = oracle_c.segment_gather_sum(off, idx, w, X)
        mag = oracle_c.segment_gather_sum(off, idx, w, np.abs(X))
        flat = torch.zeros(n_src * F + 1, dtype=torch.float32, device=dev())
        flat[1:] = torch.from_numpy(X).to(dev()).reshape(-1)
        xv = flat[1:].view(n_src, F)
        assert xv.data_ptr() % 16 != 0
        oflat = torch.ones(n_rows * F + shift, dtype=torch.float32, device=dev())
        ov = oflat[shift:].view(n_rows, F)
        run(plan, xv, ov)
        run(plan, xv, ov)                                      # accumulates, like every aggregation entry
        row_close(ov.cpu().numpy(), 1.0 + 2.0 * ref, rtol=2e-4, scale=1.0 + 2.0 * mag)
        assert float(oflat[:shift].sum()) == shift              # nothing written before the view


def test_tuned_plan_prefilter_keeps_uniform_graphs_hub_free():
    """A uniform graph has no row or column dense enough to be a hub candidate: the measured plan has no hubs."""
    from neutronstarlite_b200 import ops
    rng = np.random.default_rng(5)
    V, E = 5000, 300000
    off, idx, w = csr(rng.integers(0, V, E), rng.integers(0, V, E), V, rng)
    plan = ops.GatherPlan(up_u32(off), up_u32(idx), torch.from_numpy(w).to(dev()), 0, V, E, V, 0, tune_for=128)
    assert (plan.hub_cols, plan.hub_rows) == (0, 0)


def test_widths_with_different_hub_counts_share_nothing_and_are_right():
    """Plans of one chunk direction are shared between widths only when slab AND hub counts agree: a width that
    settled on a hybrid plan and one that settled on a plain plan with the same slab count keep their own arrays,
    and both compute the aggregation."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    rng = np.random.default_rng(11)
    V, E = 3000, 200000
    edges = np.stack([rng.zipf(1.5, E) % V, rng.zipf(1.5, E) % V], 1).astype(np.uint32)
    pg = PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev())
    c = pg.graph_chunks[0]
    real = ops.GatherPlan
    picks = {602: (64, 32), 128: (0, 0)}

    def forced(*a, tune_for=0, **kw):      # what measurement might pick per width, forced
        return real(*a[:7], 2, hubs=picks[tune_for], **kw)
    ops.GatherPlan = forced
    ops.set_plan_mode("on", 0)
    try:
        res = {}
        for F in picks:
            x = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).to(dev())
            y = ops.gather_by_dst_from_src(c, torch.zeros_like(x), x)
            torch.cuda.synchronize()
            res[F] = (x.cpu().numpy(), y.cpu().numpy())
    finally:
        ops.GatherPlan = real
        ops.set_plan_mode("auto", 0)
    assert c._gather_plan_for[("fwd", "F", 602)] is not c._gather_plan_for[("fwd", "F", 128)]
    assert ("fwd", 2, 64, 32) in c._gather_plans and ("fwd", 2) in c._gather_plans
    for F, (x, y) in res.items():
        agg_close(y, c.column_offset, c.row_indices, c.edge_weight_forward, x)


@pytest.mark.parametrize("hubs", [(10 ** 6, 0), (0, 10 ** 6)])
def test_dense_blocks_are_bit_identical_across_builds(hubs):
    """With every gathered row a hub column (or every output row a hub row) the run is the dense block times an
    identity matrix, i.e. the block itself, exactly: two builds must agree bit for bit, and each cell must be the sum
    of its multi-edges' weights."""
    rng = np.random.default_rng(9)
    n_rows, n_src = 300, 200
    off, idx, w = hub_graph(rng, n_rows, n_src, 30000)
    eye = np.eye(n_src, dtype=np.float32)
    a = run(make_plan(off, idx, w, 0, n_src, 1, hubs), eye).cpu().numpy()
    b = run(make_plan(off, idx, w, 0, n_src, 1, hubs), eye).cpu().numpy()
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    dense = np.zeros((n_rows, n_src), dtype=np.float64)
    np.add.at(dense, (np.repeat(np.arange(n_rows), np.diff(off.astype(np.int64))), idx), w)
    row_close(a, dense, rtol=1e-5)
