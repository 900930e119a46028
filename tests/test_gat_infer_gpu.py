"""Full-neighbour inference of sampled GAT on the GPU (K10: nts_gat_softmax_stats_sharded and
nts_gat_aggregate_sharded, ShardedFeatureTable.gat_aggregate, GATSampleImpl.infer / evaluate_full), against the
float64 restatement of gat_infer_oracle.py:

  * the kernels on torch.cat(shards) at H in {1, 2, 4, 8, 16, 32} x D in {8, 64}, 4 x 32, and one head at widths 1,
    3, 41 and 602; FP32 and BF16 row shards; 1, 3 and 32 shards (some empty); empty rows, a hub row of 3 000
    in-edges, multi-edges, logits up to +-90 (exp overflows without the max subtraction) and offsets that start
    inside the edge arrays.  seg_max must equal the float32 computation of the same expression; seg_sum and the
    output are held to per-row bounds (1e-4, 2^-7 for BF16 rows);
  * the entries' refusals, before any launch, and their empty no-ops;
  * infer at world 1 with a tensor, FP32 and BF16 tables and a ShardedTopology, on Cora and the synth9k hub graph;
    at fanouts >= the largest in-degree it equals Forward over every vertex and the full-graph GATImpl;
  * world 2 and 3 as processes sharing one GPU (world 3 with an empty rank), replicated graph and ShardedTopology;
  * infer leaves training bit-identical, and evaluate_full after 20 Cora epochs is within 0.05 of full-graph GAT."""
import numpy as np
import pytest

import gat_infer_oracle as go
from test_infer_gpu import SHARDINGS, cora, dev, host_csc, kernel_graph, make_shards, synth9k, whole_graph

torch = pytest.importorskip("torch")
import torch.distributed as dist

pytestmark = pytest.mark.gpu


def ptr(t):
    return t if t is None or isinstance(t, int) else t.data_ptr()


def run_stats(m, z, sptrs, offs, n_shards, spitch, dst, idx, col, n_rows, eb, ee, H):
    from neutronstarlite_b200 import _lib
    return _lib.load().nts_gat_softmax_stats_sharded(ptr(m), ptr(z), ptr(sptrs), ptr(offs), n_shards, spitch,
                                                     ptr(dst), ptr(idx), ptr(col), n_rows, eb, ee, H, 0.2,
                                                     torch.cuda.current_stream().cuda_stream)


def run_agg(out, ptrs, dtype, offs, n_shards, pitch, sptrs, spitch, dst, m, z, idx, col, n_rows, eb, ee, F, H):
    from neutronstarlite_b200 import _lib
    return _lib.load().nts_gat_aggregate_sharded(ptr(out), ptr(ptrs), dtype, ptr(offs), n_shards, pitch, ptr(sptrs),
                                                 spitch, ptr(dst), ptr(m), ptr(z), ptr(idx), ptr(col), n_rows, eb, ee,
                                                 F, H, 0.2, torch.cuda.current_stream().cuda_stream)


SHAPES = [(H, D) for H in (2, 4, 8, 16, 32) for D in (8, 64)] + [(4, 32)] + [(1, F) for F in (1, 3, 8, 41, 64, 602)]


@pytest.mark.parametrize("H,D", SHAPES, ids=["%dx%d" % s for s in SHAPES])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_kernels_match_float64_on_the_concatenated_shards(H, D, dtype):
    if dtype == torch.bfloat16 and H > 1 and D % 8:
        pytest.skip("a BF16 head must be whole 16-byte loads")
    d = dev()
    V, F = 1500, H * D
    col, row, _ = kernel_graph(V, H * 100 + D)
    rng = np.random.default_rng(F)
    T = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    S = rng.uniform(-45, 45, (V, H)).astype(np.float32)
    Dd = rng.uniform(-45, 45, (V, H)).astype(np.float32)
    g_col = torch.from_numpy(col.astype(np.uint32).view(np.int32)).to(d)
    g_row = torch.from_numpy(row.astype(np.uint32).view(np.int32)).to(d)
    code = 1 if dtype == torch.bfloat16 else 0
    for n_shards, cut in SHARDINGS.items():
        off = cut(V)
        shards, ptrs, offs, pitch, seen = make_shards(T, off, dtype, d)
        sshards, sptrs, _, spitch, _ = make_shards(S, off, torch.float32, d)
        for r0, r1 in ((0, V), (V // 3 - 5, V - 3)):
            eb, ee = int(col[r0]), int(col[r1])
            n = r1 - r0
            dst = torch.from_numpy(Dd[r0:r1]).to(d)
            seg = torch.full((2, n, H), float("nan"), device=d)
            out = torch.zeros((n, F), device=d)
            assert run_stats(seg[0], seg[1], sptrs, offs, n_shards, spitch, dst, g_row, g_col[r0:], n, eb, ee, H) == 0
            assert run_agg(out, ptrs, code, offs, n_shards, pitch, sptrs, spitch, dst, seg[0], seg[1], g_row,
                           g_col[r0:], n, eb, ee, F, H) == 0
            torch.cuda.synchronize()
            c = col[r0:r1 + 1]
            # seg_max: the float32 expression, exactly
            logit32, dsti, _, _ = go.stats(c, row, S.astype(np.float64), Dd[r0:r1].astype(np.float64))
            x = S[row[c[0]:c[-1]]] + Dd[r0:r1][dsti]
            x = np.where(x > 0, x, x * np.float32(0.2))
            m32 = np.full((n, H), -np.inf, dtype=np.float32)
            np.maximum.at(m32, dsti, x)
            m32[np.diff(c) == 0] = 0
            assert np.array_equal(seg[0].cpu().numpy(), m32), (n_shards, r0)
            _, _, m64, z64 = go.stats(c, row, S, Dd[r0:r1])
            zg = seg[1].cpu().numpy().astype(np.float64)
            assert (np.abs(zg - z64) <= 1e-4 * z64).all(), (n_shards, r0, float(np.abs(zg / z64 - 1).max()))
            assert (zg[np.diff(c) == 0] == 1).all()
            ref = go.aggregate(c, row, S, Dd[r0:r1], seen, H)
            bound = go.aggregate_abs(c, row, S, Dd[r0:r1], seen, H).max(1, keepdims=True)
            err = np.abs(out.cpu().numpy().astype(np.float64) - ref)
            tol = (2.0 ** -7 if code else 1e-4) * bound
            assert (err <= tol + 1e-30).all(), (n_shards, r0, float((err / (bound + 1e-30)).max()))
            assert (out[torch.from_numpy(np.diff(c) == 0).to(d)] == 0).all()
        del shards, sshards


def test_kernel_refusals_and_empty_no_ops():
    from neutronstarlite_b200 import _lib
    d = dev()
    V, H, D = 300, 4, 8
    F = H * D
    col, row, _ = kernel_graph(V, 3)
    g_col = torch.from_numpy(col.astype(np.uint32).view(np.int32)).to(d)
    g_row = torch.from_numpy(row.astype(np.uint32).view(np.int32)).to(d)
    _, ptrs, offs, pitch, _ = keep = make_shards(np.ones((V, F), np.float32), [0, V], torch.float32, d)
    _, sptrs, _, spitch, _ = skeep = make_shards(np.ones((V, H), np.float32), [0, V], torch.float32, d)
    dst = torch.zeros((V, H), device=d)
    seg = torch.zeros((2, V + 1, H), device=d)
    out = torch.zeros((V + 1, F), device=d)
    E = int(col[-1])
    lib = _lib.load()
    s_ok = dict(m=seg[0], z=seg[1], sptrs=sptrs, offs=offs, n_shards=1, spitch=spitch, dst=dst, idx=g_row, col=g_col,
                n_rows=V, eb=0, ee=E, H=H)
    a_ok = dict(out=out, ptrs=ptrs, dtype=0, offs=offs, n_shards=1, pitch=pitch, sptrs=sptrs, spitch=spitch, dst=dst,
                m=seg[0], z=seg[1], idx=g_row, col=g_col, n_rows=V, eb=0, ee=E, F=F, H=H)
    launches = lib.nts_kernel_launch_count()

    def refused(fn, ok, why, **kw):
        assert fn(*dict(ok, **kw).values()) != 0, kw
        assert why in lib.nts_last_error().decode(), lib.nts_last_error()

    for fn, ok in ((run_stats, s_ok), (run_agg, a_ok)):
        refused(fn, ok, "1..32 shards", n_shards=33)
        refused(fn, ok, "1..32 shards", n_shards=0)
        refused(fn, ok, "score_pitch", spitch=2)             # < heads
        refused(fn, ok, "score_pitch", spitch=6)             # % 4 != 0
        refused(fn, ok, "null pointer", idx=None)
        refused(fn, ok, "null pointer", dst=None)
        refused(fn, ok, "aligned", sptrs=sptrs.data_ptr() + 4)
        refused(fn, ok, "reversed", eb=E, ee=0)
        refused(fn, ok, "uint32", ee=1 << 32)
    refused(run_stats, s_ok, "divide 32", H=3, spitch=4)
    refused(run_stats, s_ok, "null pointer", z=None)
    refused(run_agg, a_ok, "shard_dtype", dtype=2)
    refused(run_agg, a_ok, "shard_pitch", pitch=30)
    refused(run_agg, a_ok, "shard_pitch", dtype=1, pitch=36)
    refused(run_agg, a_ok, "multiple of heads", F=30)
    refused(run_agg, a_ok, "head width", F=24, H=8, spitch=8)   # D = 3: a load would span two heads
    refused(run_agg, a_ok, "head width", dtype=1, F=16)     # BF16 D = 4
    refused(run_agg, a_ok, "null pointer", m=None)
    refused(run_agg, a_ok, "aligned", out=out.data_ptr() + 2)
    torch.cuda.synchronize()
    assert lib.nts_kernel_launch_count() == launches       # nothing was launched
    assert int(torch.count_nonzero(seg)) == 0 and int(torch.count_nonzero(out)) == 0
    # empty calls look at no pointer
    assert run_stats(None, None, None, None, 99, 3, None, None, None, 0, 0, 5, 3) == 0
    assert run_agg(None, None, 7, None, 99, 3, None, 1, None, None, None, None, None, 0, 0, 5, F, 3) == 0
    assert run_agg(None, None, 7, None, 99, 3, None, 1, None, None, None, None, None, 10, 5, 5, F, 3) == 0
    assert run_agg(None, None, 7, None, 99, 3, None, 1, None, None, None, None, None, 10, 0, 5, 0, 3) == 0
    assert lib.nts_kernel_launch_count() == launches
    # rows without edges: only the init pass runs, and every segment gets (0, 1)
    flat = torch.full((4,), E, dtype=torch.int32, device=d)
    assert run_stats(seg[0], seg[1], sptrs, offs, 1, spitch, dst, g_row, flat, 3, E, E, H) == 0
    torch.cuda.synchronize()
    assert (seg[0, :3] == 0).all() and (seg[1, :3] == 1).all() and int(torch.count_nonzero(seg[1, 3:])) == 0
    seg.zero_()
    assert run_stats(*s_ok.values()) == 0 and run_agg(*a_ok.values()) == 0
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(out)) > 0
    del keep, skeep


def test_table_gat_aggregate_refusals():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    d = dev()
    rows = ShardedFeatureTable(torch.ones((10, 8), device=d), [0, 10])
    scores = ShardedFeatureTable(torch.zeros((10, 2), device=d), [0, 10])
    col = torch.tensor([0, 2, 3], dtype=torch.int32, device=d)
    idx = torch.tensor([1, 9, 4], dtype=torch.int32, device=d)
    dst = torch.zeros((2, 2), device=d)
    out = torch.zeros((2, 8), device=d)
    rows.gat_aggregate(out, scores, dst, col, idx, 0, 3, 2)
    torch.cuda.synchronize()
    assert out.tolist() == [[1.0] * 8, [1.0] * 8]             # equal logits: a mean of ones
    bf = ShardedFeatureTable(torch.zeros((10, 2), device=d), [0, 10], dtype=torch.bfloat16)
    wide = ShardedFeatureTable(torch.zeros((10, 3), device=d), [0, 10])
    before = out.clone()
    for args, why in (((out, bf, dst, col, idx, 0, 3, 2), "float32 ShardedFeatureTable"),
                      ((out, wide, dst, col, idx, 0, 3, 2), "float32 ShardedFeatureTable"),
                      ((out, scores, dst.t().contiguous()[:1], col, idx, 0, 3, 2), "dst_score"),
                      ((out, scores, dst.double(), col, idx, 0, 3, 2), "dst_score"),
                      ((out, scores, dst.cpu(), col, idx, 0, 3, 2), "dst_score"),
                      ((out, scores, dst, col.long(), idx, 0, 3, 2), "column_offset"),
                      ((out, scores, dst, col, idx, 0, 4, 2), "edge_begin"),
                      ((torch.zeros((2, 7), device=d), scores, dst, col, idx, 0, 3, 2), "out must be")):
        with pytest.raises(_lib.NtsError, match=why):
            rows.gat_aggregate(*args)
    for F, H, dt, why in ((9, 3, torch.float32, "divide 32"), (6, 2, torch.float32, "multiple of 4"),
                          (8, 2, torch.bfloat16, "multiple of 8"), (12, 8, torch.float32, "not a multiple")):
        t = ShardedFeatureTable(torch.ones((10, F), device=d), [0, 10], dtype=dt)
        s = ShardedFeatureTable(torch.zeros((10, H), device=d), [0, 10])
        with pytest.raises(_lib.NtsError, match=why):
            t.gat_aggregate(torch.zeros((2, F), device=d), s, torch.zeros((2, H), device=d), col, idx, 0, 3, H)
        t.close()
        s.close()
    other = ShardedFeatureTable(torch.zeros((10, 2), device=d), [0, 10])
    other.offsets = np.array([0, 9])                             # a table over other offsets
    with pytest.raises(_lib.NtsError, match="same ranks and offsets"):
        rows.gat_aggregate(out, other, dst, col, idx, 0, 3, 2)
    scores.close()
    with pytest.raises(_lib.NtsError, match="closed"):
        rows.gat_aggregate(out, scores, dst, col, idx, 0, 3, 2)
    torch.cuda.synchronize()
    assert torch.equal(out, before)
    for t in (rows, bf, wide, other):
        t.close()


# ---- infer at world 1 ----------------------------------------------------------------------------------------------

def make_model(pg, layers, features, V, d, fanout, heads, gather_dtype=None, seed=3, batch_size=256):
    from neutronstarlite_b200.toolkits import GATSampleImpl
    gen = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, layers[-1], (V,), generator=gen)
    mask = torch.arange(V) % 3
    return GATSampleImpl(pg, layers, features, labels.to(d), mask, fanout=fanout, batch_size=batch_size, heads=heads,
                         seed=seed, sample_seed=1, gather_dtype=gather_dtype)


def params(model):
    return [[p.W.detach().cpu().double().numpy() for p in ps] for ps in (model.P, model.al, model.ar)]


def check_outputs(out, csc, X, model, bf16=False, rows=None, rtol=1e-4):
    """out (this rank's rows `rows` of the last layer) against the float64 restatement with the model's weights."""
    Ws, als, ars = params(model)
    rnd = (lambda T: go.bf16(T.astype(np.float32))) if bf16 else None
    ref, bound = go.infer(csc[0], csc[1], X.astype(np.float64), Ws, als, ars, model.heads, round_rows=rnd,
                          with_bound=True)
    if rows is not None:
        ref, bound = ref[rows], bound[rows]
    got = out.cpu().numpy().astype(np.float64) if torch.is_tensor(out) else out
    assert got.shape == ref.shape
    err = np.abs(got - ref)
    assert (err <= (2.0 ** -7 if bf16 else rtol) * bound + 1e-30).all(), float((err / (bound + 1e-30)).max())
    return ref


@pytest.mark.parametrize("kind", ["tensor", "table", "table_bf16", "topology"])
@pytest.mark.parametrize("graph,layers,heads", [("cora", [1433, 64, 7], 8), ("synth9k", [37, 32, 5], 4)])
def test_world_1_infer_matches_float64(kind, graph, layers, heads):
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    from neutronstarlite_b200.topology import ShardedTopology
    d = dev()
    edges, V = cora() if graph == "cora" else synth9k()
    pg = whole_graph(edges, V, d)
    csc = host_csc(pg)
    X = np.random.default_rng(layers[0]).uniform(-1, 1, (V, layers[0])).astype(np.float32)
    x = torch.from_numpy(X).to(d)
    features, topo, gather_dtype = x, pg, None
    if kind.startswith("table"):
        gather_dtype = torch.bfloat16 if kind == "table_bf16" else None
        features = ShardedFeatureTable(x, [0, V], dtype=gather_dtype or torch.float32)
    if kind == "topology":
        c = pg.graph_chunks[0]
        topo = ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu,
                                     [0, V // 3, V // 3, V])
    m = make_model(topo, layers, features, V, d, [4, 9], heads, gather_dtype=gather_dtype)
    lo, out = m.infer()
    assert lo == 0 and out.shape == (V, layers[-1]) and out.dtype == torch.float32 and m.step == 0
    # a BF16 table's rows are rounded once at the input, as the model reads them
    Xin = go.bf16(X) if kind == "table_bf16" else X
    check_outputs(out, csc, Xin, m, bf16=kind == "table_bf16")
    if kind.startswith("table"):
        features.close()
    if kind == "topology":
        topo.close()


def test_refused_head_shape_raises_before_any_collective():
    from neutronstarlite_b200 import _lib
    d = dev()
    edges, V = synth9k()
    m = make_model(whole_graph(edges, V, d), [37, 24, 5], torch.zeros((V, 37), device=d), V, d, [4, 4], 8)
    with pytest.raises(_lib.NtsError, match="layer 0"):
        m.infer()                                                # 8 heads x 3: a load would span two heads


def test_fanouts_above_the_largest_in_degree_give_forward_and_full_graph_gat():
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    rng = np.random.default_rng(12)
    V = 3000
    edges = np.stack([rng.integers(0, V, 30000), rng.integers(0, V, 30000)], 1).astype(np.uint32)
    pg = whole_graph(edges, V, d)
    csc = host_csc(pg)
    assert np.diff(csc[0]).max() <= 40
    X = rng.uniform(-1, 1, (V, 48)).astype(np.float32)
    x = torch.from_numpy(X).to(d)
    layers = [48, 64, 6]
    m = make_model(pg, layers, x, V, d, [40, 40], 8, batch_size=V)
    _, out = m.infer()
    _, bound = go.infer(csc[0], csc[1], X, *params(m), m.heads, with_bound=True)
    tol = torch.from_numpy(1e-4 * bound).to(d)
    with torch.no_grad():
        fwd = m.Forward(torch.arange(V), False)
    seeds = m.subgraph.seeds().long()
    assert ((fwd - out[seeds]).abs() <= tol[seeds]).all()
    fpg = PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=d, dist=True)
    full = GATImpl(fpg, layers, x.clone(), m.L_GT, torch.arange(V).to(d) % 3, heads=8, seed=0, fused_kernel=True)
    with torch.no_grad():
        for dst_ps, src_ps in ((full.P, m.P), (full.al, m.al), (full.ar, m.ar)):
            for a, b in zip(dst_ps, src_ps):
                a.W.copy_(b.W)
    full.Forward()
    assert ((full.X[-1].detach() - out).abs() <= tol).all()


def test_infer_leaves_training_alone():
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges
    from neutronstarlite_b200.toolkits import GATSampleImpl
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    feats, labels, masks = cora_tables()
    x = torch.from_numpy(feats).to(d)
    runs = []
    for with_infer in (False, True):
        m = GATSampleImpl(pg, [1433, 64, 7], x, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                          fanout=[10, 10], batch_size=64, heads=8, seed=0, sample_seed=0)
        res = []
        for _ in range(2):
            res.append(m.run_epoch(test=False))
            if with_infer:
                step, grads = m.step, [None if p.W.grad is None else p.W.grad.clone() for p in m.params()]
                m.infer()
                m.evaluate_full(1)
                assert m.step == step
                for p, g in zip(m.params(), grads):
                    assert (p.W.grad is None and g is None) or torch.equal(p.W.grad, g)
        runs.append((res, m.step, [p.W.detach().clone() for p in m.params()]))
    (ra, sa, wa), (rb, sb, wb) = runs
    assert ra == rb and sa == sb
    for a, b in zip(wa, wb):
        assert torch.equal(a, b)


def test_evaluate_full_on_cora_reaches_full_graph_gat_accuracy():
    from test_gat_sample_gpu import graph
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GATImpl, GATSampleImpl
    d = dev()
    feats, labels, masks = cora_tables()
    layers = [1433, 64, 7]
    m = GATSampleImpl(graph(cora_edges(), 2708), layers, torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                      torch.from_numpy(masks), fanout=[10, 10], batch_size=64, heads=8, seed=0, sample_seed=0)
    for _ in range(20):
        m.run_epoch(test=False)
    _, out = m.infer()
    ids = torch.from_numpy(np.nonzero(masks == 2)[0]).to(d)
    want = float((out[ids].argmax(1).cpu() == torch.from_numpy(labels)[ids.cpu()]).sum()) / ids.numel()
    got = m.evaluate_full(2)
    assert got == want
    fpg = PartitionedGraph(HostGraph(cora_edges(), 2708), 1, 0).generate_all(device=d, dist=True)
    full = GATImpl(fpg, layers, torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                   torch.from_numpy(masks).to(d), heads=8, seed=0, fused_kernel=True)
    for _ in range(20):
        full.run_epoch()
    full.Forward()
    test = torch.from_numpy(masks).to(d) == 2
    full_acc = float((full.X[-1].argmax(1) == full.L_GT)[test].float().mean())
    assert got >= full_acc - 0.05, (got, full_acc)


# ---- world 2 and 3 ---------------------------------------------------------------------------------------------------

CASE_LAYERS, CASE_FANOUT, CASE_HEADS = [37, 32, 5], [8, 12], 4


def _worker(rank, world, port, per_gpu, q):
    try:
        from test_dist_sample_gpu import _init, table_offsets
        from test_infer_gpu import dist_case
        from test_sharded_topology_gpu import shard_slices
        dev_ = _init(rank, world, port, per_gpu)
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        from neutronstarlite_b200.topology import ShardedTopology
        hg, pg, X = dist_case(dev_)
        V = hg.vertices
        off = table_offsets(hg, world)
        x = torch.from_numpy(X[off[rank]:off[rank + 1]]).to(dev_)
        res = {}
        for kind in ("replicated", "topology"):
            table = ShardedFeatureTable(x, off)
            graph = pg
            if kind == "topology":
                t_off = [0] + [min(V, o + 17) for o in off[1:-1]] + [V]
                graph = ShardedTopology(*shard_slices(pg, t_off[rank], t_off[rank + 1]), t_off)
            m = make_model(graph, CASE_LAYERS, table, V, dev_, CASE_FANOUT, CASE_HEADS)
            lo, out = m.infer()
            acc = [m.evaluate_full(s) for s in (1, 2)]
            res[kind] = (lo, out.cpu().numpy(), acc, params(m), m.step)
            table.close()
            if kind == "topology":
                graph.close()
        q.put((rank, "ok", res))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def run_dist(world, per_gpu, port):
    from test_dist_sample_gpu import spawn
    from test_infer_gpu import dist_case
    d = dev()
    ranks = spawn(_worker, world, port, per_gpu)
    hg, pg, X = dist_case(d)
    csc = host_csc(pg)
    V = hg.vertices
    heads = [CASE_HEADS, 1]
    for kind in ("replicated", "topology"):
        P = ranks[0][kind][3]
        ref, bound = go.infer(csc[0], csc[1], X.astype(np.float64), *P, heads, with_bound=True)
        rows = np.zeros(V, dtype=int)
        empty = 0
        for r in ranks:
            lo, out, acc, Pr, step = r[kind]
            assert step == 0 and acc == ranks[0][kind][2]
            for a, b in zip(sum(Pr, []), sum(P, [])):
                assert np.array_equal(a, b)
            err = np.abs(out - ref[lo:lo + out.shape[0]])
            assert (err <= 1e-4 * bound[lo:lo + out.shape[0]] + 1e-30).all(), kind
            rows[lo:lo + out.shape[0]] += 1
            empty += out.shape[0] == 0
        assert (rows == 1).all(), kind
        assert empty == (1 if world == 3 else 0)


@pytest.mark.parametrize("world", [2, 3])
def test_infer_on_ranks_sharing_one_gpu_matches_float64(world):
    run_dist(world, False, 29730 + world)


def test_infer_with_one_rank_per_gpu_matches_float64():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_dist(2, True, 29740)
