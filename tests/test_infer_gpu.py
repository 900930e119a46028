"""Full-neighbour inference of sampled GCN on the GPU (nts_segment_gather_sum_sharded, ShardedFeatureTable.aggregate,
GCNSampleImpl.infer / evaluate_full), against the float64 restatement of infer_oracle.py:

  * the kernel on torch.cat(shards) in float64 at widths 1..602, FP32 and BF16 shards, 1, 3 and 32 shards (some
    empty), empty rows, hub rows longer than an edge quantum, offsets that start inside the edge arrays and no weight;
    its refusals and its empty no-ops;
  * infer at world 1 with a tensor, an FP32 table, a BF16 table and a ShardedTopology, on Cora, the synth9k hub graph
    and a widening model; with fanouts >= the largest in-degree it is the full-graph GCN;
  * world 2 and 3 as processes sharing one GPU (world 3 with an empty rank), with the replicated graph and with a
    ShardedTopology, and world 2 with one rank per GPU (skipped below 2 GPUs);
  * infer leaves training alone: the same losses and weights, bit for bit, with and without infer between epochs."""
import numpy as np
import pytest

import golden_store
import infer_oracle

torch = pytest.importorskip("torch")
import torch.distributed as dist

pytestmark = pytest.mark.gpu


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def whole_graph(edges, V, d):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    return PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=d)


def host_csc(pg):
    c = pg.graph_chunks[0]
    col = c.column_offset_gpu.cpu().numpy().view(np.uint32).astype(np.int64)
    E = int(col[-1])
    return col, c.row_indices_gpu[:E].cpu().numpy().view(np.uint32).astype(np.int64), \
        c.edge_weight_forward_gpu[:E].cpu().numpy().astype(np.float64)


# ---- the kernel ----------------------------------------------------------------------------------------------------

def kernel_graph(V, seed):
    """A CSC with empty rows, a hub row of 3 000 in-edges (several edge quanta) and a few rows of 700."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 12, V)
    deg[rng.choice(V, V // 10, replace=False)] = 0
    deg[V // 3] = 3000
    deg[[5, V - 7]] = 700
    col = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(deg, out=col[1:])
    row = rng.integers(0, V, int(col[-1]))
    w = rng.uniform(-1, 1, int(col[-1])).astype(np.float32)
    return col, row, w


def make_shards(X, offsets, dtype, d):
    """Device shards of X's rows [offsets[o], offsets[o+1]) at the table's pitch, the pointer array, the offsets array
    and the float64 rows the kernel reads (BF16-rounded for BF16 shards)."""
    V, F = X.shape
    bf16 = dtype == torch.bfloat16
    pitch = (F + 7) // 8 * 8 if bf16 else (F + 3) // 4 * 4
    full = torch.zeros((V, pitch), dtype=torch.float32)
    full[:, :F] = torch.from_numpy(X)
    shards = [full[offsets[o]:offsets[o + 1]].to(d, dtype).contiguous() for o in range(len(offsets) - 1)]
    seen = torch.cat([s.float().cpu() for s in shards])[:, :F].double().numpy()
    ptrs = torch.tensor([s.data_ptr() for s in shards], dtype=torch.int64, device=d)
    offs = torch.tensor(np.asarray(offsets, dtype=np.int64).astype(np.uint32).view(np.int32), device=d)
    return shards, ptrs, offs, pitch, seen


def run_kernel(out, ptrs, dtype, offs, n_shards, pitch, w, idx, col, n_rows, eb, ee, F):
    from neutronstarlite_b200 import _lib
    return _lib.load().nts_segment_gather_sum_sharded(
        out if out is None or isinstance(out, int) else out.data_ptr(),
        ptrs if ptrs is None or isinstance(ptrs, int) else ptrs.data_ptr(), dtype,
        offs if offs is None or isinstance(offs, int) else offs.data_ptr(), n_shards, pitch,
        w if w is None or isinstance(w, int) else w.data_ptr(), idx if idx is None or isinstance(idx, int) else
        idx.data_ptr(), col if col is None or isinstance(col, int) else col.data_ptr(), n_rows, eb, ee, F,
        torch.cuda.current_stream().cuda_stream)


SHARDINGS = {1: lambda V: [0, V], 3: lambda V: [0, V // 3, V // 3, V],
             32: lambda V: [0] + sorted(np.random.default_rng(V).integers(0, V, 30).tolist()) + [V, V]}


@pytest.mark.parametrize("F", [1, 3, 4, 8, 37, 41, 64, 128, 602])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_kernel_matches_float64_on_the_concatenated_shards(F, dtype):
    d = dev()
    V = 2500
    col, row, w = kernel_graph(V, F)
    X = np.random.default_rng(F + 1).uniform(-1, 1, (V, F)).astype(np.float32)
    g_col = torch.from_numpy(col.astype(np.uint32).view(np.int32)).to(d)
    g_row = torch.from_numpy(row.astype(np.uint32).view(np.int32)).to(d)
    g_w = torch.from_numpy(w).to(d)
    code = 1 if dtype == torch.bfloat16 else 0
    for n_shards, cut in SHARDINGS.items():
        off = cut(V)
        assert len(off) == n_shards + 1
        shards, ptrs, offs, pitch, seen = make_shards(X, off, dtype, d)
        # the whole CSC, and rows [r0, r1) with offsets starting inside the edge arrays; with and without weights
        for r0, r1, weighted in ((0, V, True), (V // 3 - 5, V - 3, True), (7, V // 2, False)):
            eb, ee = int(col[r0]), int(col[r1])
            assert r0 == 0 or eb != 0
            out = torch.zeros((r1 - r0, F), dtype=torch.float32, device=d)
            assert run_kernel(out, ptrs, code, offs, n_shards, pitch, g_w if weighted else None, g_row,
                              g_col[r0:], r1 - r0, eb, ee, F) == 0
            torch.cuda.synchronize()
            wt = w.astype(np.float64) if weighted else None
            ref = infer_oracle.aggregate(col[r0:r1 + 1], row, wt, seen)
            bound = infer_oracle.aggregate(col[r0:r1 + 1], row, None if wt is None else np.abs(wt), np.abs(seen))
            # FP32 accumulation: at most (terms + pieces) roundings of 2^-24 relative to sum |w x| per row
            deg = np.diff(col[r0:r1 + 1])[:, None]
            err = np.abs(out.cpu().numpy().astype(np.float64) - ref)
            assert (err <= (deg + 8) * 2.0 ** -24 * bound + 1e-30).all(), (n_shards, r0, r1, weighted)
        del shards


def test_kernel_refusals_and_empty_no_ops():
    from neutronstarlite_b200 import _lib
    d = dev()
    V, F = 300, 41
    col, row, w = kernel_graph(V, 3)
    g_col = torch.from_numpy(col.astype(np.uint32).view(np.int32)).to(d)
    g_row = torch.from_numpy(row.astype(np.uint32).view(np.int32)).to(d)
    X = np.ones((V, F), dtype=np.float32)
    shards, ptrs, offs, pitch, _ = make_shards(X, [0, V], torch.float32, d)
    out = torch.zeros((V + 1, F), dtype=torch.float32, device=d)
    E = int(col[-1])
    ok = dict(out=out, ptrs=ptrs, dtype=0, offs=offs, n_shards=1, pitch=pitch, w=None, idx=g_row, col=g_col,
              n_rows=V, eb=0, ee=E, F=F)

    def refused(why, **kw):
        a = dict(ok, **kw)
        assert run_kernel(*a.values()) != 0, kw
        assert why in _lib.load().nts_last_error().decode(), _lib.load().nts_last_error()

    refused("shard_dtype", dtype=2)
    refused("shard_pitch", pitch=42)                    # FP32 pitch % 4 != 0
    refused("shard_pitch", pitch=40)                    # pitch < F
    refused("shard_pitch", dtype=1, pitch=44)           # BF16 pitch % 8 != 0
    refused("1..32 shards", n_shards=33)
    refused("1..32 shards", n_shards=0)
    refused("aligned", out=out.data_ptr() + 2)
    refused("aligned", ptrs=ptrs.data_ptr() + 4)
    refused("null pointer", idx=None)
    refused("reversed", eb=E, ee=0)
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(out)) == 0          # nothing was launched
    # empty no-ops look at no pointer
    launches = _lib.load().nts_kernel_launch_count()
    assert run_kernel(None, None, 7, None, 99, 3, None, None, None, 0, 0, 5, F) == 0
    assert run_kernel(None, None, 7, None, 99, 3, None, None, None, 10, 5, 5, F) == 0
    assert _lib.load().nts_kernel_launch_count() == launches
    assert run_kernel(*ok.values()) == 0
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(out)) > 0


def test_table_aggregate_refusals():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    d = dev()
    t = ShardedFeatureTable(torch.ones((10, 6), device=d), [0, 10])
    col = torch.tensor([0, 2, 3], dtype=torch.int32, device=d)
    row = torch.tensor([1, 9, 4], dtype=torch.int32, device=d)
    out = torch.zeros((2, 6), device=d)
    t.aggregate(out, col, row, None, 0, 3)
    torch.cuda.synchronize()
    assert out.tolist() == [[2.0] * 6, [1.0] * 6]
    for args in ((out.cpu(), col, row, None), (out, col.long(), row, None), (out, col, row.float(), None),
                 (out, col, row, torch.ones(3, device=d, dtype=torch.float64)), (torch.zeros((2, 5), device=d), col,
                                                                                 row, None)):
        with pytest.raises(_lib.NtsError):
            t.aggregate(*args, 0, 3)
    with pytest.raises(_lib.NtsError):
        t.aggregate(out, col, row, None, 0, 4)          # past the edge arrays
    t.close()
    with pytest.raises(_lib.NtsError, match="closed"):
        t.aggregate(out, col, row, None, 0, 3)


# ---- infer at world 1 ----------------------------------------------------------------------------------------------

def synth9k():
    z = golden_store.load("synth9k_P1_F2")
    return z["edges"], int(z["case"][0])


def cora():
    from test_sample_gpu import cora_edges
    return cora_edges(), 2708


def make_model(pg, layers, features, V, d, fanout, gather_dtype=None, classes=None, seed=3):
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    gen = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, classes or layers[-1], (V,), generator=gen)
    mask = torch.arange(V) % 3
    return GCNSampleImpl(pg, layers, features, labels.to(d), mask, fanout=fanout, batch_size=256, drop_rate=0.0,
                         seed=seed, sample_seed=1, gather_dtype=gather_dtype)


def check_outputs(out, csc, X, model, bf16=False, rows=None, rtol=1e-4):
    """out (this rank's rows `rows` of the last layer) against the float64 restatement with the model's weights."""
    Ws = [p.W.detach().cpu().double().numpy() for p in model.P]
    fanout = model.sampler.fanout
    X = infer_oracle.bf16(X) if bf16 else X.astype(np.float64)
    rnd = (lambda l, a: infer_oracle.bf16(a.astype(np.float32))) if bf16 else None
    ref = infer_oracle.infer(*csc, X, Ws, fanout, round_operand=rnd)
    bound = infer_oracle.magnitude(*csc, X, Ws, fanout)
    if rows is not None:
        ref, bound = ref[rows], bound[rows]
    got = out.cpu().numpy().astype(np.float64) if torch.is_tensor(out) else out
    assert got.shape == ref.shape
    tol = (2.0 ** -7 if bf16 else rtol) * bound
    err = np.abs(got - ref)
    assert (err <= tol + 1e-30).all(), float((err / (bound + 1e-30)).max())
    return ref


@pytest.mark.parametrize("kind", ["tensor", "table", "table_bf16", "topology"])
@pytest.mark.parametrize("graph,layers", [("cora", [1433, 32, 7]), ("synth9k", [37, 16, 5]),
                                          ("synth9k", [8, 32, 4])])
def test_world_1_infer_matches_float64(kind, graph, layers):
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    from neutronstarlite_b200.topology import ShardedTopology
    d = dev()
    edges, V = cora() if graph == "cora" else synth9k()
    pg = whole_graph(edges, V, d)
    csc = host_csc(pg)
    X = np.random.default_rng(len(layers) + layers[0]).uniform(-1, 1, (V, layers[0])).astype(np.float32)
    x = torch.from_numpy(X).to(d)
    features, topo, gather_dtype = x, pg, None
    if kind.startswith("table"):
        gather_dtype = torch.bfloat16 if kind == "table_bf16" else None
        features = ShardedFeatureTable(x, [0, V], dtype=gather_dtype or torch.float32)
    if kind == "topology":
        c = pg.graph_chunks[0]
        topo = ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu,
                                     [0, V // 3, V // 3, V])
    m = make_model(topo, layers, features, V, d, fanout=[4, 9], gather_dtype=gather_dtype)
    step = m.step
    lo, out = m.infer()
    assert lo == 0 and out.shape == (V, layers[-1]) and out.dtype == torch.float32
    assert m.step == step
    check_outputs(out, csc, X, m, bf16=kind == "table_bf16")
    if kind.startswith("table"):
        features.close()
    if kind == "topology":
        topo.close()


def test_fanouts_above_the_largest_in_degree_give_the_full_graph_gcn():
    from neutronstarlite_b200 import ops
    d = dev()
    rng = np.random.default_rng(12)
    V = 3000
    edges = np.stack([rng.integers(0, V, 30000), rng.integers(0, V, 30000)], 1).astype(np.uint32)
    pg = whole_graph(edges, V, d)
    csc = host_csc(pg)
    assert np.diff(csc[0]).max() <= 40
    x = torch.from_numpy(rng.uniform(-1, 1, (V, 64)).astype(np.float32)).to(d)
    for layers in ([64, 16, 6], [64, 96, 6]):
        m = make_model(pg, layers, x, V, d, fanout=[64, 40])
        _, out = m.infer()
        op = ops.ForwardSingleGPUfuseOp(pg)
        h = x
        for l, p in enumerate(m.P):
            h = op.forward(h.contiguous()).mm(p.W.detach())
            if l < len(m.P) - 1:
                h = torch.relu(h)
        bound = infer_oracle.magnitude(*csc, x.cpu().double().numpy(), [p.W.detach().cpu().double().numpy()
                                                                         for p in m.P], [64, 40])
        err = (out - h).abs().cpu().double().numpy()
        assert (err <= 1e-5 * bound + 1e-30).all()


def test_infer_leaves_training_alone():
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    feats, labels, masks = cora_tables()
    x = torch.from_numpy(feats).to(d)
    runs = []
    for with_infer in (False, True):
        torch.manual_seed(0)                            # the same dropout masks in both runs
        m = GCNSampleImpl(pg, [1433, 64, 7], x, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                          fanout=[10, 10], batch_size=64, seed=0, sample_seed=0)
        res = []
        for _ in range(3):
            res.append(m.run_epoch(test=True))
            if with_infer:
                step, grads = m.step, [p.W.grad.clone() for p in m.P]
                m.infer()
                m.evaluate_full(1)
                assert m.step == step
                assert all(torch.equal(p.W.grad, g) for p, g in zip(m.P, grads))
        runs.append((res, m.step, [p.W.detach().clone() for p in m.P]))
    (ra, sa, wa), (rb, sb, wb) = runs
    assert ra == rb and sa == sb
    for a, b in zip(wa, wb):
        assert torch.equal(a, b)


def test_evaluate_full_on_cora_after_training():
    """evaluate_full counts argmax hits of infer's outputs over the mask; after training it tracks the sampled
    accuracy."""
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    feats, labels, masks = cora_tables()
    m = GCNSampleImpl(pg, [1433, 64, 7], torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                      torch.from_numpy(masks), fanout=[10, 10], batch_size=64, seed=0, sample_seed=0)
    for _ in range(5):
        m.run_epoch(test=False)
    _, out = m.infer()
    for s in (1, 2):
        ids = torch.from_numpy(np.nonzero(masks == s)[0]).to(d)
        want = float((out[ids].argmax(1).cpu() == torch.from_numpy(labels)[ids.cpu()]).sum()) / ids.numel()
        assert m.evaluate_full(s) == want
        assert abs(m.evaluate_full(s) - m.evaluate(s)) < 0.15


# ---- world 2 and 3 ---------------------------------------------------------------------------------------------------

CASE_LAYERS, CASE_FANOUT = [37, 16, 5], [8, 12]


def dist_case(d):
    from neutronstarlite_b200.graph import HostGraph
    edges, V = synth9k()
    hg = HostGraph(edges, V)
    X = np.random.default_rng(21).uniform(-1, 1, (V, CASE_LAYERS[0])).astype(np.float32)
    return hg, whole_graph(edges, V, d), X


def _worker(rank, world, port, per_gpu, q):
    try:
        from test_dist_sample_gpu import _init, table_offsets
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
                # the topology's own ranges: the table's, shifted, so that ownership comes from the topology
                t_off = [0] + [min(V, o + 17) for o in off[1:-1]] + [V]
                graph = ShardedTopology(*shard_slices(pg, t_off[rank], t_off[rank + 1]), t_off)
            m = make_model(graph, CASE_LAYERS, table, V, dev_, CASE_FANOUT)
            lo, out = m.infer()
            acc = [m.evaluate_full(s) for s in (1, 2)]
            res[kind] = (lo, out.cpu().numpy(), acc, [p.W.detach().cpu().numpy() for p in m.P], m.step)
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
    d = dev()
    ranks = spawn(_worker, world, port, per_gpu)
    hg, pg, X = dist_case(d)
    csc = host_csc(pg)
    V = hg.vertices
    mask = (torch.arange(V) % 3).numpy()
    labels = torch.randint(0, CASE_LAYERS[-1], (V,), generator=torch.Generator().manual_seed(3)).numpy()
    Ws = [torch.from_numpy(w).double().numpy() for w in ranks[0]["replicated"][3]]
    ref = infer_oracle.infer(*csc, X.astype(np.float64), Ws, CASE_FANOUT)
    bound = infer_oracle.magnitude(*csc, X.astype(np.float64), Ws, CASE_FANOUT)
    top2 = np.sort(ref, 1)[:, -2:]
    sure = top2[:, 1] - top2[:, 0] >= 1e-4
    for kind in ("replicated", "topology"):
        rows = np.zeros(V, dtype=int)
        got = np.zeros_like(ref)
        empty = 0
        for r in ranks:
            lo, out, acc, W, step = r[kind]
            assert step == 0 and acc == ranks[0][kind][2]
            for a, b in zip(W, ranks[0][kind][3]):
                assert np.array_equal(a, b)
            got[lo:lo + out.shape[0]] = out
            rows[lo:lo + out.shape[0]] += 1
            empty += out.shape[0] == 0
        assert (rows == 1).all(), kind
        assert empty == (1 if world == 3 else 0)
        err = np.abs(got - ref)
        assert (err <= 1e-4 * bound + 1e-30).all(), (kind, float((err / (bound + 1e-30)).max()))
        assert (got.argmax(1) == ref.argmax(1))[sure].all()
        for s, acc in zip((1, 2), ranks[0][kind][2]):
            sel = mask == s
            hits = got.argmax(1) == labels
            assert acc == hits[sel].sum() / sel.sum()
            assert abs(acc * sel.sum() - (ref.argmax(1) == labels)[sel & sure].sum()) <= (sel & ~sure).sum()


@pytest.mark.parametrize("world", [2, 3])
def test_infer_on_ranks_sharing_one_gpu_matches_float64(world):
    run_dist(world, False, 29710 + world)


def test_infer_with_one_rank_per_gpu_matches_float64():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_dist(2, True, 29720)
