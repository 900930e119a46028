"""A sharded topology on the GPU (topology.ShardedTopology, nts_merge_chunk_csc, nts_sampler_create_sharded):

  * nts_merge_chunk_csc is bit-exact against the numpy merge (test_topology_merge_cpu.merge_chunks) on host-built and
    device-built partitions, with empty partitions and destinations without in-edges, and refuses a wrong edge count
    and a chunk with edges but no arrays;
  * the constructor from tensors gives the whole-graph blocks, and refuses malformed shards (offsets that are global,
    fall, or disagree with the edge count; source ids >= V) before any copy, as does ShardedTopology.split;
  * the sharded sampler over 1, 3, 8 and 32 shards of one process (ShardedTopology.split, some empty) gives the blocks of NeighborSampler(pg)
    and of the numpy sampler bit for bit, in both modes, on Cora and the 9k hub graph, with fanouts 1 and 64; the
    bad-seed error and the argument refusals behave as in the whole-graph sampler;
  * the topology over CUDA IPC with 2 and 3 processes sharing one GPU (gloo; an empty shard at world 3), merged from
    the rank's partition and built from tensors: every rank's blocks equal the whole-graph sampler's, and every
    process ends by itself;
  * world 1: a one-shard topology gives the losses, accuracies and weights of the PartitionedGraph on Cora (GCN, GAT);
  * one data-parallel round at world 2 and 3 with topology and table: the blocks equal the replicated-topology run's,
    and the weights meet the float64 restatement of test_dist_sample_gpu.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import golden_store
import sample_oracle as so
from test_sample_gpu import KEYS, cora_edges
from test_sample_include_dst import sample_include_dst
from test_topology_merge_cpu import merge_chunks

torch = pytest.importorskip("torch")
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYNTH = "synth9k_P1_F2"     # the 9k-vertex graph with hubs


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def graph_edges(name):
    if name == "cora":
        return cora_edges(), 2708
    z = golden_store.load(SYNTH)
    return z["edges"], int(z["case"][0])


def whole_graph(edges, V, d):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    return PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=d)


def shard_offsets(V, n, rng):
    """n + 1 offsets over [0, V) with some empty shards: random cuts, a repeated cut, and the last shard empty."""
    cuts = np.sort(rng.integers(0, V, max(n - 2, 0)))
    off = np.concatenate([[0], cuts, [V]] + ([[V]] if n > 1 else []))[:n + 1]
    if n > 3:
        off[2] = off[1]
    return np.maximum.accumulate(off).astype(np.int64)


def local_topology(pg, off):
    """Every shard of pg's single-partition CSC at `off` in this process (ShardedTopology.split)."""
    from neutronstarlite_b200.topology import ShardedTopology
    c = pg.graph_chunks[0]
    return ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, off)


def shard_slices(pg, lo, hi):
    """(column_offset, row_indices, weight) of destinations [lo, hi) cut from pg's single-partition CSC, with local
    column offsets: what a rank passes to the ShardedTopology constructor."""
    c = pg.graph_chunks[0]
    col = c.column_offset_gpu.long()
    e0, e1 = int(col[lo]), int(col[hi])
    return ((col[lo:hi + 1] - e0).to(torch.int32), c.row_indices_gpu[e0:e1].clone(),
            c.edge_weight_forward_gpu[e0:e1].clone())


def assert_same_blocks(a, b, include_dst, what=""):
    assert a.hops == b.hops
    keys = KEYS + (("dst_pos",) if include_dst else ())
    for h, (x, y) in enumerate(zip(a.blocks, b.blocks)):
        gx, gy = x.to_numpy(), y.to_numpy()
        for k in keys:
            assert np.array_equal(gx[k].view(np.uint32), gy[k].view(np.uint32)), "%s hop %d %s differs" % (what, h, k)


def assert_oracle(sg, pg, seeds, fanout, seed, step, include_dst):
    c = pg.graph_chunks[0]
    fn = sample_include_dst if include_dst else so.sample
    ref = fn(c.column_offset, c.row_indices, c.edge_weight_forward, seeds, fanout, seed, step)
    keys = KEYS + (("dst_pos",) if include_dst else ())
    for h, (b, r) in enumerate(zip(sg.blocks, ref)):
        got = b.to_numpy()
        for k in keys:
            assert np.array_equal(got[k].view(np.uint32), r[k].view(np.uint32)), "hop %d %s differs" % (h, k)


# ---- nts_merge_chunk_csc --------------------------------------------------------------------------------------

def merge_on_gpu(pg):
    from neutronstarlite_b200 import _lib
    chunks = pg.graph_chunks
    P, n_dst, E = len(chunks), int(pg.owned_vertices), sum(int(c.edge_size) for c in chunks)
    d = chunks[0].column_offset_gpu.device
    col = torch.full((n_dst + 1,), -1, dtype=torch.int32, device=d)
    row = torch.full((E,), -1, dtype=torch.int32, device=d)
    w = torch.full((E,), float("nan"), dtype=torch.float32, device=d)

    def ptrs(name):
        return (C.c_void_p * P)(*[getattr(c, name).data_ptr() if getattr(c, name).numel() else None for c in chunks])

    _lib.call("nts_merge_chunk_csc", ptrs("column_offset_gpu"), ptrs("row_indices_gpu"),
              ptrs("edge_weight_forward_gpu"), P, n_dst, E, col.data_ptr(), row.data_ptr() if E else None,
              w.data_ptr() if E else None, torch.cuda.current_stream().cuda_stream)
    return col.cpu().numpy().view(np.uint32), row.cpu().numpy().view(np.uint32), w.cpu().numpy()


@pytest.mark.parametrize("name,P", [("cora", 4), ("cora", 3), ("synth", 3), ("synth", 8)])
def test_merge_matches_numpy_on_host_and_device_built_partitions(name, P):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    d = dev()
    edges, V = graph_edges(name)
    keep = np.ones(len(edges), bool)
    keep[edges[:, 1] % 97 == 3] = False        # destinations without in-edges
    edges = edges[keep]
    hg = HostGraph(edges, V)
    po = hg.partition_offsets(P)
    src = torch.from_numpy(edges[:, 0].astype(np.int64)).to(d)
    dst = torch.from_numpy(edges[:, 1].astype(np.int64)).to(d)
    empty = 0
    for p in range(P):
        host = PartitionedGraph(hg, P, p).generate_all(device=d)
        ref = merge_chunks([c.column_offset for c in host.graph_chunks], [c.row_indices for c in host.graph_chunks],
                           [c.edge_weight_forward for c in host.graph_chunks])
        devb = PartitionedGraph.from_device_edges(src, dst, V, P, p, partition_offset=po)
        for pg in (host, devb):
            col, row, w = merge_on_gpu(pg)
            assert np.array_equal(col, ref[0]) and np.array_equal(row, ref[1])
            assert np.array_equal(w.view(np.uint32), ref[2].view(np.uint32))
        empty += int(po[p + 1] == po[p])
        assert (np.diff(ref[0].astype(np.int64)) == 0).any() or ref[0].size == 1
    if name == "cora" and P == 4:
        assert empty >= 1


def test_merge_refuses_a_wrong_edge_count_and_missing_chunk_arrays():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    d = dev()
    edges, V = graph_edges("synth")
    pg = PartitionedGraph(HostGraph(edges, V), 2, 1).generate_all(device=d)
    chunks, n_dst = pg.graph_chunks, int(pg.owned_vertices)
    E = sum(int(c.edge_size) for c in chunks)
    L = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    col = torch.empty(n_dst + 1, dtype=torch.int32, device=d)
    row = torch.empty(E + 64, dtype=torch.int32, device=d)
    w = torch.empty(E + 64, dtype=torch.float32, device=d)

    def ptrs(name, drop=None):
        return (C.c_void_p * 2)(*[None if i == drop else getattr(c, name).data_ptr() for i, c in enumerate(chunks)])

    def merge(n_edges, drop=None):
        return L.nts_merge_chunk_csc(ptrs("column_offset_gpu"), ptrs("row_indices_gpu", drop),
                                     ptrs("edge_weight_forward_gpu"), 2, n_dst, n_edges, col.data_ptr(),
                                     row.data_ptr(), w.data_ptr(), st)

    for n_edges in (E - 1, E + 1, 0):
        assert merge(n_edges) != 0
        assert b"n_edges" in L.nts_last_error()
    assert merge(E, drop=1) != 0
    assert b"null row" in L.nts_last_error()
    assert merge(E) == 0


# ---- the sharded sampler in one process ------------------------------------------------------------------------

CASES = [("cora", [1, 1], 0, 0), ("cora", [64, 64], 1, 3), ("cora", [5, 10, 3], 2, 7),
         ("synth", [1, 1], 3, 1), ("synth", [64, 64], 4, 12), ("synth", [25, 10], 5, 2)]


@pytest.mark.parametrize("include_dst", [False, True])
@pytest.mark.parametrize("name,fanout,seed,step", CASES)
def test_sharded_sampler_equals_the_whole_graph_sampler(name, fanout, seed, step, include_dst):
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    edges, V = graph_edges(name)
    pg = whole_graph(edges, V, d)
    deg = np.diff(pg.graph_chunks[0].column_offset.astype(np.int64))
    rng = np.random.default_rng(seed)
    hubs = np.nonzero(deg > max(fanout))[0][:8]
    seeds = np.unique(np.concatenate([rng.choice(V, 120, replace=False), hubs])).astype(np.int64)
    whole = NeighborSampler(pg, fanout, len(seeds), include_dst=include_dst)
    ref = whole.sample(seeds, seed, step).clone()
    assert_oracle(ref, pg, seeds, fanout, seed, step, include_dst)
    for n in (1, 3, 8, 32):
        topo = local_topology(pg, shard_offsets(V, n, rng))
        s = NeighborSampler(topo, fanout, len(seeds), include_dst=include_dst)
        assert s._graph is topo and s.V == V
        assert_same_blocks(s.sample(seeds, seed, step), ref, include_dst, "%d shards" % n)


def test_sharded_sampler_bad_seed_and_argument_refusals():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    topo = local_topology(pg, np.array([0, 1000, 1000, 2708]))
    s = NeighborSampler(topo, [5, 10], 64)
    L = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    # a device seed >= V reaches the kernels: the bad-seed flag reports it after hop 0, as in the whole-graph sampler
    bad = torch.tensor([3, 2708], dtype=torch.int32, device=d)
    assert L.nts_sampler_sample(s.handle, bad.data_ptr(), 2, 0, 0, st) != 0
    assert b"seed vertex id" in L.nts_last_error()
    with pytest.raises(_lib.NtsError):
        s.sample(np.array([3, 2708]), 0, 0)
    with pytest.raises(_lib.NtsError):
        s.sample(np.arange(65), 0, 0)
    for fan in ([0, 10], [5, 65]):
        with pytest.raises(_lib.NtsError):
            NeighborSampler(topo, fan, 64)
    ks = (C.c_int * 2)(5, 10)
    cols, rows, ws = ((C.c_void_p * 3)(*a) for a in topo.shard_arrays)

    def create(n=3, offs=(0, 1000, 1000, 2708), flags=0, c=cols):
        o = (C.c_uint32 * len(offs))(*offs)
        return L.nts_sampler_create_sharded(c, rows, ws, o, n, 64, 2, ks, flags, st)

    h = create()
    assert h
    L.nts_sampler_destroy(h)
    for kw, msg in ((dict(n=0), b"1..32"), (dict(n=33), b"1..32"), (dict(offs=(0, 1000, 900, 2708)), b"non-decreasing"),
                    (dict(offs=(1, 1000, 1000, 2708)), b"start at 0"), (dict(flags=2), b"flag"),
                    (dict(c=(C.c_void_p * 3)(cols[0], cols[1], None)), b"null")):
        assert not create(**kw), kw
        assert msg in L.nts_last_error(), (kw, L.nts_last_error())
    # an empty shard may have null arrays
    h = create(c=(C.c_void_p * 3)(cols[0], None, cols[2]))
    assert h
    L.nts_sampler_destroy(h)


@pytest.mark.parametrize("name", ["cora", "synth"])
def test_constructor_from_tensors_equals_the_whole_graph_sampler(name):
    from neutronstarlite_b200.sample import NeighborSampler
    from neutronstarlite_b200.topology import ShardedTopology
    d = dev()
    edges, V = graph_edges(name)
    pg = whole_graph(edges, V, d)
    topo = ShardedTopology(*shard_slices(pg, 0, V), [0, V])
    assert topo.world == 1 and topo.local_edges == pg.graph_chunks[0].edge_size
    seeds = np.random.default_rng(3).choice(V, 300, replace=False)
    for include_dst in (False, True):
        for fanout in ([1, 64], [25, 10, 3]):
            a = NeighborSampler(topo, fanout, 300, include_dst=include_dst).sample(seeds, 4, 9)
            b = NeighborSampler(pg, fanout, 300, include_dst=include_dst).sample(seeds, 4, 9)
            assert_same_blocks(a, b, include_dst)
    topo.close()


def test_malformed_shards_are_refused_before_any_copy():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.topology import ShardedTopology
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    c = pg.graph_chunks[0]
    col, row, w = shard_slices(pg, 0, 2708)
    lo, hi = 1000, 2000
    g_col = c.column_offset_gpu[lo:hi + 1]          # a slice with global offsets: the mistake to catch
    falling = col.clone()
    falling[5] = falling[7] + 1
    wide = row.clone()
    wide[3] = 2708
    bad = [((col + 5, row, w), "start at 0"),                     # offsets not starting at 0
           ((col, row[:-1], w[:-1]), "edge count"),               # one edge fewer than column_offset says
           ((falling, row, w), "decrease"),
           ((col, wide, w), "source id"),                         # a source id >= V
           ((col, row, w[:-1]), "same edge count"),
           ((col.long(), row, w), "int32")]
    for args, msg in bad:
        with pytest.raises(_lib.NtsError, match=msg):
            ShardedTopology(*args, [0, 2708])
        with pytest.raises(_lib.NtsError, match=msg):
            ShardedTopology.split(*args, [0, 1000, 2708])
    with pytest.raises(_lib.NtsError):
        ShardedTopology(col, row, w, [0, 2000])                  # V_r differs from the offsets
    with pytest.raises(_lib.NtsError, match="start at 0"):
        ShardedTopology(g_col.contiguous(), c.row_indices_gpu[int(c.column_offset[lo]):int(c.column_offset[hi])].clone(),
                        c.edge_weight_forward_gpu[int(c.column_offset[lo]):int(c.column_offset[hi])].clone(),
                        [0, hi - lo])
    with pytest.raises(_lib.NtsError):
        ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, [0, 1000])
    with pytest.raises(_lib.NtsError):
        ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, [0] * 34 + [2708])


# ---- processes sharing one GPU over CUDA IPC (the spawn pattern of test_dist_sample_gpu.py) ----------------------

def spawn(target, world, port, extra, timeout=420):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world, port, extra, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(world):
            results.append(q.get(timeout=timeout))
    finally:
        ended = []
        for p in procs:
            p.join(timeout=30)
            ended.append(not p.is_alive())
            if p.is_alive():
                p.kill()
    for rank, msg, _ in sorted(results, key=lambda r: r[0]):
        assert msg == "ok", "rank %d: %s" % (rank, msg)
    assert all(ended), "a rank did not end by itself"
    return [r[2] for r in sorted(results, key=lambda r: r[0])]


def _init(rank, world, port, per_gpu):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if per_gpu else 0)
    torch.cuda.set_device(dev)
    if per_gpu:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    return dev


def rank_partition(hg, world, rank, d):
    """Rank `rank`'s PartitionedGraph at the reference's offsets; at world 3 the middle partition is made empty."""
    from neutronstarlite_b200.graph import PartitionedGraph
    from test_dist_sample_gpu import table_offsets
    off = np.asarray(table_offsets(hg, world), dtype=np.uint32)
    return PartitionedGraph(hg, world, rank, off).generate_all(device=d), off


def _ipc_worker(rank, world, port, extra, q):
    try:
        d = _init(rank, world, port, False)
        from neutronstarlite_b200.graph import HostGraph
        from neutronstarlite_b200.sample import NeighborSampler
        from neutronstarlite_b200.topology import ShardedTopology
        edges, V = graph_edges("synth")
        hg = HostGraph(edges, V)
        pg, off = rank_partition(hg, world, rank, d)
        merged = ShardedTopology.from_partitioned_graph(pg)
        del pg
        assert merged.world == world and merged.rank == rank and merged.vertices == V
        assert list(merged.offsets) == [int(o) for o in off]
        whole = whole_graph(edges, V, d)
        # the same shard from tensors cut out of the whole-graph CSC
        sliced = ShardedTopology(*shard_slices(whole, int(off[rank]), int(off[rank + 1])), off)
        assert sliced.local_bytes == merged.local_bytes
        seeds = np.random.default_rng(rank).choice(V, 200, replace=False)
        remote = 0
        for topo in (merged, sliced):
            for include_dst in (False, True):
                for fanout, seed, step in (([1, 64], 1, 2), ([25, 10], 7, 5)):
                    a = NeighborSampler(topo, fanout, 200, include_dst=include_dst).sample(seeds, seed, step)
                    b = NeighborSampler(whole, fanout, 200, include_dst=include_dst).sample(seeds, seed, step)
                    assert_same_blocks(a, b, include_dst)
                    dst = a.blocks[-1].dst.cpu().numpy().view(np.uint32)
                    remote += int(((dst < off[rank]) | (dst >= off[rank + 1])).sum())
        assert remote > 0
        sliced.close()
        merged.close()
        q.put((rank, "ok", remote))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_topology_over_ipc_with_ranks_sharing_one_gpu(world):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    spawn(_ipc_worker, world, 29650 + world, None)


# ---- toolkits ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gcn", "gat"])
def test_world_1_topology_equals_the_partitioned_graph_on_cora(kind):
    from test_gather_plan_bf16 import cora_tables
    from neutronstarlite_b200.topology import ShardedTopology
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    d = dev()
    pg = whole_graph(cora_edges(), 2708, d)
    topo = ShardedTopology.from_partitioned_graph(pg)
    assert topo.world == 1 and topo.local_edges == pg.graph_chunks[0].edge_size
    feats, labels, masks = cora_tables()
    x = torch.from_numpy(feats).to(d)
    runs = []
    for g in (pg, topo):
        if kind == "gcn":
            m = GCNSampleImpl(g, [1433, 128, 7], x, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                              fanout=[5, 10], batch_size=64, drop_rate=0.0, seed=0, sample_seed=0)
        else:
            m = GATSampleImpl(g, [1433, 64, 7], x, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                              fanout=[5, 10], batch_size=64, heads=8, seed=0, sample_seed=0)
        res = [m.run_epoch(test=True) for _ in range(2)]
        runs.append((res, m.step, [p.W.detach().clone() for p in m.params()]))
    (res_a, step_a, w_a), (res_b, step_b, w_b) = runs
    assert res_a == res_b and step_a == step_b
    for a, b in zip(w_a, w_b):
        assert torch.equal(a, b)
    topo.close()


def record_blocks(model):
    """Host copies of every sample the model's sampler takes, appended to the returned list."""
    seen, sample = [], model.sampler.sample

    def recorded(*args):
        sg = sample(*args)
        seen.append([b.to_numpy() for b in sg.blocks])
        return sg

    model.sampler.sample = recorded
    return seen


def _round_worker(rank, world, port, per_gpu, q):
    try:
        d = _init(rank, world, port, per_gpu)
        import test_dist_sample_gpu as ds
        from neutronstarlite_b200 import _lib
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        from neutronstarlite_b200.topology import ShardedTopology
        hg, pg1, feats, labels = ds.graph_and_data(d)
        pg, _ = rank_partition(hg, world, rank, d)
        topo = ShardedTopology.from_partitioned_graph(pg)
        del pg
        off = [int(o) for o in hg.partition_offsets(world)]      # the table's offsets differ at world 3
        table = ShardedFeatureTable(feats[off[rank]:off[rank + 1]].to(d), off)
        try:
            ds.make_model("gcn", topo, feats.to(d), labels, ds.round_mask(hg.vertices, 10), d)
            raise AssertionError("a tensor was accepted with a sharded topology")
        except _lib.NtsError:
            pass
        out = {}
        for kind in ds.MODELS:
            for n_batches in (world, world - 1):
                n_train = n_batches * ds.BATCH - (7 if n_batches == world else 0)
                mask = ds.round_mask(hg.vertices, n_train)
                runs = []
                for g in (topo, pg1):
                    m = ds.make_model(kind, g, table, labels, mask, d)
                    runs.append(record_blocks(m))
                    loss, acc = m.run_epoch(test=True)
                    if g is topo:
                        res = (loss, acc, m.step, [p.W.detach().cpu().numpy() for p in m.params()],
                               [p.W_gradient.cpu().numpy() for p in m.params()])
                assert len(runs[0]) == len(runs[1]) > 0
                for x, y in zip(*runs):
                    for bx, by in zip(x, y):
                        for k in bx:
                            assert np.array_equal(bx[k].view(np.uint32), by[k].view(np.uint32)), (kind, k)
                out[(kind, n_batches)] = res
        table.close()
        topo.close()
        q.put((rank, "ok", out))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def run_round_test(world, per_gpu, port):
    import test_dist_sample_gpu as ds
    ranks = spawn(_round_worker, world, port, per_gpu)
    d = torch.device("cuda:0")
    for kind in ds.MODELS:
        for n_batches in (world, world - 1):
            ds.check_round(kind, n_batches, ranks, d)


@pytest.mark.parametrize("world", [2, 3])
def test_one_round_with_a_sharded_topology_on_ranks_sharing_one_gpu(world):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    run_round_test(world, False, 29660 + world)


def test_one_round_with_a_sharded_topology_one_rank_per_gpu():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_round_test(2, True, 29670)
