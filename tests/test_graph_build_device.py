"""Chunk construction on the GPU (nts_graph_build: PartitionedGraph.from_edge_file / from_device_edges) against the
golden artefacts of the reference and, bit for bit, against the host builder (nts_graph_host.cpp): degrees, partition
offsets, every chunk's CSC / CSR arrays and weights, source_active, MirrorIndex and the whole-partition CSC.  Then the
streaming reader (block sizes, permuted files), random multigraphs, the call shape bench.py uses, the errors, and end
to end runs of GCNImpl, GATImpl and the two-rank exchange on graphs built from a file."""
import multiprocessing as mp
import os
import sys

import numpy as np
import pytest

import golden_store
from neutronstarlite_b200 import _lib
from neutronstarlite_b200.graph import HostGraph, PartitionedGraph, partition_offsets_from_out_degree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def rows_as_multisets(offsets, idx):
    out = idx.copy()
    off = offsets.astype(np.int64)
    for r in range(off.shape[0] - 1):
        out[off[r]:off[r + 1]] = np.sort(out[off[r]:off[r + 1]])
    return out


def write_edges(path, edges):
    np.ascontiguousarray(edges, dtype=np.uint32).tofile(str(path))
    return str(path)


def u32(t):
    return t.cpu().numpy().view(np.uint32)


def arrays(pg):
    """Every array a device-built PartitionedGraph holds, as host numpy (u32 views; weights as their bits)."""
    out = {"partition_offset": np.asarray(pg.partition_offset), "owned": np.array([pg.owned_edges, pg.owned_mirrors]),
           "out_degree": u32(pg.out_degree_gpu), "in_degree": u32(pg.in_degree_gpu)}
    for i, c in enumerate(pg.graph_chunks):
        for name in ("column_offset", "row_indices", "edge_weight_forward", "row_offset", "column_indices",
                     "edge_weight_backward", "source_active"):
            t = getattr(c, name + "_gpu")
            out["c%d_%s" % (i, name)] = t.cpu().numpy() if name == "source_active" else u32(t)
    if pg.mirror_index_gpu is not None:
        out["mirror_index"] = u32(pg.mirror_index_gpu)
        out["whole_column_offset"] = u32(pg.column_offset_gpu)
        out["whole_row_indices"] = u32(pg.row_indices_gpu)
    return out


def assert_same_arrays(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def assert_equals_host(dpg, hg, P, r, po=None, dist=True):
    """The device-built rank r equals the host builder's rank r bit for bit."""
    hpg = PartitionedGraph(hg, P, r, po).generate_all(dist=dist)
    out_d, in_d = hg.degrees()
    assert np.array_equal(u32(dpg.out_degree_gpu), out_d) and np.array_equal(u32(dpg.in_degree_gpu), in_d)
    assert np.array_equal(dpg.partition_offset, hpg.partition_offset)
    assert dpg.owned_vertices == hpg.owned_vertices and dpg.owned_edges == hpg.owned_edges
    assert dpg.global_vertices == hg.vertices
    assert dpg.graph is None and dpg.MirrorIndex is None
    for c, h in zip(dpg.graph_chunks, hpg.graph_chunks):
        assert (c.edge_size, c.batch_size_forward, c.batch_size_backward) == \
            (h.edge_size, h.batch_size_forward, h.batch_size_backward)
        assert c.src_range == h.src_range and c.dst_range == h.dst_range
        assert c.column_offset is None and c.row_indices is None
        for name in ("column_offset", "row_indices", "row_offset", "column_indices", "edge_weight_forward",
                     "edge_weight_backward"):
            assert np.array_equal(u32(getattr(c, name + "_gpu")), getattr(h, name).view(np.uint32)), name
        assert np.array_equal(c.source_active_gpu.cpu().numpy(), h.source_active)
    if dist:
        assert dpg.owned_mirrors == hpg.owned_mirrors
        assert np.array_equal(u32(dpg.mirror_index_gpu), hpg.MirrorIndex)
        assert np.array_equal(u32(dpg.column_offset_gpu), hpg.column_offset)
        assert np.array_equal(u32(dpg.row_indices_gpu), hpg.row_indices)


# ---------------------------------------------------------------------------------------------------------------------
# 1. goldens
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_goldens_from_edge_file(golden, tmp_path):
    g = golden
    d = dev()
    path = write_edges(tmp_path / "g.edges", g.edges)
    hg = HostGraph(g.edges, g.V)
    for r in range(g.P):
        pg = PartitionedGraph.from_edge_file(path, g.V, g.P, r, device=d, dist=True)
        assert np.array_equal(u32(pg.out_degree_gpu), g.get(0, "out_degree"))
        assert np.array_equal(u32(pg.in_degree_gpu), g.get(0, "in_degree"))
        assert np.array_equal(pg.partition_offset, g.partition_offset)
        meta = g.get(r, "meta")
        assert (pg.owned_vertices, pg.owned_edges, pg.owned_mirrors) == (int(meta[4]), int(meta[5]), int(meta[6]))
        for i, c in enumerate(pg.graph_chunks):
            t = "chunk%d_" % i
            m = g.get(r, t + "meta")
            assert (m[0], m[1], m[2]) == (c.edge_size, c.batch_size_forward, c.batch_size_backward)
            assert (m[3], m[4]) == c.src_range and (m[5], m[6]) == c.dst_range
            assert np.array_equal(u32(c.column_offset_gpu), g.get(r, t + "column_offset"))
            assert np.array_equal(u32(c.row_indices_gpu), g.get(r, t + "row_indices"))
            assert np.array_equal(u32(c.edge_weight_forward_gpu), g.get(r, t + "edge_weight_forward").view(np.uint32))
            ro = u32(c.row_offset_gpu)
            assert np.array_equal(ro, g.get(r, t + "row_offset"))
            ci = u32(c.column_indices_gpu)
            ref_ci = g.get(r, t + "column_indices")
            assert np.array_equal(rows_as_multisets(ro, ci), rows_as_multisets(ro, ref_ci))
            ref_w = g.get(r, t + "edge_weight_backward").view(np.uint32).astype(np.uint64)
            mine_w = u32(c.edge_weight_backward_gpu).astype(np.uint64)
            assert np.array_equal(rows_as_multisets(ro, (ci.astype(np.uint64) << np.uint64(32)) | mine_w),
                                  rows_as_multisets(ro, (ref_ci.astype(np.uint64) << np.uint64(32)) | ref_w))
            assert np.array_equal(c.source_active_gpu.cpu().numpy(), g.get(r, t + "source_active"))
        assert np.array_equal(u32(pg.mirror_index_gpu), g.get(r, "mirror_index"))
        assert np.array_equal(u32(pg.column_offset_gpu), g.get(r, "whole_column_offset"))
        assert np.array_equal(u32(pg.row_indices_gpu), g.get(r, "whole_row_indices"))
        assert_equals_host(pg, hg, g.P, r)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the streaming reader: block sizes and record order do not show in the outputs
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_block_sizes_and_permuted_file_give_identical_arrays(tmp_path):
    d = dev()
    z = golden_store.load("cora_self_P2_F4")
    edges, V = z["edges"], int(z["case"][0])
    E = edges.shape[0]
    path = write_edges(tmp_path / "cora.edges", edges)
    ref = [arrays(PartitionedGraph.from_edge_file(path, V, 2, r, device=d, dist=True)) for r in range(2)]
    for block in (1, 7, 4096, E - 1, E, 2 * E):
        for r in range(2):
            assert_same_arrays(arrays(PartitionedGraph.from_edge_file(path, V, 2, r, device=d, dist=True,
                                                                      block_edges=block)), ref[r])
    perm = np.random.default_rng(3).permutation(E)
    ppath = write_edges(tmp_path / "cora_perm.edges", edges[perm])
    for r in range(2):
        assert_same_arrays(arrays(PartitionedGraph.from_edge_file(ppath, V, 2, r, device=d, dist=True,
                                                                  block_edges=1000)), ref[r])


# ---------------------------------------------------------------------------------------------------------------------
# 3. random multigraphs against the host builder, every rank
# ---------------------------------------------------------------------------------------------------------------------
def zipf_multigraph(V, E, seed, isolated=500):
    """Zipf destinations, uniform and hub sources, duplicate edges, self loops; the top `isolated` ids never occur."""
    rng = np.random.default_rng(seed)
    W = V - isolated
    src = rng.integers(0, W, E)
    dst = rng.zipf(1.4, E) % W
    src[: E // 20] = rng.integers(0, W)                  # a hub source
    src[E // 20: E // 10] = dst[E // 20: E // 10]        # self loops
    e = np.stack([src, dst], 1)
    e[E - E // 10:] = e[: E // 10]                       # exact duplicates
    return e.astype(np.uint32)


@gpu
@pytest.mark.parametrize("V,E,P", [(200_003, 2_000_000, 1), (200_003, 2_000_000, 3), (200_003, 2_000_000, 8),
                                   (3000, 40_000, 8)])
def test_random_multigraph_equals_host_builder(tmp_path, V, E, P):
    d = dev()
    edges = zipf_multigraph(V, E, seed=V + P)
    path = write_edges(tmp_path / "z.edges", edges)
    hg = HostGraph(edges, V)
    po = hg.partition_offsets(P)
    if V == 3000:
        assert (np.diff(po.astype(np.int64)) == 0).any()   # page rounding leaves a partition empty
    for r in range(P):
        pg = PartitionedGraph.from_edge_file(path, V, P, r, device=d, dist=True, block_edges=1 << 19)
        assert_equals_host(pg, hg, P, r)


# ---------------------------------------------------------------------------------------------------------------------
# 4. from_device_edges in the call shape of bench.py
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_from_device_edges_owned_edges_int64_degrees():
    import torch
    d = dev()
    V, E, P = 100_003, 600_000, 4
    edges = zipf_multigraph(V, E, seed=11)
    hg = HostGraph(edges, V)
    src = torch.from_numpy(edges[:, 0].astype(np.int64)).to(d)
    dst = torch.from_numpy(edges[:, 1].astype(np.int64)).to(d)
    out_raw = torch.bincount(src, minlength=V)
    in_raw = torch.bincount(dst, minlength=V)
    po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E, P)
    for r in range(P):
        keep = (dst >= int(po[r])) & (dst < int(po[r + 1]))
        pg = PartitionedGraph.from_device_edges(src[keep], dst[keep], V, P, r, po, out_raw.clamp(min=1),
                                                in_raw.clamp(min=1), dist=(r % 2 == 1))
        assert_equals_host(pg, hg, P, r, po, dist=(r % 2 == 1))
    # int32 edges, degrees computed from the edges, P = 1
    pg = PartitionedGraph.from_device_edges(src.to(torch.int32), dst.to(torch.int32), V, dist=True)
    assert_equals_host(pg, hg, 1, 0)


# ---------------------------------------------------------------------------------------------------------------------
# 5. errors
# ---------------------------------------------------------------------------------------------------------------------
def _abi_error(fn, *args):
    L = _lib.load()
    h = getattr(L, fn)(*args)
    assert not h
    return L.nts_last_error().decode()


def test_argument_errors_are_caught_before_any_cuda_call(tmp_path):
    """No GPU needed: every rejection below happens before the builder touches CUDA."""
    good = write_edges(tmp_path / "ok.edges", np.array([[0, 1], [1, 2]]))
    odd = tmp_path / "odd.edges"
    odd.write_bytes(b"\0" * 12)
    f = "nts_graph_build_from_file"
    assert "cannot open" in _abi_error(f, str(tmp_path / "missing.edges").encode(), 4, 1, 0, None, 1 << 26, 0, None)
    assert "multiple of 8" in _abi_error(f, str(odd).encode(), 4, 1, 0, None, 1 << 26, 0, None)
    assert "rank" in _abi_error(f, good.encode(), 4, 2, 2, None, 1 << 26, 0, None)
    assert "partitions" in _abi_error(f, good.encode(), 4, 0, 0, None, 1 << 26, 0, None)
    assert "2^31" in _abi_error(f, good.encode(), 1 << 31, 1, 0, None, 1 << 26, 0, None)
    assert "block_edges" in _abi_error(f, good.encode(), 4, 1, 0, None, 0, 0, None)
    bad_po = np.array([0, 3, 2], dtype=np.uint32)
    assert "decreases" in _abi_error(f, good.encode(), 2, 2, 0, bad_po.ctypes.data, 1 << 26, 0, None)
    g = "nts_graph_build_from_device"
    assert "index_dtype" in _abi_error(g, None, None, 5, 0, 4, 1, 0, None, None, None, 0, None)
    assert "both degree" in _abi_error(g, None, None, 0, 0, 4, 1, 0, None, 16, None, 0, None)
    assert "partition_offset is required" in _abi_error(g, None, None, 0, 0, 4, 2, 0, None, 16, 16, 0, None)
    assert _lib.load().nts_graph_build_destroy(None) == 0


@gpu
def test_errors_raise_with_a_message_naming_the_problem(tmp_path):
    d = dev()
    good = write_edges(tmp_path / "ok.edges", np.array([[0, 1], [1, 2]]))
    with pytest.raises(_lib.NtsError, match="cannot open"):
        PartitionedGraph.from_edge_file(tmp_path / "missing.edges", 4, device=d)
    odd = tmp_path / "odd.edges"
    odd.write_bytes(b"\0" * 20)
    with pytest.raises(_lib.NtsError, match="multiple of 8"):
        PartitionedGraph.from_edge_file(odd, 4, device=d)
    e = np.stack([np.arange(100) % 50, np.arange(100) % 49], 1)
    e[73] = (3, 50)                                         # id >= V in the 10th block of 8 records
    bad = write_edges(tmp_path / "bad.edges", e)
    with pytest.raises(_lib.NtsError, match="vertex id >= V"):
        PartitionedGraph.from_edge_file(bad, 50, device=d, block_edges=8)
    with pytest.raises(_lib.NtsError, match="rank"):
        PartitionedGraph.from_edge_file(good, 4, 2, 2, device=d)
    with pytest.raises(_lib.NtsError, match="partitions"):
        PartitionedGraph.from_edge_file(good, 4, 0, 0, device=d)
    with pytest.raises(_lib.NtsError, match="2\\^31"):
        PartitionedGraph.from_edge_file(good, 1 << 31, device=d)
    import torch
    s = torch.tensor([0, 7], device=d)
    with pytest.raises(_lib.NtsError, match="vertex id >= V"):
        PartitionedGraph.from_device_edges(s, s.flip(0), 5)
    # the builder leaves nothing behind after a failure: the next build works
    assert PartitionedGraph.from_edge_file(good, 4, device=d).owned_edges == 2


@gpu
def test_empty_file_builds_empty_chunks_with_unit_degrees(tmp_path):
    d = dev()
    path = tmp_path / "empty.edges"
    path.write_bytes(b"")
    for P, r in ((1, 0), (3, 2)):
        pg = PartitionedGraph.from_edge_file(path, 2500, P, r, device=d, dist=True)
        assert pg.owned_edges == 0 and pg.owned_mirrors == 0
        assert (u32(pg.out_degree_gpu) == 1).all() and (u32(pg.in_degree_gpu) == 1).all()
        assert_equals_host(pg, HostGraph(np.zeros((0, 2), dtype=np.uint32), 2500), P, r)


# ---------------------------------------------------------------------------------------------------------------------
# 6. end to end on graphs built from a file
# ---------------------------------------------------------------------------------------------------------------------
def _cora(tmp_path):
    z = golden_store.load("cora_self_P1_F8")
    V = int(z["case"][0])
    return z["edges"], V, write_edges(tmp_path / "cora.edges", z["edges"])


@gpu
def test_gcn_epochs_on_a_graph_built_from_the_file(tmp_path):
    import torch
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    edges, V, path = _cora(tmp_path)
    layers = [64, 16, 7]
    gen = torch.Generator().manual_seed(5)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    losses = []
    for pg in (PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=d, dist=True),
               PartitionedGraph.from_edge_file(path, V, device=d, dist=True)):
        model = GCNImpl(pg, layers, feats.clone(), labels, mask, drop_rate=0.0)
        losses.append([model.run_epoch()[0].item() for _ in range(3)])
    np.testing.assert_allclose(losses[1], losses[0], rtol=1e-6, atol=0)


@gpu
def test_fused_gat_epoch_on_a_graph_built_from_the_file(tmp_path):
    import torch
    from neutronstarlite_b200.toolkits import GATImpl
    d = dev()
    edges, V, path = _cora(tmp_path)
    layers = [32, 16, 7]
    gen = torch.Generator().manual_seed(6)
    feats = (torch.rand((V, layers[0]), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    losses = []
    for pg in (PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=d, dist=True),
               PartitionedGraph.from_edge_file(path, V, device=d, dist=True)):
        model = GATImpl(pg, layers, feats.clone(), labels, mask, heads=4, fused_kernel=True, two_pass_backward=True)
        losses.append(model.run_epoch().item())
    np.testing.assert_allclose(losses[1], losses[0], rtol=1e-6, atol=0)


def _shared_worker(rank, world, port, case, path, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["NTS_EXCHANGE_TIMEOUT_MS"] = "120000"   # ranks time-slice one GPU: waits are long but bounded
    torch.cuda.set_device(0)
    d = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from neutronstarlite_b200 import ops
        from neutronstarlite_b200.exchange import GpuExchange
        z = golden_store.load(case)
        V, E, P, F = (int(x) for x in z["case"])
        pg = PartitionedGraph.from_edge_file(path, V, P, rank, device=d, dist=True)
        ex = GpuExchange(pg, transport="p2p")
        op = ops.ForwardGPUfuseOp(pg, None, exchange=ex)
        x = torch.from_numpy(z["r%d/X" % rank].reshape(-1, F)).to(d)
        g = torch.from_numpy(z["r%d/G" % rank].reshape(-1, F)).to(d)
        for _ in range(2):
            y = op.forward(x)
            dx = op.backward(g)
            torch.cuda.synchronize()
            np.testing.assert_allclose(y.cpu().numpy(), z["r%d/gcn_Y" % rank].reshape(-1, F), rtol=1e-4, atol=1e-5)
            np.testing.assert_allclose(dx.cpu().numpy(), z["r%d/gcn_dX" % rank].reshape(-1, F), rtol=1e-4, atol=2e-5)
        dist.barrier()
        ex.close()
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@gpu
def test_two_ranks_sharing_one_gpu_give_the_golden_forward(tmp_path):
    dev()
    case = "synth9k_P2_F2"
    path = write_edges(tmp_path / "synth.edges", golden_store.load(case)["edges"])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shared_worker, args=(r, 2, 29400 + os.getpid() % 100, case, path, q))
             for r in range(2)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(2):
            results.append(q.get(timeout=420))
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, msg in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)
