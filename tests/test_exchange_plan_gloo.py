"""Host-side logic of the multi-GPU exchange on CPU: world_size 2 and 4 over gloo.

Every rank builds its chunks with the product's host builder, builds the `ExchangePlan` (need lists, slot-remapped
CSC, compacted CSR, and the all-to-all of row lists), then the test walks the plan's data path in numpy - exactly
the gathers / scatters the CUDA kernels perform - and checks the assembled Y / dX against the golden vectors of
the reference run at the same P.  The CUDA data path itself is covered by tests/test_multi_gpu.py (-m gpu)."""
import os
import sys

import golden_store
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gather_sum(offsets, idx, w, X, n_rows):
    out = np.zeros((n_rows, X.shape[1]), dtype=np.float64)
    off = offsets.astype(np.int64)
    rows = np.repeat(np.arange(n_rows), np.diff(off))
    np.add.at(out, rows, X[idx.astype(np.int64)].astype(np.float64) * w[:, None].astype(np.float64))
    return out


def _a2a(parts_out, counts_in, F):
    """list all-to-all over all_to_all_single (gloo has no list variant)."""
    send = torch.cat([t.reshape(-1, F).to(torch.float32) for t in parts_out]) if parts_out else torch.zeros(0, F)
    recv = torch.zeros((int(sum(counts_in)), F), dtype=torch.float32)
    dist.all_to_all_single(recv, send, output_split_sizes=list(counts_in),
                           input_split_sizes=[int(t.shape[0]) for t in parts_out])
    out, pos = [], 0
    for n in counts_in:
        out.append(recv[pos:pos + n])
        pos += n
    return out


def _check_cxx_plan(pg, plan, rank, P):
    """The C++ plan builder (nts_exchange_plan_*, what the reference's C++ host uses) must produce exactly the arrays
    of the Python ExchangePlan: the wire form of the need lists travels over gloo here, over MPI_Bcast there."""
    import ctypes as C
    from neutronstarlite_b200 import _lib
    L = _lib.load()
    arr = (_lib.HostChunk * P)()
    for i, c in enumerate(pg.graph_chunks):
        h = arr[i]
        for name in ("column_offset", "row_indices", "row_offset", "column_indices", "edge_weight_forward",
                     "edge_weight_backward"):
            setattr(h, name, getattr(c, name).ctypes.data_as(C.c_void_p))
        h.src_start, h.src_end = int(c.src_range[0]), int(c.src_range[1])
        h.dst_start, h.dst_end = int(c.dst_range[0]), int(c.dst_range[1])
        h.edges = int(c.edge_size)
    cp = L.nts_exchange_plan_create(arr, P, rank)
    assert cp, L.nts_last_error()
    try:
        n = int(L.nts_exchange_plan_packed_rows(cp))
        counts = np.zeros(P, dtype=np.uint32)
        rows = np.zeros(max(n, 1), dtype=np.uint32)
        assert L.nts_exchange_plan_pack_needs(cp, counts.ctypes.data_as(C.c_void_p), rows.ctypes.data_as(C.c_void_p)) == 0
        packs = [None] * P
        dist.all_gather_object(packs, (counts, rows[:n]))
        for j, (cj, rj) in enumerate(packs):
            rj = np.ascontiguousarray(np.concatenate([rj, np.zeros(1, dtype=np.uint32)]))
            assert L.nts_exchange_plan_set_peer_needs(cp, j, cj.ctypes.data_as(C.c_void_p),
                                                      rj.ctypes.data_as(C.c_void_p)) == 0, L.nts_last_error()
        assert L.nts_exchange_plan_finalize(cp) == 0, L.nts_last_error()
        v = _lib.ExchangePlanView()
        assert L.nts_exchange_plan_get_view(cp, C.byref(v)) == 0

        def arr_of(ptr, m, dt):
            return np.ctypeslib.as_array(ptr, shape=(m,)).astype(dt, copy=True) if m and ptr else np.zeros(0, dtype=dt)

        assert (v.recv_total, v.send_total, int(v.remote_edges)) == (plan.recv_total, plan.send_total, plan.remote_edges)
        assert list(arr_of(v.need_count, P, np.uint32)) == [plan.need_count[i] if i != rank else 0 for i in range(P)]
        assert list(arr_of(v.send_count, P, np.uint32)) == [plan.send_count[j] if j != rank else 0 for j in range(P)]
        u32 = lambda t: t.numpy().view(np.uint32) if t.dtype == torch.int32 else t.numpy()
        E = plan.remote_edges
        if E:
            assert np.array_equal(arr_of(v.remote_column_offset, pg.owned_vertices + 1, np.uint32), u32(plan.remote_col_offset))
            assert np.array_equal(arr_of(v.remote_slots, E, np.uint32), u32(plan.remote_slots))
            assert np.array_equal(arr_of(v.remote_weight, E, np.float32).view(np.uint32), plan.remote_w.numpy().view(np.uint32))
            assert np.array_equal(arr_of(v.backward_indices, E, np.uint32), u32(plan.bwd_indices))
            assert np.array_equal(arr_of(v.backward_weight, E, np.float32).view(np.uint32), plan.bwd_w.numpy().view(np.uint32))
        assert np.array_equal(arr_of(v.backward_offsets, v.backward_rows + 1, np.uint32), u32(plan.bwd_offsets))
        assert np.array_equal(arr_of(v.send_rows_all, v.send_total, np.uint32), u32(plan.send_rows_all))
        # peer_bwd_offset as exchange.py::_PeerWindows derives it
        allc = [None] * P
        dist.all_gather_object(allc, [plan.need_count[i] if i != rank else 0 for i in range(P)])
        assert list(arr_of(v.peer_bwd_offset, P, np.uint32)) == [int(sum(allc[j][:rank])) for j in range(P)]
        # push offsets as exchange.py::ExchangePlan.push_offsets derives them (own entries are unused)
        fwd, bwd = plan.push_offsets()
        assert [int(x) if j != rank else 0 for j, x in enumerate(arr_of(v.fwd_push_offset, P, np.uint32))] == fwd
        assert [int(x) if j != rank else 0 for j, x in enumerate(arr_of(v.bwd_push_offset, P, np.uint32))] == bwd
        # per-chunk arrays of the engine == the Python plan's
        for i in range(P):
            if i == rank:
                continue
            sl, oc = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint32)()
            assert L.nts_exchange_plan_chunk(cp, i, C.byref(sl), C.byref(oc)) == 0
            Ei = int(pg.graph_chunks[i].edge_size)
            assert np.array_equal(arr_of(sl, Ei, np.uint32), u32(plan.csc_slots[i]))
            assert np.array_equal(arr_of(oc, plan.need_count[i] + 1, np.uint32), u32(plan.csr_offsets_compact[i]))
    finally:
        L.nts_exchange_plan_destroy(cp)


def _worker(rank, world, port, case, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from neutronstarlite_b200.exchange import ExchangePlan
        from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
        z = golden_store.load(case)
        V, E, P, F = (int(x) for x in z["case"])
        assert P == world
        hg = HostGraph(z["edges"], V)
        pg = PartitionedGraph(hg, P, rank).generate_all(dist=True)
        plan = ExchangePlan(pg)
        po = pg.partition_offset
        X = np.concatenate([z["r%d/X" % r].reshape(-1, F) for r in range(P)])
        G = np.concatenate([z["r%d/G" % r].reshape(-1, F) for r in range(P)])
        Xl = X[int(po[rank]):int(po[rank + 1])]
        Gl = G[int(po[rank]):int(po[rank + 1])]
        # ---- forward: what peers read from me, what I read from them
        send = [Xl[plan.send_rows[j].numpy().astype(np.int64)] if j != rank else None for j in range(P)]
        outs = [None] * P
        bufs = [torch.from_numpy(np.ascontiguousarray(s)) if s is not None else torch.zeros(0, F) for s in send]
        recv = _a2a(bufs, [plan.need_count[i] if i != rank else 0 for i in range(P)], F)
        Vp = pg.owned_vertices
        c = pg.graph_chunks[rank]
        Y = _gather_sum(c.column_offset, c.row_indices - c.src_range[0], c.edge_weight_forward, Xl, Vp)
        for i in plan.ring():
            c = pg.graph_chunks[i]
            staged = recv[i].numpy()
            # the staged rows must be exactly the needed rows of partition i, in slot order
            assert np.array_equal(staged, X[int(po[i]):int(po[i + 1])][plan.need[i].numpy().astype(np.int64)])
            Y += _gather_sum(c.column_offset, plan.csc_slots[i].numpy(), c.edge_weight_forward, staged, Vp)
        ref_Y = z["r%d/gcn_Y" % rank].reshape(-1, F)
        np.testing.assert_allclose(Y, ref_Y, rtol=1e-5, atol=1e-5)
        # the merged remote CSC (one launch for all remote chunks) gives the same result
        if plan.remote_edges:
            staged_all = np.concatenate([recv[i].numpy() for i in range(P) if i != rank])
            c = pg.graph_chunks[rank]
            Y2 = _gather_sum(c.column_offset, c.row_indices - c.src_range[0], c.edge_weight_forward, Xl, Vp)
            Y2 += _gather_sum(plan.remote_col_offset.numpy(), plan.remote_slots.numpy(), plan.remote_w.numpy(),
                              staged_all, Vp)
            np.testing.assert_allclose(Y2, ref_Y, rtol=1e-5, atol=1e-5)
        # ---- backward: compact partials per remote chunk, returned to the owners, unique-row scatter-add
        parts = []
        for i in range(P):
            c = pg.graph_chunks[i]
            if i == rank:
                parts.append(torch.zeros(0, F))
                continue
            offc = plan.csr_offsets_compact[i].numpy()
            part = _gather_sum(offc, c.column_indices - c.dst_range[0], c.edge_weight_backward, Gl, plan.need_count[i])
            parts.append(torch.from_numpy(part.astype(np.float32)))
        got = _a2a(parts, [plan.send_count[j] if j != rank else 0 for j in range(P)], F)
        # merged compact CSR == concatenation of the per-chunk partials, in send-staging order
        if plan.remote_edges:
            merged = _gather_sum(plan.bwd_offsets.numpy(), plan.bwd_indices.numpy().view(np.uint32) - pg.graph_chunks[rank].dst_range[0],
                                 plan.bwd_w.numpy(), Gl, plan.recv_total)
            np.testing.assert_allclose(merged, np.concatenate([t.numpy() for t in parts]), rtol=1e-5, atol=1e-6)
            rows_all = np.concatenate([plan.send_rows[j].numpy() for j in range(P) if j != rank])
            assert np.array_equal(rows_all, plan.send_rows_all.numpy())
        c = pg.graph_chunks[rank]
        dX = _gather_sum(c.row_offset, c.column_indices - c.dst_range[0], c.edge_weight_backward, Gl, Vp)
        for j in range(P):
            if j != rank and plan.send_count[j]:
                rows = plan.send_rows[j].numpy().astype(np.int64)
                assert np.unique(rows).shape[0] == rows.shape[0]
                dX[rows] += got[j].numpy()
        ref_dX = z["r%d/gcn_dX" % rank].reshape(-1, F)
        np.testing.assert_allclose(dX, ref_dX, rtol=2e-5, atol=2e-5)
        # plan bookkeeping agrees with the reference's mirror bitmaps
        for i in range(P):
            act = z["r%d/chunk%d_source_active" % (rank, i)]
            assert np.array_equal(np.nonzero(act)[0], plan.need[i].numpy())
            if i != rank:
                mirror_bits = z["r%d/chunk%d_has_mirror_at" % (rank, i)]  # my rows partition i needs
                assert np.array_equal(np.nonzero(mirror_bits)[0], plan.send_rows[i].numpy())
        _check_cxx_plan(pg, plan, rank, P)
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover - surfaced in the parent
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("case,world,port", [("synth9k_P2_F2.npz", 2, 29611), ("cora_self_P2_F4.npz", 2, 29612),
                                             ("synth9k_P4_F2.npz", 4, 29613), ("cora_self_P4_F2.npz", 4, 29614),
                                             ("synth9k_P3_F2.npz", 3, 29615)])
def test_exchange_plan_matches_reference(case, world, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=240) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, msg in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)
