"""BF16 gathers across partitions (ForwardGPUfuseOp(gather_dtype=torch.bfloat16) on GpuExchange): the p2p engine
(nts_exchange_forward_bf16 / nts_exchange_backward_bf16) with ranks time-sharing one GPU (gloo control plane), and
both transports one rank per GPU.  Every rank's result is checked against a float64 aggregation of the whole graph on
the bf16-rounded operand, per row at 1e-4 of the row's sum of |w| * |x| (FP32 accumulation in another order)."""
import multiprocessing as mp
import os
import sys

import numpy as np
import pytest

import golden_store

torch = pytest.importorskip("torch")
dist = pytest.importorskip("torch.distributed")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dense(c, x64, forward):
    """float64 Y = A X (forward, CSC) or dX = A^T dY (backward, CSR) of a single-partition chunk."""
    if forward:
        off, idx, w, base = c.column_offset_gpu.long(), c.row_indices_gpu.long(), c.edge_weight_forward_gpu, 0
        n = c.batch_size_forward
    else:
        off, idx, w = c.row_offset_gpu.long(), c.column_indices_gpu.long(), c.edge_weight_backward_gpu
        base, n = c.dst_range[0], c.batch_size_backward
    rows = torch.repeat_interleave(torch.arange(off.numel() - 1, device=off.device), off[1:] - off[:-1])
    return torch.zeros((n, x64.shape[1]), dtype=torch.float64, device=x64.device).index_add_(
        0, rows, x64[idx - base] * w.double()[:, None])


def _check(got, c1, X, lo, hi, forward):
    xr = X.to(torch.bfloat16).double()
    ref = _dense(c1, xr, forward)[lo:hi]
    mag = _dense(c1, xr.abs(), forward)[lo:hi]
    err = (got.double() - ref).abs().amax(1) if got.numel() else torch.zeros(0, device=got.device)
    scale = mag.amax(1) if mag.numel() else torch.zeros(0, device=got.device)
    bad = torch.nonzero(err > 1e-4 * scale + 1e-30).view(-1)
    assert bad.numel() == 0, "rows %s: err %s scale %s" % (bad[:4].tolist(), err[bad[:4]].tolist(),
                                                         scale[bad[:4]].tolist())


def _run_rank(rank, world, dev, case, transport, po, iters):
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.exchange import GpuExchange
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    z = golden_store.load(case)
    V = int(z["case"][0])
    host = HostGraph(z["edges"], V)
    pg = PartitionedGraph(host, world, rank, po).generate_all(device=dev, dist=True)
    c1 = PartitionedGraph(HostGraph(z["edges"], V), 1, 0).generate_all(device=dev).graph_chunks[0]
    ex = GpuExchange(pg, transport=transport)
    op = ops.ForwardGPUfuseOp(pg, None, exchange=ex, gather_dtype=torch.bfloat16)
    pof = pg.partition_offset
    lo, hi = int(pof[rank]), int(pof[rank + 1])
    for F in (2, 41, 602):
        gen = torch.Generator().manual_seed(F)
        X = (torch.rand((V, F), generator=gen) * 2 - 1).to(dev)
        G = (torch.rand((V, F), generator=gen) * 2 - 1).to(dev)
        for it in range(iters):   # repeated calls: buffer reuse and the epoch protocol
            xin = X[lo:hi].contiguous()
            if it % 2:
                xin = xin.to(torch.bfloat16)
            y = op.forward(xin)
            dx = op.backward(G[lo:hi].contiguous())
            torch.cuda.synchronize()
            assert y.dtype == torch.float32 and dx.dtype == torch.float32
            _check(y, c1, X, lo, hi, True)
            _check(dx, c1, G, lo, hi, False)
    dist.barrier()
    ex.close()


def _shared_worker(rank, world, port, case, env, po, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["NTS_EXCHANGE_TIMEOUT_MS"] = "120000"   # ranks time-slice one GPU: waits are long but bounded
    os.environ.update(env)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _run_rank(rank, world, torch.device("cuda", 0), case, "p2p", po, 3)
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def _gpu_worker(rank, world, port, case, transport, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        _run_rank(rank, world, dev, case, transport, None, 2)
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


def _launch(target, world, args, timeout):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world) + args + (q,)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(world):
            results.append(q.get(timeout=timeout))
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, msg in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)


SHARED = [
    ("pipeline_w2", "synth9k_P2_F2", 2, {"NTS_EXCHANGE_MODE": "pipeline"}, None),
    ("merged_w3_plan_all", "synth9k_P3_F2", 3, {"NTS_EXCHANGE_MODE": "merged", "NTS_EXCHANGE_PLAN_MIN_EDGES": "1"},
     None),
    ("measured_w3", "synth9k_P3_F2", 3, {}, None),
    ("empty_partition_w2", "synth9k_P2_F2", 2, {}, "empty"),
]


@pytest.mark.parametrize("name,case,world,env,po", SHARED, ids=[s[0] for s in SHARED])
def test_p2p_bf16_ranks_sharing_one_gpu(name, case, world, env, po):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    if po == "empty":   # rank 1 owns no vertex: it pushes and reads nothing but takes part in the protocol
        V = int(golden_store.load(case)["case"][0])
        po = np.array([0, V, V], dtype=np.uint32)
    port = 29500 + (hash(name) % 150)
    _launch(_shared_worker, world, (port, case, env, po), 420)


@pytest.mark.parametrize("transport", ["nccl", "p2p"])
def test_bf16_exchange_one_rank_per_gpu(transport):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = 29650 + (hash(transport) % 40)
    _launch(_gpu_worker, 2, (port, "synth9k_P2_F2", transport), 300)
