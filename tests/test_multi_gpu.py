"""CUDA data path of the distributed fused aggregation against the golden vectors of the reference run at the same P.

  * test_distributed_fused_aggregation: one rank per GPU on 2 (or 4) GPUs of one box, both transports ("nccl" =
    one all-to-all + merged remote chunk, "p2p" = the peer-memory push engine, csrc/nts_exchange.cu).  Skipped when fewer GPUs are
    visible; run with `pytest -m gpu tests/test_multi_gpu.py` on a machine with that many GPUs.
  * test_p2p_engine_ranks_sharing_one_gpu: the SAME engine, flag protocol and CUDA-IPC windows with 2 / 3 / 4 ranks
    as separate processes time-slicing ONE GPU (control plane over gloo), so the single-GPU round-end run exercises
    the cross-process epoch protocol, window double-buffering, empty partitions and the planned-aggregation path
    under real concurrency too."""
import os
import sys

import golden_store
import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, case, transport, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from neutronstarlite_b200 import ops
        from neutronstarlite_b200.exchange import GpuExchange
        from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
        z = golden_store.load(case)
        V, E, P, F = (int(x) for x in z["case"])
        pg = PartitionedGraph(HostGraph(z["edges"], V), P, rank).generate_all(device=dev, dist=True)
        ex = GpuExchange(pg, transport=transport)
        op = ops.ForwardGPUfuseOp(pg, None, exchange=ex)
        x = torch.from_numpy(z["r%d/X" % rank].reshape(-1, F)).to(dev)
        g = torch.from_numpy(z["r%d/G" % rank].reshape(-1, F)).to(dev)
        ref_y = z["r%d/gcn_Y" % rank].reshape(-1, F)
        ref_dx = z["r%d/gcn_dX" % rank].reshape(-1, F)
        for it in range(3):  # repeated calls exercise buffer reuse and the p2p epoch protocol
            y = op.forward(x)
            dx = op.backward(g)
            torch.cuda.synchronize()
            np.testing.assert_allclose(y.cpu().numpy(), ref_y, rtol=1e-4, atol=1e-5)
            np.testing.assert_allclose(dx.cpu().numpy(), ref_dx, rtol=1e-4, atol=2e-5)
        # mirror fetch / return (DistGPUGetDepNbrOp) against the reference's DistGetDepNbrOp at the same P
        dep = ops.DistGPUGetDepNbrOp(pg, None, exchange=ex)
        mirror = dep.forward(x)
        torch.cuda.synchronize()
        assert np.array_equal(mirror.cpu().numpy(), z["r%d/dep_mirror" % rank].reshape(-1, F))
        gm = torch.from_numpy(z["r%d/dep_Gm" % rank].reshape(-1, F)).to(dev)
        dxm = dep.backward(gm)
        torch.cuda.synchronize()
        np.testing.assert_allclose(dxm.cpu().numpy(), z["r%d/dep_dX" % rank].reshape(-1, F), rtol=1e-4, atol=2e-5)
        # a wider feature matrix (second width through the same exchange object)
        F2 = 40
        gen = torch.Generator().manual_seed(1)
        Xg = torch.rand((V, F2), generator=gen) * 2 - 1
        po = pg.partition_offset
        y2 = op.forward(Xg[int(po[rank]):int(po[rank + 1])].contiguous().to(dev))
        torch.cuda.synchronize()
        # single-partition truth with the same kernels on this GPU
        pg1 = PartitionedGraph(HostGraph(z["edges"], V), 1, 0).generate_all(device=dev)
        y_full = ops.ForwardSingleGPUfuseOp(pg1).forward(Xg.to(dev))
        torch.testing.assert_close(y2, y_full[int(po[rank]):int(po[rank + 1])], rtol=1e-4, atol=1e-5)
        dist.barrier()
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


CASES = [("synth9k_P2_F2.npz", 2), ("cora_self_P2_F4.npz", 2), ("synth9k_P4_F2.npz", 4), ("cora_self_P4_F2.npz", 4)]


@pytest.mark.parametrize("transport", ["nccl", "p2p"])
@pytest.mark.parametrize("case,world", CASES)
def test_distributed_fused_aggregation(case, world, transport):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    port = 29700 + (hash((case, transport)) % 200)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, transport, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(world):
            results.append(q.get(timeout=300))
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, msg in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)


def _shared_gpu_worker(rank, world, port, case, plan_all, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["NTS_EXCHANGE_TIMEOUT_MS"] = "120000"   # ranks time-slice one GPU: waits are long but bounded
    if plan_all:
        os.environ["NTS_EXCHANGE_PLAN_MIN_EDGES"] = "1"  # every chunk through nts_gather_plan (tuned slab count)
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from neutronstarlite_b200 import ops
        from neutronstarlite_b200.exchange import GpuExchange
        from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
        z = golden_store.load(case)
        V, E, P, F = (int(x) for x in z["case"])
        pg = PartitionedGraph(HostGraph(z["edges"], V), P, rank).generate_all(device=dev, dist=True)
        ex = GpuExchange(pg, transport="p2p")
        op = ops.ForwardGPUfuseOp(pg, None, exchange=ex)
        x = torch.from_numpy(z["r%d/X" % rank].reshape(-1, F)).to(dev)
        g = torch.from_numpy(z["r%d/G" % rank].reshape(-1, F)).to(dev)
        ref_y = z["r%d/gcn_Y" % rank].reshape(-1, F)
        ref_dx = z["r%d/gcn_dX" % rank].reshape(-1, F)
        for it in range(4):  # > n_buffers epochs: the consumed-flag wait of the push kernel is exercised
            y = op.forward(x)
            dx = op.backward(g)
            torch.cuda.synchronize()
            np.testing.assert_allclose(y.cpu().numpy(), ref_y, rtol=1e-4, atol=1e-5)
            np.testing.assert_allclose(dx.cpu().numpy(), ref_dx, rtol=1e-4, atol=2e-5)
        # mirror fetch / return (DistGPUGetDepNbrOp) on the same windows, against the reference's DistGetDepNbrOp
        dep = ops.DistGPUGetDepNbrOp(pg, None, exchange=ex)
        mirror = dep.forward(x)
        torch.cuda.synchronize()
        assert np.array_equal(mirror.cpu().numpy(), z["r%d/dep_mirror" % rank].reshape(-1, F))
        gm = torch.from_numpy(z["r%d/dep_Gm" % rank].reshape(-1, F)).to(dev)
        dxm = dep.backward(gm)
        torch.cuda.synchronize()
        np.testing.assert_allclose(dxm.cpu().numpy(), z["r%d/dep_dX" % rank].reshape(-1, F), rtol=1e-4, atol=2e-5)
        # a wider matrix through the same engine: the window is re-reserved (release -> barrier -> reallocate)
        F2 = 602
        gen = torch.Generator().manual_seed(3)
        Xg = torch.rand((V, F2), generator=gen) * 2 - 1
        po = pg.partition_offset
        lo, hi = int(po[rank]), int(po[rank + 1])
        y2 = op.forward(Xg[lo:hi].contiguous().to(dev))
        dx2 = op.backward(Xg[lo:hi].contiguous().to(dev))
        torch.cuda.synchronize()
        pg1 = PartitionedGraph(HostGraph(z["edges"], V), 1, 0).generate_all(device=dev)
        one = ops.ForwardSingleGPUfuseOp(pg1)
        y_full = one.forward(Xg.to(dev))
        dx_full = one.backward(Xg.to(dev))
        torch.testing.assert_close(y2, y_full[lo:hi], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(dx2, dx_full[lo:hi], rtol=1e-4, atol=2e-5)
        dist.barrier()
        ex.close()
        q.put((rank, "ok"))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc())))
    finally:
        dist.destroy_process_group()


# (world 4 on one time-sliced GPU takes minutes and timed out; the 4-way split with its two EMPTY partitions runs in
# test_distributed_fused_aggregation on 4 GPUs)
SHARED = [("synth9k_P2_F2.npz", 2, False), ("synth9k_P3_F2.npz", 3, True)]


@pytest.mark.parametrize("case,world,plan_all", SHARED)
def test_p2p_engine_ranks_sharing_one_gpu(case, world, plan_all):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    port = 29900 + (hash((case, world)) % 90)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shared_gpu_worker, args=(r, world, port, case, plan_all, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(world):
            results.append(q.get(timeout=420))
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, msg in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)
