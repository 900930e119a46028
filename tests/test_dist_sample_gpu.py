"""Data-parallel sampled training over a ShardedFeatureTable (feature_table.py, toolkits._SampledRounds):

  * the table over CUDA IPC with 2 and 3 ranks as processes sharing one GPU (control plane over gloo): every rank's
    gather of random ids equals the whole table's rows bit for bit, and close() lets every process end by itself;
  * world 1: a one-shard table gives the same losses and weights as the tensor, bit for bit, on Cora (GCN and GAT);
  * one data-parallel round of GCNSampleImpl and GATSampleImpl at world 2 and 3 on one shared GPU, and at world 2 with
    one rank per GPU (skipped below 2 GPUs): every rank ends with the same weights, and they match a float64
    restatement (the same blocks from a single-GPU sampler, summed batch gradients, Parameter's Adam arithmetic), also
    when the last rank has no batch in the round; losses and accuracies agree on every rank."""
import os
import sys

import numpy as np
import pytest

import golden_store

torch = pytest.importorskip("torch")
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASE = "synth9k_P3_F2.npz"       # the 9k-vertex graph with hubs
F_IN, BATCH, FANOUT = 37, 128, [8, 12]
MODELS = {"gcn": [F_IN, 16, 5], "gat": [F_IN, 32, 5]}
GAT_HEADS = 4


def graph_and_data(dev):
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    z = golden_store.load(CASE)
    V = int(z["case"][0])
    hg = HostGraph(z["edges"], V)
    pg = PartitionedGraph(hg, 1, 0).generate_all(device=dev)
    gen = torch.Generator().manual_seed(11)
    feats = torch.rand((V, F_IN), generator=gen) * 2 - 1
    labels = torch.randint(0, 5, (V,), generator=gen)
    return hg, pg, feats, labels


def table_offsets(hg, world):
    """The reference's partitioner; at world 3 the middle shard is made empty."""
    if world == 3:
        a = int(hg.partition_offsets(2)[1])
        return [0, a, a, hg.vertices]
    return [int(o) for o in hg.partition_offsets(world)]


def round_mask(V, n_train):
    """Train ids: the first n_train multiples of 3; the other vertices alternate between validation and test."""
    mask = 1 + (torch.arange(V) % 2)
    mask[torch.arange(0, 3 * n_train, 3)] = 0
    return mask


def make_model(kind, pg, features, labels, mask, dev):
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    kw = dict(fanout=FANOUT, batch_size=BATCH, seed=5, sample_seed=9)
    if kind == "gcn":
        return GCNSampleImpl(pg, MODELS[kind], features, labels.to(dev), mask, drop_rate=0.0, **kw)
    return GATSampleImpl(pg, MODELS[kind], features, labels.to(dev), mask, heads=GAT_HEADS, **kw)


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


# ---- the table over CUDA IPC ----------------------------------------------------------------------------------

def _table_worker(rank, world, port, extra, q):
    try:
        dev = _init(rank, world, port, False)
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        hg, _, _, _ = graph_and_data(dev)
        V = hg.vertices
        off = table_offsets(hg, world)
        out = []
        for F in (3, 602):
            full = torch.rand((V, F), generator=torch.Generator().manual_seed(F)).to(dev)
            t = ShardedFeatureTable(full[off[rank]:off[rank + 1]].clone(), off)
            ids = torch.from_numpy(np.random.default_rng(rank).integers(0, V, 20000)).to(dev)
            ids[:len(off)] = torch.tensor([min(o, V - 1) for o in off], device=dev)
            got = t.gather(ids)
            torch.cuda.synchronize()
            assert torch.equal(got, full[ids]), "F=%d" % F
            remote = int(((ids < off[rank]) | (ids >= off[rank + 1])).sum())
            assert remote > 0
            out.append(remote)
            t.close()
        q.put((rank, "ok", out))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_table_over_ipc_with_ranks_sharing_one_gpu(world):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    spawn(_table_worker, world, 29610 + world, None)


# ---- world 1 ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gcn", "gat"])
def test_world_1_table_equals_the_tensor_on_cora(kind):
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges, graph
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    d = torch.device("cuda:0")
    pg = graph(cora_edges(), 2708)
    feats, labels, masks = cora_tables()
    x = torch.from_numpy(feats).to(d)
    table = ShardedFeatureTable(x, [0, 2708])
    runs = []
    for features in (x, table):
        if kind == "gcn":
            m = GCNSampleImpl(pg, [1433, 128, 7], features, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                              fanout=[5, 10], batch_size=64, drop_rate=0.0, seed=0, sample_seed=0)
        else:
            m = GATSampleImpl(pg, [1433, 64, 7], features, torch.from_numpy(labels).to(d), torch.from_numpy(masks),
                              fanout=[5, 10], batch_size=64, heads=8, seed=0, sample_seed=0)
        res = [m.run_epoch(test=True) for _ in range(2)]
        runs.append((res, m.step, [p.W.detach().clone() for p in m.params()]))
    (res_a, step_a, w_a), (res_b, step_b, w_b) = runs
    assert res_a == res_b and step_a == step_b
    for a, b in zip(w_a, w_b):
        assert torch.equal(a, b)
    table.close()


# ---- one data-parallel round ----------------------------------------------------------------------------------

def _round_worker(rank, world, port, per_gpu, q):
    try:
        dev = _init(rank, world, port, per_gpu)
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        hg, pg, feats, labels = graph_and_data(dev)
        off = table_offsets(hg, world)
        table = ShardedFeatureTable(feats[off[rank]:off[rank + 1]].to(dev), off)
        out = {}
        for kind in MODELS:
            for n_batches in (world, world - 1):        # every rank busy (last batch partial) / the last rank idle
                n_train = n_batches * BATCH - (7 if n_batches == world else 0)
                m = make_model(kind, pg, table, labels, round_mask(hg.vertices, n_train), dev)
                loss, acc = m.run_epoch(test=True)
                # numpy, not tensors: a tensor in a queue is shared through a file descriptor of this process
                out[(kind, n_batches)] = (loss, acc, m.step, [p.W.detach().cpu().numpy() for p in m.params()],
                                          [p.W_gradient.cpu().numpy() for p in m.params()])
        table.close()
        q.put((rank, "ok", out))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def adam_first_step(W, g, lr=0.01, wd=1e-4, beta1=0.9, beta2=0.999, eps=1e-9):
    """Parameter.learn_with_decay_Adam from zero moments, before any next() (alpha = learn_rate), in float64."""
    W_g = W * wd + g
    M = (1 - beta1) * W_g
    Vm = (1 - beta2) * W_g * W_g
    return W - lr * M / (torch.sqrt(Vm) + eps), W_g


def check_round(kind, n_batches, ranks, d):
    import test_gat_sample_gpu as gat_ref
    import test_sample_gpu as gcn_ref
    hg, pg, feats, labels = graph_and_data(d)
    n_train = n_batches * BATCH - (7 if n_batches == len(ranks) else 0)
    mask = round_mask(hg.vertices, n_train)
    ref = make_model(kind, pg, feats.to(d), labels, mask, d)      # initial weights, sampler, ids of one GPU
    W0 = [p.W.detach().double() for p in ref.params()]
    ids = ref.nids[0]
    grads, losses = [torch.zeros_like(w) for w in W0], []
    for b in range(n_batches):
        sg = ref.sampler.sample(ids[b * BATCH:(b + 1) * BATCH], ref.sample_seed, b)
        blocks = [blk.to_numpy() for blk in sg.blocks]
        if kind == "gcn":
            loss, gs = gcn_ref.float64_step(blocks, feats.to(d), labels.to(d), W0)
        else:
            loss, gs = gat_ref.float64_step(blocks, feats.to(d), labels.to(d), W0, ref.heads, MODELS[kind])
        losses.append(float(loss))
        grads = [a + g for a, g in zip(grads, gs)]
    r0 = ranks[0][(kind, n_batches)]
    for r in ranks[1:]:
        loss, acc, step, Ws, _ = r[(kind, n_batches)]
        assert loss == r0[0] and acc == r0[1] and step == r0[2]
        for a, b in zip(Ws, r0[3]):
            assert np.array_equal(a, b)
    loss, acc, step, Ws, Gs = r0
    Ws, Gs = [torch.from_numpy(w) for w in Ws], [torch.from_numpy(g) for g in Gs]
    assert step == sum(-(-int((mask == s).sum()) // BATCH) for s in (0, 1, 2))      # one step per batch of a pass
    assert abs(loss - float(np.mean(losses))) <= 1e-5 * abs(loss)
    for W, G, w0, g in zip(Ws, Gs, W0, grads):
        g = g.cpu()
        scale = g.abs().amax(1, keepdim=True).clamp_min(1e-30)
        assert ((G.double() - g).abs() <= 1e-4 * scale).all(), kind
        W_ref, W_g = adam_first_step(w0.cpu(), g)
        # Adam's first step is lr * sign(W_g) wherever |W_g| >> eps: an element whose W_g is within the float32
        # rounding of the summed gradient can take either sign, so only elements clear of it are compared
        sure = W_g.abs() > 1e-5 * W_g.abs().max()
        err = ((W.double() - W_ref).abs() * sure).amax(1)
        assert (err <= 1e-4 * W_ref.abs().amax(1)).all(), kind
    # the evaluation passes after the round: the same accuracies as one GPU with the round's weights and steps
    with torch.no_grad():
        for p, W in zip(ref.params(), Ws):
            p.W.copy_(W.to(d))
    ref.step = n_batches
    assert acc[1:] == [ref.evaluate(1), ref.evaluate(2)]


def run_round_test(world, per_gpu, port):
    ranks = spawn(_round_worker, world, port, per_gpu)
    d = torch.device("cuda:0")
    for kind in MODELS:
        for n_batches in (world, world - 1):
            check_round(kind, n_batches, ranks, d)


@pytest.mark.parametrize("world", [2, 3])
def test_one_round_on_ranks_sharing_one_gpu_matches_float64(world):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    run_round_test(world, False, 29630 + world)


def test_one_round_with_one_rank_per_gpu_matches_float64():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_round_test(2, True, 29640)
