"""The learnable embedding on the GPU (feature_table.ShardedEmbedding, K11 = nts_embedding_step):

  * world 1: after a step, touched rows and their moments equal nts_adam_update on the same rows bit for bit,
    untouched rows keep their bits, an empty step changes nothing;
  * over CUDA IPC with 2 and 3 ranks as processes sharing one GPU (gloo control plane; at world 3 the middle shard is
    empty): rows touched by 0, 1, 2 and 3 ranks on both sides of every shard boundary equal the float32 rank-order sum
    followed by nts_adam_update, bit for bit, over three steps, each gathering rows peers updated in the one before;
  * GCNSampleImpl (FP32 and BF16 gathers) and GATSampleImpl on a ShardedEmbedding: one step at world 1 and one round
    at world 2 and 3 with an idle last rank (and with one rank per GPU, skipped below 2 GPUs) match a float64 torch
    restatement with autograd through the gathered rows; infer() then reads the learned rows;
  * argument errors raise NtsError before any device work."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from embedding_oracle import rank_order_sum
from test_dist_sample_gpu import BATCH, FANOUT, GAT_HEADS, MODELS, adam_first_step, graph_and_data, round_mask, \
    spawn, table_offsets, _init

pytestmark = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def _adam_reference(W, M, V, g, table):
    """nts_adam_update on contiguous copies of the rows, with the table's current schedule values."""
    from neutronstarlite_b200 import _lib
    W, M, V, g = (t.contiguous().clone() for t in (W, M, V, g))
    if W.numel():
        _lib.call("nts_adam_update", W.data_ptr(), M.data_ptr(), V.data_ptr(), g.data_ptr(), W.numel(),
                  float(table.weight_decay), float(table.beta1), float(table.beta2), float(table.alpha),
                  float(table.epsilon), _lib.stream())
    return W, M, V


# ---- K11 at world 1 -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("F", [22, 128])
def test_k11_world_1_is_nts_adam_update_bit_for_bit(F):
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedEmbedding
    _need_gpu()
    d = torch.device("cuda:0")
    Vn = 3000
    gen = torch.Generator().manual_seed(F)
    x0 = (torch.rand((Vn, F), generator=gen) * 2 - 1).to(d)
    t = ShardedEmbedding(x0, [0, Vn], capacity=1000)
    W, M, V = x0.clone(), torch.zeros_like(x0), torch.zeros_like(x0)
    for s in range(3):
        ids = torch.randperm(Vn, generator=gen)[:700 + 100 * s].sort().values
        g = torch.randn((ids.numel(), F), generator=gen).to(d) * 1e-2
        idd = ids.to(d)
        Wr, Mr, Vr = _adam_reference(W[idd], M[idd], V[idd], g, t)
        W[idd], M[idd], V[idd] = Wr, Mr, Vr
        n0 = _lib.load().nts_kernel_launch_count()
        t.step(idd.to(torch.int32), g)
        assert _lib.load().nts_kernel_launch_count() - n0 == 2
        torch.cuda.synchronize()
        assert torch.equal(t.gather(torch.arange(Vn)), W)
        assert torch.equal(t.M[:, :F], M) and torch.equal(t.V[:, :F], V)
        assert not t.M[:, F:].any() and not t.V[:, F:].any() and not t._mask.any()
    before = (t.gather(torch.arange(Vn)), t.M.clone(), t.V.clone(), t.curr_epoch)
    t.step(torch.empty(0, dtype=torch.int32, device=d), torch.empty((0, F), device=d))
    torch.cuda.synchronize()
    assert torch.equal(t.gather(torch.arange(Vn)), before[0])
    assert torch.equal(t.M, before[1]) and torch.equal(t.V, before[2]) and t.curr_epoch == before[3] + 1
    t.close()


def test_errors_are_raised_before_device_work():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedEmbedding
    _need_gpu()
    d = torch.device("cuda:0")
    x0 = torch.rand((50, 8), device=d)
    with pytest.raises(_lib.NtsError, match="float32"):
        ShardedEmbedding(x0, [0, 50], dtype=torch.bfloat16)
    t = ShardedEmbedding(x0, [0, 50], capacity=4)
    g = lambda n: torch.ones((n, 8), device=d)
    n0 = _lib.load().nts_kernel_launch_count()
    for ids, what in (([3, 1], "ascending"), ([1, 1], "ascending"), ([1, 50], r"\[0, 50\)"), ([-1], r"\[0, 50\)"),
                      ([0, 1, 2, 3, 4], "capacity")):
        with pytest.raises(_lib.NtsError, match=what):
            t.step(torch.tensor(ids, dtype=torch.int32, device=d), g(len(ids)))
    with pytest.raises(_lib.NtsError, match="int32"):
        t.step(torch.tensor([1, 2], device=d), g(2))
    with pytest.raises(_lib.NtsError, match="grad"):
        t.step(torch.tensor([1, 2], dtype=torch.int32, device=d), g(3))
    assert _lib.load().nts_kernel_launch_count() == n0
    assert torch.equal(t.gather(torch.arange(50)), x0) and t.curr_epoch == 0
    t.close()
    with pytest.raises(_lib.NtsError, match="closed"):
        t.step(torch.tensor([1], dtype=torch.int32, device=d), g(1))


# ---- K11 over IPC ---------------------------------------------------------------------------------------------------

IPC_V, IPC_F = 4000, 12


def ipc_plan(world, off, step):
    """The ids each rank sends at `step`: rows on both sides of every shard boundary and random rows, each sent by
    0, 1, 2, ... up to `world` ranks (row g by the ranks (g + step + j) % world for j < its count)."""
    rng = np.random.default_rng(100 + step)
    rows = set(rng.choice(IPC_V, 400, replace=False).tolist())
    for o in off:
        rows.update(g for g in range(o - 3, o + 3) if 0 <= g < IPC_V)
    sent = [[] for _ in range(world)]
    counts = np.zeros(world + 1, dtype=np.int64)
    for g in sorted(rows):
        k = (g + step) % (world + 1)
        counts[k] += 1
        for j in range(k):
            sent[(g + step + j) % world].append(g)
    assert (counts > 0).all()
    grads = [torch.randn((len(ids), IPC_F), generator=torch.Generator().manual_seed(1000 * step + q)) * 1e-2
             for q, ids in enumerate(sent)]
    return [np.array(sorted(ids), dtype=np.int64) for ids in sent], grads


def _ipc_worker(rank, world, port, extra, q):
    try:
        dev = _init(rank, world, port, False)
        from neutronstarlite_b200.feature_table import ShardedEmbedding
        off = [0, IPC_V // 3, IPC_V // 3, IPC_V] if world == 3 else [0, IPC_V // 2, IPC_V]
        lo, hi = off[rank], off[rank + 1]
        x0 = (torch.rand((IPC_V, IPC_F), generator=torch.Generator().manual_seed(3)) * 2 - 1).to(dev)
        t = ShardedEmbedding(x0[lo:hi].clone(), off)
        W, M, V = x0.clone(), torch.zeros_like(x0), torch.zeros_like(x0)
        all_ids = torch.arange(IPC_V, device=dev)
        for step in range(3):
            # every rank reads every row, peers' rows updated by the previous step included
            assert torch.equal(t.gather(all_ids), W), "step %d: gather before the step" % step
            sent, grads = ipc_plan(world, off, step)
            ids, g = sent[rank], grads[rank]
            t.step(torch.from_numpy(ids.astype(np.int32)).to(dev), g.to(dev))
            # the restatement: the float32 rank-order sum, then nts_adam_update, on the rows of every rank
            touched = sorted(set(np.concatenate(sent).tolist()))
            gsum = []
            for r in touched:
                rows = [grads[p][int(np.searchsorted(sent[p], r))].numpy() for p in range(world) if r in set(sent[p])]
                gsum.append(rank_order_sum(rows))
            tid = torch.tensor(touched, device=dev)
            # the schedule values this step used (the table's own have advanced past them)
            from neutronstarlite_b200.adam import AdamSchedule
            s = AdamSchedule()
            s._init_schedule(0.01, 0.9, 0.999, 1e-9, 0.0001)
            s.set_decay(0.97, 100)
            for _ in range(step):
                s.next()
            Wr, Mr, Vr = _adam_reference(W[tid], M[tid], V[tid], torch.from_numpy(np.stack(gsum)).to(dev), s)
            W[tid], M[tid], V[tid] = Wr, Mr, Vr
            torch.cuda.synchronize()
            assert torch.equal(t.gather(torch.arange(lo, hi, device=dev)), W[lo:hi]), "step %d: own rows" % step
            assert torch.equal(t.M[:, :IPC_F], M[lo:hi]) and torch.equal(t.V[:, :IPC_F], V[lo:hi]), step
        t.close()
        q.put((rank, "ok", None))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_k11_over_ipc_is_the_rank_order_sum_then_adam_bit_for_bit(world):
    _need_gpu()
    spawn(_ipc_worker, world, 29710 + world, None)


# ---- models ---------------------------------------------------------------------------------------------------------

class _Agg(torch.autograd.Function):
    """y[dst(e)] += w_e x[src(e)] in float64, with K1's BF16 operand rounding when bf16: the forward rounds x, the
    backward rounds dy, as ops.MiniBatchFuseOp does under gather_dtype=torch.bfloat16."""

    @staticmethod
    def forward(ctx, x, e_dst, e_src, w, n_dst, bf16):
        ctx.save_for_backward(e_dst, e_src, w)
        ctx.n_src, ctx.bf16 = x.shape[0], bf16
        xr = x.float().bfloat16().double() if bf16 else x
        return torch.zeros((n_dst, x.shape[1]), dtype=x.dtype, device=x.device).index_add(0, e_dst,
                                                                                           xr[e_src] * w[:, None])

    @staticmethod
    def backward(ctx, dy):
        e_dst, e_src, w = ctx.saved_tensors
        dyr = dy.float().bfloat16().double() if ctx.bf16 else dy
        dx = torch.zeros((ctx.n_src, dy.shape[1]), dtype=dy.dtype, device=dy.device).index_add(
            0, e_src, dyr[e_dst] * w[:, None])
        return dx, None, None, None, None, None


def gcn_float64_step(blocks, table, labels, Ws, bf16):
    """One GCNSampleImpl step in float64 autograd with the table as a leaf: (W grads, table grad)."""
    Wd = [W.detach().double().requires_grad_(True) for W in Ws]
    tab = table.detach().double().requires_grad_(True)
    L = len(Wd)
    dv = table.device
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dv)
    h = tab[t(blocks[L - 1]["src"])]
    for l in range(L):
        b = blocks[L - 1 - l]
        n = b["column_offset"].size - 1
        e_dst = torch.repeat_interleave(torch.arange(n, device=dv), t(np.diff(b["column_offset"].astype(np.int64))))
        y = _Agg.apply(h, e_dst, t(b["row_indices"]), torch.from_numpy(b["weight"]).to(dv).double(), n, bf16)
        h = y @ Wd[l]
        if l < L - 1:
            h = torch.relu(h)
    loss = torch.nn.functional.nll_loss(h.log_softmax(1), labels[t(blocks[0]["dst"])])
    loss.backward()
    return [W.grad for W in Wd], tab.grad


def gat_table_grad(blocks, table, labels, params, heads, layers):
    """The gradient of one GATSampleImpl step's loss with respect to the table, in float64 autograd through the
    gathered rows (test_gat_sample_gpu.float64_step's layers, which give the parameters' gradients)."""
    feats = table.detach().double().requires_grad_(True)
    dv, dd = feats.device, torch.float64
    leaves = [p.detach().to(dd) for p in params]
    L = len(layers) - 1
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dv)
    x = None
    for l in range(L):
        b = blocks[L - 1 - l]
        W, al, ar = leaves[l], leaves[L + l], leaves[2 * L + l]
        H, D = heads[l], layers[l + 1] // heads[l]
        if l == 0:
            x = feats[t(b["src"])]
        xt = x @ W
        s = (xt.view(-1, H, D) * al).sum(-1)
        dsc = (xt[t(b["dst_pos"])].view(-1, H, D) * ar).sum(-1)
        n_dst = b["dst"].size
        dst = torch.repeat_interleave(torch.arange(n_dst, device=dv), t(np.diff(b["column_offset"].astype(np.int64))))
        srci = t(b["row_indices"])
        logit = torch.nn.functional.leaky_relu(s[srci] + dsc[dst], 0.2)
        mx = torch.full((n_dst, H), -float("inf"), dtype=dd, device=dv).scatter_reduce(
            0, dst[:, None].expand(-1, H), logit.detach(), "amax")
        ex = torch.exp(logit - mx[dst])
        a = ex / torch.zeros((n_dst, H), dtype=dd, device=dv).index_add(0, dst, ex)[dst]
        out = torch.zeros((n_dst, H, D), dtype=dd, device=dv).index_add(
            0, dst, xt[srci].view(-1, H, D) * a[:, :, None]).reshape(n_dst, H * D)
        x = out.log_softmax(1) if l == L - 1 else torch.relu(out)
    torch.nn.functional.nll_loss(x, labels[t(blocks[0]["dst"])]).backward()
    return feats.grad


def make_model(kind, pg, features, labels, mask, gather_dtype=None):
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    kw = dict(fanout=FANOUT, batch_size=BATCH, seed=5, sample_seed=9)
    if kind == "gcn":
        return GCNSampleImpl(pg, MODELS[kind], features, labels, mask, drop_rate=0.0, gather_dtype=gather_dtype, **kw)
    return GATSampleImpl(pg, MODELS[kind], features, labels, mask, heads=GAT_HEADS, **kw)


def reference_round(kind, n_batches, world, bf16, d):
    """The float64 restatement of one round of n_batches batches, the blocks from a single-GPU sampler: the initial
    weights, their summed gradients, the summed table gradient and the rows the round touches (its batches' deepest-hop
    sources, sent and stepped even where their gradient is zero)."""
    hg, pg, feats, labels = graph_and_data(d)
    n_train = n_batches * BATCH - 7
    mask = round_mask(hg.vertices, n_train)
    ref = make_model(kind, pg, feats.to(d), labels.to(d), mask)
    W0 = [p.W.detach().double() for p in ref.params()]
    ids = ref.nids[0]
    gW, gT = [torch.zeros_like(w) for w in W0], torch.zeros(feats.shape, dtype=torch.float64, device=d)
    touched = torch.zeros(feats.shape[0], dtype=torch.bool)
    for b in range(n_batches):
        sg = ref.sampler.sample(ids[b * BATCH:(b + 1) * BATCH], ref.sample_seed, b)
        blocks = [blk.to_numpy() for blk in sg.blocks]
        if kind == "gcn":
            gs, gt = gcn_float64_step(blocks, feats.to(d), labels.to(d), W0, bf16)
        else:
            import test_gat_sample_gpu as gat_ref
            _, gs = gat_ref.float64_step(blocks, feats.to(d), labels.to(d), W0, ref.heads, MODELS[kind])
            gt = gat_table_grad(blocks, feats.to(d), labels.to(d), W0, ref.heads, MODELS[kind])
        gW = [a + g for a, g in zip(gW, gs)]
        gT += gt
        touched[torch.from_numpy(blocks[-1]["src"].astype(np.int64))] = True
    return hg, pg, feats, labels, mask, W0, gW, gT, touched


def check_adam_first_step(got, w0, g, tol, what):
    """got = Parameter's first Adam step from w0 with gradient g (float64), on the elements clear of the float32
    rounding of g (Adam's first step is about lr * sign(W_g))."""
    W_ref, W_g = adam_first_step(w0.cpu(), g.cpu())
    sure = W_g.abs() > tol * W_g.abs().amax(1, keepdim=True)
    err = ((got.double().cpu() - W_ref).abs() * sure).amax(1)
    assert (err <= 1e-4 * W_ref.abs().amax(1).clamp_min(1e-30)).all(), what


def check_round(kind, n_batches, world, bf16, rows, Ws, d):
    hg, pg, feats, labels, mask, W0, gW, gT, touched = reference_round(kind, n_batches, world, bf16, d)
    tol = 3e-2 if bf16 else 1e-5
    for W, w0, g in zip(Ws, W0, gW):
        check_adam_first_step(W, w0, g, tol, "%s weights" % kind)
    assert touched.any() and (~touched).any()
    assert torch.equal(rows[~touched], feats[~touched]), "untouched rows changed"
    check_adam_first_step(rows[touched], feats[touched].double(), gT[touched.to(d)], tol, "%s rows" % kind)
    return hg, pg, labels, mask


@pytest.mark.parametrize("kind,bf16", [("gcn", False), ("gcn", True), ("gat", False)])
def test_one_model_step_at_world_1_matches_float64(kind, bf16):
    from neutronstarlite_b200.feature_table import ShardedEmbedding
    _need_gpu()
    d = torch.device("cuda:0")
    hg, pg, feats, labels = graph_and_data(d)
    mask = round_mask(hg.vertices, BATCH - 7)
    table = ShardedEmbedding(feats.to(d), [0, hg.vertices])
    m = make_model(kind, pg, table, labels.to(d), mask, torch.bfloat16 if bf16 else None)
    m.run_epoch(test=False)
    rows = table.gather(torch.arange(hg.vertices)).cpu()
    Ws = [p.W.detach() for p in m.params()]
    check_round(kind, 1, 1, bf16, rows, Ws, d)
    # full-neighbour inference reads the learned rows: the same model on a tensor of them gives the same outputs
    lo, out = m.infer()
    twin = make_model(kind, pg, rows.to(d), labels.to(d), mask, torch.bfloat16 if bf16 else None)
    with torch.no_grad():
        for p, q in zip(twin.params(), m.params()):
            p.W.copy_(q.W)
    lo2, out2 = twin.infer()
    assert lo == lo2
    torch.testing.assert_close(out, out2, rtol=1e-5, atol=1e-6)
    table.close()


def _round_worker(rank, world, port, per_gpu, q):
    try:
        dev = _init(rank, world, port, per_gpu)
        from neutronstarlite_b200.feature_table import ShardedEmbedding
        hg, pg, feats, labels = graph_and_data(dev)
        off = table_offsets(hg, world)
        out = {}
        for kind in MODELS:
            table = ShardedEmbedding(feats[off[rank]:off[rank + 1]].to(dev), off)
            m = make_model(kind, pg, table, labels.to(dev), round_mask(hg.vertices, (world - 1) * BATCH - 7))
            m.run_epoch(test=False)                    # one round, the last rank idle
            own = table.gather(torch.arange(off[rank], off[rank + 1])).cpu().numpy()
            out[kind] = (own, [p.W.detach().cpu().numpy() for p in m.params()])
            table.close()
        q.put((rank, "ok", out))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.destroy_process_group()


def run_round_test(world, per_gpu, port):
    ranks = spawn(_round_worker, world, port, per_gpu)
    d = torch.device("cuda:0")
    for kind in MODELS:
        for r in ranks[1:]:
            for a, b in zip(r[kind][1], ranks[0][kind][1]):
                assert np.array_equal(a, b), "ranks disagree on %s weights" % kind
        rows = torch.from_numpy(np.concatenate([r[kind][0] for r in ranks]))
        check_round(kind, world - 1, world, False, rows, [torch.from_numpy(w) for w in ranks[0][kind][1]], d)


@pytest.mark.parametrize("world", [2, 3])
def test_one_round_on_ranks_sharing_one_gpu_matches_float64(world):
    _need_gpu()
    run_round_test(world, False, 29730 + world)


def test_one_round_with_one_rank_per_gpu_matches_float64():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_round_test(2, True, 29740)
