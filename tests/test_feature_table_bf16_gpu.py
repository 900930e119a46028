"""BF16 feature tables (feature_table.ShardedFeatureTable(..., dtype=torch.bfloat16)) and their gather
(nts_gather_rows_sharded_bf16):

  * in one process, P local buffers stand for the shards: both outputs (BF16 rows, widened FP32) equal
    torch.cat(shards).to(bfloat16)[ids] and its .float() bit for bit, at widths that change the lane count and the
    store width, for 1, 3 and 32 shards with empty ones, with boundary, repeated and unsorted ids;
  * a table larger than 4 GiB: its last rows gather exactly and K1-BF16 reads them by global id (64-bit row addresses);
  * over CUDA IPC with 2 and 3 ranks sharing one GPU (gloo control plane); ranks whose dtypes differ are refused on
    every rank;
  * world 1: a one-shard BF16 table gives GCNSampleImpl(gather_dtype=bf16) the losses and weights of BF16 tensor
    features bit for bit, and GATSampleImpl the result of features rounded to BF16;
  * one data-parallel round at world 2 and 3 on one GPU (and one rank per GPU, skipped below 2 GPUs): GCN with BF16
    gathers from a BF16 table, GAT on a BF16 table; every rank ends with the same weights, within 1e-4 per row of the
    float64 restatement at the rounded operands."""
import numpy as np
import pytest

from test_dist_sample_gpu import (BATCH, GAT_HEADS, MODELS, _init, adam_first_step, graph_and_data, round_mask, spawn,
                                  table_offsets)
from test_gather_rows_sharded_gpu import SPLITS, V, boundary_ids

torch = pytest.importorskip("torch")
import torch.distributed as dist

pytestmark = pytest.mark.gpu
BF16_WIDTHS = [1, 3, 8, 37, 41, 64, 128, 602]


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def bf16_shards(table, offsets):
    """Each shard a separate [rows, 8*ceil(F/8)] BF16 buffer whose padding holds NaN."""
    F = table.shape[1]
    pitch = (F + 7) // 8 * 8
    out = []
    for o in range(len(offsets) - 1):
        s = torch.full((offsets[o + 1] - offsets[o], pitch), float("nan"), dtype=torch.bfloat16, device=table.device)
        s[:, :F] = table[offsets[o]:offsets[o + 1]].to(torch.bfloat16)
        out.append(s)
    return out, pitch


def gather_bf16(dst, dtype_code, ld, shards, offsets, pitch, ids, F):
    from neutronstarlite_b200 import _lib
    d = dst.device
    ptrs = torch.tensor([s.data_ptr() for s in shards], dtype=torch.int64, device=d)
    off = torch.tensor(np.asarray(offsets, np.int64).astype(np.uint32).view(np.int32), device=d)
    _lib.call("nts_gather_rows_sharded_bf16", dst.data_ptr(), dtype_code, ld, ptrs.data_ptr(), off.data_ptr(),
              len(shards), pitch, ids.data_ptr() if ids.numel() else None, ids.numel(), F,
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dst


@pytest.mark.parametrize("split", list(SPLITS))
@pytest.mark.parametrize("F", BF16_WIDTHS)
def test_bf16_gather_equals_the_rounded_table_rows(F, split):
    d = dev()
    offsets = SPLITS[split]
    table = (torch.rand((V, F), generator=torch.Generator().manual_seed(F)) * 200 - 100).to(d)
    shards, pitch = bf16_shards(table, offsets)
    ids = boundary_ids(offsets, np.random.default_rng(F)).to(d)
    want = table.to(torch.bfloat16)[ids.long()]
    n = ids.numel()
    for ld in (pitch, pitch + 8):
        out = torch.full((n, ld), float("inf"), dtype=torch.bfloat16, device=d)
        gather_bf16(out, 1, ld, shards, offsets, pitch, ids, F)
        assert torch.equal(out[:, :F], want)
        assert bool(torch.isinf(out[:, pitch:].float()).all())      # columns past the shard pitch are not written
    for shift in (0, 1):                                             # 16- and 4-byte aligned FP32 rows
        flat = torch.full((n * F + shift,), float("nan"), device=d)
        out = flat[shift:].view(n, F)
        gather_bf16(out, 0, F, shards, offsets, pitch, ids, F)
        assert torch.equal(out, want.float())
    empty = torch.empty((0, pitch), dtype=torch.bfloat16, device=d)
    gather_bf16(empty, 1, pitch, shards, offsets, pitch, ids[:0], F)


def test_bf16_gather_refusals():
    from neutronstarlite_b200 import _lib
    L = _lib.load()
    assert L.nts_gather_rows_sharded_bf16(None, 2, 8, None, None, 1, 8, None, 4, 8, None) != 0
    assert L.nts_gather_rows_sharded_bf16(None, 1, 8, None, None, 1, 12, None, 4, 8, None) != 0
    assert b"shard_pitch" in L.nts_last_error()
    assert L.nts_gather_rows_sharded_bf16(None, 1, 12, None, None, 1, 16, None, 4, 8, None) != 0
    assert L.nts_gather_rows_sharded_bf16(None, 0, 9, None, None, 1, 16, None, 4, 8, None) != 0
    assert L.nts_gather_rows_sharded_bf16(None, 1, 16, None, None, 1, 16, None, 0, 8, None) == 0


def test_bf16_table_refuses_a_bf16_output_from_an_fp32_table():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    d = dev()
    x = torch.rand((50, 41), device=d)
    t32 = ShardedFeatureTable(x, [0, 50])
    t16 = ShardedFeatureTable(x, [0, 50], dtype=torch.bfloat16)
    try:
        assert t32.dtype == torch.float32 and t32.pitch == 44 and t32.local_bytes == 50 * 44 * 4
        assert t16.dtype == torch.bfloat16 and t16.pitch == 48 and t16.local_bytes == 50 * 48 * 2
        with pytest.raises(_lib.NtsError):
            t32.gather([1, 2], dtype=torch.bfloat16)
        ids = [49, 0, 7, 7]
        assert torch.equal(t32.gather(ids), x[ids])
        g16 = t16.gather(ids)
        assert g16.dtype == torch.bfloat16 and g16.shape == (4, 41) and g16.stride(0) == 48
        assert torch.equal(g16, x[ids].to(torch.bfloat16))
        assert torch.equal(t16.gather(ids, dtype=torch.float32), x[ids].to(torch.bfloat16).float())
        with pytest.raises(_lib.NtsError):
            ShardedFeatureTable(x, [0, 50], dtype=torch.float16)
    finally:
        t32.close()
        t16.close()


def test_table_larger_than_4_gib():
    """A [17.5 M, 128] BF16 table (4.48 GB): the last rows gather exactly from one and from two shards, and K1-BF16 sums
    them by global id."""
    from neutronstarlite_b200 import _lib
    d = dev()
    free, _ = torch.cuda.mem_get_info(d)
    if free < 8 * 2 ** 30:
        pytest.skip("needs 8 GB of free device memory")
    F, n = 128, 17_500_000
    big = torch.zeros((n, F), dtype=torch.bfloat16, device=d)
    assert big.numel() * 2 > 4 * 2 ** 30
    tail = torch.randint(-8, 9, (64, F), generator=torch.Generator().manual_seed(3)).float().to(d)
    big[-64:] = tail.to(torch.bfloat16)
    ids = torch.arange(n - 64, n, dtype=torch.int64, device=d).flip(0).to(torch.int32)
    for offsets, shards in (([0, n], [big]), ([0, n // 2, n], [big[:n // 2], big[n // 2:]])):
        out = torch.empty((64, F), dtype=torch.bfloat16, device=d)
        gather_bf16(out, 1, F, shards, offsets, F, ids, F)
        assert torch.equal(out.float(), tail.flip(0))
    # K1-BF16 on global ids: row r sums tail rows r and 63 - r with weights 1 and 2
    E = 128
    idx = torch.cat([ids[:, None], torch.arange(n - 64, n, device=d, dtype=torch.int64).to(torch.int32)[:, None]], 1)
    w = torch.tensor([1.0, 2.0], device=d).repeat(64)
    offs = torch.arange(0, E + 1, 2, dtype=torch.int32, device=d)
    y = torch.zeros((64, F), device=d)
    _lib.call("nts_segment_gather_sum_bf16", big.data_ptr(), F, y.data_ptr(), w.data_ptr(), idx.reshape(-1).data_ptr(),
              offs.data_ptr(), 64, E, F, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y, tail.flip(0) + 2 * tail)
    del big


# ---- over CUDA IPC -----------------------------------------------------------------------------------------------------
def _table_worker(rank, world, port, extra, q):
    try:
        dev_ = _init(rank, world, port, False)
        from neutronstarlite_b200 import _lib
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        hg, _, _, _ = graph_and_data(dev_)
        Vg = hg.vertices
        off = table_offsets(hg, world)
        out = []
        for F in (3, 41, 602):
            full = torch.rand((Vg, F), generator=torch.Generator().manual_seed(F)).to(dev_)
            t = ShardedFeatureTable(full[off[rank]:off[rank + 1]].clone(), off, dtype=torch.bfloat16)
            ids = torch.from_numpy(np.random.default_rng(rank).integers(0, Vg, 20000)).to(dev_)
            ids[:len(off)] = torch.tensor([min(o, Vg - 1) for o in off], device=dev_)
            got16, got32 = t.gather(ids), t.gather(ids, dtype=torch.float32)
            torch.cuda.synchronize()
            assert torch.equal(got16, full[ids].to(torch.bfloat16)), "F=%d" % F
            assert torch.equal(got32, full[ids].to(torch.bfloat16).float()), "F=%d" % F
            out.append(int(((ids < off[rank]) | (ids >= off[rank + 1])).sum()))
            t.close()
        # a dtype mismatch between ranks is refused on every rank
        x = torch.rand((off[rank + 1] - off[rank], 8), device=dev_)
        try:
            ShardedFeatureTable(x, off, dtype=torch.bfloat16 if rank == 0 else torch.float32)
            raise AssertionError("a dtype mismatch was accepted")
        except _lib.NtsError as exc:
            assert "dtype" in str(exc)
        q.put((rank, "ok", out))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_bf16_table_over_ipc_with_ranks_sharing_one_gpu(world):
    dev()
    remote = spawn(_table_worker, world, 29660 + world, None)
    assert all(r > 0 for rr in remote for r in rr)


# ---- world 1 -------------------------------------------------------------------------------------------------------------
def test_world_1_bf16_table_equals_bf16_tensor_features_on_cora():
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges, graph
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    d = dev()
    pg = graph(cora_edges(), 2708)
    feats, labels, masks = cora_tables()
    x = torch.from_numpy(feats).to(d)
    table = ShardedFeatureTable(x, [0, 2708], dtype=torch.bfloat16)
    lab, msk = torch.from_numpy(labels).to(d), torch.from_numpy(masks)
    try:
        runs = []
        for features in (x, table):
            m = GCNSampleImpl(pg, [1433, 128, 7], features, lab, msk, fanout=[5, 10], batch_size=64, drop_rate=0.0,
                              seed=0, sample_seed=0, gather_dtype=torch.bfloat16)
            res = [m.run_epoch(test=True) for _ in range(2)]
            runs.append((res, m.step, [p.W.detach().clone() for p in m.P]))
        (ra, sa, wa), (rb, sb, wb) = runs
        assert ra == rb and sa == sb
        for a, b in zip(wa, wb):
            assert torch.equal(a, b)
        runs = []
        for features in (x.to(torch.bfloat16).float(), table):
            m = GATSampleImpl(pg, [1433, 64, 7], features, lab, msk, fanout=[5, 10], batch_size=64, heads=8, seed=0,
                              sample_seed=0)
            res = [m.run_epoch(test=True) for _ in range(2)]
            runs.append((res, m.step, [p.W.detach().clone() for p in m.params()]))
        (ra, sa, wa), (rb, sb, wb) = runs
        assert ra == rb and sa == sb
        for a, b in zip(wa, wb):
            assert torch.equal(a, b)
    finally:
        table.close()


# ---- one data-parallel round ------------------------------------------------------------------------------------------
def make_model(kind, pg, features, labels, mask, dev_):
    from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl
    kw = dict(fanout=[8, 12], batch_size=BATCH, seed=5, sample_seed=9)
    if kind == "gcn":
        return GCNSampleImpl(pg, MODELS[kind], features, labels.to(dev_), mask, drop_rate=0.0,
                             gather_dtype=torch.bfloat16, **kw)
    return GATSampleImpl(pg, MODELS[kind], features, labels.to(dev_), mask, heads=GAT_HEADS, **kw)


def _round_worker(rank, world, port, per_gpu, q):
    try:
        dev_ = _init(rank, world, port, per_gpu)
        from neutronstarlite_b200.feature_table import ShardedFeatureTable
        hg, pg, feats, labels = graph_and_data(dev_)
        off = table_offsets(hg, world)
        table = ShardedFeatureTable(feats[off[rank]:off[rank + 1]].to(dev_), off, dtype=torch.bfloat16)
        out = {}
        for kind in MODELS:
            for n_batches in (world, world - 1):
                n_train = n_batches * BATCH - (7 if n_batches == world else 0)
                m = make_model(kind, pg, table, labels, round_mask(hg.vertices, n_train), dev_)
                loss, acc = m.run_epoch(test=True)
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


def check_round_bf16(kind, n_batches, ranks, d):
    """check_round of test_dist_sample_gpu at the rounded operands: GCN through the BF16-gather restatement, GAT through
    its float64 step on the BF16-rounded features."""
    import test_gat_sample_gpu as gat_ref
    from test_minibatch_bf16_gpu import float64_step_bf16
    hg, pg, feats, labels = graph_and_data(d)
    n_train = n_batches * BATCH - (7 if n_batches == len(ranks) else 0)
    mask = round_mask(hg.vertices, n_train)
    ref = make_model(kind, pg, feats.to(d), labels, mask, d)
    W0 = [p.W.detach().double() for p in ref.params()]
    ids = ref.nids[0]
    grads = [torch.zeros_like(w) for w in W0]
    f16 = feats.to(torch.bfloat16).float().to(d)
    for b in range(n_batches):
        sg = ref.sampler.sample(ids[b * BATCH:(b + 1) * BATCH], ref.sample_seed, b)
        blocks = [blk.to_numpy() for blk in sg.blocks]
        if kind == "gcn":
            _, gs = float64_step_bf16(blocks, feats.to(d), labels.to(d), W0)
        else:
            _, gs = gat_ref.float64_step(blocks, f16, labels.to(d), W0, ref.heads, MODELS[kind])
        grads = [a + g for a, g in zip(grads, gs)]
    r0 = ranks[0][(kind, n_batches)]
    for r in ranks[1:]:
        loss, acc, step, Ws, _ = r[(kind, n_batches)]
        assert loss == r0[0] and acc == r0[1] and step == r0[2]
        for a, b in zip(Ws, r0[3]):
            assert np.array_equal(a, b)
    _, _, _, Ws, Gs = r0
    for W, G, w0, g in zip(Ws, Gs, W0, grads):
        W, G, g = torch.from_numpy(W).double(), torch.from_numpy(G).double(), g.cpu()
        scale = g.abs().amax(1, keepdim=True).clamp_min(1e-30)
        assert ((G - g).abs() <= 1e-4 * scale).all(), kind
        W_ref, W_g = adam_first_step(w0.cpu(), g)
        sure = W_g.abs() > 1e-3 * W_g.abs().max()
        err = ((W - W_ref).abs() * sure).amax(1)
        assert (err <= 1e-4 * W_ref.abs().amax(1)).all(), kind


def run_round_test(world, per_gpu, port):
    ranks = spawn(_round_worker, world, port, per_gpu)
    d = torch.device("cuda:0")
    for kind in MODELS:
        for n_batches in (world, world - 1):
            check_round_bf16(kind, n_batches, ranks, d)


@pytest.mark.parametrize("world", [2, 3])
def test_one_bf16_round_on_ranks_sharing_one_gpu_matches_float64(world):
    dev()
    run_round_test(world, False, 29670 + world)


def test_one_bf16_round_with_one_rank_per_gpu_matches_float64():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    run_round_test(2, True, 29680)
