"""Sampled GCN with BF16 gathers: K1 on BF16 rows (segment_gather_sum_kernel, head mode 0, T = __nv_bfloat16, through
nts_segment_gather_sum_bf16), ops.MiniBatchFuseOp(gather_dtype=torch.bfloat16) and
toolkits.GCNSampleImpl(gather_dtype=torch.bfloat16), against float64.

K1-BF16 runs at every NTS_BF16_CASE point of `K1_BF16_CASES` on the structured graph of test_gat_fp32_reference cut to
E % 4 = 0..3 edges (empty rows, hub rows of 4 096 to 20 011 edges), by local ids into the sources' rows and by global
id into a table with more rows than sources, with both index-staging variants:
  * exact mode: integer features in [-8, 8], weights in quarters, integer init; every partial sum is exact in FP32, and
    the features are exact in BF16, so the output must equal init + A X in float64 (torch.equal);
  * random mode: per element |y - y64| <= 1e-4 (|init| + |A| |X|), y64 taken at X.to(bfloat16).
A virtual-warp point (G > 1) exists under the bulk-staged variant only; the shuffle variant runs the same width at
G = 1.  Every launch asserts the point (nts_aggregate_last_shape) and the grid and shared memory, which show G."""
import ctypes as C
import os

import numpy as np
import pytest

from test_aggregate_reference import (check_exact, check_random, exact_inputs, hooks, random_inputs, reference,
                                      sm_count, trimmed)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

RTOL = 1e-4


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream().cuda_stream


def cdiv(a, b):
    return -(-a // b)


# ---- the dispatch, mirrored ------------------------------------------------------------------------------------------
def bf16_point(F, variant=2, tune=None):
    """((K, U, MINB, G), tiles) that segment_gather_sum_bf16 picks for F output columns under staging variant
    `variant` (1 shuffle, 2 bulk) and NTS_K1_BF16_TUNE = tune (U, MINB, G)."""
    nvec = cdiv(F, 8)
    tiles = cdiv(cdiv(nvec, 32), 4)
    tv = cdiv(nvec, tiles)
    k = cdiv(tv, 32)
    tiles = cdiv(nvec, tv)
    narrow = variant != 1 and k == 1 and tiles == 1
    g = 2 if narrow and nvec <= 16 else 1
    u = 4 if k <= 3 else 2
    minb = 1 if k == 4 else 2
    if tune is not None:
        u, minb = tune[0], tune[1]
        if narrow and tune[2] >= 1 and 32 // tune[2] >= nvec:
            g = tune[2]
    return (k, u, minb, g), tiles


def bf16_launch(n_edges, tiles, g, variant, Q=0, sms=None):
    """(grid, smem) of a K1-BF16 launch over n_edges edges (nts_aggregate_set_variant(variant, Q))."""
    if Q == 0:
        Q = 512 // g
        while Q > 32 and cdiv(n_edges, Q) * tiles < sms * 64:
            Q >>= 1
    Q = cdiv(Q, 32) * 32
    if g > 1 and Q * g > 1024:
        Q = (1024 // g) // 32 * 32
    grid = cdiv(cdiv(n_edges, Q) * tiles, 8 * g)
    return grid, (16 + 2 * (8 * g * Q + 8) * 4) if variant != 1 else 0


# (K, U, MINB, G), F, NTS_K1_BF16_TUNE (U, MINB, G).  F = 41 / 37 are 6 / 5 chunks, 128 is 16, 602 is 76.
K1_BF16_CASES = [
    # default points
    ((1, 4, 2, 2), 41, None),
    ((1, 4, 2, 1), 200, None),
    ((2, 4, 2, 1), 400, None),
    ((3, 4, 2, 1), 602, None),
    ((4, 2, 1, 1), 1000, None),
    # NTS_K1_BF16_TUNE points
    ((1, 4, 4, 4), 41, (4, 4, 4)),
    ((1, 4, 4, 2), 128, (4, 4, 2)),
    ((1, 4, 4, 1), 200, (4, 4, 1)),
    ((1, 2, 4, 4), 37, (2, 4, 4)),
    ((1, 8, 2, 4), 64, (8, 2, 4)),
    ((1, 4, 2, 4), 8, (4, 2, 4)),
    ((1, 2, 4, 2), 100, (2, 4, 2)),
    ((1, 8, 2, 2), 128, (8, 2, 2)),
    ((3, 2, 2, 1), 602, (2, 2, 1)),
    ((3, 2, 1, 1), 520, (2, 1, 1)),
    ((3, 4, 1, 1), 700, (4, 1, 1)),
]


def last_k1():
    from neutronstarlite_b200 import _lib
    rec = [C.c_int() for _ in range(4)]
    _lib.call("nts_aggregate_last_launch", *[C.byref(r) for r in rec])
    shape = [C.c_int() for _ in range(5)]
    _lib.call("nts_aggregate_last_shape", *[C.byref(r) for r in shape])
    return tuple(r.value for r in rec), tuple(r.value for r in shape)


def bf16_rows(X, ld):
    """X (float32 [n, F]) rounded to BF16 as [n, ld] rows whose pad columns hold NaN (never to be added)."""
    r = torch.full((X.shape[0], ld), float("nan"), dtype=torch.bfloat16, device=X.device)
    r[:, :X.shape[1]] = X.to(torch.bfloat16)
    return r


def run_bf16(rows, ld, out, w, idx, off, n_rows, n_edges, F, variant, Q=0):
    from neutronstarlite_b200 import _lib
    _lib.call("nts_aggregate_set_variant", variant, Q)
    _lib.call("nts_segment_gather_sum_bf16", rows.data_ptr(), ld, out.data_ptr(), None if w is None else w.data_ptr(),
              idx.data_ptr(), off.data_ptr(), n_rows, n_edges, F, stream())
    torch.cuda.synchronize()
    return out, last_k1()


def operands(g, X, addr, extra_rows=1000):
    """(rows X', indices) of an addressing mode: 'local' reads the sources' own rows by slot (mi[id]), 'global' reads a
    table of Vg + extra_rows rows by global id."""
    d = dev()
    a = g.device()
    if addr == "local":
        Xl = torch.from_numpy(X).to(d)[torch.from_numpy(g.ids).to(d)].contiguous()
        return Xl, torch.from_numpy(g.mi[g.idx].astype(np.int64).astype(np.uint32).view(np.int32)).to(d)
    T = torch.from_numpy(np.concatenate([X, np.full((extra_rows, X.shape[1]), 3.0, np.float32)])).to(d)
    return T, a["idx"]


@pytest.mark.parametrize("case", range(len(K1_BF16_CASES)), ids=["k%du%db%dg%d" % c[0] for c in K1_BF16_CASES])
def test_every_bf16_point_exact_and_random(case, monkeypatch):
    point, F, tune = K1_BF16_CASES[case]
    g = trimmed(case % 4)
    a = g.device()
    sms = sm_count()
    if tune is not None:
        monkeypatch.setenv("NTS_K1_BF16_TUNE", "%d,%d,%d" % tune)
    want, tiles = bf16_point(F, 2, tune)
    assert want == point
    ld = cdiv(F, 8) * 8 + (8 if case % 3 == 0 else 0)       # some rows with a pitch past 8*ceil(F/8)
    with hooks():
        for mode, make in (("exact", exact_inputs), ("random", random_inputs)):
            X, w, init = make(g, F, seed=700 + case)
            d = dev()
            Xb = torch.from_numpy(X).to(d).to(torch.bfloat16).float()
            wd, initd = torch.from_numpy(w).to(d), torch.from_numpy(init).to(d)
            unweighted = mode == "random" and case % 2 == 1
            ref, mag = reference(a["dst64"], a["src64"], None if unweighted else wd, Xb, initd)
            ops = {addr: operands(g, X, addr) for addr in ("local", "global")}
            ops = {addr: (bf16_rows(rows, ld), idx) for addr, (rows, idx) in ops.items()}
            for variant in (1, 2):
                # a virtual-warp point runs under the bulk variant; the shuffle variant runs its width at G = 1,
                # without the tuning hook (whose U and MINB need not exist at G = 1)
                vtune = tune if (variant == 2 or point[3] == 1) else None
                if vtune is None:
                    monkeypatch.delenv("NTS_K1_BF16_TUNE", raising=False)
                else:
                    monkeypatch.setenv("NTS_K1_BF16_TUNE", "%d,%d,%d" % vtune)
                vpoint, vt = bf16_point(F, variant, vtune)
                assert variant == 1 or vpoint == point
                for addr, (rows, idx) in ops.items():
                    for Q in (0, 64):
                        out, (rec, shape) = run_bf16(rows, ld, initd.clone(), None if unweighted else wd, idx,
                                                     a["off"], g.n_rows, g.E, F, variant, Q)
                        assert shape == (8, vpoint[0], vpoint[1], vpoint[2], vt), (variant, addr, shape, vpoint)
                        assert rec[3] == variant and rec[1] == 256
                        assert (rec[0], rec[2]) == bf16_launch(g.E, vt, vpoint[3], variant, Q, sms), (variant, Q, rec)
                        if mode == "exact":
                            check_exact(out, ref)
                        else:
                            check_random(out, ref, mag, RTOL)


def test_refusals_and_empty_launches():
    """An unpadded pitch, ld < F and a misaligned input are refused before any launch; n_rows = 0 and n_edges = 0
    launch nothing (even with null pointers)."""
    from neutronstarlite_b200 import _lib
    d = dev()
    L = _lib.load()
    g = trimmed(0)
    a = g.device()
    out = torch.zeros((g.n_rows, 41), device=d)
    rows = torch.zeros((g.Vg + 1, 48), dtype=torch.bfloat16, device=d)
    args = lambda x, ld, F: (x, ld, out.data_ptr(), None, a["idx"].data_ptr(), a["off"].data_ptr(), g.n_rows, g.E, F,
                             stream())
    n0 = L.nts_kernel_launch_count()
    assert L.nts_segment_gather_sum_bf16(*args(rows.data_ptr(), 41, 41)) != 0
    assert b"input_ld" in L.nts_last_error()
    assert L.nts_segment_gather_sum_bf16(*args(rows.data_ptr(), 40, 41)) != 0
    assert L.nts_segment_gather_sum_bf16(*args(rows.data_ptr() + 2, 48, 41)) != 0
    assert b"aligned" in L.nts_last_error()
    assert L.nts_segment_gather_sum_bf16(None, 48, None, None, None, None, 0, 100, 41, None) == 0
    assert L.nts_segment_gather_sum_bf16(None, 48, None, None, None, None, 10, 0, 41, None) == 0
    assert L.nts_kernel_launch_count() == n0
    from neutronstarlite_b200 import ops
    with pytest.raises(_lib.NtsError, match="pitch"):
        ops._check_bf16_operand(torch.zeros((10, 41), dtype=torch.bfloat16, device=d), "input")
    with pytest.raises(_lib.NtsError, match="pitch"):
        ops._check_bf16_operand(torch.zeros((10, 49), dtype=torch.bfloat16, device=d)[:, 1:], "input")


# ---- MiniBatchFuseOp ------------------------------------------------------------------------------------------------
def hub_graph():
    import golden_store
    z = golden_store.load("synth9k_P3_F2.npz")
    return z["edges"], int(z["case"][0])


def block_float64(b, h, transposed=False):
    """float64 A h (or A^T h) of one block (numpy arrays of SampledBlock.to_numpy), on h's device."""
    t = {k: torch.from_numpy(v.astype(np.int64) if v.dtype == np.uint32 else v).to(h.device) for k, v in b.items()}
    if not transposed:
        n = t["column_offset"].numel() - 1
        dst = torch.repeat_interleave(torch.arange(n, device=h.device), t["column_offset"].diff())
        src, w = t["row_indices"], t["weight"]
    else:
        n = t["row_offset"].numel() - 1
        dst = torch.repeat_interleave(torch.arange(n, device=h.device), t["row_offset"].diff())
        src, w = t["column_indices"], t["weight_backward"]
    y = torch.zeros((n, h.shape[1]), dtype=torch.float64, device=h.device)
    return y.index_add(0, dst, h[src] * w.double()[:, None])


def rnd(t):
    return t.to(torch.bfloat16).double()


@pytest.mark.parametrize("graph_name", ["cora", "hub9k"])
def test_minibatch_op_bf16_forward_backward_against_float64(graph_name):
    """Forward from a BF16 tensor, an FP32 tensor and the [V, F] table (table=True); backward with dY rounded once.
    Per element within 1e-4 (|A| |bf16(X)|) of float64 at the rounded operands."""
    from test_sample_gpu import cora_edges, graph
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    edges, V = (cora_edges(), 2708) if graph_name == "cora" else hub_graph()
    pg = graph(edges, V)
    sg = NeighborSampler(pg, [10, 25], 256).sample(np.arange(0, V, max(1, V // 256))[:256], 3, 1)
    gen = torch.Generator().manual_seed(5)
    for F in (41, 128, 37):
        table = (torch.rand((V, F), generator=gen) * 2 - 1).to(d)
        ld = cdiv(F, 8) * 8
        t16 = torch.zeros((V, ld), dtype=torch.bfloat16, device=d)
        t16[:, :F] = table.to(torch.bfloat16)
        for hop in (1, 0):
            b = sg.blocks[hop]
            bn = b.to_numpy()
            src = b.src.long()
            x32 = table[src].contiguous()
            x16 = t16[src][:, :F]
            ref = block_float64(bn, rnd(x32))
            mag = block_float64({**bn, "weight": np.abs(bn["weight"])}, rnd(x32).abs())
            inputs = [("fp32", x32, False), ("bf16", x16, False)] + ([("table", t16[:, :F], True)] if hop == 1 else [])
            for name, x, table_mode in inputs:
                op = ops.MiniBatchFuseOp(sg, hop, table=table_mode, gather_dtype=torch.bfloat16)
                y = op.forward(x)
                torch.cuda.synchronize()
                assert y.dtype == torch.float32 and y.shape == (b.n_dst, F)
                check_random(y, ref, mag, RTOL)
            op = ops.MiniBatchFuseOp(sg, hop, gather_dtype=torch.bfloat16)
            op.forward(x32)
            dy = (torch.rand((b.n_dst, F), generator=gen) * 2 - 1).to(d)
            dx = op.backward(dy)
            ref_b = block_float64(bn, rnd(dy), transposed=True)
            mag_b = block_float64({**bn, "weight_backward": np.abs(bn["weight_backward"])}, rnd(dy).abs(),
                                  transposed=True)
            assert dx.dtype == torch.float32 and dx.shape == (b.n_src, F)
            check_random(dx, ref_b, mag_b, RTOL)


def test_minibatch_op_bf16_refuses_before_device_work():
    from test_sample_gpu import cora_edges, graph
    from neutronstarlite_b200 import _lib, ops
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    pg = graph(cora_edges(), 2708)
    sg = NeighborSampler(pg, [5, 5], 64).sample(np.arange(64), 0, 0)
    with pytest.raises(_lib.NtsError, match="gather_dtype"):
        ops.MiniBatchFuseOp(sg, 0, gather_dtype=torch.float16)
    op = ops.MiniBatchFuseOp(sg, 0, gather_dtype=torch.bfloat16)
    n = sg.blocks[0].n_src
    with pytest.raises(_lib.NtsError, match="pitch"):
        op.forward(torch.zeros((n, 41), dtype=torch.bfloat16, device=d))
    with pytest.raises(_lib.NtsError, match="rows"):
        op.forward(torch.zeros((n + 1, 48), dtype=torch.bfloat16, device=d))
    with pytest.raises(_lib.NtsError):
        op.forward(torch.zeros((n, 48), dtype=torch.float16, device=d))


# ---- GCNSampleImpl ----------------------------------------------------------------------------------------------------
class _AggBF16(torch.autograd.Function):
    """float64 A bf16(h) forward, A^T bf16(dY) backward: the BF16 gathers of one sampled layer."""

    @staticmethod
    def forward(ctx, h, b):
        ctx.b = b
        return block_float64(b, rnd(h))

    @staticmethod
    def backward(ctx, g):
        return block_float64(ctx.b, rnd(g), transposed=True), None


def float64_step_bf16(blocks, table, labels, Ws):
    """One GCNSampleImpl(gather_dtype=bf16) step in float64: every aggregation gathers bf16 of its operand (the table
    rows, the activations, dY), weights and the rest in float64.  Returns the loss and the weight gradients."""
    Wd = [W.detach().double().requires_grad_(True) for W in Ws]
    L = len(Wd)
    h = table.double()
    for l in range(L):
        b = blocks[L - 1 - l]
        if l == 0:          # the first layer reads the table by global id
            b = {**b, "row_indices": b["row_global"]}
        h = _AggBF16.apply(h, b) @ Wd[l]
        if l < L - 1:
            h = torch.relu(h)
    seeds = torch.from_numpy(blocks[0]["dst"].astype(np.int64)).to(h.device)
    loss = torch.nn.functional.nll_loss(h.log_softmax(1), labels[seeds])
    loss.backward()
    return loss.detach(), [W.grad for W in Wd]


def test_gcn_sample_bf16_three_steps_match_float64():
    from test_sample_gpu import graph, zipf_hub_edges
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    edges, V = zipf_hub_edges(V=5000, E=60000)
    pg = graph(edges, V)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, 37), generator=gen) * 2 - 1).to(d)
    keep = feats.clone()
    labels = torch.randint(0, 5, (V,), generator=gen).to(d)
    mask = torch.arange(V) % 3
    model = GCNSampleImpl(pg, [37, 16, 5], feats, labels, mask, fanout=[8, 12], batch_size=128, drop_rate=0.0,
                          gather_dtype=torch.bfloat16)
    assert torch.equal(feats, keep)
    ids = model.nids[0]
    for step in range(3):
        Ws = [p.W.detach().clone() for p in model.P]
        loss, _ = model.train_step(ids[step * 128:(step + 1) * 128])
        blocks = [b.to_numpy() for b in model.subgraph.blocks]
        ref_loss, ref_grads = float64_step_bf16(blocks, feats, labels, Ws)
        torch.testing.assert_close(loss.double(), ref_loss, rtol=1e-5, atol=0)
        for p, g, W0 in zip(model.P, ref_grads, Ws):
            scale = float(g.abs().max())
            torch.testing.assert_close(p.W_gradient.double(), g, rtol=1e-4, atol=1e-4 * scale)


def cora_run(gather_dtype, epochs, drop_rate=0.5, test=False):
    from test_gather_plan_bf16 import cora_tables
    from test_sample_gpu import cora_edges, graph
    from neutronstarlite_b200.toolkits import GCNSampleImpl
    d = dev()
    pg = graph(cora_edges(), 2708)
    feats, labels, masks = cora_tables()
    torch.manual_seed(0)
    m = GCNSampleImpl(pg, [1433, 128, 7], torch.from_numpy(feats).to(d), torch.from_numpy(labels).to(d),
                      torch.from_numpy(masks), fanout=[5, 10], batch_size=64, drop_rate=drop_rate, seed=0,
                      sample_seed=0, gather_dtype=gather_dtype)
    res = [m.run_epoch(test=test) for _ in range(epochs)]
    return res, [p.W.detach().clone() for p in m.P]


def test_gcn_sample_bf16_runs_are_bit_identical_on_cora():
    """Fanouts 5-10 on Cora batches: no aggregation row is cut into three or more pieces by K1's edge quanta (DESIGN.md
    §3 K8), so two runs with the same seeds give the same losses and weights bit for bit."""
    (ra, wa), (rb, wb) = cora_run(torch.bfloat16, 1), cora_run(torch.bfloat16, 1)
    assert ra == rb
    for a, b in zip(wa, wb):
        assert torch.equal(a, b)


def test_gcn_sample_bf16_accuracy_within_002_of_fp32_on_cora():
    res32, _ = cora_run(None, 20, test=True)
    res16, _ = cora_run(torch.bfloat16, 20, test=True)
    acc32, acc16 = res32[-1][1][2], res16[-1][1][2]
    assert abs(acc16 - acc32) <= 0.02, (acc32, acc16)
