"""The passes around the planned gather (csrc/nts_plan.cu) that do no aggregation work, and what replaces them:

  * overwrite runs (nts_gather_plan_run_ex / _run_bf16_ex with NTS_PLAN_OVERWRITE, GatherPlan.run(accumulate=False)):
    out = A x into an output that may hold anything, instead of a zero fill followed by out += A x.  The hub column
    block stores its tiles; plans without hub columns zero the output inside the run.
  * row-pitched inputs: x[:, :F] of a [V, ld] tensor is gathered in place when ld % 4 == 0 (FP32) and its storage runs
    to the last row's ld-th value, else through the padded copy; the pad columns never reach an output.

Exactness: the comparisons of two modes use integer features and weights in quarters, so every partial sum is exact
in FP32 (and every feature exact in BF16) and the order in which split partials reach an output (`red` flushes) cannot
change a bit; overwrite and accumulate-into-zeros then agree with `==` (only the sign of a zero may differ)."""
import ctypes as C

import numpy as np
import pytest

from test_gather_plan_hubs import agg_close, dev, hub_graph, make_plan, row_close

torch = pytest.importorskip("torch")

WIDTHS = [1, 2, 3, 4, 5, 6, 7, 8, 41, 128, 602]


def exact_graph(rng, n_rows=700, n_src=900):
    off, idx, w = hub_graph(rng, n_rows, n_src)
    w = (rng.integers(1, 5, w.shape[0]) / 4).astype(np.float32)
    return off, idx, w


def exact_features(rng, n, F):
    return rng.integers(-8, 9, (n, F)).astype(np.float32)


def run_mode(plan, x, bf16, accumulate):
    out = torch.full((plan.n_rows, x.shape[1]), float("nan") if not accumulate else 0.0, dtype=torch.float32,
                     device=dev())
    plan.run(x, out, gather_dtype=torch.bfloat16 if bf16 else None, accumulate=accumulate)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_same(a, b):
    assert not np.isnan(a).any() and not np.isnan(b).any()
    assert np.array_equal(a, b), "max |diff| %g" % np.abs(a - b).max()


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("hubs", [(0, 0), (0, 32), (64, 0), (64, 32)])
@pytest.mark.parametrize("slabs", [1, 3, 16])
@pytest.mark.parametrize("bf16", [False, True])
def test_overwrite_matches_accumulate_into_zeros(bf16, slabs, hubs, overlap):
    """Output pre-filled with NaN: no NaN survives, and the result is what accumulating into zeros gives."""
    rng = np.random.default_rng(1000 + 100 * slabs + hubs[0] + hubs[1] + 7 * overlap + bf16)
    off, idx, w = exact_graph(rng)
    plan = make_plan(off, idx, w, 0, 900, slabs, hubs)
    assert (plan.slabs, plan.hub_cols, plan.hub_rows) == (slabs,) + hubs
    plan.set_overlap(overlap)
    for F in WIDTHS:
        x = torch.from_numpy(exact_features(rng, 900, F)).to(dev())
        assert_same(run_mode(plan, x, bf16, accumulate=False), run_mode(plan, x, bf16, accumulate=True))


@pytest.mark.gpu
@pytest.mark.parametrize("hubs", [(0, 0), (64, 32)])
def test_overwrite_against_oracle(hubs):
    """Random FP32 features and weights, overwrite run into NaN against the C oracle of the reference's loop."""
    rng = np.random.default_rng(77 + hubs[0])
    off, idx, w = hub_graph(rng)
    plan = make_plan(off, idx, w, 0, 900, 3, hubs)
    for F in (3, 41, 602):
        X = rng.uniform(-1, 1, (900, F)).astype(np.float32)
        agg_close(run_mode(plan, torch.from_numpy(X).to(dev()), False, accumulate=False), off, idx, w, X)


@pytest.mark.gpu
def test_overwrite_of_a_plan_without_edges_zeroes_the_output():
    from neutronstarlite_b200 import ops
    from test_gather_plan_hubs import up_u32
    plan = ops.GatherPlan(up_u32(np.zeros(11, dtype=np.uint32)), None, None, 0, 10, 0, 5, 2)
    x = torch.ones((5, 6), dtype=torch.float32, device=dev())
    for bf16 in (False, True):
        assert np.array_equal(run_mode(plan, x, bf16, accumulate=False), np.zeros((10, 6), dtype=np.float32))


def pitched(X, ld, pad_value=float("nan")):
    """X as the [:, :F] view of a [V, ld] tensor whose pad columns hold pad_value."""
    n, F = X.shape
    buf = torch.full((n, ld), pad_value, dtype=torch.float32, device=dev())
    buf[:, :F] = torch.from_numpy(X).to(dev())
    return buf[:, :F]


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("F,ld", [(602, 608), (602, 604), (41, 44), (41, 48)])
def test_row_pitched_input_matches_contiguous(F, ld, overlap):
    """NaN in the pad columns: the in-place gather (FP32) and the BF16 conversion read them, no output sees them."""
    rng = np.random.default_rng(F + ld)
    off, idx, w = exact_graph(rng)
    plan = make_plan(off, idx, w, 0, 900, 3, (64, 32))
    plan.set_overlap(overlap)
    X = exact_features(rng, 900, F)
    xp = pitched(X, ld)
    assert not xp.is_contiguous() and xp.stride(0) == ld
    xc = torch.from_numpy(X).to(dev())
    for bf16 in (False, True):
        for accumulate in (False, True):
            assert_same(run_mode(plan, xp, bf16, accumulate), run_mode(plan, xc, bf16, accumulate))


@pytest.mark.gpu
def test_row_pitched_input_against_oracle():
    rng = np.random.default_rng(5)
    off, idx, w = hub_graph(rng)
    plan = make_plan(off, idx, w, 0, 900, 3, (64, 32))
    for F, ld in ((602, 604), (41, 44), (5, 8)):
        X = rng.uniform(-1, 1, (900, F)).astype(np.float32)
        agg_close(run_mode(plan, pitched(X, ld), False, accumulate=False), off, idx, w, X)


@pytest.mark.gpu
def test_pitched_view_without_storage_for_the_last_pad_takes_the_padded_copy():
    """torch.empty_strided((V, 602), (608, 1)) ends at the last row's 602nd value: reading that row to 608 would leave
    the allocation, so the run gathers through the padded copy (the plan's workspace appears) with the same result;
    a view with the storage behind it is gathered in place (no workspace)."""
    rng = np.random.default_rng(9)
    off, idx, w = exact_graph(rng)
    X = exact_features(rng, 900, 602)
    ref_plan = make_plan(off, idx, w, 0, 900, 3, (64, 32))
    ref = run_mode(ref_plan, torch.from_numpy(X).to(dev()), False, accumulate=False)

    short = torch.empty_strided((900, 602), (608, 1), dtype=torch.float32, device=dev())
    assert short.untyped_storage().nbytes() == (899 * 608 + 602) * 4
    short.as_strided((short.untyped_storage().nbytes() // 4,), (1,)).fill_(float("nan"))
    short.copy_(torch.from_numpy(X))
    plan = make_plan(off, idx, w, 0, 900, 3, (64, 32))
    before = plan.bytes()
    for accumulate in (False, True):
        assert_same(run_mode(plan, short, False, accumulate), ref if not accumulate else
                    run_mode(ref_plan, torch.from_numpy(X).to(dev()), False, True))
    assert plan.bytes() - before == 900 * 604 * 4

    inplace = make_plan(off, idx, w, 0, 900, 3, (64, 32))
    before = inplace.bytes()
    assert_same(run_mode(inplace, pitched(X, 608), False, accumulate=False), ref)
    assert inplace.bytes() == before


class _AccumulatingSingleGPUOp:
    """The single-GPU aggregation with the previous semantics: contiguous input, zero-filled outputs, accumulating
    runs (not a ForwardSingleGPUfuseOp subclass, so GCNImpl keeps X[0] contiguous for it)."""

    def __init__(self, partitioned_graph, active=None):
        self.pg = partitioned_graph

    def forward(self, x, f_input1=None):
        from neutronstarlite_b200 import ops
        c = self.pg.graph_chunks[0]
        y = torch.zeros((c.batch_size_forward, x.shape[1]), dtype=torch.float32, device=x.device)
        return ops.gather_by_dst_from_src(c, y, x.contiguous())

    def backward(self, g):
        from neutronstarlite_b200 import ops
        c = self.pg.graph_chunks[0]
        dx = torch.zeros((c.batch_size_backward, g.shape[1]), dtype=torch.float32, device=g.device)
        return ops.gather_by_src_from_dst(c, dx, g.contiguous())


def zipf_edges(rng, V, E):
    src = np.minimum(rng.zipf(1.5, E) - 1, V - 1)
    dst = np.minimum(rng.zipf(1.5, E) - 1, V - 1)
    e = np.stack([rng.permutation(V)[src], rng.permutation(V)[dst]], 1)
    return np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1)]).astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("F0", [602, 41])
def test_gcn_epochs_match_the_accumulating_contiguous_op(F0):
    """GCNImpl with its row-pitched X[0] and overwriting runs against the same model on the previous semantics, on
    measured plans (forced on for this small graph): loss and last-layer rows within 1e-5 of each row's magnitude."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    from neutronstarlite_b200.toolkits import GCNImpl
    d = dev()
    rng = np.random.default_rng(F0)
    V = 4000
    layers = [F0, 64, 41]
    pg = PartitionedGraph(HostGraph(zipf_edges(rng, V, 120000), V), 1, 0).generate_all(device=d, dist=True)
    gen = torch.Generator().manual_seed(1)
    feats = (torch.rand((V, F0), generator=gen) * 2 - 1).to(d)
    labels = torch.randint(0, layers[-1], (V,), generator=gen).to(d)
    mask = (torch.arange(V) % 3).to(d)
    mode = (ops._plan_mode, ops._plan_slabs)
    ops.set_plan_mode("on")
    try:
        new = GCNImpl(pg, layers, feats, labels, mask, drop_rate=0.0)
        old = GCNImpl(pg, layers, feats, labels, mask, drop_rate=0.0, op_class=_AccumulatingSingleGPUOp)
        x0 = new.X[0]
        assert x0.data_ptr() != feats.data_ptr() and x0.stride() == ((F0 + 3) // 4 * 4, 1)
        assert torch.equal(x0, feats) and old.X[0].is_contiguous()
        for _ in range(3):
            loss_new, _ = new.run_epoch()
            loss_old, _ = old.run_epoch()
            torch.testing.assert_close(loss_new, loss_old, rtol=1e-5, atol=0)
            row_close(new.X[-1].detach().cpu().numpy(), old.X[-1].detach().cpu().numpy(), rtol=1e-5)
        assert new.X[0] is x0
    finally:
        ops.set_plan_mode(*mode)


def test_run_ex_rejects_a_pitch_below_the_width_and_a_null_output():
    """Argument checks of the new entries, before any device work (no GPU needed)."""
    from neutronstarlite_b200 import _lib
    L = _lib.load()
    out = C.c_void_p(16)   # never dereferenced: the checks fail first
    for name, args in (("nts_gather_plan_run_ex", lambda ld, o: (None, None, ld, o, 602, 1, None)),
                       ("nts_gather_plan_run_bf16_ex", lambda ld, o: (None, None, 0, ld, o, 602, 1, None))):
        fn = getattr(L, name)
        assert fn(*args(600, out)) != 0
        assert b"pitch" in L.nts_last_error()
        assert fn(*args(608, None)) != 0
        assert b"null output" in L.nts_last_error()
        assert fn(*args(608, out)) != 0
        assert b"null plan" in L.nts_last_error()
    assert L.nts_gather_plan_create_tuned_ex(None, None, None, None, 0, 1, 1, 1, 8, 0, 2, None) is None
    assert b"run_flags" in L.nts_last_error()


def test_ops_accept_row_pitched_views_only_where_the_pitch_is_passed_on():
    from neutronstarlite_b200 import _lib, ops
    buf = torch.zeros((6, 8))
    assert ops.row_pitched(buf[:, :5]) and ops.row_pitched(buf)
    assert not ops.row_pitched(buf.t()) and not ops.row_pitched(buf[:, ::2])
    with pytest.raises(_lib.NtsError):
        ops._check_input(torch.zeros(4, 4)[:, :3], pitched=True)    # CPU tensors stay refused
