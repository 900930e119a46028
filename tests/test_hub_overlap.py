"""The fused schedule of hybrid plans (nts_gather_plan_set_overlap / nts_gather_plan_overlap, csrc/nts_plan.cu): the
hub-row block's tiles run inside the slab launches (planned_slab_hub_kernel) with their split-K cut at the slab
boundaries.  Both schedules against the C oracle per row (1e-4 of the row's sum of |w| * |x|), against each other
(1e-5: only the order in which the row block's split-K partials reach a hub row changes), on FP32 and BF16 gathers."""
import ctypes as C

import numpy as np
import pytest

import oracle_c
from test_gather_plan_hubs import agg_close, csr, dev, hub_graph, make_plan, row_close, run

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

WIDTHS = [4, 41, 128, 602]


def bf16_round(X):
    return torch.from_numpy(X).to(torch.bfloat16).float().numpy()


def run_dtype(plan, X, bf16):
    x = torch.from_numpy(X).to(dev())
    out = torch.zeros((plan.n_rows, X.shape[1]), dtype=torch.float32, device=dev())
    plan.run(x, out, gather_dtype=torch.bfloat16 if bf16 else None)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def both_schedules(plan, X, bf16=False):
    plan.set_overlap(False)
    assert not plan.overlap
    seq = run_dtype(plan, X, bf16)
    plan.set_overlap(True)
    assert plan.overlap
    fused = run_dtype(plan, X, bf16)
    return seq, fused


def last_launch(plan):
    from neutronstarlite_b200 import _lib
    v = [C.c_int(0) for _ in range(5)]
    _lib.call("nts_gather_plan_last_launch", plan.handle, *[C.byref(x) for x in v])
    return v[0].value, v[1].value


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("hub_cols", [0, 64])
@pytest.mark.parametrize("hub_rows", [0, 32, 200])
@pytest.mark.parametrize("slabs", [1, 3, 4])
def test_fused_and_sequential_match_oracle_and_each_other(slabs, hub_rows, hub_cols, bf16):
    """900 gathered rows: 3 and 4 slabs put the slab boundaries at rows 300 / 225, not multiples of the 16-row K tile."""
    rng = np.random.default_rng(500 + slabs * 10 + hub_rows + hub_cols + bf16)
    n_rows, n_src = 700, 900
    off, idx, w = hub_graph(rng, n_rows, n_src)
    plan = make_plan(off, idx, w, 0, n_src, slabs, (hub_cols, hub_rows))
    assert (plan.slabs, plan.hub_cols, plan.hub_rows) == (slabs, hub_cols, hub_rows)
    for F in WIDTHS:
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        Xg = bf16_round(X) if bf16 else X
        seq, fused = both_schedules(plan, X, bf16)
        agg_close(seq, off, idx, w, Xg)
        agg_close(fused, off, idx, w, Xg)
        row_close(fused, seq, rtol=1e-5, scale=oracle_c.segment_gather_sum(off, idx, w, np.abs(Xg)))


def test_slab_with_empty_residual_runs_its_row_block_tiles():
    """Gathered rows 30..59 (slab 1 of 3) feed only the hub row: slab 1 has no residual edge, its launch runs row-block
    tiles only, and the sequential schedule skips it."""
    rng = np.random.default_rng(17)
    n_rows, n_src = 50, 90
    dst, src = [np.zeros(n_src, dtype=np.int64)], [np.arange(n_src)]          # row 0: every source, the hub row
    for r in range(1, n_rows):
        s = rng.choice(np.r_[0:30, 60:90], 12)
        dst.append(np.full(12, r)), src.append(s)
    off, idx, w = csr(np.concatenate(dst), np.concatenate(src), n_rows, rng)
    plan = make_plan(off, idx, w, 0, n_src, 3, (0, 1))
    assert plan.hub_rows == 1
    for F in (41, 602):
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        plan.set_overlap(False)
        seq = run_dtype(plan, X, False)
        assert last_launch(plan)[0] == 2
        plan.set_overlap(True)
        fused = run_dtype(plan, X, False)
        launches, grid = last_launch(plan)
        assert launches == 3
        agg_close(seq, off, idx, w, X)
        agg_close(fused, off, idx, w, X)


@pytest.mark.parametrize("hubs", [(10 ** 6, 10 ** 6), (0, 10 ** 6)])
@pytest.mark.parametrize("bf16", [False, True])
def test_all_hub_plans(hubs, bf16):
    """Every gathered row a hub column and every output row a hub row, or every output row a hub row alone: no residual
    edge is left, every fused launch is GEMM-only."""
    rng = np.random.default_rng(23)
    n_rows, n_src = 300, 400
    off, idx, w = hub_graph(rng, n_rows, n_src, 20000)
    plan = make_plan(off, idx, w, 0, n_src, 3, hubs)
    for F in (4, 128, 602):
        X = rng.uniform(-1, 1, (n_src, F)).astype(np.float32)
        Xg = bf16_round(X) if bf16 else X
        seq, fused = both_schedules(plan, X, bf16)
        agg_close(seq, off, idx, w, Xg)
        agg_close(fused, off, idx, w, Xg)


def test_identity_plus_hub_rows_against_float64():
    """out = X on the non-hub rows (one edge of weight 1: exact), the hub rows a dense row of weights times X, which
    the fused row-block tiles (split-K cut at the slab boundaries) must compute to 1e-5 of the float64 product."""
    rng = np.random.default_rng(31)
    n, hubs = 600, 12
    dst = [np.arange(n)]
    src = [np.arange(n)]
    for h in range(hubs):
        dst.append(np.full(n, h)), src.append(np.arange(n))
    dst, src = np.concatenate(dst), np.concatenate(src)
    off, idx, w = csr(dst, src, n, rng)
    w[np.repeat(np.arange(n), np.diff(off.astype(np.int64))) >= hubs] = 1.0    # identity rows: weight 1
    plan = make_plan(off, idx, w, 0, n, 3, (0, hubs))
    plan.set_overlap(True)
    for F in (41, 128, 602):
        X = rng.uniform(-1, 1, (n, F)).astype(np.float32)
        y = run_dtype(plan, X, False)
        assert np.array_equal(y[hubs:], X[hubs:])
        dense = np.zeros((hubs, n), dtype=np.float64)
        rows = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
        sel = rows < hubs
        np.add.at(dense, (rows[sel], idx[sel]), w[sel].astype(np.float64))
        ref = dense @ X.astype(np.float64)
        row_close(y[:hubs], ref, rtol=1e-5, scale=np.abs(dense) @ np.abs(X.astype(np.float64)))


def test_overlap_env_forces_sequential_and_query_reports_launches(monkeypatch):
    """NTS_PLAN_OVERLAP=0 keeps measured plans sequential; the query reflects what runs: the fused schedule's slab
    launches carry the row-block tiles (a larger grid) and the sequential one does not."""
    from neutronstarlite_b200 import ops
    rng = np.random.default_rng(3)
    n_rows, n_src = 700, 900
    off, idx, w = hub_graph(rng, n_rows, n_src)
    monkeypatch.setenv("NTS_PLAN_OVERLAP", "0")
    tuned = ops.GatherPlan(torch.from_numpy(off.view(np.int32)).to(dev()), torch.from_numpy(idx.view(np.int32)).to(dev()),
                           torch.from_numpy(w).to(dev()), 0, n_rows, idx.shape[0], n_src, 0, tune_for=128)
    assert not tuned.overlap
    assert "overlap" not in tuned.key()
    plan = make_plan(off, idx, w, 0, n_src, 1, (0, 64))
    X = rng.uniform(-1, 1, (n_src, 128)).astype(np.float32)
    plan.set_overlap(False)
    run_dtype(plan, X, False)
    seq_launches, seq_grid = last_launch(plan)
    plan.set_overlap(True)
    assert plan.key() == (1, 0, 64, "overlap")
    run_dtype(plan, X, False)
    launches, grid = last_launch(plan)
    assert (launches, seq_launches) == (1, 1)
    assert grid > seq_grid
