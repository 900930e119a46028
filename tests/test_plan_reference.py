"""The planned GCN aggregation (K1P: planned_gather_sum_kernel, planned_slab_hub_kernel, planned_gather_sum_tma_kernel
and hub_block_gemm_kernel, csrc/nts_plan.cu, through nts_gather_plan_run_ex / _run_bf16_ex) against float64, at every
NTS_PLAN_CASE, NTS_PLAN_CASE_G, NTS_PLAN_FUSED_CASE and NTS_PLAN_TMA_CASE instantiation.

The references, the exact and random modes and the graph are those of test_aggregate_reference: integer features,
weights in quarters and an integer initial output make every partial sum exact in FP32 and every feature exact in BF16,
so the plan must reproduce float64 bit for bit, whatever the slab order, split K or `red` flush order.

Every point of `PLAN_CASES` runs at OUTV 4, 2 and 1 (F % 4 == 0, F = 2 mod 4, and F odd or an output view one float
into its allocation; the gathered row length, and so the point, is the same for all three).  Plain points run on plans
of 1 and 3 slabs, BF16 points from FP32 and from BF16 inputs, fused points on plans with 200 hub rows (two 128-row M
tiles) and 17 or 64 hub columns over 3 slabs.  Points that are not a default are reached with
nts_gather_plan_set_tuning(u, minb, 0).  nts_gather_plan_last_launch must report the point's (k, u, outv), the number of
launches (slabs with residual edges; fused plans also launch slabs that only carry row-block tiles) and the last
launch's grid.  `test_plan_tables_match_the_source` keeps the table equal to the macro lines of run_gather."""
import ctypes as C

import numpy as np
import pytest

from test_aggregate_reference import (BASE, cdiv, check_exact, check_random, dev, exact_inputs, hooks, random_inputs,
                                      read_source, reference, shifted, sm_count, source_cases, trimmed)

torch = pytest.importorskip("torch")

HUB_ROWS = 200


# ---- the dispatch of run_gather, mirrored ------------------------------------------------------------------------------
def plan_point(F, bf16, out_align=16, tuning=(0, 0), variant=0):
    """What run_gather picks for F columns (gathered rows padded to 4 floats or 8 BF16 values) into an output whose rows
    are out_align-byte aligned, under nts_gather_plan_set_tuning(tuning[0], tuning[1], .) and set_variant(variant)."""
    V = 8 if bf16 else 4
    ldc = cdiv(F, V)
    tiles = cdiv(cdiv(ldc, 32), 5)
    tile_vecs = cdiv(ldc, tiles)
    k = cdiv(tile_vecs, 32)
    tiles = cdiv(ldc, tile_vecs)
    outv = 4 if F % 4 == 0 and out_align % 16 == 0 else (2 if F % 2 == 0 and out_align % 8 == 0 else 1)
    g = 1 if variant == 1 else (4 if ldc <= 8 else (2 if ldc <= 16 else 1))
    if bf16:
        minb, u = (2 if k >= 4 else (3 if k >= 2 else 4)), (4 if k == 1 else 2)
    else:
        minb, u = (2 if k >= 3 else (3 if k == 2 else 4)), (2 if k == 4 else 4)
    if tuning[0]:
        u = tuning[0]
    if tuning[1]:
        minb = tuning[1]
    stages = 8 if u >= 8 else (4 if u >= 4 else 2)
    return dict(k=k, u=u, minb=minb, g=g, outv=outv, tiles=tiles, stages=stages)


def case_point(kind, p):
    """The macro arguments of the instantiation that point p runs."""
    if kind == "g":
        return (p["u"], p["minb"], p["g"])
    if kind == "plain":
        return (p["k"], p["u"], p["minb"])
    if kind == "fused":
        return (p["k"], p["u"], p["minb"], p["g"])
    return (p["k"], p["stages"], p["minb"])


# kind, gather dtype, macro arguments, F (a multiple of 4 for FP32 and of 8 for BF16), (u, minb) of set_tuning.
# plain: NTS_PLAN_CASE(k, u, minb); g: NTS_PLAN_CASE_G(u, minb, g); fused: NTS_PLAN_FUSED_CASE(k, u, minb, g);
# tma: NTS_PLAN_TMA_CASE(k, stages, minb) under set_variant(1).
PLAN_CASES = [
    # FP32 gathers, defaults
    ("g", "f32", (4, 4, 4), 24, (0, 0)),
    ("g", "f32", (4, 4, 2), 48, (0, 0)),
    ("plain", "f32", (1, 4, 4), 128, (0, 0)),
    ("plain", "f32", (2, 4, 3), 200, (0, 0)),
    ("plain", "f32", (3, 4, 2), 380, (0, 0)),
    ("plain", "f32", (4, 2, 2), 1436, (0, 0)),          # 3 column tiles
    ("plain", "f32", (5, 4, 2), 604, (0, 0)),
    # FP32 gathers, tuning points
    ("g", "f32", (8, 3, 2), 56, (8, 3)),
    ("g", "f32", (8, 3, 4), 16, (8, 3)),
    ("plain", "f32", (1, 8, 4), 100, (8, 4)),
    ("plain", "f32", (1, 8, 3), 80, (8, 3)),
    ("plain", "f32", (1, 16, 2), 120, (16, 2)),
    ("plain", "f32", (2, 8, 2), 256, (8, 2)),
    ("plain", "f32", (3, 4, 3), 300, (4, 3)),
    ("plain", "f32", (4, 4, 2), 448, (4, 2)),
    ("plain", "f32", (5, 2, 2), 1280, (2, 2)),           # 2 column tiles
    ("plain", "f32", (5, 1, 3), 560, (1, 3)),
    ("plain", "f32", (5, 2, 3), 640, (2, 3)),
    ("plain", "f32", (5, 4, 1), 520, (4, 1)),
    # BF16 gathers, defaults
    ("g", "bf16", (4, 4, 4), 64, (0, 0)),
    ("g", "bf16", (4, 4, 2), 96, (0, 0)),
    ("plain", "bf16", (1, 4, 4), 200, (0, 0)),
    ("plain", "bf16", (2, 2, 3), 400, (0, 0)),
    ("plain", "bf16", (3, 2, 3), 1432, (0, 0)),          # 2 column tiles
    ("plain", "bf16", (4, 2, 2), 1000, (0, 0)),
    ("plain", "bf16", (5, 2, 2), 1280, (0, 0)),
    # BF16 gathers, tuning points
    ("g", "bf16", (8, 2, 2), 120, (8, 2)),
    ("g", "bf16", (8, 2, 4), 40, (8, 2)),
    ("plain", "bf16", (1, 8, 2), 256, (8, 2)),
    ("plain", "bf16", (2, 4, 2), 320, (4, 2)),
    ("plain", "bf16", (3, 4, 2), 600, (4, 2)),
    ("plain", "bf16", (3, 6, 1), 544, (6, 1)),
    ("plain", "bf16", (4, 4, 2), 800, (4, 2)),
    # fused slab + hub-row launches (every point is a default)
    ("fused", "f32", (1, 4, 4, 4), 24, (0, 0)),
    ("fused", "f32", (1, 4, 4, 2), 48, (0, 0)),
    ("fused", "f32", (1, 4, 4, 1), 128, (0, 0)),
    ("fused", "f32", (2, 4, 3, 1), 256, (0, 0)),
    ("fused", "f32", (3, 4, 2, 1), 760, (0, 0)),          # 2 column tiles
    ("fused", "f32", (4, 2, 2, 1), 500, (0, 0)),
    ("fused", "f32", (5, 4, 2, 1), 604, (0, 0)),
    ("fused", "bf16", (1, 4, 4, 4), 32, (0, 0)),
    ("fused", "bf16", (1, 4, 4, 2), 96, (0, 0)),
    ("fused", "bf16", (1, 4, 4, 1), 248, (0, 0)),
    ("fused", "bf16", (2, 2, 3, 1), 512, (0, 0)),
    ("fused", "bf16", (3, 2, 3, 1), 608, (0, 0)),
    ("fused", "bf16", (4, 2, 2, 1), 1024, (0, 0)),
    ("fused", "bf16", (5, 2, 2, 1), 1200, (0, 0)),
    # TMA row staging (FP32 only)
    ("tma", "f32", (1, 4, 4), 100, (0, 0)),
    ("tma", "f32", (2, 4, 3), 200, (0, 0)),
    ("tma", "f32", (3, 4, 2), 300, (0, 0)),
    ("tma", "f32", (4, 2, 2), 400, (0, 0)),
    ("tma", "f32", (5, 4, 2), 604, (0, 0)),
    ("tma", "f32", (1, 8, 4), 128, (8, 0)),
    ("tma", "f32", (1, 8, 3), 64, (8, 3)),
    ("tma", "f32", (2, 4, 2), 160, (0, 2)),
    ("tma", "f32", (4, 4, 2), 448, (4, 0)),
    ("tma", "f32", (5, 2, 2), 560, (2, 0)),
    ("tma", "f32", (5, 4, 1), 520, (0, 1)),
    ("tma", "f32", (5, 8, 1), 640, (8, 1)),
]


def case_id(c):
    return "%s-%s-%s-F%d" % (c[0], c[1], "_".join(map(str, c[2])), c[3])


# ---- plans on the structured graph ---------------------------------------------------------------------------------------
def top_ids(cnt, h):
    """The h ids of largest count, ties to the smaller id (top_ids of the plan builder)."""
    order = np.lexsort((np.arange(cnt.size), -cnt.astype(np.int64)))
    return order[:min(h, cnt.size)]


class Plan:
    """A GatherPlan of the E % 4 == 1 structured graph with what a run must report: addressing 'base' (indices global id
    + BASE, gathered row = global id) or 'slot' (global ids through the MirrorIndex), slab count and hub counts."""

    def __init__(self, addr, slabs, hubs, w):
        from neutronstarlite_b200 import ops
        g = self.g = trimmed(1)
        a = g.device()
        wd = torch.from_numpy(w).to(dev())
        self.addr, self.slabs = addr, slabs
        if addr == "base":
            self.G, grow = g.Vg, g.idx
            self.plan = ops.GatherPlan(a["off"], a["idx_base"], wd, BASE, g.n_rows, g.E, self.G, slabs, hubs=hubs)
        else:
            self.G, grow = g.M, g.mi[g.idx].astype(np.int64)
            self.plan = ops.GatherPlan(a["off"], a["idx"], wd, 0, g.n_rows, g.E, self.G, slabs, slot_of=a["mi"],
                                       hubs=hubs)
        assert (self.plan.slabs, self.plan.hub_cols, self.plan.hub_rows) == (slabs,) + tuple(hubs)
        cols = top_ids(np.bincount(grow, minlength=self.G), hubs[0])
        rows = top_ids(g.deg, hubs[1])
        resid = ~np.isin(grow, cols) & ~np.isin(g.dst, rows)
        self.slab_rows = cdiv(self.G, slabs)
        slab = np.minimum(grow // self.slab_rows, slabs - 1)
        self.slab_edges = np.bincount(slab[resid], minlength=slabs)
        self.hub_rows = hubs[1]

    def inputs(self, Xg):
        """The gathered matrix in this plan's row space."""
        return Xg if self.addr == "base" else Xg[torch.from_numpy(self.g.ids).to(Xg.device)].contiguous()

    def expected(self, F, p, fused, Q_req=0):
        """(launches, grid of the last launch) of a run at point p (plan_point) over F columns."""
        G = p["g"]
        Q = Q_req or 512 // G
        if not Q_req:
            per_slab = int(self.slab_edges.sum()) // self.slabs + 1
            while Q > 32 and cdiv(per_slab, Q) * p["tiles"] < sm_count() * 64 * G:
                Q >>= 1
        Q = cdiv(Q, 32) * 32
        if Q * G > 1024:
            Q = (1024 // G) // 32 * 32
        grids = []
        for s in range(self.slabs):
            blocks = cdiv(cdiv(int(self.slab_edges[s]), Q) * p["tiles"], 8 * G)
            if fused and self.hub_rows:
                TN = 8 if p["minb"] <= 2 else 4
                m_tiles, n_tiles = cdiv(self.hub_rows, 128), cdiv(F, 16 * TN)
                splits = cdiv(sm_count() * 8, m_tiles * n_tiles)
                k_split = max(cdiv(cdiv(self.G, splits), 16) * 16, 256)
                k_lo = min(s * self.slab_rows, self.G)
                k_hi = self.G if s == self.slabs - 1 else min((s + 1) * self.slab_rows, self.G)
                blocks += (cdiv(k_hi - k_lo, k_split) if k_hi > k_lo else 0) * m_tiles * n_tiles
            if blocks:
                grids.append(blocks)
        return len(grids), grids[-1]


@pytest.fixture(scope="module")
def plans():
    """Plans with exact weights ('exact') and with uniform weights ('random') of the same graph."""
    g = trimmed(1)
    rng = np.random.default_rng(11)
    w_exact = exact_inputs(g, 1, seed=12)[1]
    w_rand = rng.uniform(-1, 1, g.E).astype(np.float32)
    out = {}
    for tag, w in (("exact", w_exact), ("random", w_rand)):
        out[tag] = dict(w=w, p1=Plan("base", 1, (0, 0), w), p3=Plan("slot", 3, (0, 0), w),
                        h64=Plan("slot", 3, (64, HUB_ROWS), w), h17=Plan("base", 3, (17, HUB_ROWS), w),
                        c64=Plan("base", 3, (64, 0), w), r200=Plan("slot", 3, (0, HUB_ROWS), w))
    yield out
    out.clear()
    torch.cuda.empty_cache()


def last_launch(plan):
    from neutronstarlite_b200 import _lib
    v = [C.c_int(0) for _ in range(5)]
    _lib.call("nts_gather_plan_last_launch", plan.handle, *[C.byref(x) for x in v])
    return tuple(x.value for x in v)     # launches, grid, k, u, outv


def run(P, X, init, F, *, bf16=False, bf16_input=False, out_shift=0, overwrite=False):
    """Run plan P on the first F columns of X (the gathered matrix in P's row space) into the first F columns of
    init (or into NaN for an overwrite run); returns the output and the launch record."""
    x = X[:, :F].contiguous()
    if bf16_input:
        x = x.to(torch.bfloat16)
    start = torch.full_like(init[:, :F], float("nan")) if overwrite else init[:, :F].contiguous()
    out = shifted(start, out_shift)
    P.plan.run(x, out, gather_dtype=torch.bfloat16 if bf16 else None, accumulate=not overwrite)
    torch.cuda.synchronize()
    return out, last_launch(P.plan)


def exact_case(plans, F, seed):
    """Exact inputs for F columns, the float64 reference A X (no init) and the device init."""
    g = trimmed(1)
    X, _, init = exact_inputs(g, F, seed)
    a = g.device()
    Xg, initd = torch.from_numpy(X).to(dev()), torch.from_numpy(init).to(dev())
    ax, _ = reference(a["dst64"], a["src64"], torch.from_numpy(plans["exact"]["w"]).to(dev()), Xg,
                      torch.zeros_like(initd))
    return Xg, initd, ax


def outv_runs(F, case):
    """(F, output shift) of the OUTV 4 / 2 / 1 runs: the gathered row length is ceil(F / 4) * 4 (ceil(F / 8) * 8) for
    all three."""
    return [(F, 0), (F - 2, 0), (F - 1, 0) if case % 2 else (F, 1)]


# ---- CPU: the tables -------------------------------------------------------------------------------------------------------
def between(text, start, end):
    i = text.index(start)
    return text[i:text.index(end, i)]


def source_plan_points():
    """{(kind, dtype, macro arguments)} of run_gather (nts_plan.cu), by the branch each macro line sits in."""
    src = read_source("nts_plan.cu")
    body = between(src, "static int run_gather(", "// Workspace of at least")
    fused = between(body, "if (fused) {", "no fused slab/hub-row instantiation")
    fused_bf16, fused_f32 = fused.split("} else {")
    rest = body[body.index("no fused slab/hub-row instantiation"):]
    bf16 = between(rest, "if constexpr (kBf16) {", "no BF16 planned-aggregation instantiation")
    f32 = rest[rest.index("no BF16 planned-aggregation instantiation"):]
    tma = between(f32, "if (g_plan_variant == 1)", "no TMA row-staging instantiation")
    f32 = f32[f32.index("no TMA row-staging instantiation"):]
    pts = []
    for kind, dtype, text, macro in (("fused", "bf16", fused_bf16, "NTS_PLAN_FUSED_CASE"),
                                     ("fused", "f32", fused_f32, "NTS_PLAN_FUSED_CASE"),
                                     ("g", "bf16", bf16, "NTS_PLAN_CASE_G"), ("plain", "bf16", bf16, "NTS_PLAN_CASE"),
                                     ("tma", "f32", tma, "NTS_PLAN_TMA_CASE"),
                                     ("g", "f32", f32, "NTS_PLAN_CASE_G"), ("plain", "f32", f32, "NTS_PLAN_CASE")):
        pts += [(kind, dtype, t) for t in source_cases(text, macro)]
    return pts


def test_plan_tables_match_the_source():
    """Every NTS_PLAN_*CASE* line of run_gather has exactly one row in PLAN_CASES and no row names a point that is not
    instantiated: a new instantiation without a test point fails here."""
    src = source_plan_points()
    assert len(src) == len(set(src)) == 19 + 14 + 14 + 12
    table = [(c[0], c[1], c[2]) for c in PLAN_CASES]
    assert len(table) == len(set(table))
    assert sorted(table) == sorted(src)


def test_plan_table_points_follow_the_dispatch_rule():
    """The mirror of run_gather reaches every table point at every OUTV run; default rows without set_tuning, tuned
    rows only with it.  Every OUTV run keeps the gathered row length of F."""
    for i, (kind, dtype, args, F, tuning) in enumerate(PLAN_CASES):
        bf16, variant = dtype == "bf16", 1 if kind == "tma" else 0
        assert F % (8 if bf16 else 4) == 0
        for outv, (Fr, shift) in zip((4, 2, 1), outv_runs(F, i)):
            p = plan_point(Fr, bf16, 16 if shift == 0 else 4, tuning, variant)
            assert p["outv"] == outv and case_point(kind, p) == args, (kind, dtype, args, Fr, shift, p)
            if kind in ("g", "plain"):
                assert (kind == "g") == (p["g"] > 1)
        if tuning != (0, 0):
            assert case_point(kind, plan_point(F, bf16, 16, (0, 0), variant)) != args, (args, "reached by default")


# ---- GPU: every instantiation ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(PLAN_CASES)), ids=[case_id(c) for c in PLAN_CASES])
def test_every_plan_point_exact(plans, case):
    from neutronstarlite_b200 import _lib
    kind, dtype, args, F, tuning = PLAN_CASES[case]
    bf16 = dtype == "bf16"
    Xg, initd, ax = exact_case(plans, F, seed=600 + case)
    ps = plans["exact"]
    runs = []
    for j, (Fr, shift) in enumerate(outv_runs(F, case)):
        if kind == "fused":
            P = ps["h64"] if case % 2 == 0 else ps["h17"]
            runs += [(P, Fr, shift, ow, j % 2 == 1) for ow in (False, True)]
        else:
            for P in (ps["p1"], ps["p3"]):
                runs.append((P, Fr, shift, P is ps["p3"] and j == 1, (j + (P is ps["p3"])) % 2 == 1))
    with hooks():
        _lib.call("nts_gather_plan_set_tuning", tuning[0], tuning[1], 0)
        _lib.call("nts_gather_plan_set_variant", 1 if kind == "tma" else 0)
        for P, Fr, shift, overwrite, bf16_input in runs:
            P.plan.set_overlap(kind == "fused")
            out, (launches, grid, k, u, outv) = run(P, P.inputs(Xg), initd, Fr, bf16=bf16,
                                                    bf16_input=bf16 and bf16_input, out_shift=shift,
                                                    overwrite=overwrite)
            p = plan_point(Fr, bf16, 16 if shift == 0 else 4, tuning, 1 if kind == "tma" else 0)
            assert case_point(kind, p) == args
            assert (k, u, outv) == (p["k"], p["u"], p["outv"]), (Fr, shift, (k, u, outv))
            want = P.expected(Fr, p, kind == "fused")
            assert (launches, grid) == want, (Fr, P.addr, P.slabs, (launches, grid), want)
            check_exact(out, ax[:, :Fr] if overwrite else ax[:, :Fr] + initd[:, :Fr])


@pytest.mark.gpu
@pytest.mark.parametrize("F", [100, 200, 300, 448, 604, 760])
def test_tma_variant_runs_at_its_default_point_for_every_chunk_count(plans, F):
    """set_variant(1) with no tuning: 1-5 chunks per lane (760: 3 chunks in 2 column tiles).  At 2 and 3 chunks the
    default occupancy used to be 4 CTAs per SM, which has no instantiation."""
    from neutronstarlite_b200 import _lib
    Xg, initd, ax = exact_case(plans, F, seed=700 + F)
    P = plans["exact"]["p3"]
    with hooks():
        _lib.call("nts_gather_plan_set_variant", 1)
        out, (launches, grid, k, u, outv) = run(P, P.inputs(Xg), initd, F)
        p = plan_point(F, False, variant=1)
        assert (k, u, outv) == (p["k"], p["u"], 4)
        assert (launches, grid) == P.expected(F, p, False)
        check_exact(out, ax + initd)


@pytest.mark.gpu
@pytest.mark.parametrize("hubs", ["h17", "c64", "r200"])
@pytest.mark.parametrize("bf16", [False, True])
def test_standalone_hub_blocks_exact(plans, hubs, bf16):
    """The sequential schedule: column block (accumulating, or storing in overwrite runs) and split-K row block as
    stand-alone GEMM launches, then the slab launches.  M tails (2609 output rows, 200 hub rows), N tails (F % 128 != 0),
    a K tail (17 hub columns), OUTV 4 / 2 / 1."""
    P = plans["exact"][hubs]
    Xg, initd, ax = exact_case(plans, 602, seed=800 + len(hubs) + bf16)
    P.plan.set_overlap(False)
    for F in (600, 602, 601, 128):
        for overwrite in (False, True):
            out, (launches, grid, k, u, outv) = run(P, P.inputs(Xg), initd, F, bf16=bf16, bf16_input=bf16 and F == 128,
                                                    overwrite=overwrite)
            assert outv == (4 if F % 4 == 0 else (2 if F % 2 == 0 else 1))
            p = plan_point(F, bf16)
            assert (launches, grid) == P.expected(F, p, False)
            check_exact(out, ax[:, :F] if overwrite else ax[:, :F] + initd[:, :F])


@pytest.mark.gpu
@pytest.mark.parametrize("Q", [32, 1024])
def test_plan_quantum_sizes_exact(plans, Q):
    """The edge quantum of set_tuning's third argument (rounded to 32, at most 1024 / G lanes' worth), on a plain plan
    and on a fused one, FP32 and BF16."""
    from neutronstarlite_b200 import _lib
    ps = plans["exact"]
    for F, bf16 in ((24, False), (48, False), (128, False), (604, False), (1436, False), (96, True), (1432, True)):
        Xg, initd, ax = exact_case(plans, F, seed=900 + F)
        with hooks():
            _lib.call("nts_gather_plan_set_tuning", 0, 0, Q)
            for P, fused in ((ps["p3"], False), (ps["h64"], True)):
                P.plan.set_overlap(fused)
                out, (launches, grid, k, u, outv) = run(P, P.inputs(Xg), initd, F, bf16=bf16)
                assert (launches, grid) == P.expected(F, plan_point(F, bf16), fused, Q), (F, bf16, fused)
                check_exact(out, ax + initd)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [i for i, c in enumerate(PLAN_CASES) if c[4] == (0, 0) and c[0] != "tma"],
                         ids=[case_id(c) for c in PLAN_CASES if c[4] == (0, 0) and c[0] != "tma"])
def test_default_points_random_within_rounding(plans, case):
    """Uniform features and weights at every default point: per element within 1e-4 (|init| + |A| |X|) of float64; BF16
    gathers against the reference at bf16(X)."""
    kind, dtype, args, F, _ = PLAN_CASES[case]
    bf16 = dtype == "bf16"
    g = trimmed(1)
    ps = plans["random"]
    X, _, init = random_inputs(g, F, seed=1000 + case)
    if bf16:
        X = torch.from_numpy(X).to(torch.bfloat16).float().numpy()
    a = g.device()
    Xg, initd = torch.from_numpy(X).to(dev()), torch.from_numpy(init).to(dev())
    ref, mag = reference(a["dst64"], a["src64"], torch.from_numpy(ps["w"]).to(dev()), Xg, initd)
    with hooks():
        for P in ((ps["h64"], ps["h17"]) if kind == "fused" else (ps["p1"], ps["p3"])):
            P.plan.set_overlap(kind == "fused")
            out, (_, _, k, u, outv) = run(P, P.inputs(Xg), initd, F, bf16=bf16)
            assert (k, u, outv) == (args[0] if kind != "g" else 1, args[1] if kind != "g" else args[0], 4)
            check_random(out, ref, mag)
