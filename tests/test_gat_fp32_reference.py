"""The FP32 fused GAT layer (K7: nts_gat_softmax_stats, nts_gat_fused_aggregate_forward, the single-pass and the
two-pass backward, ops.DistGPUFusedGATOp) against float64, at every dispatch branch the (H, D) grid below reaches.

Reference: `analytic_reference`, float64 and computed in edge chunks (so that it also runs on a graph of 11 M edges):
    a = exp(leaky(s + d) - max) / sum,  out = sum a m,  d_mirror = sum a g[dst],
    d_pre = a (<m, g> - <out, g>) leaky'(s + d),  ds / dd = sums of d_pre over a slot's out-edges / a destination's
    in-edges.
It is checked against float64 torch autograd of the layer (test_gat_bf16.layer_reference) to 1e-12 on the structured
graph, including edges with s + d == 0 exactly, where leaky' follows torch (pre > 0).

Tolerances are per row (and head) and scaled by the magnitudes of the summed terms, not by the sum: a hub row's terms
cancel, and FP32 rounding scales with the terms.
    out, d_mirror:  row_close(rtol=1e-4, scale=sum a |m| / sum a |g[dst]|)
    ds, dd:         |err| <= 1e-4 sum a (<|m|,|g|> + |<out,g>|) |leaky'|  +  FLT_MIN sum (<|m|,|g|> + |<out,g>|) |leaky'|
The second term only matters for weights below FLT_MIN (scores of +-40), which FP32 cannot carry: such a weight is 0 or
a subnormal in the kernel.  The sensitivity tests show that the bounds reject a reference with one edge dropped or
doubled, in the hub segment and just after a quantum boundary.

GPU tests are marked one by one; the reference self-check, the sensitivity tests and the graph invariants run on the
CPU."""
import ctypes
import time

import numpy as np
import pytest

from test_gat_bf16 import layer_reference, stub_graph
from test_gather_plan_bf16 import row_close

torch = pytest.importorskip("torch")

SLOPES = [0.2, 0.0, 1.0]
FLT_MIN = float(np.finfo(np.float32).tiny)


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return t.data_ptr()


# ---- a structured whole-partition CSC + MirrorIndex ----------------------------------------------------------------
HUB_SRC, ONE_SRC = 7, 11        # global ids: the hub source, the only source of ONE_ROW
EMPTY_SLOT_IDS = (5990, 5995, 5999)   # marked in the MirrorIndex, never a source: mirror slots without out-edges


class Structured:
    """off [Vp+1], idx [E] (global source ids), mi [Vg+1] (MirrorIndex), slot [E] (mi[idx]) and the rows of note."""

    def __init__(self, seed=0):
        rng = np.random.default_rng(seed)
        Vg = 6000
        # rows 0, 1, 5 empty; 2-4 end exactly on 64, 256, 512; 6 starts on 512 with exactly kHubDegree = 4096 edges
        # (warp path of both row kernels), 7 has 4097 (whole-CTA path), 8 is a hub of 20 011 edges
        head = [0, 0, 64, 192, 256, 0, 4096, 4097, 20011]
        small = rng.integers(0, 41, 2600)
        small[rng.random(small.size) < 0.1] = 0
        self.one_row = len(head) + 1300
        small[1300] = 300                  # every in-edge from ONE_SRC; spans a 256-edge boundary
        deg = np.concatenate([head, small]).astype(np.int64)
        off = np.zeros(deg.size + 1, dtype=np.int64)
        np.cumsum(deg, out=off[1:])
        E = int(off[-1])
        idx = rng.integers(0, EMPTY_SLOT_IDS[0], E)
        dst = np.repeat(np.arange(deg.size), deg)
        same_row = np.nonzero((dst[1:] == dst[:-1]) & (rng.random(E - 1) < 0.05))[0] + 1
        idx[same_row] = idx[same_row - 1]  # explicit duplicate edges
        idx[idx == HUB_SRC] = HUB_SRC + 1
        idx[idx == ONE_SRC] = ONE_SRC + 1
        b, e = off[self.one_row], off[self.one_row + 1]
        idx[b:e] = ONE_SRC
        small_edges = np.nonzero((dst >= len(head)) & (dst != self.one_row))[0]
        idx[rng.choice(small_edges, 1000, replace=False)] = HUB_SRC   # a hub SOURCE: > 3 x 256 out-edges
        marked = np.zeros(Vg + 1, dtype=np.uint32)
        marked[np.unique(idx) + 1] = 1
        marked[np.array(EMPTY_SLOT_IDS) + 1] = 1
        self.mi = np.cumsum(marked, dtype=np.uint32)
        self.off, self.idx = off.astype(np.uint32), idx.astype(np.uint32)
        self.slot = self.mi[self.idx].astype(np.int64)
        self.Vp, self.E, self.M = deg.size, E, int(self.mi[-1])
        self.hub_row = 8
        self.empty_rows = np.nonzero(deg == 0)[0]
        self.empty_slots = self.mi[list(EMPTY_SLOT_IDS)].astype(np.int64)
        self.hub_slot = int(self.mi[HUB_SRC])

    def graph(self):
        return stub_graph(self.off, self.idx, self.mi)

    def torch_csc(self, device):
        return (torch.from_numpy(self.off.astype(np.int64)).to(device),
                torch.from_numpy(self.slot).to(device))


_STRUCTURED = None


def structured():
    global _STRUCTURED
    if _STRUCTURED is None:
        _STRUCTURED = Structured()
    return _STRUCTURED


# ---- float64 references ----------------------------------------------------------------------------------------------
def analytic_reference(off, slot, m, s, d, g, H, slope, chunk=1 << 20):
    """float64 K7 layer in edge chunks (off int64 [V+1], slot int64 [E], all on one device).  A NaN logit makes its
    whole (destination, head) NaN, as torch's max does.  Returns a dict of float64 tensors: out, dm, ds, dd, the
    magnitudes out_mag, dm_mag, ds_mag, dd_mag, the underflow floors ds_floor, dd_floor, and the statistics mx, z."""
    f8 = torch.float64
    dv = m.device
    V, M, F = off.numel() - 1, m.shape[0], m.shape[1]
    D = F // H
    E = slot.numel()
    m64, s64, d64, g64 = (t.to(f8) for t in (m, s, d, g))

    def edges():
        for e0 in range(0, E, chunk):
            e1 = min(E, e0 + chunk)
            dst = torch.searchsorted(off, torch.arange(e0, e1, device=dv), right=True) - 1
            src = slot[e0:e1]
            pre = s64[src] + d64[dst]
            yield src, dst, pre, torch.where(pre > 0, pre, pre * slope)

    mx = torch.full((V, H), -float("inf"), dtype=f8, device=dv)
    has_nan = torch.zeros((V, H), dtype=f8, device=dv)
    for _, dst, _, lg in edges():
        mx.scatter_reduce_(0, dst[:, None].expand(-1, H), lg, "amax")
        has_nan.index_add_(0, dst, torch.isnan(lg).to(f8))
    mx[has_nan > 0] = float("nan")
    z = torch.zeros((V, H), dtype=f8, device=dv)
    for _, dst, _, lg in edges():
        z.index_add_(0, dst, torch.exp(lg - mx[dst]))
    out = torch.zeros((V, H, D), dtype=f8, device=dv)
    out_mag = torch.zeros_like(out)
    for src, dst, _, lg in edges():
        a = (torch.exp(lg - mx[dst]) / z[dst])[:, :, None]
        ms = m64[src].view(-1, H, D)
        out.index_add_(0, dst, ms * a)
        out_mag.index_add_(0, dst, ms.abs() * a)
    og = (out * g64.view(V, H, D)).sum(-1)
    r = {"dm": torch.zeros((M, H, D), dtype=f8, device=dv), "ds": torch.zeros((M, H), dtype=f8, device=dv),
         "dd": torch.zeros((V, H), dtype=f8, device=dv)}
    r["dm_mag"] = torch.zeros_like(r["dm"])
    for k in ("ds", "dd"):
        r[k + "_mag"] = torch.zeros_like(r[k])
        r[k + "_floor"] = torch.zeros_like(r[k])
    for src, dst, pre, lg in edges():
        a = torch.exp(lg - mx[dst]) / z[dst]
        ms, gd = m64[src].view(-1, H, D), g64[dst].view(-1, H, D)
        lp = torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, slope))
        r["dm"].index_add_(0, src, gd * a[:, :, None])
        r["dm_mag"].index_add_(0, src, gd.abs() * a[:, :, None])
        d_pre = a * ((ms * gd).sum(-1) - og[dst]) * lp
        t0 = ((ms.abs() * gd.abs()).sum(-1) + og[dst].abs()) * lp.abs()
        for k, rows in (("ds", src), ("dd", dst)):
            r[k].index_add_(0, rows, d_pre)
            r[k + "_mag"].index_add_(0, rows, a * t0)
            r[k + "_floor"].index_add_(0, rows, t0)
    r.update(out=out.reshape(V, F), out_mag=out_mag.reshape(V, F), mx=mx, z=z)
    r["dm"], r["dm_mag"] = r["dm"].reshape(M, F), r["dm_mag"].reshape(M, F)
    return r


def np64(t):
    return t.detach().double().cpu().numpy()


def check_layer(got, ref, rtol=1e-4):
    """got = (out, dm, ds, dd) of the kernel.  NaN entries must be exactly the reference's; everything else is held to
    the per-row bounds of the module docstring."""
    for name, x in zip(("out", "dm", "ds", "dd"), got):
        a, b = np64(x), np64(ref[name])
        nan = np.isnan(b)
        assert np.array_equal(np.isnan(a), nan), "%s: NaN at %s, reference NaN at %s" % (
            name, np.argwhere(np.isnan(a) & ~nan)[:4].tolist(), np.argwhere(nan & ~np.isnan(a))[:4].tolist())
        a, b = np.where(nan, 0.0, a), np.where(nan, 0.0, b)
        if name in ("out", "dm"):
            row_close(a, b, rtol, scale=np.nan_to_num(np64(ref[name + "_mag"])))
        else:
            bound = rtol * np64(ref[name + "_mag"]) + FLT_MIN * np64(ref[name + "_floor"])
            err = np.abs(a - b)
            bad = np.argwhere(err > np.nan_to_num(bound) + 1e-30)
            assert bad.size == 0, "%s at (row, head) %s: err %s vs bound %s" % (
                name, bad[:4].tolist(), err[tuple(bad[:4].T)], bound[tuple(bad[:4].T)])


def check_stats(seg_max, seg_sum, ref, empty_rows):
    """Segment statistics: exactly (0, 1) on empty destinations, otherwise the float64 max (up to the FP32 rounding of
    s + d) and sum of exp(logit - max)."""
    mx, z = np64(seg_max), np64(seg_sum)
    assert (mx[empty_rows] == 0).all() and (z[empty_rows] == 1).all()
    rm, rz = np64(ref["mx"]), np64(ref["z"])
    live = np.isfinite(rm)
    assert np.all(np.abs(mx[live] - rm[live]) <= 1e-6 * (1 + np.abs(rm[live])))
    assert np.all(np.abs(z[live] - rz[live]) <= 1e-5 * rz[live])


def layer_inputs(M, V, H, D, seed, score=2.0, device="cpu"):
    rng = np.random.default_rng(seed)
    F = H * D
    mk = lambda a: torch.from_numpy(a.astype(np.float32)).to(device)
    return (mk(rng.uniform(-1, 1, (M, F))), mk(rng.uniform(-score, score, (M, H))),
            mk(rng.uniform(-score, score, (V, H))), mk(rng.uniform(-1, 1, (V, F))))


def run_k7(pg, mirror, s, d, g, slope, two_pass, gather_dtype=None):
    """(out, dm, ds, dd), (seg_max, seg_sum) and the forward's launch record (grid, block, smem, variant)."""
    from neutronstarlite_b200 import _lib, ops
    op = ops.DistGPUFusedGATOp(pg, negative_slope=slope, two_pass_backward=two_pass, gather_dtype=gather_dtype)
    out = op.forward(mirror, s, d)
    rec = [ctypes.c_int() for _ in range(4)]
    _lib.call("nts_aggregate_last_launch", *[ctypes.byref(r) for r in rec])
    dm, ds, dd = op.backward(g)
    torch.cuda.synchronize()
    return (out, dm, ds, dd), op._saved[3:5], tuple(r.value for r in rec)


def sm_count():
    from neutronstarlite_b200 import _lib
    n = ctypes.c_int()
    _lib.call("nts_device_sm_count", ctypes.byref(n))
    return n.value


def expected_launch(E, tiles, G, variant=0, Q=0):
    """(grid, smem, variant) that segment_gather_sum picks for the fused forward over E edges in `tiles` column tiles
    with G virtual warps (set by nts_aggregate_set_variant(variant, Q) when non-zero)."""
    bulk = variant != 1
    if Q == 0:
        Q = 512 // G
        while Q > 32 and -(-E // Q) * tiles < sm_count() * 64:
            Q >>= 1
    Q = (Q + 31) // 32 * 32
    if G > 1 and Q * G > 1024:
        Q = (1024 // G) // 32 * 32
    warps = -(-E // Q) * tiles
    if bulk and G == 2:
        return -(-warps // 16), 16 + 2 * (16 * Q + 8) * 4, 2
    return -(-warps // 8), (16 + 2 * (8 * Q + 8) * 4) if bulk else 0, 2 if bulk else 1


# ---- CPU: the graph, the reference and the comparator ------------------------------------------------------------------
def test_structured_graph_has_the_edges_kernels_go_wrong_at():
    st = structured()
    off, deg = st.off.astype(np.int64), np.diff(st.off.astype(np.int64))
    assert st.empty_rows.size > 100 and deg[st.hub_row] > 20000
    assert (deg == 4096).any() and (deg == 4097).any()
    for q in (64, 256, 512):
        starts_on = (off[:-1] % q == 0) & (deg > 0) & (off[:-1] > 0)
        straddles = (off[:-1] // q < (off[1:] - 1) // q) & (deg > 0)
        assert starts_on.any() and straddles.sum() > 10, q
    dst = np.repeat(np.arange(st.Vp), deg)
    pairs = dst.astype(np.int64) * (1 << 32) + st.idx
    assert np.unique(pairs).size < pairs.size                      # duplicate edges
    out_deg = np.bincount(st.slot, minlength=st.M)
    slot_off = np.concatenate([[0], np.cumsum(out_deg)])
    assert out_deg[st.hub_slot] > 3 * 256 and slot_off[st.hub_slot] % 256 != 0
    assert (out_deg[st.empty_slots] == 0).all()
    b, e = off[st.one_row], off[st.one_row + 1]
    assert np.unique(st.idx[b:e]).tolist() == [ONE_SRC] and b // 256 < (e - 1) // 256


@pytest.mark.parametrize("slope", SLOPES)
def test_analytic_reference_equals_float64_autograd(slope):
    """The chunked analytic reference against autograd (layer_reference) on the structured graph, with dyadic scores
    so that s + d == 0 exactly on about a fifth of the edges (leaky' there is torch's: the negative slope)."""
    st = structured()
    H, D = 2, 3
    m, _, _, g = layer_inputs(st.M, st.Vp, H, D, seed=1)
    rng = np.random.default_rng(2)
    grid = np.array([-1.0, -0.5, 0.0, 0.5, 1.0], dtype=np.float32)
    s = torch.from_numpy(rng.choice(grid, (st.M, H)))
    d = torch.from_numpy(rng.choice(grid, (st.Vp, H)))
    off, slot = st.torch_csc("cpu")
    pre = s[slot] + d[torch.repeat_interleave(torch.arange(st.Vp), torch.diff(off))]
    assert (pre == 0).float().mean() > 0.1
    ref = analytic_reference(off, slot, m, s, d, g, H, slope, chunk=10007)
    want = layer_reference(st.off, st.slot, m, s, d, g, H, slope)
    # elementwise against the magnitude of the summed terms (at slope 1, dd = <out,g> - <out,g> sums to ~1e-16)
    for name, w in zip(("out", "dm", "ds", "dd", "out_mag", "dm_mag"), want):
        scale = ref[name.split("_")[0] + "_mag"]
        assert bool(((ref[name] - w).abs() <= 1e-12 * scale).all()), name


def reference_without(st, edge, H, inputs, slope, double=False):
    """The analytic reference on the structured graph with `edge` dropped (or doubled)."""
    off = st.off.astype(np.int64).copy()
    r = np.searchsorted(off, edge, side="right") - 1
    off[r + 1:] += 1 if double else -1
    slot = np.insert(st.slot, edge, st.slot[edge]) if double else np.delete(st.slot, edge)
    m, s, d, g = inputs
    return analytic_reference(torch.from_numpy(off), torch.from_numpy(slot), m, s, d, g, H, slope)


@pytest.mark.parametrize("where", ["hub", "quantum_boundary"])
@pytest.mark.parametrize("double", [False, True])
def test_comparator_rejects_a_reference_with_one_edge_dropped_or_doubled(where, double):
    """The bounds are tight enough to see one edge: the FP32-rounded full reference passes check_layer, a reference
    built without (or with twice) one edge of the hub segment - the one with the largest weight - or the first edge of
    a 512-edge quantum in an ordinary segment is rejected."""
    st = structured()
    H, D, slope = 2, 4, 0.2
    inputs = layer_inputs(st.M, st.Vp, H, D, seed=3)
    off, slot = st.torch_csc("cpu")
    full = analytic_reference(off, slot, *inputs, H, slope)
    got = [full[k].float() for k in ("out", "dm", "ds", "dd")]
    check_layer(got, full)
    if where == "hub":
        b, e = int(st.off[st.hub_row]), int(st.off[st.hub_row + 1])
        m, s, d, g = inputs
        edge = b + int((s[slot[b:e], 0] + d[st.hub_row, 0]).argmax())
    else:
        edge = next(q for q in range(512 * 40, st.E, 512)
                    if np.diff(st.off.astype(np.int64))[np.searchsorted(st.off, q, side="right") - 1] > 1)
    with pytest.raises(AssertionError):
        check_layer(got, reference_without(st, edge, H, inputs, slope, double))


# ---- GPU: the (H, D) grid ----------------------------------------------------------------------------------------------
# (H, D, forward column tiles, forward virtual warps).  Branches, read from the dispatch code (forward:
# segment_gather_sum / pick_shape; statistics: nts_gat_softmax_stats; backward: nts_gat_fused_aggregate_backward and
# _two_pass).  "single" = two_pass_backward=False, "two-pass" = the default.
GRID = [
    # F 64, VEC 4, 16 vectors: two 16-lane virtual warps (Q 256). stats edge kernel H 8. two-pass VEC 2 KB 1 (4 vectors
    # per head); single seg kernel VEC 2 KB 1
    (8, 8, 1, 2),
    # the operator pads 41 -> 44 columns: VEC 4, 11 vectors, two virtual warps. stats H 1. backward on 41 columns:
    # VEC 1, two-pass ONEHEAD KB 2; single generic kernel VEC 1 (41 vectors per head is not a power of two)
    (1, 41, 1, 2),
    # F 64, VEC 2 (D = 2), 32 vectors: one warp. stats edge kernel H 32 (one edge per warp step). two-pass VEC 2 KB 1,
    # 1 vector per head; single seg kernel VEC 2 KB 1
    (32, 2, 1, 1),
    # F 40, VEC 4, 10 vectors: two virtual warps. stats ROW kernel (5 does not divide 32). two-pass VEC 1 KB 2 (8 per
    # head); single seg kernel VEC 1 KB 2
    (5, 8, 1, 2),
    # F 15, VEC 1, two virtual warps. stats ROW kernel. 5 vectors per head: two-pass falls back to single; generic VEC 1
    (3, 5, 1, 2),
    # F 128, VEC 4, 32 vectors, one tile K 1. stats H 4. two-pass VEC 4 KB 1 (8 per head); single seg VEC 4 KB 1
    (4, 32, 1, 1),
    # F 256, VEC 4, K 2. stats H 2. two-pass VEC 4 KB 2 (32 per head); single seg VEC 4 KB 2
    (2, 128, 1, 1),
    # F 512, VEC 4, K 4. stats H 1. two-pass ONEHEAD VEC 4 KB 4; single generic VEC 4 (128 vectors per head > 32)
    (1, 512, 1, 1),
    # F 201, VEC 1 (D odd), 201 vectors: 2 tiles of 101 (K 4), the head boundary at column 67 / 134 falls inside a
    # lane's chunks. stats ROW kernel. kb 7: two-pass falls back; generic VEC 1
    (3, 67, 2, 1),
    # F 600, VEC 4, 150 vectors: 2 tiles of 75 (K 3), head boundaries at vectors 50 / 100 inside a tile. stats ROW
    # kernel. kb 5: two-pass falls back; single generic VEC 4 (50 vectors per head)
    (3, 200, 2, 1),
    # F 1024, VEC 4, 256 vectors: 2 tiles of 128 (K 4). stats H 8. kb 8: two-pass falls back; single: 32 vectors per
    # head but kb 8 > 4, so generic VEC 4
    (8, 128, 2, 1),
    # padded to 1436: VEC 4, 359 vectors, 3 tiles of 120 (K 4). stats H 1. backward on 1433 columns: VEC 1, kb 45,
    # falls back; generic VEC 1 (ONEHEAD)
    (1, 1433, 3, 1),
    # F 24, VEC 2 (D = 6), 12 vectors: two virtual warps. stats H 4. backward VEC 1 (24 < 32 lanes at VEC 2), 6
    # vectors per head: two-pass falls back; generic VEC 1
    (4, 6, 1, 2),
]


def check_exact_zeros(st, got):
    """Empty destinations: out row and dd exactly 0.  Slots with no out-edges: d_mirror row and ds exactly 0."""
    out, dm, ds, dd = (np64(x) for x in got)
    assert not out[st.empty_rows].any() and not dd[st.empty_rows].any()
    assert not dm[st.empty_slots].any() and not ds[st.empty_slots].any()


@pytest.mark.gpu
@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("H,D,tiles,G", GRID)
def test_fused_gat_layer_vs_float64(H, D, tiles, G, slope):
    dv = dev()
    st = structured()
    pg = st.graph()
    inputs = layer_inputs(st.M, st.Vp, H, D, seed=H * 1000 + D, device=dv)
    ref = analytic_reference(*st.torch_csc(dv), *inputs, H, slope)
    Fk = (H * D + 3) // 4 * 4 if H == 1 else H * D
    want = expected_launch(st.E, tiles, G)
    for two_pass in (True, False):
        got, (seg_max, seg_sum), (grid, block, smem, variant) = run_k7(pg, *inputs, slope, two_pass)
        assert (grid, smem, variant) == want, (Fk, (grid, smem, variant), want)
        check_stats(seg_max, seg_sum, ref, st.empty_rows)
        check_layer(got, ref)
        check_exact_zeros(st, got)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D,tiles,G", [GRID[0], GRID[1], GRID[8], GRID[9], GRID[12]])
def test_forward_quantum_and_staging_sweep(H, D, tiles, G):
    """Both index-staging variants at Q = 32, 64 and the production 512 (the test graph alone would shrink Q to 32).
    Variant 1 runs the shuffle-staged head-mode-2 kernel, without virtual warps."""
    from neutronstarlite_b200 import _lib
    dv = dev()
    st = structured()
    pg = st.graph()
    inputs = layer_inputs(st.M, st.Vp, H, D, seed=H * 1000 + D + 1, device=dv)
    ref = analytic_reference(*st.torch_csc(dv), *inputs, H, 0.2)
    try:
        for v in (1, 2):
            for Q in (32, 64, 512):
                _lib.call("nts_aggregate_set_variant", v, Q)
                got, _, (grid, _, smem, variant) = run_k7(pg, *inputs, 0.2, True)
                assert (grid, smem, variant) == expected_launch(st.E, tiles, G, v, Q), (v, Q)
                row_close(np64(got[0]), np64(ref["out"]), scale=np64(ref["out_mag"]))
    finally:
        _lib.call("nts_aggregate_set_variant", 0, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", [(8, 8), (3, 5), (1, 41), (3, 200), (2, 128)])
def test_c_abi_with_mirror_index(H, D):
    """Statistics, forward and both backwards through the C ABI with global row_indices and a non-NULL mirror_index
    (the operator always passes precomputed slots).  F = 41 is not padded here: a VEC 1 forward."""
    from neutronstarlite_b200 import _lib, ops
    dv = dev()
    st = structured()
    pg = st.graph()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=H * 31 + D, device=dv)
    slope, F, V = 0.2, H * D, st.Vp
    ref = analytic_reference(*st.torch_csc(dv), m, s, d, g, H, slope)
    ri, co, mi = pg.row_indices_gpu, pg.column_offset_gpu, pg.mirror_index_gpu
    seg_max = torch.full((V, H), 7.0, device=dv)
    seg_sum = torch.full((V, H), 7.0, device=dv)
    _lib.call("nts_gat_softmax_stats", ptr(seg_max), ptr(seg_sum), ptr(s), ptr(d), ptr(ri), ptr(co), ptr(mi), V, H,
              slope, stream())
    out = torch.zeros((V, F), device=dv)
    _lib.call("nts_gat_fused_aggregate_forward", ptr(m), ptr(out), ptr(s), ptr(d), ptr(seg_max), ptr(seg_sum), ptr(ri),
              ptr(co), ptr(mi), V, st.E, F, H, slope, stream())
    og = (out * g).view(V, H, D).sum(-1).contiguous()
    slot_off, slot_dst = ops.DistGPUFusedGATOp.slot_csr(pg)
    for two_pass in (True, False):
        dm, ds, dd = torch.zeros_like(m), torch.zeros_like(s), torch.zeros_like(d)
        if two_pass:
            pack = torch.empty((V, H, 4), device=dv)
            _lib.call("nts_gat_fused_aggregate_backward_two_pass", ptr(dm), ptr(ds), ptr(dd), ptr(pack), ptr(m),
                      ptr(s), ptr(d), ptr(seg_max), ptr(seg_sum), ptr(og), ptr(g), ptr(ri), ptr(co), ptr(mi),
                      ptr(slot_off), ptr(slot_dst), V, st.M, F, H, slope, stream())
        else:
            _lib.call("nts_gat_fused_aggregate_backward", ptr(dm), ptr(ds), ptr(dd), ptr(m), ptr(s), ptr(d),
                      ptr(seg_max), ptr(seg_sum), ptr(og), ptr(g), ptr(ri), ptr(co), ptr(mi), V, F, H, slope,
                      stream())
        torch.cuda.synchronize()
        check_stats(seg_max, seg_sum, ref, st.empty_rows)
        check_layer((out, dm, ds, dd), ref)
        check_exact_zeros(st, (out, dm, ds, dd))


# ---- GPU: edge semantics -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41), (3, 5), (3, 200)])
def test_equal_logits_give_uniform_weights(H, D):
    """One source score for every slot: all logits of a segment are equal, so the statistics are exactly
    (leaky(s + d), deg) and out is the mean of the segment's mirror rows."""
    dv = dev()
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=5, device=dv)
    s = torch.full_like(s, 0.375)
    ref = analytic_reference(*st.torch_csc(dv), m, s, d, g, H, 0.2)
    for two_pass in (True, False):
        got, (seg_max, seg_sum), _ = run_k7(st.graph(), m, s, d, g, 0.2, two_pass)
        deg = torch.from_numpy(np.diff(st.off.astype(np.int64))).to(dv)
        live = deg > 0
        pre = s[0] + d
        assert torch.equal(seg_max[live], torch.where(pre > 0, pre, pre * 0.2)[live])
        assert torch.equal(seg_sum[live], deg[live, None].float().expand(-1, H))
        check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", [0.2, 0.0])
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41), (3, 67)])
def test_zero_preactivation_uses_the_negative_slope(H, D, slope):
    """Dyadic scores make s + d == 0 exactly on about a fifth of the edges; leaky'(0) must be the negative slope
    (torch's convention, pinned by the reference self-check), in both backwards."""
    dv = dev()
    st = structured()
    m, _, _, g = layer_inputs(st.M, st.Vp, H, D, seed=6, device=dv)
    rng = np.random.default_rng(7)
    grid = np.array([-1.0, -0.5, 0.0, 0.5, 1.0], dtype=np.float32)
    s = torch.from_numpy(rng.choice(grid, (st.M, H))).to(dv)
    d = torch.from_numpy(rng.choice(grid, (st.Vp, H))).to(dv)
    ref = analytic_reference(*st.torch_csc(dv), m, s, d, g, H, slope)
    for two_pass in (True, False):
        got, _, _ = run_k7(st.graph(), m, s, d, g, slope, two_pass)
        check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", [0.2, 1.0])
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41), (3, 200), (5, 8)])
def test_large_scores_underflow_without_inf_or_nan(H, D, slope):
    """Scores in +-40: most weights underflow in FP32 (logits span up to 160).  No inf or NaN, bounds hold."""
    dv = dev()
    st = structured()
    inputs = layer_inputs(st.M, st.Vp, H, D, seed=8, score=40.0, device=dv)
    ref = analytic_reference(*st.torch_csc(dv), *inputs, H, slope)
    for two_pass in (True, False):
        got, _, _ = run_k7(st.graph(), *inputs, slope, two_pass)
        assert all(bool(torch.isfinite(x).all()) for x in got)
        check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41), (3, 5), (3, 200), (2, 128)])
def test_one_nan_source_score_stays_in_its_rows(H, D):
    """One NaN source score (of the slot that is the only source of one row, and one of the hub source's heads): every
    output is NaN exactly where the float64 reference is - the (destination, head) pairs that slot feeds and what
    their gradients reach - and nowhere else, although the statistics drop NaN from the maximum."""
    dv = dev()
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=9, device=dv)
    s[int(st.mi[ONE_SRC]), H - 1] = float("nan")
    s[st.hub_slot, 0] = float("nan")
    ref = analytic_reference(*st.torch_csc(dv), m, s, d, g, H, 0.2)
    assert bool(torch.isnan(ref["out"]).any()) and not bool(torch.isnan(ref["out"]).all())
    for two_pass in (True, False):
        got, _, _ = run_k7(st.graph(), m, s, d, g, 0.2, two_pass)
        check_layer(got, ref)


# ---- GPU: a graph past the grid-stride boundary --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zipf_graph():
    """A Zipf multigraph with E >= 1.25 x (16 CTAs x 8 warps x SMs x 512) edges: every warp of the 512-edge statistics
    kernel, and so of every edge kernel with a smaller quantum, reaches its second quantum."""
    from neutronstarlite_b200 import ops, synth
    from neutronstarlite_b200.graph import PartitionedGraph
    dv = dev()
    free, _ = torch.cuda.mem_get_info()
    if free < 20e9:
        pytest.skip("needs ~12 GB of free device memory")
    t0 = time.perf_counter()
    threshold = 16 * 8 * sm_count() * 512
    V = 200_000
    src, dst = synth.zipf_edges(V, int(1.3 * threshold) - V, dv)
    pg = PartitionedGraph.from_device_edges(src, dst, V, dist=True)
    del src, dst
    assert pg.owned_edges >= 1.25 * threshold, (pg.owned_edges, threshold)
    off = pg.column_offset_gpu.long()
    slot = ops.DistGPUFusedGATOp.slot_indices(pg).long()
    torch.cuda.synchronize()
    print("zipf graph: %d edges (threshold %d), built in %.1f s" % (pg.owned_edges, threshold,
                                                                    time.perf_counter() - t0))
    yield pg, off, slot
    del pg, off, slot
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41)])
def test_fused_gat_layer_past_the_grid_stride_boundary(zipf_graph, H, D):
    """Config D's 8 x 8 hidden layer and 41-wide output layer on > 10 M edges (the production quantum Q = 512 / 256),
    both backwards, against the chunked float64 reference."""
    pg, off, slot = zipf_graph
    t0 = time.perf_counter()
    inputs = layer_inputs(pg.owned_mirrors, pg.owned_vertices, H, D, seed=10 + H, device=off.device)
    ref = analytic_reference(off, slot, *inputs, H, 0.2)
    for two_pass in (True, False):
        got, (seg_max, seg_sum), _ = run_k7(pg, *inputs, 0.2, two_pass)
        check_stats(seg_max, seg_sum, ref, np.nonzero(np.diff(np64(off)) == 0)[0])
        check_layer(got, ref)
    print("large-graph K7 %dx%d: %.1f s" % (H, D, time.perf_counter() - t0))
