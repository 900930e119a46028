"""The GCN aggregation on the reference layout (K1: segment_gather_sum_kernel in head mode 0, csrc/nts_aggregate.cu,
through nts_segment_gather_sum, _slots and _range) against float64, at every NTS_CASE instantiation.

Reference: `reference`, float64 `init + A X` by index_add_ in edge chunks, on the device of the inputs.

Exact mode (the main check): weights in {+-1/4, +-1/2, +-1, +-2}, integer features in [-8, 8], an integer initial
output, and max_row(deg * max|w| * max|x|) + max|init| < 2^22 asserted for every input.  Every partial sum is then a
multiple of 1/4 below 2^22, exact in FP32 whatever the order (`red` flushes, quantum cuts, split K, slab order), and
every feature is exact in BF16.  The kernel must give the reference bit for bit (`torch.equal`): a dropped, doubled or
misplaced edge or column chunk fails anywhere, inside the 20 011-edge hub row too.

Random mode (rounding): uniform features and weights, per element |y - y64| <= 1e-4 (|init| + |A| |X|).  For BF16
gathers the reference is evaluated at X.to(bfloat16).  The CPU tests show that this bound rejects one edge dropped from
a row of at most 64 edges and a BF16 result computed at the unrounded X.

The graph is `Structured` of test_gat_fp32_reference (empty rows, rows ending on 64 / 256 / 512 edges, rows of 4096,
4097 and 20 011 edges, duplicate edges, a hub source), cut to E % 4 = 0, 1, 2 and 3 edges: the bulk-staged variant
copies whole 16-byte units and loads the last 1-3 indices one by one.

Every (VEC, K, U, MINB) point of `K1_CASES` runs with both index-staging variants (nts_aggregate_set_variant 1 and 2),
through a non-zero index base and through a slot table, and nts_aggregate_last_shape must report that point.  Default
points are reached by width and by input / output views offset by 1 or 2 floats (4- or 8-byte aligned rows), the
others by NTS_AGG_TUNE; `test_k1_table_matches_the_source` keeps the table equal to the NTS_CASE lines."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from test_gat_fp32_reference import structured

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "neutronstarlite_b200", "csrc")
EXACT_LIMIT = 2.0 ** 22
WEIGHTS = np.array([-2.0, -1.0, -0.5, -0.25, 0.25, 0.5, 1.0, 2.0], dtype=np.float32)
BASE = 3 * (1 << 20) + 5          # index base of the base-addressed runs: indices are global id + BASE
RTOL = 1e-4


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream().cuda_stream


def cdiv(a, b):
    return -(-a // b)


# ---- the graph ---------------------------------------------------------------------------------------------------------
class Trimmed:
    """The structured graph cut to its first E edges, E % 4 == r (the last rows lose up to 3 edges).
    idx: global source ids; mi: the MirrorIndex (slot of id g = mi[g]); ids: the global id of every slot."""

    def __init__(self, r):
        st = structured()
        self.E = st.E - (st.E - r) % 4
        self.off = np.minimum(st.off.astype(np.int64), self.E)
        self.idx = st.idx[:self.E].astype(np.int64)
        self.mi = st.mi
        self.ids = np.nonzero(np.diff(st.mi.astype(np.int64)))[0]
        self.n_rows, self.Vg, self.M = st.Vp, st.mi.size - 1, st.M
        self.deg = np.diff(self.off)
        self.hub_row = st.hub_row
        self.dst = np.repeat(np.arange(self.n_rows), self.deg)
        self._dev = None

    def device(self):
        """Device arrays: off, idx + BASE, idx (global), mi (uint32 as int32), and dst / idx as int64."""
        if self._dev is None:
            d = dev()
            self._dev = dict(off=u32(self.off, d), idx_base=u32(self.idx + BASE, d), idx=u32(self.idx, d),
                             mi=u32(self.mi, d), dst64=torch.from_numpy(self.dst).to(d),
                             src64=torch.from_numpy(self.idx).to(d))
        return self._dev


_TRIMMED = {}


def trimmed(r):
    if r not in _TRIMMED:
        _TRIMMED[r] = Trimmed(r)
    return _TRIMMED[r]


def u32(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64).astype(np.uint32).view(np.int32)).to(device)


# ---- references and comparators --------------------------------------------------------------------------------------
def reference(dst, src, w, X, init, chunk_elems=1 << 24):
    """float64 (init + A X, |init| + |A| |X|): row dst[e] gets w[e] * X[src[e]] (w None: 1), on X's device."""
    f8 = torch.float64
    X64 = X.to(f8)
    out = init.to(f8).clone()
    mag = init.to(f8).abs()
    chunk = max(1024, chunk_elems // max(1, X.shape[1]))
    for e0 in range(0, dst.numel(), chunk):
        e1 = min(dst.numel(), e0 + chunk)
        x = X64[src[e0:e1]]
        d = dst[e0:e1]
        if w is None:
            out.index_add_(0, d, x)
            mag.index_add_(0, d, x.abs())
        else:
            ww = w[e0:e1].to(f8)[:, None]
            out.index_add_(0, d, x * ww)
            mag.index_add_(0, d, x.abs() * ww.abs())
    return out, mag


def assert_exact_range(deg, w, X, init):
    """Every partial sum of every row is a multiple of 1/4 below 2^22: exact in FP32 in any order."""
    mw = 1.0 if w is None else float(np.abs(w).max())
    bound = float(deg.max()) * mw * float(np.abs(X).max()) + float(np.abs(init).max())
    assert bound < EXACT_LIMIT, bound
    assert np.all(X == np.round(X)) and np.all(init == np.round(init))
    assert w is None or np.all(w * 4 == np.round(w * 4))


def exact_inputs(g, F, seed, rows=None):
    """Integer features [rows or Vg, F], weights in quarters [E], integer initial output [n_rows, F]."""
    rng = np.random.default_rng(seed)
    X = rng.integers(-8, 9, (rows or g.Vg, F)).astype(np.float32)
    w = rng.choice(WEIGHTS, g.E).astype(np.float32)
    init = rng.integers(-64, 65, (g.n_rows, F)).astype(np.float32)
    assert_exact_range(g.deg, w, X, init)
    return X, w, init


def random_inputs(g, F, seed, rows=None):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (rows or g.Vg, F)).astype(np.float32)
    w = rng.uniform(-1, 1, g.E).astype(np.float32)
    init = rng.uniform(-1, 1, (g.n_rows, F)).astype(np.float32)
    return X, w, init


def check_exact(got, ref, rows=None):
    """got (FP32) == ref (float64) element for element, on `rows` (default all)."""
    a = got.double() if rows is None else got[rows].double()
    b = ref if rows is None else ref[rows]
    if not torch.equal(a, b):
        bad = torch.nonzero(a != b)
        r, c = bad[0].tolist()
        raise AssertionError("%d elements differ, first at (row %d, col %d): %r vs %r; rows %s" % (
            bad.shape[0], r, c, float(a[r, c]), float(b[r, c]), torch.unique(bad[:, 0])[:8].tolist()))


def check_random(got, ref, mag, rtol=RTOL):
    """|got - ref| <= rtol * (|init| + |A| |X|) per element (a NaN fails)."""
    err = (got.double() - ref).abs()
    bad = torch.nonzero(~(err <= rtol * mag))
    if bad.numel():
        r, c = bad[0].tolist()
        raise AssertionError("%d elements out of bound, first (row %d, col %d): err %g vs bound %g" % (
            bad.shape[0], r, c, float(err[r, c]), rtol * float(mag[r, c])))


# ---- the K1 dispatch, mirrored -----------------------------------------------------------------------------------------
def k1_point(F, align, tune=None, tiles=None):
    """((VEC, K, U, MINB, tiles), tile_major) that segment_gather_sum picks in head mode 0 for F columns whose input and
    output rows are `align`-byte aligned, under NTS_AGG_TUNE = tune and NTS_AGG_TILES = tiles."""
    vec = 4 if F % 4 == 0 and align % 16 == 0 else (2 if F % 2 == 0 and align % 8 == 0 else 1)
    nvec = F // vec
    chunks = cdiv(nvec, 32)
    kmax = 4 if vec == 4 else 5
    n_tiles, tile_major = cdiv(chunks, kmax), 0
    if tiles is not None and 1 <= tiles[0] <= chunks and cdiv(chunks, tiles[0]) <= kmax:
        n_tiles, tile_major = tiles[0], int(bool(tiles[1]))
    tile_vecs = cdiv(nvec, n_tiles)
    k = cdiv(tile_vecs, 32)
    n_tiles = cdiv(nvec, tile_vecs)
    budget = 40 // (k * vec)
    u, minb = (8 if budget >= 8 else (4 if budget >= 4 else 2)), 1
    if (vec, k) == (2, 5):
        u, minb = 2, 2
    elif (vec, k) == (4, 1):
        u, minb = 4, 4
    if tune is not None:
        u, minb = tune
    return (vec, k, u, minb, n_tiles), tile_major


def k1_launch(n_edges, tiles, tile_major, variant, Q=0, sms=None):
    """(grid, smem, variant) of a head-mode-0 launch over n_edges edges (nts_aggregate_set_variant(variant, Q))."""
    if Q == 0:
        Q = 512
        while Q > 32 and cdiv(n_edges, Q) * tiles < sms * 64:
            Q >>= 1
    Q = cdiv(Q, 32) * 32
    quanta = cdiv(n_edges, Q)
    warps = cdiv(quanta, 8) * 8 * tiles if tile_major else quanta * tiles
    bulk = variant != 1
    return cdiv(warps, 8), (16 + 2 * (8 * Q + 8) * 4) if bulk else 0, 2 if bulk else 1


# (VEC, K, U, MINB), F, (input, output) view offsets in floats, NTS_AGG_TUNE.  An offset of 1 float leaves rows 4-byte
# aligned (VEC 1), 2 floats 8-byte aligned (VEC 2 at most).
K1_CASES = [
    # default points
    ((4, 1, 4, 4), 128, (0, 0), None),
    ((4, 2, 4, 1), 200, (0, 0), None),
    ((4, 3, 2, 1), 300, (0, 0), None),
    ((4, 4, 2, 1), 500, (0, 0), None),
    ((2, 1, 8, 1), 42, (0, 0), None),
    ((2, 2, 8, 1), 128, (2, 0), None),
    ((2, 3, 4, 1), 150, (0, 0), None),
    ((2, 4, 4, 1), 256, (0, 2), None),
    ((2, 5, 2, 2), 602, (0, 0), None),
    ((1, 1, 8, 1), 7, (0, 0), None),
    ((1, 2, 8, 1), 64, (1, 0), None),
    ((1, 3, 8, 1), 95, (0, 0), None),
    ((1, 4, 8, 1), 100, (1, 1), None),
    ((1, 5, 8, 1), 133, (0, 0), None),
    # NTS_AGG_TUNE points
    ((4, 1, 8, 1), 124, (0, 0), (8, 1)),
    ((4, 1, 8, 4), 4, (0, 0), (8, 4)),
    ((4, 1, 16, 2), 96, (0, 0), (16, 2)),
    ((4, 1, 8, 3), 112, (0, 0), (8, 3)),
    ((2, 5, 4, 1), 602, (0, 0), (4, 1)),
    ((2, 5, 2, 3), 578, (0, 0), (2, 3)),
    ((2, 5, 4, 2), 320, (2, 2), (4, 2)),
    ((2, 4, 2, 3), 250, (0, 0), (2, 3)),
    ((2, 4, 4, 2), 200, (2, 0), (4, 2)),
    ((2, 3, 2, 3), 190, (0, 0), (2, 3)),
    ((2, 3, 4, 3), 162, (0, 0), (4, 3)),
    ((2, 3, 4, 2), 192, (0, 2), (4, 2)),
    ((2, 2, 4, 3), 98, (0, 0), (4, 3)),
    ((2, 2, 4, 4), 66, (0, 0), (4, 4)),
    ((2, 2, 8, 2), 120, (2, 2), (8, 2)),
    ((2, 2, 8, 3), 126, (0, 0), (8, 3)),
    ((2, 1, 8, 4), 62, (0, 0), (8, 4)),
    ((2, 1, 8, 3), 2, (0, 0), (8, 3)),
    ((2, 1, 16, 2), 64, (2, 2), (16, 2)),
]


def view_align(shifts):
    """Byte alignment of both row views offset by `shifts` floats from 16-byte aligned allocations."""
    a = 16
    for s in shifts:
        a = min(a, 16 if s % 4 == 0 else (8 if s % 2 == 0 else 4))
    return a


def shifted(t, shift):
    """t as a view that starts `shift` floats into a fresh allocation."""
    flat = torch.empty(t.numel() + shift, dtype=t.dtype, device=t.device)
    v = flat[shift:].view(t.shape)
    v.copy_(t)
    return v


def last_k1():
    from neutronstarlite_b200 import _lib
    rec = [C.c_int() for _ in range(4)]
    _lib.call("nts_aggregate_last_launch", *[C.byref(r) for r in rec])
    shape = [C.c_int() for _ in range(5)]
    _lib.call("nts_aggregate_last_shape", *[C.byref(r) for r in shape])
    return tuple(r.value for r in rec), tuple(r.value for r in shape)


def run_k1(g, X, w, init, addr, variant, Q=0, shifts=(0, 0), idx_shift=0):
    """init + A X through nts_segment_gather_sum (addr 'base': indices global id + BASE) or _slots (addr 'slot':
    indices global ids through the MirrorIndex, X given per slot).  X, w, init: device tensors (w may be None).
    Returns the output and the launch record ((grid, block, smem, variant), (vec, k, u, minb, tiles))."""
    from neutronstarlite_b200 import _lib
    a = g.device()
    x = shifted(X, shifts[0])
    out = shifted(init, shifts[1])
    idx = a["idx_base"] if addr == "base" else a["idx"]
    if idx_shift:
        idx = shifted(idx, idx_shift)
    wp = None if w is None else w.data_ptr()
    _lib.call("nts_aggregate_set_variant", variant, Q)
    if addr == "base":
        _lib.call("nts_segment_gather_sum", x.data_ptr(), out.data_ptr(), wp, idx.data_ptr(), a["off"].data_ptr(),
                  BASE, g.n_rows, g.E, X.shape[1], stream())
    else:
        _lib.call("nts_segment_gather_sum_slots", x.data_ptr(), out.data_ptr(), wp, idx.data_ptr(),
                  a["off"].data_ptr(), a["mi"].data_ptr(), g.n_rows, g.E, X.shape[1], stream())
    torch.cuda.synchronize()
    return out, last_k1()


class hooks:
    """Restores the K1 and K1P measurement hooks on exit, whatever happened inside."""

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        from neutronstarlite_b200 import _lib
        _lib.call("nts_aggregate_set_variant", 0, 0)
        _lib.call("nts_gather_plan_set_tuning", 0, 0, 0)
        _lib.call("nts_gather_plan_set_variant", 0)
        return False


def sm_count():
    from test_gat_fp32_reference import sm_count as sms
    return sms()


def device_inputs(g, X, w, init, weighted=True):
    """Device copies: X per global id, X per slot, w (or None), init."""
    d = dev()
    Xg = torch.from_numpy(X).to(d)
    return Xg, Xg[torch.from_numpy(g.ids).to(d)].contiguous(), torch.from_numpy(w).to(d) if weighted else None, \
        torch.from_numpy(init).to(d)


# ---- CPU: inputs, comparators, tables ------------------------------------------------------------------------------------
def test_trimmed_graphs_keep_the_structure_and_every_tail_length():
    st = structured()
    for r in range(4):
        g = trimmed(r)
        assert g.E % 4 == r and st.E - 3 <= g.E <= st.E
        assert g.deg[g.hub_row] == 20011 and (g.deg == 0).sum() > 100
        assert (g.deg == 4096).any() and (g.deg == 4097).any()
        X, w, init = exact_inputs(g, 8, seed=r)
        assert_exact_range(g.deg, w, X, init)
        # the largest row stays far below the exact range: 20 011 edges x 2 x 8 + 64
        assert float(g.deg.max()) * 2 * 8 + 64 < EXACT_LIMIT / 8


def test_exact_range_assertion_refuses_inputs_that_could_round():
    g = trimmed(0)
    X, w, init = exact_inputs(g, 4, seed=0)
    with pytest.raises(AssertionError):
        assert_exact_range(g.deg, w * 64, X, init)
    with pytest.raises(AssertionError):
        assert_exact_range(g.deg, w, X + 0.5, init)


def cpu_reference(g, X, w, init):
    return reference(torch.from_numpy(g.dst), torch.from_numpy(g.idx), None if w is None else torch.from_numpy(w),
                     torch.from_numpy(X), torch.from_numpy(init))


def test_random_bound_accepts_fp32_rounding_and_rejects_one_dropped_edge():
    """The float32 rounding of the float64 result passes; the same result with one edge dropped from a row of at most
    64 edges fails, in every such row tried."""
    g = trimmed(1)
    X, w, init = random_inputs(g, 16, seed=3)
    ref, mag = cpu_reference(g, X, w, init)
    check_random(ref.float(), ref, mag)
    rows = np.nonzero((g.deg > 0) & (g.deg <= 64))[0]
    rng = np.random.default_rng(4)
    for r in rng.choice(rows, 5, replace=False).tolist() + [int(rows[-1])]:
        e = int(g.off[r] + rng.integers(0, g.deg[r]))
        dropped = ref.clone()
        dropped[r] -= float(w[e]) * torch.from_numpy(X[g.idx[e]]).double()
        with pytest.raises(AssertionError):
            check_random(dropped.float(), ref, mag)


def test_random_bound_rejects_a_bf16_result_taken_at_the_unrounded_features():
    """BF16 gathers are checked against the reference at bf16(X): a result computed at X itself fails the bound."""
    g = trimmed(2)
    X, w, init = random_inputs(g, 16, seed=5)
    Xb = torch.from_numpy(X).to(torch.bfloat16).float().numpy()
    ref_b, mag_b = cpu_reference(g, Xb, w, init)
    check_random(ref_b.float(), ref_b, mag_b)
    unrounded, _ = cpu_reference(g, X, w, init)
    with pytest.raises(AssertionError):
        check_random(unrounded.float(), ref_b, mag_b)


def read_source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def source_cases(text, macro):
    """The integer argument tuples of every `macro(...)` use in text (the #define line excluded)."""
    return [tuple(int(v) for v in m.split(","))
            for m in re.findall(r"^\s*%s\(\s*([0-9,\s]+)\)" % re.escape(macro), text, flags=re.M)]


def test_k1_table_matches_the_source():
    """Every NTS_CASE instantiation of segment_gather_sum has exactly one row in K1_CASES, and no row names a point that
    is not instantiated: a new instantiation without a test point fails here."""
    src = source_cases(read_source("nts_aggregate.cu"), "NTS_CASE")
    assert len(src) == len(set(src)) >= 33
    table = [c[0] for c in K1_CASES]
    assert len(table) == len(set(table))
    assert sorted(table) == sorted(src)


def test_k1_table_points_follow_the_dispatch_rule():
    """The mirror of pick_shape reaches every table point from its width, alignment and tuning hook; default rows need
    no hook, tuned rows would not be reached without it."""
    for point, F, shifts, tune in K1_CASES:
        (got, _) = k1_point(F, view_align(shifts), tune)
        assert got[:4] == point, (point, F, shifts, tune, got)
        if tune is not None:
            assert k1_point(F, view_align(shifts))[0][:4] != point, (point, "reached without the hook")


# ---- GPU: every instantiation ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(K1_CASES)), ids=["v%dk%du%db%d" % c[0] for c in K1_CASES])
def test_every_k1_point_exact(case, monkeypatch):
    """Both staging variants x (index base, slot table), one of the four without weights; bit-exact results and the
    launch record of the point."""
    point, F, shifts, tune = K1_CASES[case]
    g = trimmed(case % 4)
    X, w, init = exact_inputs(g, F, seed=100 + case)
    Xg, Xs, wd, initd = device_inputs(g, X, w, init)
    a = g.device()
    ref, _ = reference(a["dst64"], a["src64"], wd, Xg, initd)
    ref_unweighted, _ = reference(a["dst64"], a["src64"], None, Xg, initd)
    if tune is not None:
        monkeypatch.setenv("NTS_AGG_TUNE", "%d,%d" % tune)
    want, tm = k1_point(F, view_align(shifts), tune)
    assert want[:4] == point
    with hooks():
        for variant in (1, 2):
            for addr in ("base", "slot"):
                unweighted = addr == "slot" and variant == 1 + case % 2
                out, (rec, shape) = run_k1(g, Xg if addr == "base" else Xs, None if unweighted else wd, initd, addr,
                                           variant, shifts=shifts)
                assert shape == want, (variant, addr, shape, want)
                assert rec[3] == variant and rec[1] == 256
                assert (rec[0], rec[2], rec[3]) == k1_launch(g.E, want[4], tm, variant, sms=sm_count())
                check_exact(out, ref_unweighted if unweighted else ref)


@pytest.mark.gpu
@pytest.mark.parametrize("F,tiles", [(602, t) for t in range(2, 11)] + [(1433, t) for t in (9, 12, 23, 45)])
def test_tile_major_order_exact(F, tiles, monkeypatch):
    """NTS_AGG_TILES = "t,1": all quanta of column tile 0 first, then tile 1, ...  (warps per tile padded to whole CTAs).
    F = 602 is VEC 2 with 2-10 tiles (K 5 down to 1), F = 1433 VEC 1 with 9-45 tiles (K 5 down to 1)."""
    g = trimmed(tiles % 4)
    X, w, init = exact_inputs(g, F, seed=200 + F + tiles)
    Xg, Xs, wd, initd = device_inputs(g, X, w, init)
    a = g.device()
    ref, _ = reference(a["dst64"], a["src64"], wd, Xg, initd)
    monkeypatch.setenv("NTS_AGG_TILES", "%d,1" % tiles)
    want, tm = k1_point(F, 16, tiles=(tiles, 1))
    assert tm == 1 and want[4] == tiles
    with hooks():
        for variant, addr in ((1, "base"), (2, "slot")):
            out, (rec, shape) = run_k1(g, Xg if addr == "base" else Xs, wd, initd, addr, variant)
            assert shape == want
            assert (rec[0], rec[2], rec[3]) == k1_launch(g.E, tiles, 1, variant, sms=sm_count())
            check_exact(out, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [128, 602, 41])
def test_quantum_sizes_and_unaligned_indices_exact(F):
    """Q = 32, 64, 512 and the default shrink, both variants.  An index array that starts one element into its
    allocation cannot be bulk-copied: the launch falls back to variant 1, and the record says so."""
    g = trimmed(3)
    X, w, init = exact_inputs(g, F, seed=300 + F)
    Xg, Xs, wd, initd = device_inputs(g, X, w, init)
    a = g.device()
    ref, _ = reference(a["dst64"], a["src64"], wd, Xg, initd)
    want, _ = k1_point(F, 16)
    sms = sm_count()
    with hooks():
        for variant in (1, 2):
            for Q in (32, 64, 512, 0):
                for addr in ("base", "slot"):
                    out, (rec, shape) = run_k1(g, Xg if addr == "base" else Xs, wd, initd, addr, variant, Q=Q)
                    assert shape == want
                    assert (rec[0], rec[2], rec[3]) == k1_launch(g.E, want[4], 0, variant, Q, sms), (variant, Q)
                    check_exact(out, ref)
        for variant in (0, 2):
            for addr in ("base", "slot"):
                out, (rec, _) = run_k1(g, Xg if addr == "base" else Xs, wd, initd, addr, variant, idx_shift=1)
                assert (rec[0], rec[2], rec[3]) == k1_launch(g.E, want[4], 0, 1, sms=sms)
                check_exact(out, ref)


def range_rows(g, kind):
    """(r0, r1) of a row range: 'unaligned' starts at an edge position with e % 4 != 0, 'boundary' at row 6 (edge 512,
    a 512-edge quantum boundary of the whole-array launch), 'hub' at the 20 011-edge row, 'tail' runs to the last row."""
    off = g.off
    if kind == "unaligned":
        r0 = next(r for r in range(20, g.n_rows) if off[r] % 4 == 3 and g.deg[r] > 0)
        return r0, r0 + 700
    if kind == "boundary":
        assert off[6] == 512
        return 6, 400
    if kind == "hub":
        assert off[g.hub_row] % 4 != 0
        return g.hub_row, g.hub_row + 300
    r0 = next(r for r in range(g.n_rows - 500, g.n_rows) if off[r] % 4 == 2)
    return r0, g.n_rows


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["unaligned", "boundary", "hub", "tail"])
@pytest.mark.parametrize("F", [128, 602, 41])
def test_row_range_launch_exact(kind, F):
    """nts_segment_gather_sum_range on rows [r0, r1): offsets and output at row r0, indices and weights the whole arrays.
    Range rows exact, every other row keeps its NaN.  Both variants, Q default and 64, index base and slot table."""
    from neutronstarlite_b200 import _lib
    g = trimmed({"unaligned": 1, "boundary": 2, "hub": 3, "tail": 1}[kind])
    r0, r1 = range_rows(g, kind)
    e0, e1 = int(g.off[r0]), int(g.off[r1])
    X, w, init = exact_inputs(g, F, seed=400 + F + r0)
    Xg, Xs, wd, initd = device_inputs(g, X, w, init)
    a = g.device()
    nan = torch.full_like(initd, float("nan"))
    start = nan.clone()
    start[r0:r1] = initd[r0:r1]
    ref, _ = reference(a["dst64"], a["src64"], wd, Xg, start)
    want, _ = k1_point(F, 16)
    sms = sm_count()
    with hooks():
        for variant in (1, 2):
            for Q in (0, 64):
                for addr in ("base", "slot"):
                    out = start.clone()
                    _lib.call("nts_aggregate_set_variant", variant, Q)
                    _lib.call("nts_segment_gather_sum_range", (Xg if addr == "base" else Xs).data_ptr(),
                              out[r0].data_ptr(), wd.data_ptr(),
                              (a["idx_base"] if addr == "base" else a["idx"]).data_ptr(),
                              a["off"][r0].data_ptr(), None if addr == "base" else a["mi"].data_ptr(), BASE, r1 - r0,
                              e0, e1, F, stream())
                    torch.cuda.synchronize()
                    rec, shape = last_k1()
                    assert shape == want
                    assert (rec[0], rec[2], rec[3]) == k1_launch(e1 - e0, want[4], 0, variant, Q, sms)
                    check_exact(out, ref, rows=slice(r0, r1))
                    outside = torch.cat([out[:r0], out[r1:]])
                    assert bool(torch.isnan(outside).all()), "a row outside the range was written"


@pytest.mark.gpu
@pytest.mark.parametrize("case", [i for i, c in enumerate(K1_CASES) if c[3] is None])
def test_default_points_random_within_rounding(case):
    """Uniform features and weights at every default point (default variant and quantum): per element within
    1e-4 (|init| + |A| |X|) of float64."""
    point, F, shifts, _ = K1_CASES[case]
    g = trimmed(case % 4)
    X, w, init = random_inputs(g, F, seed=500 + case)
    Xg, Xs, wd, initd = device_inputs(g, X, w, init)
    a = g.device()
    ref, mag = reference(a["dst64"], a["src64"], wd, Xg, initd)
    with hooks():
        for addr in ("base", "slot"):
            out, (rec, shape) = run_k1(g, Xg if addr == "base" else Xs, wd, initd, addr, 0, shifts=shifts)
            assert shape[:4] == point and rec[3] == 2
            check_random(out, ref, mag)
