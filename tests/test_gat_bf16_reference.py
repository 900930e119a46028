"""The BF16 fused GAT layer (K7: nts_gat_fused_aggregate_forward_bf16, nts_gat_fused_aggregate_backward_two_pass_bf16,
ops.DistGPUFusedGATOp / MiniBatchGATOp with gather_dtype=torch.bfloat16) against float64, at every dispatch branch the
(H, D) grid below reaches.

Precision contract (DESIGN §3 K7 with BF16 gathers): with m~ = bf16(mirror) and g~ = bf16(grad_out), the layer IS the
FP32 layer evaluated at m~ and g~.  So the reference is test_gat_fp32_reference.analytic_reference at the rounded
operands, and the bounds are check_layer's FP32 bounds, unchanged: nothing about BF16 gathers loosens the FP32
accumulation.  The CPU tests show that those bounds see the contract broken (a result at the unrounded mirror or the
unrounded gradient, out_dot_g from g instead of g~, one edge dropped or doubled), and pin the shape rule of both entries
without a device.

The structured graph, the float64 reference, the comparators and the Zipf graph fixture are those of
test_gat_fp32_reference.py; the sampled hub block is test_gat_sample_gpu.hub_block()."""
import ctypes
import time

import numpy as np
import pytest

from test_gat_fp32_reference import (ONE_SRC, SLOPES, analytic_reference, check_exact_zeros, check_layer, check_stats,
                                     layer_inputs, np64, ptr, reference_without, run_k7, sm_count, stream, structured,
                                     zipf_graph)  # noqa: F401  (zipf_graph is a fixture)
from test_gather_plan_bf16 import row_close

torch = pytest.importorskip("torch")

BF16 = torch.bfloat16


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def rounded(t):
    return t.to(BF16).float()


# ---- the (H, D) grid -------------------------------------------------------------------------------------------------
# (H, D, forward column tiles, forward virtual warps G).  Branches, read from the dispatch code, on rows of
# ld = ceil(H*D / 8) * 8 BF16 values:
#   forward (gat_forward_bf16): nvec = ld / 8 chunks; tiles from ceil(nvec / 32) lane chunks, at most 4 per tile;
#     K = ceil(tile_vecs / 32); U = 2 / 4 / 2 / 2 at K = 1 / 2 / 3 / 4; G = 4 / 2 / 1 at nvec <= 8 / <= 16 / more
#     (one tile of K = 1 only).  Its edge quantum Q = 512 / G, halved down to 32 while the grid would not fill the GPU
#     (always 32 on the structured graph), is its own: nts_aggregate_set_variant does not reach it.
#   backward (nts_gat_fused_aggregate_backward_two_pass_bf16): VEC 8, halved (down to 2) while ld / VEC < 32;
#     nvec = ld / VEC, hv = nvec / H, kb = ceil(nvec / 32): NTS_GAT2B(VEC, KB, U dst-major, U src-major, ONEHEAD) of
#     NTS_GAT2B_ONE; kb 3 runs the KB 4 instantiation with its 4th chunk inactive.  No fallback.
# Every NTS_GAT16 line with U = 2 / 4 at its default point, and all 14 NTS_GAT2B calls (7 per ONEHEAD value), are
# reached below; the U = 4 / 8 one-chunk points that only NTS_GAT_BF16_TUNE reaches are in test_tune_points.
GRID = [
    # ld 8: fwd K 1 U 2 G 4 (NTS_GAT16(1, 2, 4)).  bwd VEC 2 nvec 4 KB 1 (U 8 / 4), ONEHEAD
    (1, 8, 1, 4),
    # ld 64: fwd K 1 U 2 G 4, 8 heads of one chunk.  bwd VEC 2 nvec 32 KB 1 (U 4 / 4), hv 4
    (8, 8, 1, 4),
    # ld 48 (7 zero pad columns): fwd K 1 U 2 G 4.  bwd VEC 2 nvec 24 KB 1 (U 8 / 4), ONEHEAD, lanes 24-31 idle
    (1, 41, 1, 4),
    # ld 96: fwd K 1 U 2 G 2 (NTS_GAT16(1, 2, 2)), 12 chunks.  bwd VEC 2 nvec 48 KB 2 (U 2 / 2), hv 16
    (3, 32, 1, 2),
    # ld 104 (4 pad): fwd K 1 U 2 G 2, 13 chunks.  bwd VEC 2 nvec 52 KB 2 (U 2 / 4), ONEHEAD, 2nd chunk partly active
    (1, 100, 1, 2),
    # ld 128: fwd K 1 U 2 G 2, 16 chunks (a full 16-lane virtual warp).  bwd VEC 4 nvec 32 KB 1 (U 4 / 4), hv 8
    (4, 32, 1, 2),
    # ld 128: fwd as above, one head.  bwd VEC 4 KB 1, ONEHEAD
    (1, 128, 1, 2),
    # ld 200: fwd K 1 U 2 G 1 (NTS_GAT16(1, 2, 1)), 25 chunks.  bwd VEC 4 nvec 50 KB 2 (U 2 / 2), ONEHEAD
    (1, 200, 1, 1),
    # ld 192: fwd K 1 U 2 G 1, 24 chunks.  bwd VEC 4 nvec 48 KB 2, hv 16
    (3, 64, 1, 1),
    # ld 256: fwd K 1 U 2 G 1, 32 chunks, one head per chunk.  bwd VEC 8 nvec 32 KB 1 (U 4 / 4), hv 1
    (32, 8, 1, 1),
    # ld 256: fwd as above, one head.  bwd VEC 8 KB 1, ONEHEAD
    (1, 256, 1, 1),
    # ld 304: fwd K 2 U 4 G 1 (NTS_GAT16(2, 4, 1)), 38 chunks.  bwd VEC 8 nvec 38 KB 2 (U 2 / 4), ONEHEAD
    (1, 300, 1, 1),
    # ld 512: fwd K 2 U 4 G 1, 64 chunks.  bwd VEC 8 nvec 64 KB 2 (U 2 / 2), hv 8
    (8, 64, 1, 1),
    # ld 512: fwd K 2.  bwd VEC 8 KB 2, hv 32 (the largest power of two a head may have)
    (2, 256, 1, 1),
    # ld 608: fwd K 3 U 2 G 1 (NTS_GAT16(3, 2, 1)), 76 chunks: the lanes' 3rd chunk partly active.  bwd VEC 8 nvec 76
    # kb 3 -> the KB 4 instantiation (U 1 / 1), ONEHEAD
    (1, 602, 1, 1),
    # ld 768: fwd K 3, 96 chunks.  bwd VEC 8 nvec 96 kb 3 -> KB 4, hv 16
    (6, 128, 1, 1),
    # ld 1000: fwd K 4 U 2 G 1 (NTS_GAT16(4, 2, 1)), 125 chunks.  bwd VEC 8 nvec 125 KB 4, ONEHEAD, the 4th chunk
    # active on 29 lanes
    (1, 1000, 1, 1),
    # ld 1024: fwd K 4, 128 chunks.  bwd VEC 8 nvec 128 KB 4, hv 16
    (8, 128, 1, 1),
]

# forward accepted, backward refused (no two-pass shape, and no fallback): (H, D, tiles, G)
FORWARD_ONLY = [
    # ld 96: fwd K 1 G 2.  bwd VEC 2 nvec 48, hv 24 is not a power of two
    (2, 48, 1, 2),
    # ld 320: fwd K 2.  bwd VEC 8 nvec 40, hv 10
    (4, 80, 1, 1),
    # ld 600: fwd K 3 (75 chunks).  bwd VEC 8 nvec 75, hv 25
    (3, 200, 1, 1),
    # ld 192: fwd K 1 G 1.  bwd VEC 4 nvec 48, hv 6
    (8, 24, 1, 1),
    # ld 1440: fwd 180 chunks, 2 tiles of 90 (K 3).  bwd kb 6 > 4
    (1, 1433, 2, 1),
    # ld 2048: fwd 256 chunks, 2 tiles of 128 (K 4).  bwd kb 8
    (8, 256, 2, 1),
    # ld 2000: fwd 250 chunks, 2 tiles of 125 (K 4); head boundaries at chunks 50 / 100 / 150 / 200 fall inside a tile
    # and inside a lane's chunks.  bwd kb 8
    (5, 400, 2, 1),
]

# both refused by the layout check (heads > 1 need D % 8 == 0): (H, D)
BOTH_REFUSED = [(3, 5), (16, 4)]

# (H, D) -> (forward accepts, backward accepts)
SHAPE_RULE = {**{(H, D): (True, True) for H, D, _, _ in GRID},
              **{(H, D): (True, False) for H, D, _, _ in FORWARD_ONLY},
              **{(H, D): (False, False) for H, D in BOTH_REFUSED}}


def expected_launch(E, tiles, G):
    """(grid, block, smem, variant) of gat_forward_bf16 over E edges in `tiles` column tiles with G virtual warps: 8 * G
    virtual warps per CTA, each over Q edges, the CTA's indices and weights staged in shared memory."""
    Q = 512 // G
    while Q > 32 and -(-E // Q) * tiles < sm_count() * 64:
        Q >>= 1
    Q = (Q + 31) // 32 * 32
    if Q * G > 1024:
        Q = (1024 // G) // 32 * 32
    kvw = 8 * G
    return -(-(-(-E // Q) * tiles) // kvw), 256, 16 + 2 * (kvw * Q + 8) * 4, 2


def bf16_entries():
    from neutronstarlite_b200 import _lib
    lib = _lib.load()
    return lib, lib.nts_gat_fused_aggregate_forward_bf16, lib.nts_gat_fused_aggregate_backward_two_pass_bf16


# ---- CPU: the comparator sees the contract broken ----------------------------------------------------------------------
def rounded_inputs(st, H, D, seed):
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=seed)
    return (m, s, d, g), (rounded(m), s, d, rounded(g))


def rejected(name, wrong, ref):
    """check_layer on the FP32-rounded reference, with only `name` taken from `wrong`, must fail (the rounded
    reference itself passes)."""
    got = [(wrong if k == name else ref)[k].float() for k in ("out", "dm", "ds", "dd")]
    with pytest.raises(AssertionError):
        check_layer(got, ref)


def test_comparator_rejects_a_result_at_the_unrounded_mirror():
    """out at m instead of m~ is off by up to 2^-9 per term: rejected in out, and through <m, g~> in ds and dd.
    d_mirror = sum a g~ does not read the mirror at all, so it must come out identical."""
    st = structured()
    H, D, slope = 2, 8, 0.2
    (m, s, d, g), (mt, _, _, gt) = rounded_inputs(st, H, D, seed=21)
    off, slot = st.torch_csc("cpu")
    ref = analytic_reference(off, slot, mt, s, d, gt, H, slope)
    check_layer([ref[k].float() for k in ("out", "dm", "ds", "dd")], ref)
    wrong = analytic_reference(off, slot, m, s, d, gt, H, slope)
    assert torch.equal(wrong["dm"], ref["dm"])
    for name in ("out", "ds", "dd"):
        rejected(name, wrong, ref)


def test_comparator_rejects_a_result_at_the_unrounded_gradient():
    """d_mirror, ds and dd at g instead of g~ are each rejected."""
    st = structured()
    H, D, slope = 2, 8, 0.2
    (m, s, d, g), (mt, _, _, gt) = rounded_inputs(st, H, D, seed=22)
    off, slot = st.torch_csc("cpu")
    ref = analytic_reference(off, slot, mt, s, d, gt, H, slope)
    wrong = analytic_reference(off, slot, mt, s, d, g, H, slope)
    for name in ("dm", "ds", "dd"):
        rejected(name, wrong, ref)


def test_comparator_rejects_out_dot_g_from_the_unrounded_gradient():
    """The bias DESIGN warns about: the passes use g~ but out_dot_g = <out, g> (not <out, g~>).  At slope 1 every
    leaky' is 1 and a segment's weights sum to 1, so dd moves by exactly <out, g~ - g>; that is rejected."""
    st = structured()
    H, D = 2, 8
    (m, s, d, g), (mt, _, _, gt) = rounded_inputs(st, H, D, seed=23)
    off, slot = st.torch_csc("cpu")
    ref = analytic_reference(off, slot, mt, s, d, gt, H, 1.0)
    out = ref["out"].view(st.Vp, H, D)
    shift = (out * (gt.double() - g.double()).view(st.Vp, H, D)).sum(-1)
    rejected("dd", {"dd": ref["dd"] - shift}, ref)


@pytest.mark.parametrize("where", ["hub", "quantum_boundary"])
@pytest.mark.parametrize("double", [False, True])
def test_comparator_rejects_one_edge_dropped_or_doubled_at_rounded_operands(where, double):
    """test_gat_fp32_reference's one-edge sensitivity, with m~ and g~ as the operands."""
    st = structured()
    H, D, slope = 2, 8, 0.2
    _, inputs = rounded_inputs(st, H, D, seed=24)
    off, slot = st.torch_csc("cpu")
    full = analytic_reference(off, slot, *inputs, H, slope)
    got = [full[k].float() for k in ("out", "dm", "ds", "dd")]
    check_layer(got, full)
    if where == "hub":
        b, e = int(st.off[st.hub_row]), int(st.off[st.hub_row + 1])
        s, d = inputs[1], inputs[2]
        edge = b + int((s[slot[b:e], 0] + d[st.hub_row, 0]).argmax())
    else:
        deg = np.diff(st.off.astype(np.int64))
        edge = next(q for q in range(512 * 40, st.E, 512) if deg[np.searchsorted(st.off, q, side="right") - 1] > 1)
    with pytest.raises(AssertionError):
        check_layer(got, reference_without(st, edge, H, inputs, slope, double))


# ---- CPU: the shape rule of both entries -------------------------------------------------------------------------------
def test_shape_table_matches_both_entries():
    """Both entries check layout and shape before their batch_size == 0 return, so batch 0 with null pointers gives
    the verdict without a device: 0 where the table accepts, an error where it refuses.  The backward names its
    two-pass rule, the forward (and the backward, which checks the layout first) the head-width rule."""
    from neutronstarlite_b200 import ops
    lib, fwd, bwd = bf16_entries()
    assert len(SHAPE_RULE) == len(GRID) + len(FORWARD_ONLY) + len(BOTH_REFUSED)
    for (H, D), (fwd_ok, bwd_ok) in SHAPE_RULE.items():
        F = H * D
        ld = (F + 7) // 8 * 8
        assert (fwd(*([None] * 9), 0, 0, F, ld, H, 0.2, None) == 0) == fwd_ok, (H, D)
        if not fwd_ok:
            assert b"head width" in lib.nts_last_error(), (H, D)
        assert (bwd(*([None] * 16), 0, 0, F, ld, H, 0.2, None) == 0) == bwd_ok, (H, D)
        if not bwd_ok:
            msg = lib.nts_last_error()
            assert (b"two-pass" in msg) if fwd_ok else (b"head width" in msg), (H, D, msg)
        why = ops.gat_bf16_shape_error(F, H)
        assert (why is None) == (fwd_ok and bwd_ok), (H, D, why)
        if why is not None:
            entry = "forward" if not fwd_ok else "backward_two_pass"
            assert why.startswith("nts_gat_fused_aggregate_%s_bf16: " % entry), why


def test_toolkits_refuse_a_bf16_layer_shape_at_construction(monkeypatch):
    """GATImpl and GATSampleImpl refuse a layer that a BF16 entry refuses before any device work (no graph, no
    device tensors are needed to see it), naming the layer and the entry's message; accepted layer lists go on."""
    from neutronstarlite_b200 import _lib, sample, toolkits
    V = 10
    feats, labels, mask = torch.zeros((V, 23)), torch.zeros(V, dtype=torch.int64), torch.zeros(V, dtype=torch.int64)
    refused = [([23, 192, 5], 8, 0, "two-pass"),          # 8 heads x 24: hv 6
               ([23, 64, 320, 5], 4, 1, "two-pass"),      # 4 heads x 80: hv 10
               ([23, 600, 5], 3, 0, "two-pass"),          # 3 heads x 200: hv 25
               ([23, 16, 1433], 2, 1, "two-pass"),        # a single-head layer wider than 1024
               ([23, 15, 5], 3, 0, "head width")]         # 3 heads x 5
    for layers, heads, bad, words in refused:
        with pytest.raises(_lib.NtsError, match="layer %d .*%s" % (bad, words)):
            toolkits.GATImpl(None, layers, feats, labels, mask, heads=heads, fused_kernel=True, gather_dtype=BF16)
        with pytest.raises(_lib.NtsError, match="layer %d .*%s" % (bad, words)):
            toolkits.GATSampleImpl(None, layers, feats, labels, mask, fanout=[5] * (len(layers) - 1), batch_size=4,
                                   heads=heads, gather_dtype=BF16)
        # FP32 gathers take every such shape
        toolkits.GATImpl(None, layers, feats, labels, mask, heads=heads, fused_kernel=True, exchange=object())

    class Reached(Exception):
        pass

    def sampler(*args, **kwargs):
        raise Reached

    monkeypatch.setattr(sample, "NeighborSampler", sampler)
    for layers, heads in (([23, 64, 64, 41], 8), ([23, 192, 5], 3), ([23, 256, 1000], 2), ([23, 128, 602], 16)):
        m = toolkits.GATImpl(None, layers, feats, labels, mask, heads=heads, fused_kernel=True, gather_dtype=BF16,
                             exchange=object())
        assert m.heads == [heads] * (len(layers) - 2) + [1]
        with pytest.raises(Reached):
            toolkits.GATSampleImpl(None, layers, feats, labels, mask, fanout=[5] * (len(layers) - 1), batch_size=4,
                                   heads=heads, gather_dtype=BF16)


# ---- GPU: the grid on the structured graph -----------------------------------------------------------------------------
def grid_case(H, D, seed, slope=0.2, dv=None, **kw):
    """Structured graph, FP32 operands and the float64 reference at m~ and g~."""
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=seed, device=dv, **kw)
    return st, (m, s, d, g), analytic_reference(*st.torch_csc(dv), rounded(m), s, d, rounded(g), H, slope)


def run_bf16(pg, inputs, slope=0.2):
    return run_k7(pg, *inputs, slope, True, gather_dtype=BF16)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("H,D,tiles,G", GRID)
def test_bf16_gat_layer_vs_float64_at_rounded_operands(H, D, tiles, G, slope):
    dv = dev()
    st, inputs, ref = grid_case(H, D, seed=H * 1000 + D + 7, slope=slope, dv=dv)
    got, (seg_max, seg_sum), rec = run_bf16(st.graph(), inputs, slope)
    assert rec == expected_launch(st.E, tiles, G), (H, D, rec)
    check_stats(seg_max, seg_sum, ref, st.empty_rows)
    check_layer(got, ref)
    check_exact_zeros(st, got)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D,tiles,G", FORWARD_ONLY)
def test_forward_only_shapes(H, D, tiles, G):
    """Multi-tile rows and head widths the backward refuses: the forward against float64; the operator's backward
    raises NtsError, and the C ABI backward returns an error without touching its output buffers."""
    from neutronstarlite_b200 import _lib, ops
    dv = dev()
    st, (m, s, d, g), ref = grid_case(H, D, seed=H * 1000 + D + 8, dv=dv)
    pg = st.graph()
    op = ops.DistGPUFusedGATOp(pg, gather_dtype=BF16)
    out = op.forward(m, s, d)
    rec = [ctypes.c_int() for _ in range(4)]
    _lib.call("nts_aggregate_last_launch", *[ctypes.byref(r) for r in rec])
    torch.cuda.synchronize()
    assert tuple(r.value for r in rec) == expected_launch(st.E, tiles, G), (H, D)
    assert not np.isnan(np64(out)).any()
    row_close(np64(out), np64(ref["out"]), scale=np64(ref["out_mag"]))
    assert not np64(out)[st.empty_rows].any()
    with pytest.raises(_lib.NtsError, match="two-pass"):
        op.backward(g)
    mt, _, _, seg_max, seg_sum, _ = op._saved
    F, ld = H * D, mt.shape[1]
    gt = ops._FusedGAT._to_bf16_rows(g, ld)
    og = torch.zeros((st.Vp, H), device=dv)
    dm, ds, dd = (torch.full(shape, 7.0, device=dv) for shape in ((st.M, ld), (st.M, H), (st.Vp, H)))
    pack = torch.full((st.Vp, H, 4), 7.0, device=dv)
    slot_off, slot_dst = ops.DistGPUFusedGATOp.slot_csr(pg)
    rc = _lib.load().nts_gat_fused_aggregate_backward_two_pass_bf16(
        ptr(dm), ptr(ds), ptr(dd), ptr(pack), ptr(mt), ptr(s), ptr(d), ptr(seg_max), ptr(seg_sum), ptr(og), ptr(gt),
        ptr(pg.row_indices_gpu), ptr(pg.column_offset_gpu), ptr(pg.mirror_index_gpu), ptr(slot_off), ptr(slot_dst),
        st.Vp, st.M, F, ld, H, 0.2, stream())
    torch.cuda.synchronize()
    assert rc != 0 and b"two-pass" in _lib.load().nts_last_error()
    assert all(bool((t == 7.0).all()) for t in (dm, ds, dd, pack))


# the one-chunk rows the tune hook applies to, with the G it takes (32 / G lanes must hold the row's chunks)
TUNE_SHAPES = [(8, 8, (1, 2, 4)), (1, 41, (1, 2, 4)), (4, 32, (1, 2)), (1, 200, (1,))]


@pytest.mark.gpu
@pytest.mark.parametrize("H,D,Gs", TUNE_SHAPES)
def test_tune_points(H, D, Gs, monkeypatch):
    """NTS_GAT_BF16_TUNE="U,G" at every (U, G) with an instantiation that the hook accepts (tools/gat_dtype_sweep.py
    --tune measures these): the launch record shows the requested G and the layer meets the bounds.  A G whose virtual
    warp is narrower than the row is ignored: the default point runs."""
    dv = dev()
    st, inputs, ref = grid_case(H, D, seed=H * 1000 + D + 9, dv=dv)
    pg = st.graph()
    default_G = next(G for h, d_, _, G in GRID if (h, d_) == (H, D))
    points = [(U, G) for U in (2, 4, 8) for G in Gs] + [(2, G) for G in (1, 2, 4) if G not in Gs]
    for U, G in points:
        monkeypatch.setenv("NTS_GAT_BF16_TUNE", "%d,%d" % (U, G))
        got, (seg_max, seg_sum), rec = run_bf16(pg, inputs)
        assert rec == expected_launch(st.E, 1, G if G in Gs else default_G), (U, G, rec)
        check_stats(seg_max, seg_sum, ref, st.empty_rows)
        check_layer(got, ref)
        check_exact_zeros(st, got)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", [(8, 8), (1, 41), (3, 64), (1, 602), (8, 128), (1, 100)])
def test_c_abi_with_mirror_index(H, D):
    """Both BF16 entries through the C ABI with global row_indices and a non-NULL mirror_index (the col_map branch of
    the destination-major pass; the operator always passes precomputed slots), on rows from nts_rows_to_bf16.  With one
    head and ld > F, the pad columns of out and d_mirror are exactly 0 (sums of a * 0)."""
    from neutronstarlite_b200 import _lib, ops
    dv = dev()
    st, (m, s, d, g), ref = grid_case(H, D, seed=H * 31 + D, dv=dv)
    pg = st.graph()
    slope, F, V, M = 0.2, H * D, st.Vp, st.M
    ld = (F + 7) // 8 * 8
    ri, co, mi = pg.row_indices_gpu, pg.column_offset_gpu, pg.mirror_index_gpu
    seg_max = torch.full((V, H), 7.0, device=dv)
    seg_sum = torch.full((V, H), 7.0, device=dv)
    _lib.call("nts_gat_softmax_stats", ptr(seg_max), ptr(seg_sum), ptr(s), ptr(d), ptr(ri), ptr(co), ptr(mi), V, H,
              slope, stream())
    mt = torch.full((M, ld), 7.0, dtype=BF16, device=dv)
    gt = torch.full((V, ld), 7.0, dtype=BF16, device=dv)
    _lib.call("nts_rows_to_bf16", ptr(m), 0, F, ptr(mt), M, F, ld, stream())
    _lib.call("nts_rows_to_bf16", ptr(g), 0, F, ptr(gt), V, F, ld, stream())
    out = torch.zeros((V, ld), device=dv)
    _lib.call("nts_gat_fused_aggregate_forward_bf16", ptr(mt), ptr(out), ptr(s), ptr(d), ptr(seg_max), ptr(seg_sum),
              ptr(ri), ptr(co), ptr(mi), V, st.E, F, ld, H, slope, stream())
    og = (out[:, :F] * gt[:, :F].float()).view(V, H, D).sum(-1).contiguous()
    slot_off, slot_dst = ops.DistGPUFusedGATOp.slot_csr(pg)
    dm, ds, dd = torch.zeros((M, ld), device=dv), torch.zeros_like(s), torch.zeros_like(d)
    pack = torch.empty((V, H, 4), device=dv)
    _lib.call("nts_gat_fused_aggregate_backward_two_pass_bf16", ptr(dm), ptr(ds), ptr(dd), ptr(pack), ptr(mt), ptr(s),
              ptr(d), ptr(seg_max), ptr(seg_sum), ptr(og), ptr(gt), ptr(ri), ptr(co), ptr(mi), ptr(slot_off),
              ptr(slot_dst), V, M, F, ld, H, slope, stream())
    torch.cuda.synchronize()
    if ld > F:
        assert not out[:, F:].any() and not dm[:, F:].any()
    got = (out[:, :F], dm[:, :F], ds, dd)
    check_stats(seg_max, seg_sum, ref, st.empty_rows)
    check_layer(got, ref)
    check_exact_zeros(st, got)


# ---- GPU: edge semantics -----------------------------------------------------------------------------------------------
SEMANTICS = [(8, 8), (1, 41), (3, 64), (1, 602), (8, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", SEMANTICS)
def test_equal_logits_give_uniform_weights(H, D):
    """One source score for every slot: the statistics are exactly (leaky(s + d), deg) and out is the mean of the
    segment's rounded mirror rows."""
    dv = dev()
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=5, device=dv)
    s = torch.full_like(s, 0.375)
    ref = analytic_reference(*st.torch_csc(dv), rounded(m), s, d, rounded(g), H, 0.2)
    got, (seg_max, seg_sum), _ = run_bf16(st.graph(), (m, s, d, g))
    deg = torch.from_numpy(np.diff(st.off.astype(np.int64))).to(dv)
    live = deg > 0
    pre = s[0] + d
    assert torch.equal(seg_max[live], torch.where(pre > 0, pre, pre * 0.2)[live])
    assert torch.equal(seg_sum[live], deg[live, None].float().expand(-1, H))
    check_layer(got, ref)
    check_exact_zeros(st, got)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", [0.2, 0.0])
@pytest.mark.parametrize("H,D", SEMANTICS)
def test_zero_preactivation_uses_the_negative_slope(H, D, slope):
    """Dyadic scores make s + d == 0 exactly on about a fifth of the edges; leaky'(0) is the negative slope."""
    dv = dev()
    st = structured()
    m, _, _, g = layer_inputs(st.M, st.Vp, H, D, seed=6, device=dv)
    rng = np.random.default_rng(7)
    grid = np.array([-1.0, -0.5, 0.0, 0.5, 1.0], dtype=np.float32)
    s = torch.from_numpy(rng.choice(grid, (st.M, H))).to(dv)
    d = torch.from_numpy(rng.choice(grid, (st.Vp, H))).to(dv)
    ref = analytic_reference(*st.torch_csc(dv), rounded(m), s, d, rounded(g), H, slope)
    got, _, _ = run_bf16(st.graph(), (m, s, d, g), slope)
    check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("slope", [0.2, 1.0])
@pytest.mark.parametrize("H,D", SEMANTICS)
def test_large_scores_underflow_without_inf_or_nan(H, D, slope):
    """Scores in +-40: most weights underflow in FP32.  No inf or NaN, and the bounds (with their FLT_MIN floor on
    ds / dd) hold."""
    dv = dev()
    st, inputs, ref = grid_case(H, D, seed=8, slope=slope, dv=dv, score=40.0)
    got, _, _ = run_bf16(st.graph(), inputs, slope)
    assert all(bool(torch.isfinite(x).all()) for x in got)
    check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", SEMANTICS)
def test_one_nan_source_score_stays_in_its_rows(H, D):
    """One NaN source score (of the only source of one row, in its last head, and of the hub source in head 0): every
    output is NaN exactly where the float64 reference is."""
    dv = dev()
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=9, device=dv)
    s[int(st.mi[ONE_SRC]), H - 1] = float("nan")
    s[st.hub_slot, 0] = float("nan")
    ref = analytic_reference(*st.torch_csc(dv), rounded(m), s, d, rounded(g), H, 0.2)
    assert bool(torch.isnan(ref["out"]).any()) and not bool(torch.isnan(ref["out"]).all())
    got, _, _ = run_bf16(st.graph(), (m, s, d, g))
    check_layer(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("H,D", SEMANTICS)
def test_a_mirror_value_that_rounds_to_inf(H, D):
    """+-3.4e38 is finite in FP32 and +-inf in BF16: the out rows it reaches are +-inf (or NaN where +inf meets -inf)
    exactly where the float64 reference at m~ has them, every other entry of out meets the bounds, and d_mirror (which
    does not read the mirror) is unaffected."""
    dv = dev()
    st = structured()
    m, s, d, g = layer_inputs(st.M, st.Vp, H, D, seed=10, device=dv)
    F = H * D
    dst = np.repeat(np.arange(st.Vp), np.diff(st.off.astype(np.int64)))
    hub_fed = np.isin(dst, dst[st.slot == st.hub_slot])
    other = int(st.slot[np.nonzero(hub_fed & (st.slot != st.hub_slot))[0][0]])
    m[st.hub_slot, 0] = 3.4e38
    m[other, 0] = -3.4e38                            # meets the hub source's +inf in column 0 of a row: NaN
    m[int(st.mi[ONE_SRC]), F - 1] = -3.4e38          # the only source of its row
    mt = rounded(m)
    assert bool(torch.isposinf(mt[st.hub_slot, 0])) and bool(torch.isneginf(mt[int(st.mi[ONE_SRC]), F - 1]))
    ref = analytic_reference(*st.torch_csc(dv), mt, s, d, rounded(g), H, 0.2)
    got, _, _ = run_bf16(st.graph(), (m, s, d, g))
    a, b = np64(got[0]), np64(ref["out"])
    fin = np.isfinite(b)
    assert np.isposinf(b).any() and np.isneginf(b).any() and np.isnan(b).any()
    assert np.array_equal(np.isnan(a), np.isnan(b))
    assert np.array_equal(a[np.isinf(b)], b[np.isinf(b)]) and np.isfinite(a[fin]).all()
    mag = np64(ref["out_mag"])
    row_close(np.where(fin, a, 0.0), np.where(fin, b, 0.0), scale=np.where(np.isfinite(mag), mag, 0.0))
    row_close(np64(got[1]), np64(ref["dm"]), scale=np64(ref["dm_mag"]))


# ---- GPU: the production quantum -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("H,D,G", [(8, 8, 4), (1, 41, 4)])
def test_bf16_gat_layer_at_the_production_quantum(zipf_graph, H, D, G):
    """Config D's 8 x 8 hidden layer and 41-wide output layer on > 10 M edges: the forward runs its production quantum
    Q = 512 / G (asserted through the launch record) and every warp of the backward passes strides past its first
    quantum; against the chunked float64 reference at m~ and g~."""
    pg, off, slot = zipf_graph
    t0 = time.perf_counter()
    m, s, d, g = layer_inputs(pg.owned_mirrors, pg.owned_vertices, H, D, seed=30 + H, device=off.device)
    ref = analytic_reference(off, slot, rounded(m), s, d, rounded(g), H, 0.2)
    got, (seg_max, seg_sum), rec = run_bf16(pg, (m, s, d, g))
    want = expected_launch(pg.owned_edges, 1, G)
    assert rec == want and want[2] == 16 + 2 * (8 * G * (512 // G) + 8) * 4, (rec, want)
    check_stats(seg_max, seg_sum, ref, np.nonzero(np.diff(np64(off)) == 0)[0])
    check_layer(got, ref)
    print("large-graph BF16 K7 %dx%d: %.1f s" % (H, D, time.perf_counter() - t0))


# ---- GPU: sampled blocks ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("gather_dtype", [None, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("H,D", [(H, D) for H, D, _, _ in GRID])
def test_minibatch_gat_op_on_the_hub_block(H, D, gather_dtype):
    """ops.MiniBatchGATOp on the sampled hub block (hub destinations of 64 kept edges, multi-edges, destinations that
    are their own sources) at every grid shape, held to check_layer against the block's float64 reference (at x~ and
    g~ for BF16 gathers)."""
    from neutronstarlite_b200 import ops
    from test_gat_sample_gpu import hub_block, operands
    dev()
    sg, b = hub_block()
    x, s, d, g = operands(b, H, D, seed=H * 100 + D + 3)
    op = ops.MiniBatchGATOp(sg, 0, gather_dtype=gather_dtype)
    out = op.forward(x, s, d)
    got = (out,) + tuple(op.backward(g))
    torch.cuda.synchronize()
    co = torch.from_numpy(b["column_offset"].astype(np.int64)).to(x.device)
    ri = torch.from_numpy(b["row_indices"].astype(np.int64)).to(x.device)
    if gather_dtype is not None:
        x, g = rounded(x), rounded(g)
    check_layer(got, analytic_reference(co, ri, x, s, d, g, H, 0.2))
