"""Merged multi-part plans (nts_gather_plan_create_parts, csrc/nts_plan.cu): several chunks in one plan, part-local row
r -> output row row_add + r, mapped index g -> index_add + g.  Checked against the C oracle of the reference's
aggregation loop on the equivalent single CSR (per row, 1e-4 of the row's magnitude), exactly on the all-ones product
(in-degree counts), and against the single-chunk builder for one part; FP32 and BF16 gathers."""
import ctypes as C

import numpy as np
import pytest

import oracle_c

torch = pytest.importorskip("torch")


class Part(C.Structure):
    _fields_ = [("offsets", C.c_void_p), ("indices", C.c_void_p), ("weight", C.c_void_p), ("slot_of", C.c_void_p),
                ("index_base", C.c_uint32), ("index_add", C.c_uint32), ("n_rows", C.c_uint32),
                ("row_add", C.c_uint32), ("n_edges", C.c_uint64)]


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def up(a):
    if a is None:
        return None
    if a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def ptr(t):
    return 0 if t is None else t.data_ptr()


def row_close(actual, desired, rtol=1e-4):
    err = np.abs(actual.astype(np.float64) - desired.astype(np.float64)).max(axis=1)
    scale = np.abs(desired).max(axis=1).astype(np.float64)
    bad = np.nonzero(err > rtol * scale + 1e-30)[0]
    assert bad.size == 0, "rows %s: err %s vs scale %s" % (bad[:5], err[bad[:5]], scale[bad[:5]])


def make_part(rng, n_rows, n_src, n_edges, mode):
    """One chunk: CSR over n_rows part-local rows gathering n_src part-local rows, with a hub row, a hub source and
    empty rows.  mode: 'base' (indices = local + 1000, index_base 1000), 'slots' (global ids through a slot table) or
    'empty' (no edges)."""
    if mode == "empty":
        return dict(off=np.zeros(n_rows + 1, np.uint32), idx=None, local=np.zeros(0, np.uint32),
                    w=np.zeros(0, np.float32), slot_of=None, base=0, n_rows=n_rows, n_src=n_src)
    dst = rng.integers(0, n_rows, n_edges)
    dst[: n_edges // 5] = n_rows // 2
    dst = dst[dst % 7 != 1]
    src = rng.integers(0, n_src, dst.shape[0])
    src[: dst.shape[0] // 10] = n_src - 1
    order = np.argsort(dst, kind="stable")             # each row keeps its own (unsorted) source order
    dst, src = dst[order], src[order].astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n_rows))]).astype(np.uint32)
    w = rng.uniform(0.1, 1.0, dst.shape[0]).astype(np.float32)
    if mode == "slots":
        ids = rng.permutation(3 * n_src)[:n_src].astype(np.uint32)
        slot_of = np.zeros(3 * n_src, np.uint32)
        slot_of[ids] = np.arange(n_src, dtype=np.uint32)
        return dict(off=off, idx=ids[src], local=src, w=w, slot_of=slot_of, base=0, n_rows=n_rows, n_src=n_src)
    return dict(off=off, idx=src + 1000, local=src, w=w, slot_of=None, base=1000, n_rows=n_rows, n_src=n_src)


def make_parts(rng, n_parts, n_out, G, E):
    """n_parts parts over n_out output rows and G gathered rows: overlapping row ranges (row_add) and gathered blocks
    (index_add), one part through a slot table and, from three parts on, one empty part."""
    modes = (["base", "slots", "empty", "base"] if n_parts >= 3 else ["base", "slots"])[:n_parts]
    parts = []
    for k, mode in enumerate(modes):
        n_rows = int(rng.integers(n_out // 2, n_out))
        n_src = int(rng.integers(G // 4, G // 2))
        p = make_part(rng, n_rows, n_src, E // n_parts, mode)
        p["row_add"] = int(rng.integers(0, n_out - n_rows + 1))
        p["index_add"] = int(rng.integers(0, G - n_src + 1))
        parts.append(p)
    return parts


def merged_csr(parts, n_out, weighted=True):
    """The single CSR the merged plan stands for: per output row the parts in order, each in its own edge order."""
    rows, cols, ws = [], [], []
    for p in parts:
        rows.append(np.repeat(np.arange(p["n_rows"]), np.diff(p["off"].astype(np.int64))) + p["row_add"])
        cols.append(p["local"].astype(np.int64) + p["index_add"])
        ws.append(p["w"] if weighted else np.ones_like(p["w"]))
    rows, cols, ws = np.concatenate(rows), np.concatenate(cols), np.concatenate(ws)
    order = np.argsort(rows, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n_out))]).astype(np.uint32)
    return off, cols[order].astype(np.uint32), ws[order].astype(np.float32)


def create_parts(parts, n_out, G, slabs, F, weighted=True):
    """Build through nts_gather_plan_create_parts; returns an ops.GatherPlan around the handle (None on refusal)."""
    from neutronstarlite_b200 import _lib, ops
    keep, arr = [], (Part * len(parts))()
    for k, p in enumerate(parts):
        d = [up(p["off"]), up(p["idx"]), up(p["w"]) if weighted else None, up(p["slot_of"])]
        keep += d
        arr[k] = Part(ptr(d[0]), ptr(d[1]), ptr(d[2]), ptr(d[3]), p["base"], p["index_add"], p["n_rows"],
                      p["row_add"], len(p["local"]))
    h = _lib.load().nts_gather_plan_create_parts(arr, len(parts), n_out, G, slabs, F, ops._stream())
    if not h:
        return None
    plan = ops.GatherPlan.__new__(ops.GatherPlan)
    plan.handle = h
    return plan


def run(plan, X, n_out, gather_dtype=None):
    out = torch.zeros((n_out, X.shape[1]), dtype=torch.float32, device=dev())
    plan.run(torch.from_numpy(X).to(dev()), out, gather_dtype=gather_dtype)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("gather_dtype", ["f32", "bf16"])
@pytest.mark.parametrize("slabs", [1, 3, 16, 0])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_merged_plan_matches_oracle(n_parts, slabs, gather_dtype):
    from neutronstarlite_b200 import _lib
    dev()
    rng = np.random.default_rng(100 * n_parts + slabs)
    # 40000 gathered rows of 128 floats exceed the 16 MB slab budget: the measured count (0) has two candidates
    n_out, G, E, F = 1500, 40000, 120000, 128
    parts = make_parts(rng, n_parts, n_out, G, E)
    L = _lib.load()
    plan = create_parts(parts, n_out, G, slabs, F)
    assert plan is not None, L.nts_last_error()
    if slabs:
        assert L.nts_gather_plan_slabs(plan.handle) == slabs
    else:
        assert L.nts_gather_plan_slabs(plan.handle) in (1, 2) and L.nts_gather_plan_tuned_ms(plan.handle) > 0
    hc, hr = C.c_int(-1), C.c_int(-1)
    _lib.call("nts_gather_plan_hubs", plan.handle, C.byref(hc), C.byref(hr))
    assert (hc.value, hr.value) == (0, 0)
    off, idx, w = merged_csr(parts, n_out)
    gd = torch.bfloat16 if gather_dtype == "bf16" else None
    for width in (F, 41):
        X = rng.uniform(-1, 1, (G, width)).astype(np.float32)
        Xr = torch.from_numpy(X).bfloat16().float().numpy() if gd else X
        row_close(run(plan, X, n_out, gd), oracle_c.segment_gather_sum(off, idx, w, Xr))
    # segment sizes exactly: all-ones input, unit weights -> in-degree counts of the merged rows
    ones = create_parts(parts, n_out, G, slabs, F, weighted=False)
    cnt = run(ones, np.ones((G, 4), np.float32), n_out, gd)
    assert np.array_equal(cnt[:, 0], np.diff(off.astype(np.int64)).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["base", "slots"])
@pytest.mark.parametrize("slabs", [1, 3, 16])
def test_one_part_merged_plan_equals_single_chunk_plan(slabs, mode):
    """A merged plan of one part (row_add = index_add = 0) is the single-chunk plan: identical results on integer-valued
    data, where every summation order gives the same sum."""
    from neutronstarlite_b200 import ops
    dev()
    rng = np.random.default_rng(7 + slabs)
    n_rows, n_src = 900, 3000
    p = make_part(rng, n_rows, n_src, 60000, mode)
    p["w"] = rng.integers(1, 4, p["w"].shape[0]).astype(np.float32)
    p["row_add"] = p["index_add"] = 0
    merged = create_parts([p], n_rows, n_src, slabs, 0)
    single = ops.GatherPlan(up(p["off"]), up(p["idx"]), up(p["w"]), p["base"], n_rows, len(p["local"]), n_src, slabs,
                            slot_of=up(p["slot_of"]), hubs=(0, 0))
    X = rng.integers(-4, 5, (n_src, 40)).astype(np.float32)
    for gd in (None, torch.bfloat16):
        a, b = run(merged, X, n_rows, gd), run(single, X, n_rows, gd)
        assert np.array_equal(a, b)
    off, idx, w = merged_csr([p], n_rows)
    assert np.array_equal(run(merged, X, n_rows), oracle_c.segment_gather_sum(off, idx, w, X))


def test_refused_parts():
    """Parts whose rows leave the output, and parts with edges but no arrays, are refused before any device work."""
    from neutronstarlite_b200 import _lib
    L = _lib.load()
    fake = 0x1000    # never dereferenced: the refusal comes first
    rows_out = (Part * 2)(Part(fake, fake, 0, 0, 0, 0, 8, 0, 10), Part(fake, fake, 0, 0, 0, 0, 8, 4, 10))
    assert not L.nts_gather_plan_create_parts(rows_out, 2, 10, 16, 1, 0, None)
    assert b"exceed the output rows" in L.nts_last_error()
    for missing in (Part(0, fake, 0, 0, 0, 0, 8, 0, 10), Part(fake, 0, 0, 0, 0, 0, 8, 0, 10)):
        arr = (Part * 2)(Part(fake, fake, 0, 0, 0, 0, 2, 0, 10), missing)
        assert not L.nts_gather_plan_create_parts(arr, 2, 10, 16, 1, 0, None)
        assert b"null graph array" in L.nts_last_error()
    assert not L.nts_gather_plan_create_parts(None, 0, 10, 16, 1, 0, None)
    assert b"no plan parts" in L.nts_last_error()
