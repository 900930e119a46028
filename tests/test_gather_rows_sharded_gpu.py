"""nts_gather_rows_sharded in one process: P local buffers stand for the shards of a table, and the gather must equal
torch.cat(shards)[ids] bit for bit at every feature width the kernel treats differently (store widths 1 / 2 / 4,
8 / 16 / 32 lanes per row), for 1, 3 and 32 shards with empty ones, ids at every shard boundary, repeated and
unsorted ids, and n = 0.  Plus the range check of ShardedFeatureTable.gather on a one-shard table."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

WIDTHS = [1, 2, 3, 4, 5, 8, 41, 64, 128, 602]
V = 1000
SPLITS = {
    "1": [0, V],
    "3_empty": [0, 400, 400, V],
    "32_empty": [0, 0] + list(range(10, 800, 30))[:24] + [800, 800, 850, 900, 900, 990, V],
}


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def shards_of(table, offsets):
    """Each shard a separate [rows, 4*ceil(F/4)] buffer whose padding holds NaN (never to be copied out)."""
    F = table.shape[1]
    pitch = (F + 3) // 4 * 4
    out = []
    for o in range(len(offsets) - 1):
        s = torch.full((offsets[o + 1] - offsets[o], pitch), float("nan"), device=table.device)
        s[:, :F] = table[offsets[o]:offsets[o + 1]]
        out.append(s)
    return out, pitch


def gather(dst, shards, offsets, pitch, ids, F):
    from neutronstarlite_b200 import _lib
    d = dst.device
    ptrs = torch.tensor([s.data_ptr() for s in shards], dtype=torch.int64, device=d)
    off = torch.tensor(offsets, dtype=torch.int32, device=d)
    _lib.call("nts_gather_rows_sharded", dst.data_ptr(), ptrs.data_ptr(), off.data_ptr(), len(shards), pitch,
              ids.data_ptr() if ids.numel() else None, ids.numel(), F, torch.cuda.current_stream().cuda_stream)
    return dst


def boundary_ids(offsets, rng):
    edge = []
    for o in offsets:
        edge += [o - 1, o, o + 1]
    edge = [i for i in edge if 0 <= i < V]
    rand = rng.integers(0, V, 3000)
    ids = np.concatenate([edge, rand, edge[::-1], rand[:50]])      # unsorted, every id of `edge` twice
    return torch.from_numpy(ids.astype(np.int32))


@pytest.mark.parametrize("split", list(SPLITS))
@pytest.mark.parametrize("F", WIDTHS)
def test_gather_equals_the_whole_table_rows(F, split):
    d = dev()
    offsets = SPLITS[split]
    assert len(offsets) - 1 == int(split.split("_")[0]) and offsets[-1] == V
    gen = torch.Generator().manual_seed(F)
    table = (torch.rand((V, F), generator=gen) * 2 - 1).to(d)
    shards, pitch = shards_of(table, offsets)
    ids = boundary_ids(offsets, np.random.default_rng(F)).to(d)
    out = gather(torch.empty((ids.numel(), F), device=d), shards, offsets, pitch, ids, F)
    assert torch.equal(out, torch.cat(shards)[:, :F][ids.long()])
    assert torch.equal(out, table[ids.long()])


@pytest.mark.parametrize("F", [2, 4, 8, 64])
def test_gather_into_an_output_that_is_only_4_byte_aligned(F):
    """The store width follows the output's alignment, not only F: a row-aligned output shifted by one float."""
    d = dev()
    offsets = SPLITS["3_empty"]
    table = torch.rand((V, F), generator=torch.Generator().manual_seed(3)).to(d)
    shards, pitch = shards_of(table, offsets)
    ids = boundary_ids(offsets, np.random.default_rng(3)).to(d)
    flat = torch.zeros(ids.numel() * F + 1, device=d)
    out = gather(flat[1:].view(ids.numel(), F), shards, offsets, pitch, ids, F)
    assert torch.equal(out, table[ids.long()]) and flat[0] == 0


def test_no_ids_launch_nothing_and_bad_arguments_are_refused():
    from neutronstarlite_b200 import _lib
    d = dev()
    table = torch.rand((V, 8), device=d)
    shards, pitch = shards_of(table, SPLITS["1"])
    L = _lib.load()
    torch.cuda.synchronize()
    n0 = L.nts_kernel_launch_count()
    empty = torch.empty((0, 8), device=d)
    gather(empty, shards, SPLITS["1"], pitch, torch.empty(0, dtype=torch.int32, device=d), 8)
    assert L.nts_kernel_launch_count() == n0
    ids = torch.arange(4, dtype=torch.int32, device=d)
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty((4, 8), device=d)
    ptrs = torch.tensor([shards[0].data_ptr()] * 33, dtype=torch.int64, device=d)
    off = torch.tensor([0] * 33 + [V], dtype=torch.int32, device=d)
    for n_shards, p in ((0, pitch), (33, pitch), (1, 6), (1, 4)):        # shard count, pitch % 4, pitch < F
        assert L.nts_gather_rows_sharded(out.data_ptr(), ptrs.data_ptr(), off.data_ptr(), n_shards, p,
                                         ids.data_ptr(), 4, 8, st) != 0
    assert L.nts_kernel_launch_count() == n0


def test_table_gather_range_checks_ids():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.feature_table import ShardedFeatureTable
    d = dev()
    x = torch.rand((V, 5), device=d)
    t = ShardedFeatureTable(x, [0, V])
    assert t.world == 1 and t.pitch == 8
    ids = torch.tensor([V - 1, 0, 17, 17], device=d)
    assert torch.equal(t.gather(ids), x[ids])
    assert torch.equal(t.gather(np.array([3, 999])), x[[3, 999]])
    assert t.gather([]).shape == (0, 5)
    for bad in (torch.tensor([1, V], device=d), torch.tensor([-1], device=d),
                torch.tensor([(1 << 32) + 3], device=d), np.array([V]), [-2], torch.tensor([0.5], device=d)):
        with pytest.raises(_lib.NtsError):
            t.gather(bad)
    with pytest.raises(_lib.NtsError):
        ShardedFeatureTable(x[:10], [0, V])
    t.close()
    with pytest.raises(_lib.NtsError):
        t.gather([0])
