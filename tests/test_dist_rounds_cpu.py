"""CPU checks of the data-parallel batch schedule of the sampled toolkits (toolkits._SampledRounds) and of the argument
checks a ShardedFeatureTable makes before it touches a device."""
import pytest

torch = pytest.importorskip("torch")

from neutronstarlite_b200 import _lib  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.toolkits import _SampledRounds  # noqa: E402


def schedule(n_ids, batch, world, rank, step):
    r = _SampledRounds()
    r.batch_size, r.world, r.rank, r.step = batch, world, rank, step
    seen = []
    for seeds in r._batches(torch.arange(n_ids)):
        seen.append(None if seeds is None else (r.step, seeds.tolist()))
    return seen, r.step


@pytest.mark.parametrize("n_ids,batch,world", [(10, 3, 1), (10, 3, 2), (10, 3, 4), (12, 3, 4), (2, 3, 3), (0, 3, 2)])
def test_rounds_cover_every_batch_once_with_the_steps_of_one_gpu(n_ids, batch, world):
    base = 7
    one, end_one = schedule(n_ids, batch, 1, 0, base)
    n_batches = -(-n_ids // batch)
    assert end_one == base + n_batches
    assert one == [(base + b, list(range(b * batch, min((b + 1) * batch, n_ids)))) for b in range(n_batches)]
    per_rank = [schedule(n_ids, batch, world, r, base) for r in range(world)]
    rounds = -(-n_batches // world)
    got = {}
    for r, (seen, end) in enumerate(per_rank):
        assert end == base + n_batches and len(seen) == rounds      # same collectives on every rank
        for t, item in enumerate(seen):
            b = t * world + r
            assert (item is None) == (b >= n_batches)
            if item is not None:
                got[b] = item
    assert [got[b] for b in range(n_batches)] == one


def test_table_arguments_are_checked_before_any_device_work():
    x = torch.zeros((4, 3))
    for offsets in ([0, 4, 4], [1, 4], [0, 5, 4], [4, 0]):
        with pytest.raises(_lib.NtsError, match="offsets"):
            ShardedFeatureTable(x, offsets)
    with pytest.raises(_lib.NtsError, match="CUDA"):
        ShardedFeatureTable(x, [0, 4])
