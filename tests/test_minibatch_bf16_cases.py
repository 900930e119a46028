"""CPU checks of the K1-BF16 test table (tests/test_minibatch_bf16_gpu.py): it lists every NTS_BF16_CASE instantiation
of nts_aggregate.cu exactly once and nothing else, and the Python mirror of the BF16 dispatch rule reaches every
listed point from its width, or from the NTS_K1_BF16_TUNE hook."""
import pytest

from test_aggregate_reference import read_source, source_cases
from test_minibatch_bf16_gpu import K1_BF16_CASES, bf16_launch, bf16_point


def test_bf16_table_matches_the_source():
    src = source_cases(read_source("nts_aggregate.cu"), "NTS_BF16_CASE")
    assert len(src) == len(set(src)) >= 16
    table = [c[0] for c in K1_BF16_CASES]
    assert len(table) == len(set(table))
    assert sorted(table) == sorted(src)


def test_bf16_points_follow_the_dispatch_rule():
    """Default rows need no hook; tuned rows would not be reached without it."""
    for point, F, tune in K1_BF16_CASES:
        assert bf16_point(F, 2, tune)[0] == point, (point, F, tune)
        if tune is not None:
            assert bf16_point(F, 2)[0] != point, (point, "reached without the hook")


def test_bf16_dispatch_of_the_model_widths():
    """Config B's 602-128-41 and the tests' 37: chunk counts, virtual warps under the bulk variant only."""
    assert bf16_point(602) == ((3, 4, 2, 1), 1)
    assert bf16_point(128) == ((1, 4, 2, 2), 1)
    assert bf16_point(41) == ((1, 4, 2, 2), 1)
    assert bf16_point(37) == ((1, 4, 2, 2), 1)
    for F in (37, 41, 128):
        assert bf16_point(F, 1)[0] == (1, 4, 2, 1)
    assert bf16_point(1025)[1] == 2                          # past 4 chunks of 32 lanes: two column tiles
    # a G the row does not fit in is ignored
    assert bf16_point(128, 2, (4, 4, 4))[0] == (1, 4, 4, 2)


@pytest.mark.parametrize("g", [1, 2, 4])
def test_bf16_launch_grid_shows_the_virtual_warps(g):
    """At a fixed quantum the grid divides by G, so the launch record tells the points apart."""
    grids = {gg: bf16_launch(64 * 8 * 4 * 10, 1, gg, 2, Q=64)[0] for gg in (1, 2, 4)}
    assert grids[g] * g == grids[1]
