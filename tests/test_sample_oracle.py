"""CPU checks of the sampler's numpy restatement (tests/sample_oracle.py), which the GPU sampler tests hold the kernels
to bit for bit: Floyd's draw is uniform over k-subsets, hops keep min(deg, k) slots that are edges of the graph, and
the blocks are self-consistent (distinct sources ascending, transposed block = the block)."""
import numpy as np
import pytest
from scipy import stats

import sample_oracle as so
from neutronstarlite_b200 import _lib
from neutronstarlite_b200.sample import check_fanout


def csc(edges, V):
    """CSC of (src, dst) edges: column_offset, row_indices ascending inside a destination, weights = a distinct float
    per slot (so that the tests can tell slots apart)."""
    order = np.lexsort((edges[:, 0], edges[:, 1]))
    e = edges[order]
    col = np.zeros(V + 1, dtype=np.uint32)
    np.cumsum(np.bincount(e[:, 1], minlength=V), out=col[1:])
    return col, e[:, 0].astype(np.uint32), np.arange(e.shape[0], dtype=np.float32) + 0.5


def star(deg):
    """Vertex 0 with `deg` in-edges from 1..deg (plus nothing else)."""
    edges = np.stack([np.arange(1, deg + 1), np.zeros(deg, dtype=np.int64)], 1)
    return csc(edges, deg + 1)


def test_floyd_is_uniform_over_all_subsets():
    col, row, w = star(6)
    counts = {}
    steps = 6000
    for step in range(steps):
        b = so.sample(col, row, w, [0], [3], seed=11, step=step)[0]
        key = tuple(b["row_global"])
        assert len(set(key)) == 3 and list(key) == sorted(key)
        counts[key] = counts.get(key, 0) + 1
    assert len(counts) == 20
    chi2, p = stats.chisquare(np.array(list(counts.values())))
    assert p > 1e-3, (chi2, p)


def test_each_slot_is_kept_with_probability_k_over_deg():
    col, row, w = star(12)
    k, steps = 5, 12000
    hits = np.zeros(13)
    for step in range(steps):
        b = so.sample(col, row, w, [0], [k], seed=3, step=step)[0]
        hits[b["row_global"]] += 1
    freq = hits[1:] / steps
    # binomial standard deviation at p = 5/12 over 12000 draws is 0.0045
    np.testing.assert_allclose(freq, k / 12, atol=0.02)
    assert stats.chisquare(hits[1:]).pvalue > 1e-3


def random_multigraph(V=400, E=5000, seed=0, self_loops=False):
    rng = np.random.default_rng(seed)
    e = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1)
    e[: E // 5, 1] = 3                                   # a hub with multi-edges
    e[E // 5: E // 5 + 50] = [7, 9]                      # one pair repeated 50 times
    if self_loops:
        e = np.concatenate([e, np.stack([np.arange(V), np.arange(V)], 1)])
    return e, V


@pytest.mark.parametrize("fanout", [[1, 1], [5, 10], [64, 64, 3]])
def test_hops_keep_min_deg_k_edges_of_the_graph(fanout):
    edges, V = random_multigraph()
    col, row, w = csc(edges, V)
    seeds = np.arange(0, V, 7)
    hops = so.sample(col, row, w, seeds, fanout, seed=5, step=2)
    dst = seeds
    for h, (b, k) in enumerate(zip(hops, fanout)):
        assert np.array_equal(b["dst"], dst)
        deg = col[dst + 1].astype(np.int64) - col[dst]
        assert np.array_equal(np.diff(b["column_offset"].astype(np.int64)), np.minimum(deg, k))
        # every kept slot is one of the destination's slots, none twice, weight copied from that slot
        for d in range(dst.size):
            lo, hi = b["column_offset"][d], b["column_offset"][d + 1]
            slots = (b["weight"][lo:hi] - 0.5).astype(np.int64)
            assert np.all((slots >= col[dst[d]]) & (slots < col[dst[d] + 1]))
            assert np.all(np.diff(slots) > 0)
            assert np.array_equal(row[slots], b["row_global"][lo:hi])
        assert np.array_equal(b["src"], np.unique(b["row_global"]))
        assert np.array_equal(b["src"][b["row_indices"]], b["row_global"])
        # transposed block: the same (dst, src, w) triples, edges of a source in edge order
        e_dst = np.repeat(np.arange(dst.size), np.diff(b["column_offset"].astype(np.int64)))
        t_src = np.repeat(np.arange(b["src"].size), np.diff(b["row_offset"].astype(np.int64)))
        fwd = sorted(zip(b["row_indices"].tolist(), e_dst.tolist(), b["weight"].tolist()))
        bwd = sorted(zip(t_src.tolist(), b["column_indices"].tolist(), b["weight_backward"].tolist()))
        assert fwd == bwd
        dst = b["src"].astype(np.int64)


def test_sample_does_not_depend_on_the_batch():
    """A destination's kept slots are a function of (seed, step, hop, destination) alone."""
    edges, V = random_multigraph(seed=1)
    col, row, w = csc(edges, V)
    whole = so.sample(col, row, w, np.arange(V), [4], seed=9, step=4)[0]
    for d in (3, 7, 100):
        one = so.sample(col, row, w, [d], [4], seed=9, step=4)[0]
        lo, hi = whole["column_offset"][d], whole["column_offset"][d + 1]
        assert np.array_equal(one["weight"], whole["weight"][lo:hi])
    other = so.sample(col, row, w, [3], [4], seed=9, step=5)[0]
    assert not np.array_equal(other["weight"], so.sample(col, row, w, [3], [4], seed=9, step=4)[0]["weight"])


def test_zero_in_degree_and_empty_inputs():
    col, row, w = star(4)
    b = so.sample(col, row, w, [1, 0, 2], [2], seed=0, step=0)[0]   # 1 and 2 have no in-edges
    assert b["column_offset"].tolist() == [0, 0, 2, 2]
    e = so.sample(col, row, w, [], [2, 3], seed=0, step=0)
    assert all(h["row_indices"].size == 0 and h["column_offset"].tolist() == [0] for h in e)


def test_fanout_limits_are_checked_without_a_gpu():
    assert check_fanout([1, 64]) == [1, 64]
    for bad in ([0], [65], [5, 0], [], [1] * 9):
        with pytest.raises(_lib.NtsError):
            check_fanout(bad)
