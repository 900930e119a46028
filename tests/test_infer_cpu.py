"""The float64 restatement of full-neighbour inference (infer_oracle.py) against its definition, without a GPU:

  * on small multigraphs with in-degrees 0..8, the restated aggregation s ⊙ A X equals the exact mean of the sampled
    aggregation over ALL k-subsets of each destination's in-edge slots, enumerated, for every fanout 1..9: this pins
    s_v = min(1, k / indeg(v)) (1 at indeg 0) to the sampling law, not to the restatement;
  * transform-first and aggregate-first give the same float64 outputs, so infer's width rule changes no result;
  * the BF16 rounding helper is round-to-nearest-even on float32 values."""
import itertools

import numpy as np
import pytest

import infer_oracle


def small_graph(V, max_deg, seed):
    """A CSC with in-degrees 0..max_deg (every value present), repeated sources (a multigraph) and weights != 1."""
    rng = np.random.default_rng(seed)
    deg = np.concatenate([np.arange(max_deg + 1), rng.integers(0, max_deg + 1, V - max_deg - 1)])
    rng.shuffle(deg)
    col = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(deg, out=col[1:])
    row = rng.integers(0, V, int(col[-1]))
    row[:4] = row[4]                       # repeated sources of one destination
    w = rng.uniform(0.25, 2.0, int(col[-1]))
    return col, row, w


def subset_mean(col, row, w, X, k):
    """Mean over every k-subset S of each destination's in-edge slots of sum_{e in S} w[e] X[row[e]] (all slots when
    indeg <= k), enumerated."""
    out = np.zeros((col.size - 1, X.shape[1]))
    for v in range(col.size - 1):
        slots = np.arange(col[v], col[v + 1])
        if slots.size <= k:
            out[v] = (w[slots, None] * X[row[slots]]).sum(0)
            continue
        subsets = list(itertools.combinations(slots, k))
        acc = np.zeros(X.shape[1])
        for S in subsets:
            S = np.array(S)
            acc += (w[S, None] * X[row[S]]).sum(0)
        out[v] = acc / len(subsets)
    return out


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 8, 9])
def test_expected_aggregation_is_the_mean_over_all_k_subsets(k, seed):
    col, row, w = small_graph(40, 8, seed)
    X = np.random.default_rng(seed + 10).standard_normal((40, 3))
    want = subset_mean(col, row, w, X, k)
    got = infer_oracle.scale(col, k)[:, None] * infer_oracle.aggregate(col, row, w, X)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    deg = np.diff(col)
    assert (infer_oracle.scale(col, k)[deg <= k] == 1).all()       # indeg 0 included


def test_a_one_layer_model_is_the_expected_sampled_layer():
    col, row, w = small_graph(30, 7, 3)
    rng = np.random.default_rng(4)
    X, W = rng.standard_normal((30, 5)), rng.standard_normal((5, 2))
    np.testing.assert_allclose(infer_oracle.infer(col, row, w, X, [W], [3]), subset_mean(col, row, w, X, 3) @ W,
                               rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("layers", [[16, 8, 3], [8, 32, 4], [5, 5, 5, 2]])
def test_transform_first_and_aggregate_first_agree(layers):
    col, row, w = small_graph(60, 8, 5)
    rng = np.random.default_rng(6)
    X = rng.standard_normal((60, layers[0]))
    Ws = [rng.standard_normal((a, b)) for a, b in zip(layers[:-1], layers[1:])]
    fanout = [2, 5, 3][:len(Ws)]
    ref = infer_oracle.infer(col, row, w, X, Ws, fanout, order="aggregate")
    for order in ("transform", "widths"):
        np.testing.assert_allclose(infer_oracle.infer(col, row, w, X, Ws, fanout, order=order), ref,
                                   rtol=1e-10, atol=1e-10)
    bound = infer_oracle.magnitude(col, row, w, X, Ws, fanout)
    assert (np.abs(ref) <= bound * (1 + 1e-12)).all()


def test_offsets_may_start_inside_the_edge_arrays():
    col, row, w = small_graph(20, 6, 7)
    X = np.random.default_rng(8).standard_normal((20, 4))
    whole = infer_oracle.aggregate(col, row, w, X)
    np.testing.assert_allclose(infer_oracle.aggregate(col[5:12], row, w, X), whole[5:11], rtol=0, atol=0)


def test_bf16_rounding_is_nearest_even():
    a = np.array([1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -9, -3.14159, 0.0], dtype=np.float32)
    got = infer_oracle.bf16(a)
    assert got[0] == 1.0 and got[1] == 1.0 and got[2] == 1 + 2 ** -6 and got[3] == 1.0
    assert got[4] == -3.140625 and got[5] == 0.0
