"""The float64 restatement of full-neighbour GAT inference (gat_infer_oracle.py) against its definition, without a GPU:

  * on multigraphs with in-degrees 0..8, the restated layer equals a dense formulation: per head, an attention matrix
    over (destination, source) with the multiplicity of every (u, v) slot pair as a factor;
  * with every fanout >= the largest in-degree it equals the GAT layer applied to sample_oracle blocks that keep every
    slot, seeded with every vertex;
  * shifting every logit of a destination by a constant leaves its output unchanged (the max subtraction)."""
import numpy as np
import pytest

import gat_infer_oracle as go
import sample_oracle


def multigraph(V, max_deg, seed):
    """A CSC with in-degrees 0..max_deg (every value present) and repeated sources of one destination."""
    rng = np.random.default_rng(seed)
    deg = np.concatenate([np.arange(max_deg + 1), rng.integers(0, max_deg + 1, V - max_deg - 1)])
    rng.shuffle(deg)
    col = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(deg, out=col[1:])
    row = rng.integers(0, V, int(col[-1]))
    v = int(np.argmax(deg))
    row[col[v]:col[v + 1]] = row[col[v]]     # one destination whose slots all come from one source
    return col, row


def model(F, layers, heads, seed):
    rng = np.random.default_rng(seed)
    Ws, als, ars = [], [], []
    for l in range(len(layers) - 1):
        Ws.append(rng.uniform(-0.5, 0.5, (layers[l], layers[l + 1])))
        D = layers[l + 1] // heads[l]
        als.append(rng.uniform(-1, 1, (heads[l], D)))
        ars.append(rng.uniform(-1, 1, (heads[l], D)))
    return Ws, als, ars


def dense_layer(col, row, T, al, ar, H):
    """Y = softmax_rows(C ⊙ exp(leaky(s_u + d_v))) T per head, C[v, u] the number of slots u -> v."""
    V = col.size - 1
    C = np.zeros((V, T.shape[0]))
    np.add.at(C, (np.repeat(np.arange(V), np.diff(col)), row[:col[-1]]), 1.0)
    D = T.shape[1] // H
    t = T.reshape(-1, H, D)
    Y = np.zeros((V, H, D))
    for h in range(H):
        s, d = t[:, h] @ al[h], t[:V, h] @ ar[h]
        Lg = go.leaky(d[:, None] + s[None, :])
        Lg = np.where(C > 0, Lg, -np.inf)
        m = np.where(C.sum(1) > 0, Lg.max(1), 0.0)
        P = C * np.exp(Lg - m[:, None])
        Z = P.sum(1)
        A = np.where(Z[:, None] > 0, P / np.where(Z > 0, Z, 1)[:, None], 0.0)
        Y[:, h] = A @ t[:, h]
    return Y.reshape(V, H * D)


@pytest.mark.parametrize("H,D", [(1, 5), (2, 4), (4, 3)])
def test_layer_matches_the_dense_attention_matrix(H, D):
    col, row = multigraph(60, 8, H * 10 + D)
    rng = np.random.default_rng(H)
    T = rng.uniform(-2, 2, (60, H * D))
    al, ar = rng.uniform(-1, 1, (H, D)), rng.uniform(-1, 1, (H, D))
    s, d = go.scores(T, al, ar, H)
    got = go.aggregate(col, row, s, d, T, H)
    want = dense_layer(col, row, T, al, ar, H)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)
    assert (got[np.diff(col) == 0] == 0).all()


def block_forward(col, row, X, Ws, als, ars, heads):
    """GATSampleImpl's layers on sample_oracle blocks at fanouts >= the largest in-degree.  Every hop's destinations
    are all the vertices (the seeds, and with destination-inclusive sampling the sources of every deeper hop), so
    every destination's own row is there for its score d."""
    V = col.size - 1
    L = len(Ws)
    k = int(np.diff(col).max()) + 1
    skey = sample_oracle.step_key(5, 0)
    hops = [sample_oracle.sample_hop(col.astype(np.uint32), row.astype(np.uint32), np.ones(row.size, np.float32),
                                     np.arange(V), k, skey, h) for h in range(L)]
    for b in hops:
        assert (np.diff(b["column_offset"].astype(np.int64)) == np.diff(col)).all()   # every slot kept
    x = np.asarray(X, dtype=np.float64)           # indexed by global id; rows not yet computed are unused
    for l in range(L):
        b = hops[L - 1 - l]
        dst = b["dst"].astype(np.int64)
        T = x @ Ws[l]
        s, d = go.scores(T, als[l], ars[l], heads[l])
        y = go.aggregate(b["column_offset"].astype(np.int64), b["row_global"].astype(np.int64), s, d[dst],
                         T, heads[l])
        out = np.zeros((V, y.shape[1]))
        out[dst] = np.maximum(y, 0) if l < L - 1 else go.log_softmax(y)
        x = out
    return x


def test_full_fanout_blocks_equal_the_restatement():
    col, row = multigraph(80, 8, 3)
    layers, heads = [6, 8, 3], [2, 1]
    X = np.random.default_rng(4).uniform(-1, 1, (80, 6))
    Ws, als, ars = model(6, layers, heads, 5)
    want = go.infer(col, row, X, Ws, als, ars, heads)
    got = block_forward(col, row, X, Ws, als, ars, heads)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_shifting_a_destinations_logits_changes_nothing():
    col, row = multigraph(50, 8, 7)
    rng = np.random.default_rng(8)
    T = rng.uniform(-1, 1, (50, 8))
    s, d = rng.uniform(1, 3, (50, 2)), rng.uniform(1, 3, (50, 2))
    # with s + d > 0 everywhere leaky_relu is the identity, so adding c to d[v] adds c to every logit of v
    base = go.aggregate(col, row, s, d, T, 2)
    for c in (-0.9, 25.0, 700.0):
        shifted = go.aggregate(col, row, s, d + c * (np.arange(50) % 2 == 0)[:, None], T, 2)
        assert np.allclose(shifted, base, rtol=1e-12, atol=1e-12)
    _, _, m, z = go.stats(col, row, s, d + 700.0, 0.2)
    assert np.isfinite(z).all() and (z >= 1).all()
