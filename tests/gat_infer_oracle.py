"""float64 numpy restatement of GATSampleImpl.infer (full-neighbour inference of sampled GAT).

Layer l of an L-layer model, with H heads of width D and weights (W, al, ar), over the in-edge CSC (col, row):

    T = X W,   s[u, h] = <T[u, h, :], al[h]>,   d[v, h] = <T[v, h, :], ar[h]>
    a[e, h] = softmax over the in-edge slots e of v of leaky_relu(s[row[e], h] + d[v, h], 0.2)
    Y[v, h, :] = sum_e a[e, h] T[row[e], h, :]      (a zero row at in-degree 0)
    X_{l+1} = relu(Y), or log_softmax(Y) on the last layer

Every slot counts, so a multi-edge counts once per slot; edge weights are ignored."""
import numpy as np

from infer_oracle import bf16  # noqa: F401  (re-exported for the tests)

SLOPE = 0.2


def leaky(x, slope=SLOPE):
    return np.where(x > 0, x, slope * x)


def stats(col, row, s, d, slope=SLOPE):
    """(logit [E, H], dst [E], m [n, H], z [n, H]) of the CSC piece col (absolute edge positions, n = col.size - 1):
    the segment maximum and the sum of exp(logit - m) of every destination and head; (0, 1) for an empty one."""
    col = np.asarray(col, dtype=np.int64)
    n = col.size - 1
    src = np.asarray(row, dtype=np.int64)[col[0]:col[-1]]
    dst = np.repeat(np.arange(n), np.diff(col))
    logit = leaky(np.asarray(s, np.float64)[src] + np.asarray(d, np.float64)[dst], slope)
    H = logit.shape[1]
    m = np.full((n, H), -np.inf)
    np.maximum.at(m, dst, logit)
    empty = np.diff(col) == 0
    m[empty] = 0.0
    z = np.zeros((n, H))
    np.add.at(z, dst, np.exp(logit - m[dst]))
    z[empty] = 1.0
    return logit, dst, m, z


def aggregate(col, row, s, d, T, heads, slope=SLOPE):
    """Y [n, H*D]: the attention-weighted sum over the piece's in-edges of the source rows T [V, H*D] (T may be the
    BF16-rounded rows while s and d come from the float32 ones)."""
    logit, dst, m, z = stats(col, row, s, d, slope)
    a = np.exp(logit - m[dst]) / z[dst]
    col = np.asarray(col, dtype=np.int64)
    src = np.asarray(row, dtype=np.int64)[col[0]:col[-1]]
    T = np.asarray(T, dtype=np.float64)
    D = T.shape[1] // heads
    y = np.zeros((col.size - 1, heads, D))
    np.add.at(y, dst, a[:, :, None] * T[src].reshape(-1, heads, D))
    return y.reshape(col.size - 1, heads * D)


def scores(T, al, ar, heads):
    """s and d of T [n, H*D] for the attention vectors al, ar [H, D]."""
    t = np.asarray(T, dtype=np.float64).reshape(T.shape[0], heads, -1)
    return (t * al).sum(-1), (t * ar).sum(-1)


def log_softmax(y):
    m = y.max(1, keepdims=True)
    return y - m - np.log(np.exp(y - m).sum(1, keepdims=True))


def aggregate_abs(col, row, s, d, B, heads, slope=SLOPE):
    """sum_e a[e, h] B[src(e), h, :] with the attention of (s, d): the size of what aggregate() sums, for bounds."""
    return aggregate(col, row, s, d, np.abs(B), heads, slope)


def infer(col, row, X, Ws, als, ars, heads, round_rows=None, slope=SLOPE, with_bound=False):
    """The last layer's [V, classes] log-probabilities.  heads: per layer.  round_rows(T) is applied to the gathered
    rows only (bf16 for BF16 tables); the scores come from the unrounded T.  with_bound=True also returns a per-row
    bound on the size of everything the float32 computation rounded: the same chain on |X| and |W| with the exact
    attention; for the log_softmax outputs 2 * its row maximum, plus the output's own size."""
    x = np.asarray(X, dtype=np.float64)
    b = np.abs(x)
    L = len(Ws)
    for l in range(L):
        W = np.asarray(Ws[l], np.float64)
        T = x @ W
        s, d = scores(T, np.asarray(als[l], np.float64), np.asarray(ars[l], np.float64), heads[l])
        rows = T if round_rows is None else round_rows(T)
        y = aggregate(col, row, s, d, rows, heads[l], slope)
        b = aggregate_abs(col, row, s, d, b @ np.abs(W), heads[l], slope)
        x = np.maximum(y, 0) if l < L - 1 else log_softmax(y)
    if with_bound:
        return x, 2 * b.max(1, keepdims=True) + np.abs(x)
    return x
