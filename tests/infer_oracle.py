"""float64 numpy restatement of GCNSampleImpl.infer (full-neighbour inference of sampled GCN).

Layer l of an L-layer model aggregates with the expectation of the sampled aggregation of hop h = L-1-l, which keeps
min(indeg(v), k_h) uniform in-edge slots of every destination v:

    X_{l+1} = relu(s ⊙ A (X_l W_l)),   s_v = min(1, k_h / indeg(v))  (1 when indeg(v) = 0),   no relu on the last layer

with A the weighted in-edge CSC (col, row, w): (A X)[v] = sum_{e in [col[v], col[v+1])} w[e] X[row[e]]."""
import numpy as np


def scale(col, k):
    """s_v = min(1, k / indeg(v)), 1 where indeg(v) == 0."""
    deg = np.diff(np.asarray(col, dtype=np.int64)).astype(np.float64)
    return np.where(deg > k, k / np.maximum(deg, 1), 1.0)


def aggregate(col, row, w, X):
    """(A X) in float64: row v sums w[e] * X[row[e]] over its in-edges."""
    col = np.asarray(col, dtype=np.int64)
    n = col.size - 1
    E = int(col[-1] - col[0])
    row = np.asarray(row, dtype=np.int64)[col[0]:col[-1]]
    w = np.ones(E) if w is None else np.asarray(w, dtype=np.float64)[col[0]:col[-1]]
    dst = np.repeat(np.arange(n), np.diff(col))
    out = np.zeros((n, X.shape[1]))
    np.add.at(out, dst, w[:, None] * np.asarray(X, dtype=np.float64)[row])
    return out


def bf16(a):
    """float32 values rounded to the nearest BF16 (ties to even), as float64: what a BF16 table stores."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16 << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def infer(col, row, w, X, Ws, fanout, order="widths", round_operand=None):
    """The last layer's [V, classes] outputs.  order: "widths" (transform first where a layer narrows, as infer
    does), "transform" or "aggregate" (every layer in that order).  round_operand(layer, rows) is applied to every
    aggregated operand (e.g. bf16 for BF16 tables)."""
    L = len(Ws)
    x = np.asarray(X, dtype=np.float64)
    for l, W in enumerate(Ws):
        W = np.asarray(W, dtype=np.float64)
        s = scale(col, fanout[L - 1 - l])[:, None]
        first = (W.shape[1] < W.shape[0]) if order == "widths" else order == "transform"
        op = x @ W if first else x
        if round_operand is not None:
            op = round_operand(l, op)
        y = s * aggregate(col, row, w, op)
        if not first:
            y = y @ W
        x = np.maximum(y, 0) if l < L - 1 else y
    return x


def magnitude(col, row, w, X, Ws, fanout):
    """The same chain on absolute values without relu: a bound on every intermediate's size, against which a float32
    or BF16 result's error is measured."""
    return infer(col, row, None if w is None else np.abs(w), np.abs(X), [np.abs(W) for W in Ws], fanout,
                 order="aggregate")
