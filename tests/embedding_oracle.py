"""Restatements of a ShardedEmbedding step (feature_table.py, K11) in numpy float32: the rank-order sum of the rows
several ranks send, and lazy row-sparse Adam with Parameter's schedule (adam.AdamSchedule)."""
import numpy as np


def rank_order_sum(rows):
    """rows[0] + rows[1] + ... in float32, left to right: the gradient of a row, its contributors in ascending rank
    order, starting from the first contributor's row."""
    acc = np.array(rows[0], dtype=np.float32, copy=True)
    for r in rows[1:]:
        acc = (acc + np.asarray(r, dtype=np.float32)).astype(np.float32)
    return acc


def adam_rows(W, M, V, g, sched):
    """Parameter.learn_with_decay_Adam's arithmetic (the host mirror's order of operations) on float32 rows W, M, V in
    place, with gradient g and the schedule's current values."""
    f = np.float32
    one = f(1)
    W_g = W * f(sched.weight_decay) + g
    M[...] = f(sched.beta1) * M + f(one - sched.beta1) * W_g
    V[...] = f(sched.beta2) * V + f(one - sched.beta2) * W_g * W_g
    W -= f(sched.alpha) * M / (np.sqrt(V) + f(sched.epsilon))


def lazy_adam(W, M, V, steps, sched):
    """Row-sparse lazy Adam: for each step (ids, grad rows), rows ids of W, M, V get adam_rows with the step-wide
    schedule values, every other row keeps its bits; sched.next() after every step, touched or not."""
    for ids, g in steps:
        ids = np.asarray(ids, dtype=np.int64)
        if ids.size:
            w, m, v = W[ids], M[ids], V[ids]
            adam_rows(w, m, v, np.asarray(g, dtype=np.float32), sched)
            W[ids], M[ids], V[ids] = w, m, v
        sched.next()
