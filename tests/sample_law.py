"""The sampling law of the neighbour sampler (K8) and the statistics that hold draws to it, shared by
tests/test_sample_law.py (the numpy restatement, CPU) and tests/test_sample_law_gpu.py (the kernels).

The law: a destination with deg <= k in-edge slots keeps every slot; one with deg > k keeps a k-subset of its slots
that is uniform over all C(deg, k) subsets, drawn independently for every destination, hop, step and seed.  The
restatement (sample_oracle.py) is bit-exact to the kernels, so it cannot show that the algorithm itself is wrong; these
statistics can.

Graph.  One CSC holds every destination class, built directly in numpy: each class has N_DST destinations with the
same degree (the `low` class has degrees 0..64), and the weight of an edge is float(its local slot), exact below
2^24, so a block's `weight` names the kept slot even where sources repeat (the `multi` class: 100 slots over 10
distinct sources).  Sources are vertices without in-edges, so a destination-inclusive second hop samples the first
hop's destinations again and nothing else.  Half of class d100 sits HIGH_BIT above the other half, so destinations one
high id bit apart are compared too.

Runs.  RUNS[k] lists the classes sampled together at fanout k: deg = k+1 (the complement law: the dropped slot must
be uniform) and 2k, the hub degrees 100 .. 70 000 (the last above 2^16), the multigraph class, and the `low`
destinations with deg <= k.  A run is STEPS steps of one hop over all its seeds, so every class gets STEPS * N_DST =
2^17 draws.  SUBSET_CLASSES add (8, 4) and (12, 6) for the subset law.  The fanouts cover every branch of select_kernel:
deg <= k, Floyd with k <= 32 (one lane pass of the hit test and the rank loop) and k > 32 (two passes).

Thresholds, fixed before any run: every statistic of the real sampler must give p >= P_PASS, every mutation of the
restatement p <= P_REJECT (or fail a hard check).  The sampler is deterministic, so each p-value is a fixed number for
(graph, SEED, steps): these seeds were chosen before any draw was looked at and are not to be tuned to results."""
from math import comb

import numpy as np
from scipy import stats

import sample_oracle as so

SEED = 20261018            # the sampler seed of every run; SEED + 1 for the seed-independence run
STEPS = 512
N_DST = 256                # STEPS * N_DST = 2^17 draws per class of a run
FANOUTS = (1, 2, 3, 25, 32, 33, 63, 64)
HUB_DEGREES = (100, 1000, 20000, 70000)
SUBSET_CLASSES = ((8, 4), (12, 6))
SUBSET_MAX = 5000          # the subset law runs where C(deg, k) <= SUBSET_MAX (>= 26 expected draws per subset)
PAIR_MAX_DEG = 100         # the pair law runs where deg <= 100 and 2 <= k <= deg / 2
MULTI_DEG, MULTI_SOURCES = 100, 10
LOW_MAX_DEG = 64
HIGH_BIT = 1 << 20
SRC_BASE, SRC_POOL = 1 << 16, 65521    # sources: SRC_BASE + [0, SRC_POOL), a prime, none with in-edges
V = HIGH_BIT + (1 << 17)
P_PASS = 1e-6
P_REJECT = 1e-12
# the CPU file: classes drawn by sample_oracle.floyd (the subset-law classes, the complement law at k = 3 and 64, k > 32
# against deg 100, hubs below and above 2^16), steps of sample_oracle.sample per run, and the calibration over seeds
RESTATED_CLASSES = ((2, 1), (4, 3), (6, 3), (8, 4), (12, 6), (65, 64), (100, 2), (100, 33), (20000, 25), (70000, 3))
SAMPLE_STEPS = 128         # 32 768 draws per class
CAL_SEED, CAL_SEEDS, CAL_STEPS = SEED + 1000, 128, 16     # seeds CAL_SEED + i, 4096 draws per seed and class
KS_MIN = 1e-3


def _run(k):
    return tuple("d%d" % d for d in sorted({k + 1, 2 * k})) + tuple("d%d" % d for d in HUB_DEGREES) + ("multi", "low")


RUNS = {k: _run(k) for k in FANOUTS}
RUNS.update({k: ("d%d" % d,) for d, k in SUBSET_CLASSES})


def _layout():
    """name -> (destination ids, degrees) of every class; ids are consecutive from 0, except d100's upper half."""
    degrees = sorted({int(n[1:]) for names in RUNS.values() for n in names if n.startswith("d")})
    out, nxt = {}, 0
    for name in ["d%d" % d for d in degrees] + ["multi", "low"]:
        ids = np.arange(nxt, nxt + N_DST, dtype=np.int64)
        nxt += N_DST
        if name == "d100":
            ids[N_DST // 2:] = ids[:N_DST // 2] + HIGH_BIT
        deg = (np.arange(N_DST) % (LOW_MAX_DEG + 1) if name == "low"
               else np.full(N_DST, MULTI_DEG if name == "multi" else int(name[1:])))
        out[name] = (ids, deg.astype(np.int64))
    assert nxt <= SRC_BASE and SRC_BASE + SRC_POOL <= HIGH_BIT and out["d100"][0].max() < V
    return out


CLASSES = _layout()


def build_csc(names):
    """CSC (column_offset uint32 [V+1], row_indices uint32, weight float32) whose only destinations are the classes
    `names`; the weight of an edge is its local slot, the source of slot j of v a fixed function of (v, j)."""
    indeg = np.zeros(V, dtype=np.int64)
    for n in names:
        ids, deg = CLASSES[n]
        indeg[ids] = deg
    col = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(indeg, out=col[1:])
    row = np.empty(int(col[-1]), dtype=np.uint32)
    w = np.empty(int(col[-1]), dtype=np.float32)
    for n in names:
        for v, d in zip(*CLASSES[n]):
            j = np.arange(d, dtype=np.int64)
            src = j % MULTI_SOURCES if n == "multi" else (v * 7919 + j * 104729) % SRC_POOL
            row[col[v]:col[v] + d] = SRC_BASE + src
            w[col[v]:col[v] + d] = j
    return col.astype(np.uint32), row, w


def plan(k):
    """[(name, ids, degrees)] of run k in seed order; the `low` class keeps only its destinations with deg <= k."""
    out = []
    for n in RUNS[k]:
        ids, deg = CLASSES[n]
        keep = deg <= k if n == "low" else np.ones(ids.size, dtype=bool)
        out.append((n, ids[keep], deg[keep]))
    return out


def seeds(k):
    return np.concatenate([ids for _, ids, _ in plan(k)])


def split_run(weights, k):
    """name -> kept slots of run k from its per-step block weights [steps, n_edges]: [steps * n, k] (draw s * n + i
    is destination i at step s) for a class with deg > k, and [steps, edges] for `low`."""
    slots = np.asarray(weights)
    assert np.array_equal(slots, np.round(slots)), "a block weight is not a slot index"
    slots = slots.astype(np.int64)
    out, e0 = {}, 0
    for n, ids, deg in plan(k):
        m = int(np.minimum(deg, k).sum())
        part = slots[:, e0:e0 + m]
        out[n] = part if n == "low" else part.reshape(-1, k)
        e0 += m
    assert e0 == slots.shape[1], (e0, slots.shape)
    return out


def low_slots(k):
    """The slots every step must keep of run k's `low` destinations: all of them, 0 .. deg-1 each."""
    (_, _, deg), = [p for p in plan(k) if p[0] == "low"]
    return np.concatenate([np.arange(d) for d in deg]).astype(np.int64)


def class_degree(name):
    return int(CLASSES[name][1][0])


# ---- draws of the restatement ------------------------------------------------------------------------------------

def draw_keys(seed, steps, hop, ids):
    """Destination keys of K8 for every (step, destination), step-major: splitmix64(step_key(seed, step) ^ (hop << 32
    | v))."""
    return np.concatenate([so.dst_keys(so.step_key(seed, s), hop, ids) for s in steps])


def restated_draws(deg, k, ids, steps, seed=SEED, hop=0, floyd=so.floyd, keys=draw_keys):
    """[len(steps) * len(ids), k] slots that sample_oracle.floyd keeps (or a mutation passed as floyd / keys)."""
    kk = keys(seed, steps, hop, np.asarray(ids, dtype=np.int64))
    return floyd(kk, np.full(kk.size, deg, dtype=np.int64), k)


# ---- hard checks ---------------------------------------------------------------------------------------------------

def check_subsets(slots, deg):
    """(e): every draw holds slots in [0, deg), distinct and ascending (the order K8 writes them in)."""
    slots = np.asarray(slots)
    assert slots.min() >= 0 and slots.max() < deg, "a kept slot lies outside [0, %d)" % deg
    if slots.shape[1] > 1:
        bad = np.nonzero((np.diff(slots, axis=1) <= 0).any(1))[0]
        assert bad.size == 0, "draw %d keeps slots %s: not distinct and ascending" % (bad[0], slots[bad[0]].tolist())


def check_kept_edges(col, row, dst, column_offset, weight, row_global):
    """(e): each kept edge of a block is the slot its weight names, of its own destination: row_global equals
    row[col[dst] + weight]."""
    cnt = np.diff(np.asarray(column_offset, dtype=np.int64))
    e_dst = np.repeat(np.asarray(dst, dtype=np.int64), cnt)
    pos = np.asarray(col, dtype=np.int64)[e_dst] + np.asarray(weight).astype(np.int64)
    assert np.array_equal(np.asarray(row)[pos], np.asarray(row_global)), "a kept weight is not the weight of its slot"


# ---- statistics (each returns a p-value) ---------------------------------------------------------------------------

def inclusion_p(slots, deg):
    """(a) Inclusion.  N draws of k slots; c_i counts draws that keep slot i, p = k/deg.  Under the law the indicator
    vector of one draw has covariance p(1-p) deg/(deg-1) (I - J/deg): rank deg-1, and the sum of its eigenvalues is
    deg p(1-p).  So

        X = (deg-1)/deg * sum_i (c_i - N p)^2 / (N p (1-p))

    has mean deg-1 and variance 2 (deg-1)(N-1)/N, those of chi2(deg-1), to which it is compared (one-sided: a large
    X rejects).  Without the (deg-1)/deg factor X is deg/(deg-1) times too large (twice at deg 2); the plain
    multinomial chi2 sum (c_i - Np)^2 / (Np) is (1-p) deg/(deg-1) times X and accepts anything at k close to deg."""
    slots = np.asarray(slots)
    n, k = slots.shape
    c = np.bincount(slots.ravel(), minlength=deg)[:deg].astype(np.float64)
    p = k / deg
    x = (deg - 1) / deg * ((c - n * p) ** 2).sum() / (n * p * (1 - p))
    return float(stats.chi2.sf(x, deg - 1))


def subset_p(slots, deg):
    """(b) Subset law.  Pearson chi2 over all C = C(deg, k) subsets, e = N / C expected draws each:
    X = sum_s (o_s - e)^2 / e, against chi2(C-1).  A subset s_0 < .. < s_{k-1} is counted at its colex rank
    sum_i C(s_i, i+1), which is < C for every k-subset of [0, deg); a larger rank is a draw outside the law's
    support (p = 0)."""
    slots = np.asarray(slots)
    n, k = slots.shape
    c = comb(deg, k)
    assert c <= SUBSET_MAX
    table = np.array([[min(comb(s, i + 1), c) for i in range(k)] for s in range(deg)], dtype=np.int64)
    rank = table[np.sort(slots, axis=1), np.arange(k)].sum(1)
    if rank.max() >= c:
        return 0.0
    e = n / c
    x = ((np.bincount(rank, minlength=c) - e) ** 2).sum() / e
    return float(stats.chi2.sf(x, c - 1))


def pair_p(slots, deg):
    """(c) Pairs.  c_ab counts draws that keep both slots a < b; under the law c_ab ~ Binomial(N, q), q =
    k(k-1)/(deg(deg-1)).  The most extreme pair, by its exact two-sided binomial tail p_ab (the normal tail of
    |z| = |c_ab - Nq| / sqrt(Nq(1-q)) is too light where Nq is small: 27 at (100, 2)), against a Bonferroni bound:
    p = min(1, M * min_ab p_ab), M = deg(deg-1)/2."""
    slots = np.asarray(slots)
    n, k = slots.shape
    ind = np.zeros((n, deg), dtype=np.float32)
    np.put_along_axis(ind, slots, 1.0, axis=1)
    both = np.rint(ind.T @ ind).astype(np.int64)[np.triu_indices(deg, 1)]   # exact: counts < 2^24
    q = k * (k - 1) / (deg * (deg - 1))
    tail = 2 * np.minimum(stats.binom.cdf(both, n, q), stats.binom.sf(both - 1, n, q))
    return float(min(1.0, both.size * tail.min()))


def contingency_p(a, b, deg):
    """(d) Independence of two single-slot draws (k = 1) taken together: the deg x deg table T[a, b] against the
    product of its margins, Pearson chi2 with (r-1)(c-1) degrees of freedom over its r non-empty rows and c columns."""
    a, b = np.asarray(a).ravel(), np.asarray(b).ravel()
    t = np.bincount(a * deg + b, minlength=deg * deg).reshape(deg, deg).astype(np.float64)
    t = t[t.sum(1) > 0][:, t.sum(0) > 0]
    e = np.outer(t.sum(1), t.sum(0)) / t.sum()
    df = (t.shape[0] - 1) * (t.shape[1] - 1)
    return float(stats.chi2.sf(((t - e) ** 2 / e).sum(), df)) if df else 0.0


def identical_p(a, b, deg):
    """(d) Independence of two k-subset draws taken together: the number of pairs that drew the same subset against
    Binomial(N, 1 / C(deg, k)), two-sided."""
    a, b = np.asarray(a), np.asarray(b)
    same = int((a == b).all(1).sum())
    return float(stats.binomtest(same, a.shape[0], 1 / comb(deg, a.shape[1])).pvalue)


def law_p_values(slots, deg):
    """Every statistic of (a)-(c) that applies to a class: {"inclusion", "subset", "pairs"} -> p."""
    k = np.asarray(slots).shape[1]
    out = {"inclusion": inclusion_p(slots, deg)}
    if comb(deg, k) <= SUBSET_MAX:
        out["subset"] = subset_p(slots, deg)
    if deg <= PAIR_MAX_DEG and 2 <= k <= deg // 2:
        out["pairs"] = pair_p(slots, deg)
    return out


def independence_p_values(draws, other_seed, other_hop, deg):
    """(d) for one class drawn as [steps, n, k] at (SEED, hop 0), at SEED + 1 and at hop 1 (the same destinations and
    steps), destinations ordered as CLASSES lists them.  Pairs: neighbouring destinations (v, v+1) at the same step,
    destinations n/2 apart in that order at the same step (for d100: one id bit, HIGH_BIT, apart), steps (2s, 2s+1)
    of one destination, the two seeds and the two hops.  Identical-subset counts for every pair; with k = 1 also the
    contingency chi2."""
    x, s, h = (np.asarray(a) for a in (draws, other_seed, other_hop))
    n, k = x.shape[1], x.shape[2]
    pairs = {"destinations": (x[:, 0::2], x[:, 1::2]), "high_bit": (x[:, :n // 2], x[:, n // 2:]),
             "steps": (x[0::2], x[1::2]), "seeds": (x, s), "hops": (x, h)}
    out = {}
    for name, (a, b) in pairs.items():
        a, b = a.reshape(-1, k), b.reshape(-1, k)
        out["identical/" + name] = identical_p(a, b, deg)
        if k == 1:
            out["contingency/" + name] = contingency_p(a, b, deg)
    return out


def failures(pvals, threshold=P_PASS):
    """The statistics of {name: p} below threshold."""
    return {n: p for n, p in pvals.items() if not p >= threshold}
