"""The sampling law (tests/sample_law.py) on the sampler's numpy restatement, on the CPU: its draws pass every
statistic, the statistics are calibrated (their p-values are uniform over independent seeds), and each of six
mutations of the restatement is rejected by the statistic named for it.  The GPU file holds the kernels to the same
statistics and thresholds."""
import numpy as np
import pytest
from scipy import stats

import sample_law as sl
import sample_oracle as so


def draws(deg, k, ids=None, steps=sl.STEPS, **kw):
    ids = np.arange(sl.N_DST) if ids is None else ids
    return sl.restated_draws(deg, k, ids, range(steps), **kw)


@pytest.mark.parametrize("deg,k", sl.RESTATED_CLASSES)
def test_restated_floyd_keeps_uniform_subsets(deg, k):
    s = draws(deg, k)
    sl.check_subsets(s, deg)
    p = sl.law_p_values(s, deg)
    assert not sl.failures(p), p


def independence(deg, k, **kw):
    """independence_p_values of class d<deg> at fanout k, drawn by the restatement (or a mutation of its keys)."""
    ids = sl.CLASSES["d%d" % deg][0]

    def one(**o):
        return draws(deg, k, ids, **kw, **o).reshape(sl.STEPS, ids.size, k)
    return sl.independence_p_values(one(), one(seed=sl.SEED + 1), one(hop=1), deg)


@pytest.mark.parametrize("deg,k", [(100, 1), (6, 3)])
def test_restated_draws_are_independent(deg, k):
    p = independence(deg, k)
    assert len(p) == (10 if k == 1 else 5)
    assert not sl.failures(p), p


@pytest.mark.parametrize("k", [3, 33])
def test_restated_sample_keeps_the_law_in_every_class(k):
    """sample_oracle.sample over the CSC of run k: kept edges name their slots, `low` keeps every slot, and each class
    passes (a)-(c) and (e)."""
    names = sl.RUNS[k]
    col, row, w = sl.build_csc(names)
    seeds = sl.seeds(k)
    weights = []
    for step in range(sl.SAMPLE_STEPS):
        b = so.sample(col, row, w, seeds, [k], sl.SEED, step)[0]
        sl.check_kept_edges(col, row, b["dst"], b["column_offset"], b["weight"], b["row_global"])
        weights.append(b["weight"])
    got = sl.split_run(np.stack(weights), k)
    assert (got["low"] == sl.low_slots(k)).all()
    for n in names[:-1]:
        deg = sl.class_degree(n)
        sl.check_subsets(got[n], deg)
        p = sl.law_p_values(got[n], deg)
        assert not sl.failures(p), (n, p)


def test_statistics_are_calibrated_over_seeds():
    """Over CAL_SEEDS independent seeds the p-values of the real restatement are uniform (KS), so p >= P_PASS is a
    test of the law, not of an approximation.  The inclusion statistic without its (deg-1)/deg factor is not."""
    inc = ((2, 1), (3, 2), (12, 6), (65, 64), (100, 33))
    sub = ((6, 3), (8, 4))
    pv = {}
    ids = np.arange(sl.N_DST)
    for i in range(sl.CAL_SEEDS):
        seed = sl.CAL_SEED + i
        for deg, k in inc:
            x = draws(deg, k, steps=sl.CAL_STEPS, seed=seed)
            pv.setdefault(("inclusion", deg, k), []).append(sl.inclusion_p(x, deg))
        for deg, k in sub:
            x = draws(deg, k, steps=sl.CAL_STEPS, seed=seed)
            pv.setdefault(("subset", deg, k), []).append(sl.subset_p(x, deg))
        x = draws(8, 1, steps=sl.CAL_STEPS, seed=seed).reshape(sl.CAL_STEPS, ids.size)
        pv.setdefault(("contingency", 8, 1), []).append(sl.contingency_p(x[:, 0::2], x[:, 1::2], 8))
    for key, p in pv.items():
        assert len(p) == sl.CAL_SEEDS
        assert stats.kstest(p, "uniform").pvalue >= sl.KS_MIN, key
    # deg 2 over 4 * CAL_SEEDS seeds, with the factor and without it: X = 2 (c_0 - N/2)^2 / (N/4), twice chi2(1)
    n = sl.CAL_STEPS * sl.N_DST
    s = [draws(2, 1, steps=sl.CAL_STEPS, seed=sl.CAL_SEED + i) for i in range(4 * sl.CAL_SEEDS)]
    good = [sl.inclusion_p(x, 2) for x in s]
    bad = [float(stats.chi2.sf(2 * ((x == 0).sum() - n / 2) ** 2 / (n / 4), 1)) for x in s]
    assert stats.kstest(good, "uniform").pvalue >= sl.KS_MIN
    assert stats.kstest(bad, "uniform").pvalue < sl.KS_MIN


# ---- mutations of the restatement --------------------------------------------------------------------------------

def mutated_floyd(bits=32, span=1, keep_t=False):
    """sample_oracle.floyd with one change: t = (h * (j + span)) >> bits from the top `bits` bits h of the hash
    (32 and 1 in K8), and, with keep_t, t kept on a hit instead of j.  mutated_floyd() is sample_oracle.floyd."""
    def floyd(keys, deg, k):
        n = keys.shape[0]
        chosen = np.zeros((n, k), dtype=np.int64)
        deg = deg.astype(np.uint64)
        for i in range(k):
            j = deg - np.uint64(k) + np.uint64(i)
            h = so.splitmix64(keys ^ j) >> np.uint64(64 - bits)
            t = ((h * (j + np.uint64(span))) >> np.uint64(bits)).astype(np.int64)
            hit = (chosen[:, :i] == t[:, None]).any(1) if i else np.zeros(n, dtype=bool)
            chosen[:, i] = t if keep_t else np.where(hit, j.astype(np.int64), t)
        return np.sort(chosen, axis=1)
    return floyd


def first_k(keys, deg, k):
    return np.tile(np.arange(k, dtype=np.int64), (keys.shape[0], 1))


def keys_without_hop(seed, steps, hop, ids):
    return sl.draw_keys(seed, steps, 0, ids)


def keys_without_step(seed, steps, hop, ids):
    return np.concatenate([so.dst_keys(so.splitmix64(np.uint64(seed)), hop, ids) for _ in steps])


def test_unmutated_floyd_is_the_restatement():
    for deg, k in ((6, 3), (100, 33), (70000, 64)):
        keys = sl.draw_keys(sl.SEED, range(4), 0, np.arange(sl.N_DST))
        d = np.full(keys.size, deg, dtype=np.int64)
        assert np.array_equal(mutated_floyd()(keys, d, k), so.floyd(keys, d, k))


def test_draw_from_the_open_range_is_rejected_by_inclusion_and_subsets():
    f = mutated_floyd(span=0)             # t in [0, j) instead of [0, j]
    for deg, k in ((6, 3), (100, 33), (65, 64)):
        s = draws(deg, k, floyd=f)
        sl.check_subsets(s, deg)          # still distinct slots: only the law tells
        assert sl.inclusion_p(s, deg) <= sl.P_REJECT, (deg, k)
        if deg != 100:
            assert sl.subset_p(s, deg) <= sl.P_REJECT, (deg, k)


def test_twelve_bit_hash_is_rejected_by_inclusion_at_a_hub():
    assert sl.inclusion_p(draws(20000, 25, floyd=mutated_floyd(bits=12)), 20000) <= sl.P_REJECT


def test_duplicate_slot_on_a_hit_fails_the_hard_check():
    with pytest.raises(AssertionError, match="distinct and ascending"):
        sl.check_subsets(draws(6, 3, floyd=mutated_floyd(keep_t=True)), 6)


@pytest.mark.parametrize("deg,k", [(100, 1), (6, 3)])
def test_key_without_the_hop_is_rejected_by_hop_independence(deg, k):
    p = independence(deg, k, keys=keys_without_hop)
    rejected = {n for n, v in p.items() if v <= sl.P_REJECT}
    assert {"identical/hops"} <= rejected and ("contingency/hops" in rejected or k > 1), p


@pytest.mark.parametrize("deg,k", [(100, 1), (6, 3)])
def test_key_without_the_step_is_rejected_by_step_independence(deg, k):
    p = independence(deg, k, keys=keys_without_step)
    rejected = {n for n, v in p.items() if v <= sl.P_REJECT}
    assert {"identical/steps"} <= rejected and ("contingency/steps" in rejected or k > 1), p


def test_first_k_slots_are_rejected_by_inclusion():
    for deg, k in ((100, 33), (70000, 3)):
        assert sl.inclusion_p(draws(deg, k, floyd=first_k), deg) <= sl.P_REJECT, (deg, k)
