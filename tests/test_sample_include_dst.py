"""CPU checks of the numpy restatement of the sampler's destination-inclusive mode (NTS_SAMPLER_INCLUDE_DST), which
the GPU tests hold the kernels to bit for bit: a hop keeps the default mode's edges, its sources are the sorted union
of kept sources and destinations, and dst_pos locates every destination among them."""
import numpy as np
import pytest

import golden_store
import sample_oracle as so
from test_sample_oracle import csc


def sample_hop_include_dst(col, row, w, dst, k, skey, hop):
    """One destination-inclusive hop: the default hop's edges (sample_oracle.sample_hop), sources = distinct ids of
    (kept sources U destinations) ascending, dst_pos = each destination's index in them."""
    b = so.sample_hop(col, row, w, dst, k, skey, hop)
    src = np.union1d(b["row_global"], b["dst"]).astype(np.uint32)
    row_local = np.searchsorted(src, b["row_global"]).astype(np.int64)
    edge_dst = np.repeat(np.arange(b["dst"].size, dtype=np.int64), np.diff(b["column_offset"].astype(np.int64)))
    order = np.argsort(row_local, kind="stable")
    r_o = np.zeros(src.size + 1, dtype=np.uint32)
    np.cumsum(np.bincount(row_local, minlength=src.size), out=r_o[1:])
    b.update({"src": src, "row_indices": row_local.astype(np.uint32), "row_offset": r_o,
              "column_indices": edge_dst[order].astype(np.uint32), "weight_backward": b["weight"][order],
              "dst_pos": np.searchsorted(src, b["dst"]).astype(np.uint32)})
    return b


def sample_include_dst(col, row, w, seeds, fanout, seed, step):
    """Every hop of one destination-inclusive sample; hop h+1's destinations are hop h's sources."""
    col = np.asarray(col, dtype=np.uint32)
    row = np.asarray(row, dtype=np.uint32)
    w = np.asarray(w, dtype=np.float32)
    skey = so.step_key(seed, step)
    hops, dst = [], np.asarray(seeds, dtype=np.int64)
    for h, k in enumerate(fanout):
        b = sample_hop_include_dst(col, row, w, dst, int(k), skey, h)
        hops.append(b)
        dst = b["src"].astype(np.int64)
    return hops


def cora():
    return golden_store.load("cora_self_P1_F8")["edges"], 2708


def zipf_hubs(V=20000, E=150000, seed=1):
    """Power-law sources and two hub destinations with 6000 and 3000 in-edges (multi-edges included)."""
    rng = np.random.default_rng(seed)
    src = np.minimum(rng.zipf(1.6, E) - 1, V - 1)
    dst = rng.integers(0, V, E)
    dst[:6000] = 5
    dst[6000:9000] = 77
    return np.stack([src, dst], 1).astype(np.int64), V


def edges_of(b):
    """{global destination: (global sources, weights)} of a block, in slot order."""
    c = b["column_offset"].astype(np.int64)
    return {int(d): (b["row_global"][c[i]:c[i + 1]], b["weight"][c[i]:c[i + 1]]) for i, d in enumerate(b["dst"])}


@pytest.mark.parametrize("graph", ["cora", "zipf"])
@pytest.mark.parametrize("fanout,seed,step", [([5, 10], 0, 0), ([64, 3], 2, 5), ([25, 10, 3], 1, 7)])
def test_include_dst_blocks_are_the_default_edges_plus_the_destinations(graph, fanout, seed, step):
    edges, V = cora() if graph == "cora" else zipf_hubs()
    col, row, w = csc(edges, V)
    rng = np.random.default_rng(seed)
    seeds = rng.choice(V, 200, replace=False)
    if graph == "zipf":
        seeds[:2] = [5, 77]
    inc = sample_include_dst(col, row, w, seeds, fanout, seed, step)
    ref = so.sample(col, row, w, seeds, fanout, seed, step)
    dst = np.asarray(seeds, dtype=np.uint32)
    for h, (b, r) in enumerate(zip(inc, ref)):
        assert np.array_equal(b["dst"], dst)
        assert np.array_equal(b["src"], np.union1d(b["row_global"], b["dst"]))
        assert np.all(np.diff(b["src"].astype(np.int64)) > 0)
        assert np.array_equal(b["src"][b["dst_pos"]], b["dst"])
        assert np.array_equal(b["src"][b["row_indices"]], b["row_global"])
        # every destination the default mode samples at this hop keeps the same edges, weights and order
        mine, theirs = edges_of(b), edges_of(r)
        assert set(theirs) <= set(mine)
        if h == 0:
            assert set(theirs) == set(mine)
        for d, (s, wt) in theirs.items():
            assert np.array_equal(mine[d][0], s) and np.array_equal(mine[d][1].view(np.uint32), wt.view(np.uint32))
        # the transposed block holds the same triples, edges of a source in edge order
        e_dst = np.repeat(np.arange(b["dst"].size), np.diff(b["column_offset"].astype(np.int64)))
        t_src = np.repeat(np.arange(b["src"].size), np.diff(b["row_offset"].astype(np.int64)))
        assert np.array_equal(t_src, np.sort(b["row_indices"].astype(np.int64), kind="stable"))
        order = np.argsort(b["row_indices"], kind="stable")
        assert np.array_equal(b["column_indices"], e_dst[order])
        dst = b["src"]
    # the destination set only grows with depth
    for a, b in zip(inc, inc[1:]):
        assert np.isin(a["dst"], b["dst"]).all()


def test_a_destination_without_in_edges_is_its_own_source():
    edges = np.array([[1, 0], [2, 0], [3, 0]])
    col, row, w = csc(edges, 5)
    b = sample_include_dst(col, row, w, [4, 0], [2], seed=0, step=0)[0]     # vertex 4 has no in-edge
    assert b["column_offset"].tolist() == [0, 0, 2]
    assert 4 in b["src"].tolist() and 0 in b["src"].tolist()
    assert np.array_equal(b["src"][b["dst_pos"]], [4, 0])
    e = sample_include_dst(col, row, w, [], [2, 3], seed=0, step=0)
    assert all(h["src"].size == 0 and h["dst_pos"].size == 0 and h["row_offset"].tolist() == [0] for h in e)
