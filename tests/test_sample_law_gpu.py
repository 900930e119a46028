"""The neighbour sampler (K8) on the GPU against its sampling law (tests/sample_law.py), with the statistics and
thresholds the CPU file calibrates on the restatement: every run of sample_law.RUNS (2^17 draws per class) keeps
uniform k-subsets, through the world-1 topology, three shards in one process and the whole-graph arrays; draws are
independent across destinations, hops, steps and seeds; one class equals the restatement bit for bit; and the
operator averaged over steps matches its float64 expectation.  Every p-value is printed (run with -s to see them)."""
import types

import numpy as np
import pytest
from scipy import stats

import sample_law as sl

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

EXPECT_FANOUT, EXPECT_PER_CLASS, EXPECT_F = 25, 32, 8


def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def graph():
    """The CSC of every class on the host (numpy) and the device (int32 / float32 tensors)."""
    d = dev()
    col, row, w = sl.build_csc(list(sl.CLASSES))
    return types.SimpleNamespace(col=col, row=row, w=w, col_t=torch.from_numpy(col.view(np.int32)).to(d),
                                 row_t=torch.from_numpy(row.view(np.int32)).to(d), w_t=torch.from_numpy(w).to(d))


@pytest.fixture(scope="module")
def world_one(graph):
    from neutronstarlite_b200.topology import ShardedTopology
    topo = ShardedTopology(graph.col_t, graph.row_t, graph.w_t, [0, sl.V])
    yield topo
    topo.close()


def whole_graph_arrays(g):
    """What NeighborSampler reads of a single-partition PartitionedGraph: the whole CSC as chunk 0, which it samples
    through nts_sampler_create_ex (K8's whole-graph instantiation) rather than a shard table."""
    chunk = types.SimpleNamespace(column_offset_gpu=g.col_t, row_indices_gpu=g.row_t, edge_weight_forward_gpu=g.w_t,
                                  edge_size=g.row.size)
    return types.SimpleNamespace(partitions=1, global_vertices=sl.V, graph_chunks=[chunk])


def sample_run(g, source, k, seed=sl.SEED):
    """Block weights [STEPS, n_edges] of run k (one hop, fanout k) over `source`.  Every step's block is checked on the
    device: its destinations are the seeds, each keeps min(deg, k) edges, each weight is a slot of its destination and
    each kept edge is the slot its weight names (row_global == row[col[dst] + weight])."""
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    seeds = sl.seeds(k)
    deg = g.col[seeds + 1].astype(np.int64) - g.col[seeds]
    cnt = np.minimum(deg, k)
    col_expect = torch.from_numpy(np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)).to(d)
    base = torch.from_numpy(np.repeat(g.col[seeds].astype(np.int64), cnt)).to(d)
    deg_e = torch.from_numpy(np.repeat(deg, cnt)).to(d)
    seeds_t = torch.from_numpy(seeds.astype(np.int32)).to(d)
    s = NeighborSampler(source, [k], seeds.size)
    out = torch.empty((sl.STEPS, int(cnt.sum())), dtype=torch.float32, device=d)
    bad = torch.zeros((), dtype=torch.int64, device=d)
    for step in range(sl.STEPS):
        b = s.sample(seeds_t, seed, step).blocks[0]
        slot = b.weight.long()
        bad += (b.dst != seeds_t).sum() + (b.column_offset != col_expect).sum()
        bad += ((slot < 0) | (slot >= deg_e) | (b.weight != slot.float())).sum()
        pos = (base + slot).clamp(0, g.row.size - 1)
        bad += (g.row_t[pos] != b.row_global).sum()
        out[step] = b.weight
    assert int(bad) == 0, "%d block entries differ from what the kept slots imply" % int(bad)
    return out.cpu().numpy()


def check_law(weights, k, what):
    """sample_law's checks of every class of run k: `low` keeps every slot, (e) for every class, (a)-(c) p >=
    P_PASS.  Prints each p-value."""
    got = sl.split_run(weights, k)
    fails = {}
    for n in sl.RUNS[k]:
        if n == "low":
            assert (got["low"] == sl.low_slots(k)).all(), "a destination with deg <= %d lost a slot" % k
            continue
        deg = sl.class_degree(n)
        sl.check_subsets(got[n], deg)
        p = sl.law_p_values(got[n], deg)
        print("sample law %s k=%d %s(deg %d): %s" % (what, k, n, deg,
                                                     " ".join("%s=%.3g" % kv for kv in sorted(p.items()))))
        fails.update({(n, s): v for s, v in sl.failures(p).items()})
    assert not fails, fails
    return got


@pytest.mark.parametrize("k", sorted(sl.RUNS))
def test_world_one_topology_keeps_the_law(graph, world_one, k):
    check_law(sample_run(graph, world_one, k), k, "world-1")


def test_three_shards_keep_the_law(graph):
    """The CSC split into 3 shards in this process, cut inside classes d66 and d70000, so count and select look up
    owners in the middle of a class (K8's sharded instantiation with a shard table of 3)."""
    from neutronstarlite_b200.topology import ShardedTopology
    cut = [int(sl.CLASSES[n][0][sl.N_DST // 2]) for n in ("d66", "d70000")]
    topo = ShardedTopology.split(graph.col_t, graph.row_t, graph.w_t, [0] + cut + [sl.V])
    try:
        check_law(sample_run(graph, topo, 33), 33, "3-shard")
    finally:
        topo.close()


def test_whole_graph_arrays_keep_the_law_and_equal_the_restatement(graph):
    k = 25
    got = check_law(sample_run(graph, whole_graph_arrays(graph), k), k, "whole-graph")
    ids = sl.CLASSES["d20000"][0]
    assert np.array_equal(got["d20000"], sl.restated_draws(20000, k, ids, range(sl.STEPS)))


def class_draws(source, name, k, seed=sl.SEED, hop=0):
    """[STEPS, n, k] slots drawn for the destinations of class `name` at fanout k: at hop 0, or (hop=1) at hop 1 of a
    destination-inclusive sample with fanout [k, k], where every hop-0 destination is a hop-1 destination too."""
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    ids = sl.CLASSES[name][0]
    n = ids.size
    ids_t = torch.from_numpy(ids.astype(np.int32)).to(d)
    s = NeighborSampler(source, [k] * (hop + 1), n, include_dst=hop > 0)
    out = torch.empty((sl.STEPS, n, k), dtype=torch.float32, device=d)
    bad = torch.zeros((), dtype=torch.int64, device=d)
    ar = torch.arange(k, device=d)
    for step in range(sl.STEPS):
        sg = s.sample(ids_t, seed, step)
        if hop == 0:
            bad += (sg.blocks[0].column_offset.long() != k * torch.arange(n + 1, device=d)).sum()
            out[step] = sg.blocks[0].weight.view(n, k)
        else:
            b1 = sg.blocks[1]
            pos = sg.blocks[0].dst_pos.long()
            c1 = b1.column_offset.long()
            bad += (b1.dst[pos] != ids_t).sum() + (c1[pos + 1] - c1[pos] != k).sum()
            out[step] = b1.weight[(c1[pos][:, None] + ar).clamp(0, b1.n_edges - 1)]
    assert int(bad) == 0
    return out.cpu().numpy().astype(np.int64)


@pytest.mark.parametrize("name,k", [("d100", 1), ("d6", 3)])
def test_draws_are_independent_across_destinations_hops_steps_and_seeds(world_one, name, k):
    deg = sl.class_degree(name)
    x, other_seed, other_hop = (class_draws(world_one, name, k, **kw) for kw in ({}, {"seed": sl.SEED + 1},
                                                                                  {"hop": 1}))
    for y in (x, other_seed, other_hop):
        sl.check_subsets(y.reshape(-1, k), deg)
    p = sl.independence_p_values(x, other_seed, other_hop, deg)
    print("sample independence k=%d %s(deg %d): %s" % (k, name, deg,
                                                       " ".join("%s=%.3g" % kv for kv in sorted(p.items()))))
    assert not sl.failures(p), p


def test_operator_mean_over_steps_matches_its_float64_expectation(graph, world_one):
    """MiniBatchFuseOp(sg, 0, table=True) on a one-hop sample of a fixed batch (the first EXPECT_PER_CLASS destinations
    of every class of run 25), averaged over STEPS steps in float64.  For deg > k the kept sum of v is a k-draw without
    replacement from the population a_j = w_j X[src_j] (j < deg): mean k * mean(a) = (k/deg) (A X)[v], variance
    k (deg-k)/(deg-1) * var(a).  The step mean is held to that mean within a z-bound (Bonferroni over every element,
    P_PASS).  For deg <= k every step is A X exactly: integer features and slot weights make every sum exact in FP32."""
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.sample import NeighborSampler
    d = dev()
    k = EXPECT_FANOUT
    batch = np.concatenate([ids[:EXPECT_PER_CLASS] for _, ids, _ in sl.plan(k)])
    gen = torch.Generator().manual_seed(sl.SEED)
    x = torch.randint(-8, 9, (sl.V, EXPECT_F), generator=gen).float()
    xh = x.double().numpy()
    deg = graph.col[batch + 1].astype(np.int64) - graph.col[batch]
    ax = np.zeros((batch.size, EXPECT_F))
    var_a = np.zeros_like(ax)
    for i, v in enumerate(batch):
        lo, hi = int(graph.col[v]), int(graph.col[v + 1])
        a = graph.w[lo:hi, None].astype(np.float64) * xh[graph.row[lo:hi].astype(np.int64)]
        if a.size:
            ax[i], var_a[i] = a.sum(0), a.var(0)
    whole = deg <= k
    batch_t = torch.from_numpy(batch.astype(np.int32)).to(d)
    x = x.to(d)
    ax_whole = torch.from_numpy(ax[whole]).to(d)
    whole_t = torch.from_numpy(whole).to(d)
    s = NeighborSampler(world_one, [k], batch.size)
    acc = torch.zeros((batch.size, EXPECT_F), dtype=torch.float64, device=d)
    bad = torch.zeros((), dtype=torch.int64, device=d)
    for step in range(sl.STEPS):
        y = ops.MiniBatchFuseOp(s.sample(batch_t, sl.SEED, step), 0, table=True).forward(x).double()
        bad += (y[whole_t] != ax_whole).sum()
        acc += y
    assert int(bad) == 0, "a destination with deg <= k is not A X exactly at some step"
    mean = acc.cpu().numpy() / sl.STEPS
    assert np.array_equal(mean[whole], ax[whole])
    part = ~whole
    assert part.sum() >= 6 * EXPECT_PER_CLASS and np.all(var_a[part] > 0)
    dd = deg[part, None]
    sd = np.sqrt(k * (dd - k) / (dd - 1) * var_a[part] / sl.STEPS)
    z = np.abs(mean[part] - k / dd * ax[part]) / sd
    z_max = stats.norm.isf(sl.P_PASS / (2 * z.size))
    print("sample expectation k=%d: max |z| %.3f over %d elements (bound %.3f)" % (k, z.max(), z.size, z_max))
    assert z.max() <= z_max, (z.max(), z_max)
