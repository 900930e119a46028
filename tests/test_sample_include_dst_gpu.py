"""The sampler's destination-inclusive mode (NTS_SAMPLER_INCLUDE_DST) on the GPU: blocks and dst_pos bit-exact against
the numpy restatement (tests/test_sample_include_dst.py), the default mode of nts_sampler_create_ex identical to
nts_sampler_create, empty and edge-less seeds, and the argument errors of the new entries."""
import ctypes as C

import numpy as np
import pytest

from test_sample_gpu import KEYS, cora_edges, dev, graph, zipf_hub_edges
from test_sample_include_dst import sample_include_dst

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def check_against_oracle(pg, seeds, fanout, seed, step):
    from neutronstarlite_b200.sample import NeighborSampler
    c = pg.graph_chunks[0]
    s = NeighborSampler(pg, fanout, max(len(seeds), 1), include_dst=True)
    sg = s.sample(seeds, seed, step)
    ref = sample_include_dst(c.column_offset, c.row_indices, c.edge_weight_forward, seeds, fanout, seed, step)
    assert sg.hops == len(fanout)
    for h, (b, r) in enumerate(zip(sg.blocks, ref)):
        got = b.to_numpy()
        for k in KEYS + ("dst_pos",):
            assert got[k].dtype == r[k].dtype, (h, k)
            assert np.array_equal(got[k].view(np.uint32), r[k].view(np.uint32)), "hop %d %s differs" % (h, k)
    return sg, ref


@pytest.mark.parametrize("self_loops", [True, False])
@pytest.mark.parametrize("fanout,seed,step", [([1, 1], 0, 0), ([64, 64], 1, 3), ([5, 10], 2, 7),
                                              ([25, 10, 3], 3, 1)])
def test_include_dst_matches_numpy_on_cora(self_loops, fanout, seed, step):
    edges = cora_edges(self_loops)
    if not self_loops:
        edges = edges[edges[:, 1] >= 10]         # vertices 0..9 keep no in-edge
    pg = graph(edges, 2708)
    rng = np.random.default_rng(seed)
    seeds = np.concatenate([np.arange(12), rng.choice(np.arange(12, 2708), 300, replace=False)])
    check_against_oracle(pg, seeds, fanout, seed, step)


@pytest.mark.parametrize("fanout,seed,step", [([1, 1], 0, 0), ([64, 64], 5, 2), ([10, 5, 3], 7, 4)])
def test_include_dst_matches_numpy_on_a_zipf_graph_with_hubs(fanout, seed, step):
    edges, V = zipf_hub_edges()
    pg = graph(edges, V)
    rng = np.random.default_rng(seed)
    seeds = np.concatenate([[5, 77, 0, 1], rng.choice(np.arange(100, V), 1020, replace=False)])
    check_against_oracle(pg, seeds, fanout, seed, step)


def test_create_ex_without_flags_is_create():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.sample import NeighborSampler
    pg = graph(cora_edges(), 2708)
    seeds = np.arange(0, 2708, 9)
    new = NeighborSampler(pg, [10, 5], 512)                 # nts_sampler_create_ex(..., flags=0)
    a = [b.to_numpy() for b in new.sample(seeds, 4, 2).clone().blocks]
    old = NeighborSampler(pg, [10, 5], 512)
    L = _lib.load()
    c = pg.graph_chunks[0]
    L.nts_sampler_destroy(old.handle)
    old.handle = L.nts_sampler_create(c.column_offset_gpu.data_ptr(), c.row_indices_gpu.data_ptr(),
                                      c.edge_weight_forward_gpu.data_ptr(), 2708, int(c.edge_size), 512, 2,
                                      (C.c_int * 2)(10, 5), torch.cuda.current_stream().cuda_stream)
    assert old.handle
    b = [blk.to_numpy() for blk in old.sample(seeds, 4, 2).blocks]
    assert new.bytes() == old.bytes()
    for x, y in zip(a, b):
        assert sorted(x) == sorted(y) and "dst_pos" not in x
        for k in x:
            assert np.array_equal(x[k].view(np.uint32), y[k].view(np.uint32)), k


def test_empty_seed_list_gives_empty_blocks():
    pg = graph(cora_edges(), 2708)
    sg, ref = check_against_oracle(pg, np.zeros(0, dtype=np.int64), [5, 10], 0, 0)
    assert all(b.n_dst == 0 and b.n_src == 0 and b.n_edges == 0 for b in sg.blocks)


def test_a_seed_without_in_edges_gets_a_dst_pos_and_a_zero_output_row():
    from neutronstarlite_b200 import ops
    d = dev()
    edges = cora_edges(False)
    edges = edges[edges[:, 1] != 7]                     # vertex 7 has no in-edge
    pg = graph(edges, 2708)
    sg, ref = check_against_oracle(pg, np.array([7, 100, 200]), [5, 5], 1, 1)
    top = sg.blocks[0]
    pos = top.dst_pos.long()
    assert int(top.src[pos[0]]) == 7 and int(top.column_offset[1]) == 0
    H, D = 2, 8
    gen = torch.Generator().manual_seed(0)
    x = (torch.rand((top.n_src, H * D), generator=gen) * 2 - 1).to(d)
    s = torch.rand((top.n_src, H), generator=gen).to(d)
    op = ops.MiniBatchGATOp(sg, 0)
    out = op.forward(x, s, s[pos].contiguous())
    assert torch.equal(out[0], torch.zeros(H * D, device=d))
    assert out[1:].abs().sum() > 0
    dx, ds, dd = op.backward(torch.ones_like(out))
    assert torch.equal(dd[0], torch.zeros(H, device=d))
    # a block without any edge: zero rows and zero gradients, no kernel needed
    sg0, _ = check_against_oracle(pg, np.array([7]), [5], 0, 0)
    assert sg0.blocks[0].n_edges == 0 and sg0.blocks[0].n_src == 1
    op0 = ops.MiniBatchGATOp(sg0, 0)
    o0 = op0.forward(torch.ones((1, 16), device=d), torch.ones((1, 2), device=d), torch.ones((1, 2), device=d))
    assert torch.equal(o0, torch.zeros((1, 16), device=d))
    assert all(torch.equal(t, torch.zeros_like(t)) for t in op0.backward(torch.ones_like(o0)))


def test_bad_flags_and_dst_pos_without_the_mode_are_refused():
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.sample import NeighborSampler
    pg = graph(cora_edges(), 2708)
    c = pg.graph_chunks[0]
    L = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    ks = (C.c_int * 2)(5, 10)
    for flags in (2, 0x80000000, 3):
        h = L.nts_sampler_create_ex(c.column_offset_gpu.data_ptr(), c.row_indices_gpu.data_ptr(),
                                    c.edge_weight_forward_gpu.data_ptr(), 2708, int(c.edge_size), 64, 2, ks, flags, st)
        assert not h
        assert b"flag" in L.nts_last_error()
    s = NeighborSampler(pg, [5, 10], 64)
    s.sample(np.arange(10), 0, 0)
    p = C.c_void_p()
    assert L.nts_sampler_hop_dst_pos(s.handle, 0, C.byref(p)) != 0
    assert b"NTS_SAMPLER_INCLUDE_DST" in L.nts_last_error()
    inc = NeighborSampler(pg, [5, 10], 64, include_dst=True)
    assert inc.bytes() > s.bytes()
    assert L.nts_sampler_hop_dst_pos(inc.handle, 0, C.byref(p)) != 0        # nothing sampled yet
    inc.sample(np.arange(10), 0, 0)
    assert L.nts_sampler_hop_dst_pos(inc.handle, 1, C.byref(p)) == 0 and p.value
    assert L.nts_sampler_hop_dst_pos(inc.handle, 2, C.byref(p)) != 0        # hop out of range
