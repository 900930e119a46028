"""The reference's own sampled blocks (tests/golden/cora_sample_B64_F8, dumped by oracle/make_sample_golden.py from
the unmodified GCNSAMPLESINGLE sampler: Cora with self loops, FANOUT 5-10, BATCH_SIZE 64, first train batch, sources in
the reference's first-appearance order): on the CPU, every block is made of Cora edges with min(indeg, k) slots per
destination and weights bit-equal to the topology golden's nts_norm_degree; on the GPU, ops.MiniBatchFuseOp on these
blocks reproduces the reference MiniBatchFuseOp forward and backward."""
import os

import numpy as np
import pytest

import golden_store

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cora_sample_B64_F8", "blocks.npz")
FANOUT = (5, 10)


def blocks():
    z = np.load(GOLDEN)
    hops, batch, F, n_train = (int(x) for x in z["meta"])
    return [{k: z["h%d/%s" % (h, k)] for k in ("dst", "c_o", "r_i", "src", "w", "X", "Y", "G", "dX")}
            for h in range(hops)], batch, F


def cora_csc():
    g = golden_store.load("cora_self_P1_F8")
    return g["r0/chunk0_column_offset"], g["r0/chunk0_row_indices"], g["r0/chunk0_edge_weight_forward"]


def test_golden_blocks_are_cora_edges_with_the_topology_weights():
    col, row, w = cora_csc()
    bs, batch, F = blocks()
    assert len(bs) == len(FANOUT) and bs[0]["dst"].size == batch
    for h, (b, k) in enumerate(zip(bs, FANOUT)):
        if h:
            assert np.array_equal(b["dst"], bs[h - 1]["src"])       # next hop's destinations = distinct sources
        assert np.unique(b["src"]).size == b["src"].size
        assert np.array_equal(np.unique(b["src"][b["r_i"]]), np.sort(b["src"]))
        deg = col[b["dst"].astype(np.int64) + 1].astype(np.int64) - col[b["dst"]]
        assert np.array_equal(np.diff(b["c_o"].astype(np.int64)), np.minimum(deg, k))
        for d in range(b["dst"].size):
            v = int(b["dst"][d])
            nbr, nw = row[col[v]:col[v + 1]], w[col[v]:col[v + 1]]
            for e in range(b["c_o"][d], b["c_o"][d + 1]):
                s = b["src"][b["r_i"][e]]
                hit = np.nonzero(nbr == s)[0]
                assert hit.size, "hop %d: (%d -> %d) is not a Cora edge" % (h, s, v)
                assert nw[hit[0]].view(np.uint32) == b["w"][e].view(np.uint32)


def test_golden_inputs_are_the_driver_inputs():
    bs, _, F = blocks()
    for b in bs:
        # gen_x / gen_g of the driver by global vertex id (float32 arithmetic, libm sinf / cosf)
        f = np.arange(F)
        ax = np.float32(0.37) * ((b["src"].astype(np.int64)[:, None] * F + f) % 100003).astype(np.float32)
        np.testing.assert_allclose(b["X"], np.sin(ax), rtol=0, atol=1e-6)
        ag = np.float32(0.11) * ((b["dst"].astype(np.int64)[:, None] * F + f) % 100019).astype(np.float32)
        np.testing.assert_allclose(b["G"], np.cos(ag), rtol=0, atol=1e-6)


@pytest.mark.gpu
def test_minibatch_op_on_the_reference_blocks_matches_the_reference():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from neutronstarlite_b200 import ops
    from neutronstarlite_b200.sample import SampledSubgraph
    d = torch.device("cuda:0")
    bs, _, _ = blocks()

    def t(a):
        return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).to(d)

    sg = SampledSubgraph.from_blocks([{"dst": t(b["dst"]), "column_offset": t(b["c_o"]), "row_indices": t(b["r_i"]),
                                       "weight": t(b["w"]), "src": t(b["src"])} for b in bs])
    for h, b in enumerate(bs):
        op = ops.MiniBatchFuseOp(sg, h)
        y = op.forward(t(b["X"]))
        dx = op.backward(t(b["G"]))
        np.testing.assert_allclose(y.cpu().numpy(), b["Y"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(dx.cpu().numpy(), b["dX"], rtol=1e-4, atol=1e-5)
