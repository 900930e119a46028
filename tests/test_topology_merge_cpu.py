"""The invariant a sharded topology rests on (topology.ShardedTopology, nts_merge_chunk_csc): merging each rank's P chunk
CSCs per destination, chunk 0 first, and concatenating the ranks gives the single-partition CSC of the same graph, bit
for bit - column offsets, source ids and edge weights.  Checked on the reference's own golden chunks of every case
with P > 1 whose P = 1 case is stored (cora_self at P = 2 and 4, where P = 4 has empty partitions; synth9k at P = 2
and 3).  merge_chunks is the numpy restatement the GPU merge is tested against (test_sharded_topology_gpu.py)."""
import numpy as np
import pytest

import golden_store

CASES = [("cora_self_P2_F4", "cora_self_P1_F8"), ("cora_self_P4_F2", "cora_self_P1_F8"),
         ("synth9k_P2_F2", "synth9k_P1_F2"), ("synth9k_P3_F2", "synth9k_P1_F2")]


def merge_chunks(cols, rows, weights):
    """One CSC from chunk CSCs over the same destinations: destination d's slots are chunk 0's, then chunk 1's, ...,
    each in its chunk's order.  Returns (column_offset uint32 [n_dst+1], row_indices uint32, weight float32)."""
    cols = [np.asarray(c, dtype=np.int64) for c in cols]
    n_dst = cols[0].size - 1
    deg = sum(np.diff(c) for c in cols)
    col = np.zeros(n_dst + 1, dtype=np.int64)
    np.cumsum(deg, out=col[1:])
    row = np.zeros(int(col[-1]), dtype=np.uint32)
    w = np.zeros(int(col[-1]), dtype=np.float32)
    cursor = col[:-1].copy()
    for c, r, x in zip(cols, rows, weights):
        d = np.diff(c)
        if not d.sum():
            continue
        dst_of_edge = np.repeat(np.arange(n_dst), d)
        within = np.arange(int(c[-1]) - int(c[0])) - np.repeat(c[:-1] - c[0], d)
        pos = cursor[dst_of_edge] + within
        row[pos] = np.asarray(r)[int(c[0]):int(c[-1])]
        w[pos] = np.asarray(x)[int(c[0]):int(c[-1])]
        cursor += d
    return col.astype(np.uint32), row, w


def rank_chunks(z, r, P):
    key = "r%d/chunk%d_%s"
    return ([z[key % (r, i, "column_offset")] for i in range(P)], [z[key % (r, i, "row_indices")] for i in range(P)],
            [z[key % (r, i, "edge_weight_forward")] for i in range(P)])


def partitions(name):
    return int(name.split("_P")[1].split("_")[0])


@pytest.mark.parametrize("case,whole", CASES)
def test_rank_merges_concatenate_to_the_single_partition_csc(case, whole):
    z, z1 = golden_store.load(case), golden_store.load(whole)
    P = partitions(case)
    po = z["r0/partition_offset"].astype(np.int64)
    assert np.array_equal(z["edges"], z1["edges"])
    cols, rows, ws = [], [], []
    empty = 0
    for r in range(P):
        col, row, w = merge_chunks(*rank_chunks(z, r, P))
        assert col.size == po[r + 1] - po[r] + 1
        empty += col.size == 1
        cols.append(np.diff(col.astype(np.int64)))
        rows.append(row)
        ws.append(w)
    if case == "cora_self_P4_F2":
        assert empty == 2
    col1 = z1["r0/chunk0_column_offset"].astype(np.int64)
    assert np.array_equal(np.concatenate(cols), np.diff(col1))
    assert np.array_equal(np.concatenate(rows), z1["r0/chunk0_row_indices"])
    w1 = z1["r0/chunk0_edge_weight_forward"]
    assert np.array_equal(np.concatenate(ws).view(np.uint32), w1.view(np.uint32))
