"""TEST INFRASTRUCTURE ONLY - CPU restatement of the reference's hot path (numpy).

This module is the *checker*.  Nothing under ``neutronstarlite_b200/`` imports it; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu-baseline legs may.

Every function restates one piece of iDC-NEU/NeutronStarLite (paths relative to the reference
root) and cites the file:line it follows.  Parity is PINNED: ``tests/test_oracle_golden.py``
checks every function here against golden vectors produced by the *unmodified* reference CPU
operators (``oracle/_ref/nts_ref_driver``, built by ``oracle/Makefile`` from the reference sources,
run at P = 1, 2, 4, 8 ranks under the MPI stand-in of ``oracle/shim``) and committed under
``tests/golden/`` by ``oracle/make_golden.py``.

Integer artefacts are bit-exact restatements.  Float results follow the reference's summation
order (CSC order per destination, CSR order per source) in float32.
"""
from __future__ import annotations

import numpy as np

PAGESIZE = 1 << 10  # dep/gemini/constants.hpp: PAGESIZE = 1024 vertices


# --------------------------------------------------------------------------------------------
# graph artefacts
# --------------------------------------------------------------------------------------------
def read_edge_file(path):
    """Binary edge list: packed {uint32 src, uint32 dst} (dep/gemini/type.hpp:100-106)."""
    return np.fromfile(path, dtype=np.uint32).reshape(-1, 2)


def degrees(edges, V):
    """out/in degree with multiplicity over the whole edge file, clamped to >= 1.

    core/graph.hpp:1160-1181 (out_degree, all-reduced), :1373,:1414-1417 (in_degree, all-reduced),
    :4396-4401 (clamp of *_degree_for_backward)."""
    out_deg = np.bincount(edges[:, 0], minlength=V).astype(np.uint32)
    in_deg = np.bincount(edges[:, 1], minlength=V).astype(np.uint32)
    return np.maximum(out_deg, 1).astype(np.uint32), np.maximum(in_deg, 1).astype(np.uint32)


def partition_offsets(edges, V, P):
    """Vertex-chunk partitioner, core/graph.hpp:1185-1211.

    Greedy prefix over (raw out_degree + alpha), alpha = 12*(P+1) (core/graph.hpp:408); a cut is
    placed at the first vertex where the running sum exceeds remaining/(P-i), then rounded DOWN to
    a multiple of PAGESIZE; the last boundary is V."""
    E = int(edges.shape[0])
    alpha = 12 * (P + 1)
    out_deg = np.bincount(edges[:, 0], minlength=V).astype(np.int64)  # un-clamped at this point
    cost = out_deg + alpha
    off = np.zeros(P + 1, dtype=np.uint32)
    remained = E + V * alpha
    prefix = np.concatenate([[0], np.cumsum(cost)])
    for i in range(P):
        parts_left = P - i
        expected = remained // parts_left
        start = int(off[i])
        if parts_left == 1:
            off[i + 1] = V
        else:
            # first v_i >= start with prefix[v_i+1]-prefix[start] > expected
            target = prefix[start] + expected
            v_i = int(np.searchsorted(prefix[1:], target, side="right"))
            # (the reference leaves the boundary unset if the sum never exceeds; with alpha>0 and
            #  expected = remained/parts_left < remained that cannot happen for parts_left > 1)
            v_i = max(v_i, start)
            off[i + 1] = (v_i // PAGESIZE) * PAGESIZE
        remained -= int(prefix[int(off[i + 1])] - prefix[start])
    assert off[P] == V
    return off


def weights_norm_degree(src, dst, out_deg, in_deg):
    """nts_norm_degree, core/ntsBaseOp.hpp:194-197:
    1 / ((float)sqrt((double)out[s]) * (float)sqrt((double)in[d])) evaluated in float32."""
    a = np.sqrt(out_deg[src].astype(np.float64)).astype(np.float32)
    b = np.sqrt(in_deg[dst].astype(np.float64)).astype(np.float32)
    return (np.float32(1.0) / (a * b)).astype(np.float32)


class Chunk:
    """One CSC_segment_pinned (core/GraphSegment.h:52-139): edges src in partition i -> dst local."""

    __slots__ = ("src_range", "dst_range", "edge_size", "column_offset", "row_indices",
                 "edge_weight_forward", "row_offset", "column_indices", "edge_weight_backward",
                 "source_active")


def build_chunks(edges, V, partition_offset, rank, out_deg=None, in_deg=None):
    """PartitionedGraph::PartitionToChunks, core/PartitionedGraph.hpp:324-420.

    Local edges = all edges whose dst is owned by `rank` (core/graph.hpp:1328-1416 shuffles edges
    to the destination owner).  Chunk i keeps those with src in partition i.
    CSC: by local dst, inside a destination ascending global src (the COO walk of
    generatePartitionedSubgraph :306-323 is src-ascending and placement is stable), duplicates kept.
    CSR: by src local to partition i; the order of destinations inside a source row is NOT
    deterministic in the reference (parallel fetch-and-add in load_directed) - we canonicalise to
    ascending dst and compare rows as multisets."""
    if out_deg is None:
        out_deg, in_deg = degrees(edges, V)
    P = len(partition_offset) - 1
    v0, v1 = int(partition_offset[rank]), int(partition_offset[rank + 1])
    src_all = edges[:, 0].astype(np.int64)
    dst_all = edges[:, 1].astype(np.int64)
    local = (dst_all >= v0) & (dst_all < v1)
    src_l, dst_l = src_all[local], dst_all[local]
    chunks = []
    for i in range(P):
        s0, s1 = int(partition_offset[i]), int(partition_offset[i + 1])
        sel = (src_l >= s0) & (src_l < s1)
        s, d = src_l[sel], dst_l[sel]
        c = Chunk()
        c.src_range = (s0, s1)
        c.dst_range = (v0, v1)
        c.edge_size = int(s.shape[0])
        # CSC
        order = np.lexsort((s, d))  # primary dst, secondary src
        cs, cd = s[order], d[order]
        c.column_offset = np.zeros(v1 - v0 + 1, dtype=np.uint32)
        np.cumsum(np.bincount(cd - v0, minlength=v1 - v0), out=c.column_offset[1:])
        c.row_indices = cs.astype(np.uint32)
        c.edge_weight_forward = weights_norm_degree(cs, cd, out_deg, in_deg)
        # CSR
        order = np.lexsort((d, s))  # primary src, secondary dst
        rs, rd = s[order], d[order]
        c.row_offset = np.zeros(s1 - s0 + 1, dtype=np.uint32)
        np.cumsum(np.bincount(rs - s0, minlength=s1 - s0), out=c.row_offset[1:])
        c.column_indices = rd.astype(np.uint32)
        c.edge_weight_backward = weights_norm_degree(rs, rd, out_deg, in_deg)
        # source_active bitmap (PartitionedGraph.hpp:397): sources of partition i with an edge into rank
        act = np.zeros(s1 - s0, dtype=np.uint8)
        act[np.unique(s - s0)] = 1
        c.source_active = act
        chunks.append(c)
    return chunks


def has_mirror_at(edges, V, partition_offset, rank):
    """hasMirrorAtPartition[i] on `rank` (PartitionedGraph::DetermineMirror, :174-209):
    bit v set iff local vertex v (owned by rank) is a source of some edge into partition i,
    i.e. partition i's chunk[rank].source_active."""
    P = len(partition_offset) - 1
    v0, v1 = int(partition_offset[rank]), int(partition_offset[rank + 1])
    src = edges[:, 0].astype(np.int64)
    dst = edges[:, 1].astype(np.int64)
    mine = (src >= v0) & (src < v1)
    out = []
    for i in range(P):
        d0, d1 = int(partition_offset[i]), int(partition_offset[i + 1])
        sel = mine & (dst >= d0) & (dst < d1)
        bits = np.zeros(v1 - v0, dtype=np.uint8)
        bits[np.unique(src[sel] - v0)] = 1
        out.append(bits)
    return out


def mirror_index(edges, V, partition_offset, rank):
    """PartitionedGraph::generateMirrorIndex, core/PartitionedGraph.hpp:295-305:
    exclusive prefix sum over 'global vertex s is the source of at least one local in-edge'.
    Returns (MirrorIndex[V+1] uint32, owned_mirrors)."""
    v0, v1 = int(partition_offset[rank]), int(partition_offset[rank + 1])
    dst = edges[:, 1].astype(np.int64)
    local = (dst >= v0) & (dst < v1)
    flag = np.zeros(V + 1, dtype=np.uint32)
    flag[edges[local, 0].astype(np.int64) + 1] = 1
    mi = np.cumsum(flag, dtype=np.uint32)
    return mi, int(mi[V])


def whole_graph_topo(edges, V, partition_offset, rank):
    """PartitionedGraph::GenerateWholeGraphTopo, core/PartitionedGraph.hpp:105-143: CSC of ALL local
    in-edges (column_offset[Vp+1], row_indices[Ep] global src ascending inside a destination) and the
    mirror-compressed CSR (compressed_row_offset[M+1], column_indices[Ep] global dst)."""
    v0, v1 = int(partition_offset[rank]), int(partition_offset[rank + 1])
    src = edges[:, 0].astype(np.int64)
    dst = edges[:, 1].astype(np.int64)
    local = (dst >= v0) & (dst < v1)
    s, d = src[local], dst[local]
    order = np.lexsort((s, d))
    cs, cd = s[order], d[order]
    col_off = np.zeros(v1 - v0 + 1, dtype=np.uint32)
    np.cumsum(np.bincount(cd - v0, minlength=v1 - v0), out=col_off[1:])
    mi, M = mirror_index(edges, V, partition_offset, rank)
    order = np.lexsort((d, s))
    rs, rd = s[order], d[order]
    crow = np.zeros(M + 1, dtype=np.uint32)
    if rs.size:
        np.cumsum(np.bincount(mi[rs].astype(np.int64), minlength=M), out=crow[1:])
    return col_off, cs.astype(np.uint32), crow, rd.astype(np.uint32)


# --------------------------------------------------------------------------------------------
# float operators (float32, reference summation order)
# --------------------------------------------------------------------------------------------
def _segment_weighted_sum(offsets, indices, weights, X, base):
    """out[r,:] = sum_{e in [offsets[r], offsets[r+1])} X[indices[e]-base,:] * w[e], sequential per
    row in float32 (nts_comp, core/ntsBaseOp.hpp:82-104: mul then add)."""
    R = offsets.shape[0] - 1
    F = X.shape[1]
    out = np.zeros((R, F), dtype=np.float32)
    deg = np.diff(offsets.astype(np.int64))
    maxdeg = int(deg.max()) if R else 0
    idx = indices.astype(np.int64) - base
    off = offsets.astype(np.int64)
    # vectorised over rows, sequential over the k-th edge of every row -> same order as the loop
    for k in range(maxdeg):
        rows = np.nonzero(deg > k)[0]
        e = off[rows] + k
        if weights is None:
            out[rows] = out[rows] + X[idx[e]]
        else:
            out[rows] = out[rows] + X[idx[e]] * weights[e][:, None]
    return out


def gather_by_dst_from_src(chunk, X_src, Y=None, with_weight=True):
    """Forward aggregation of one chunk: Y[d,:] += sum_{e->d} X_src[row_indices[e]-src_start,:]*w_fwd[e].
    core/ntsCPUFusedGraphOp.hpp:81-106 (the sparse_slot); GPU twin cuda/ntsCUDAFuseKernel.cuh:272-309."""
    part = _segment_weighted_sum(chunk.column_offset, chunk.row_indices,
                                 chunk.edge_weight_forward if with_weight else None,
                                 X_src, chunk.src_range[0])
    return part if Y is None else (Y + part).astype(np.float32)


def gather_by_src_from_dst(chunk, G_dst, with_weight=True):
    """Backward aggregation of one chunk: P[s,:] = sum_{s->d} G_dst[column_indices[e]-dst_start,:]*w_bwd[e].
    core/ntsCPUFusedGraphOp.hpp:123-143; GPU twin cuda/ntsCUDAFuseKernel.cuh:450-487."""
    return _segment_weighted_sum(chunk.row_offset, chunk.column_indices,
                                 chunk.edge_weight_backward if with_weight else None,
                                 G_dst, chunk.dst_range[0])


def gcn_forward_all(edges, V, P, X):
    """Y = A_hat X over the whole graph, assembled the way the P ranks do it: rank p accumulates
    chunk after chunk in ring order (core/graph.hpp:3678-3719).  Returns [V,F]."""
    po = partition_offsets(edges, V, P)
    out_deg, in_deg = degrees(edges, V)
    Y = np.zeros_like(X, dtype=np.float32)
    for p in range(P):
        chunks = build_chunks(edges, V, po, p, out_deg, in_deg)
        v0, v1 = int(po[p]), int(po[p + 1])
        acc = np.zeros((v1 - v0, X.shape[1]), dtype=np.float32)
        for step in range(P):
            i = (p + step) % P
            acc = gather_by_dst_from_src(chunks[i], X[int(po[i]):int(po[i + 1])], acc)
        Y[v0:v1] = acc
    return Y


def gcn_backward_all(edges, V, P, G):
    """dX = A_hat^T G: rank p computes a partial for every source partition j from its chunk j
    (core/graph.hpp:3455-3622), partials are summed at the owner (nts_acc, ntsBaseOp.hpp:114-126)."""
    po = partition_offsets(edges, V, P)
    out_deg, in_deg = degrees(edges, V)
    dX = np.zeros_like(G, dtype=np.float32)
    for p in range(P):
        chunks = build_chunks(edges, V, po, p, out_deg, in_deg)
        v0, v1 = int(po[p]), int(po[p + 1])
        for j in range(P):
            part = gather_by_src_from_dst(chunks[j], G[v0:v1])
            dX[int(po[j]):int(po[j + 1])] += part
    return dX


# ---- edge-granular operators (GAT building blocks) --------------------------------------------
def scatter_src_mirror_to_msg(col_off, row_idx, mirror_idx, mirror):
    """DistScatterSrc::forward, core/ntsDistCPUGraphOp.hpp:139-163: msg[e,:] = mirror[MirrorIndex[src(e)],:]."""
    return mirror[mirror_idx[row_idx.astype(np.int64)].astype(np.int64)].astype(np.float32)


def gather_msg_to_src_mirror(col_off, row_idx, mirror_idx, msg_grad, M):
    """DistScatterSrc::backward, :165-189: mirror_grad[MirrorIndex[src(e)],:] += msg_grad[e,:] (edge order)."""
    out = np.zeros((M, msg_grad.shape[1]), dtype=np.float32)
    slot = mirror_idx[row_idx.astype(np.int64)].astype(np.int64)
    np.add.at(out, slot, msg_grad)
    return out


def _edge_dst(col_off):
    deg = np.diff(col_off.astype(np.int64))
    return np.repeat(np.arange(deg.shape[0], dtype=np.int64), deg)


def scatter_dst_to_msg(col_off, x):
    """DistScatterDst::forward, :200-222: msg[e,:] = x[dst(e),:]."""
    return x[_edge_dst(col_off)].astype(np.float32)


def gather_msg_to_dst(col_off, msg):
    """DistAggregateDst::forward, :258-284 (== DistScatterDst::backward :224-249):
    y[d,:] = sum_{e->d} msg[e,:], sequential in edge order."""
    Vp = col_off.shape[0] - 1
    out = np.zeros((Vp, msg.shape[1]), dtype=np.float32)
    deg = np.diff(col_off.astype(np.int64))
    off = col_off.astype(np.int64)
    for k in range(int(deg.max()) if Vp else 0):
        rows = np.nonzero(deg > k)[0]
        out[rows] = out[rows] + msg[off[rows] + k]
    return out


def edge_softmax_forward(col_off, m):
    """DistEdgeSoftMax::forward, :449-470: per destination segment, column-wise softmax(0) of m[seg,:]
    (libtorch Tensor::softmax = max-subtracted exp / sum; the reference GPU kernel
    cuda/ntsCUDADistKernel.cuh:166-213 omits the max subtraction and is NOT the oracle)."""
    out = np.zeros_like(m, dtype=np.float32)
    off = col_off.astype(np.int64)
    for d in range(off.shape[0] - 1):
        a, b = off[d], off[d + 1]
        if b > a:
            seg = m[a:b].astype(np.float32)
            mx = seg.max(axis=0, keepdims=True)
            ex = np.exp(seg - mx, dtype=np.float32)
            out[a:b] = ex / ex.sum(axis=0, keepdims=True, dtype=np.float32)
    return out


def edge_softmax_backward(col_off, a_cached, g):
    """DistEdgeSoftMax::backward, :472-492: g_in = a*g - a*(sum_seg g*a), per destination segment and
    per column (the reference expression `imr*(d.t().mm(imr))` is only well-formed for one column;
    the column-wise form is its natural multi-head extension)."""
    out = np.zeros_like(g, dtype=np.float32)
    off = col_off.astype(np.int64)
    for d in range(off.shape[0] - 1):
        a0, b0 = off[d], off[d + 1]
        if b0 > a0:
            a = a_cached[a0:b0]
            gg = g[a0:b0]
            dot = (a * gg).sum(axis=0, keepdims=True, dtype=np.float32)
            out[a0:b0] = a * gg - a * dot
    return out


def aggregate_dst_fuse_weight_forward(col_off, row_idx, mirror_idx, mirror, e_weight):
    """DistAggregateDstFuseWeight::forward, :516-546: y[d,:] = sum_{e->d} mirror[MirrorIndex[src(e)],:]*a[e]."""
    Vp = col_off.shape[0] - 1
    out = np.zeros((Vp, mirror.shape[1]), dtype=np.float32)
    deg = np.diff(col_off.astype(np.int64))
    off = col_off.astype(np.int64)
    slot = mirror_idx[row_idx.astype(np.int64)].astype(np.int64)
    w = e_weight.reshape(-1).astype(np.float32)
    for k in range(int(deg.max()) if Vp else 0):
        rows = np.nonzero(deg > k)[0]
        e = off[rows] + k
        out[rows] = out[rows] + mirror[slot[e]] * w[e][:, None]
    return out


def aggregate_dst_fuse_weight_backward(col_off, row_idx, mirror_idx, mirror, e_weight, g, M,
                                       reference_double_count=False):
    """DistAggregateDstFuseWeight::backward, :548-589.
    d_mirror[slot(e),:] += g[dst(e),:]*a[e];  d_a[e] = <mirror[slot(e),:], g[dst(e),:]>.
    The reference ALSO adds the unweighted g[dst(e),:] once (`nts_acc` at :572 before `nts_comp`),
    which is a bug (the mathematical gradient has no such term); `reference_double_count=True`
    reproduces it so the golden vectors of the unmodified reference can be matched."""
    dst = _edge_dst(col_off)
    slot = mirror_idx[row_idx.astype(np.int64)].astype(np.int64)
    w = e_weight.reshape(-1).astype(np.float32)
    dm = np.zeros((M, g.shape[1]), dtype=np.float32)
    contrib = g[dst] * w[:, None]
    if reference_double_count:
        contrib = contrib + g[dst]
    np.add.at(dm, slot, contrib.astype(np.float32))
    dw = (mirror[slot] * g[dst]).sum(axis=1, dtype=np.float32).reshape(-1, 1)
    return dm, dw


def get_dep_neighbor(edges, V, partition_offset, rank, X_global):
    """DistGetDepNbrOp::forward, :48-86: mirror[MirrorIndex[s],:] = X[s,:] for every global source s
    of a local in-edge."""
    mi, M = mirror_index(edges, V, partition_offset, rank)
    srcs = np.nonzero(mi[1:] != mi[:-1])[0]
    out = np.zeros((M, X_global.shape[1]), dtype=np.float32)
    out[mi[srcs].astype(np.int64)] = X_global[srcs]
    return out


def message_bytes_fp32(F):
    """Size of one (vid, row) record: comm/network.h:143-149 sizeofM = sizeof(VertexId) + F*sizeof(float)."""
    return 4 + 4 * F
