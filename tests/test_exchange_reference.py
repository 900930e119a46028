"""The peer-memory exchange engine (csrc/nts_exchange.cu) against float64 at every branch it takes: push widths
(VEC 1, 2, 4), kernel and copy-engine pushes, flag-only pushes, pipeline and merged receive (FP32 and BF16), planned
and K1 chunks, one and two window buffers, re-reservation, an empty partition, BF16 input taken as it is, mirror
fetch and return.

Three ranks share one GPU as spawned processes (gloo control plane).  Every rank builds the same purpose-made graph,
partitioned at explicit offsets so that each branch is reached on purpose (see `make_graph`).  In exact mode the edge
weights are q/4 with q in 1..8 and the features are integers in [-8, 8] that change with every call, so every
partial sum is exact in FP32 and every result must equal its float64 reference bit for bit: a stale epoch buffer, a
row in the wrong slot or a dropped edge cannot pass.  One configuration keeps the real GCN weights and uniform
inputs, checked per element against 1e-4 * (|A| |X|).  After every call the engine's path record
(`nts_exchange_last_paths`) must match what the graph and the configuration predict.

The CPU tests show that the comparator rejects a stale epoch, a misplaced mirror row and a dropped edge, that the
graph has the properties the branches need, and that the path prediction agrees with `ExchangePlan` built for all
three ranks in one process."""
import ctypes as C
import multiprocessing as mp
import os
import sys
import threading

import numpy as np
import pytest

torch = pytest.importorskip("torch")
dist = pytest.importorskip("torch.distributed")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---- the graph ------------------------------------------------------------------------------------------------------
V = 2600
PO = {"a": (0, 1003, 1850, V),   # 1003 is not a multiple of 4
      "b": (0, 1003, 1003, V)}   # rank 1 owns no vertex
HUB = 1010                       # in partition 1 of layout a
SRC_1_TO_0 = (1014,)             # the only row partition 1 sends to partition 0
SRC_1_TO_2 = (1006, 1103, 1203, 1303, 1849)   # the five rows partition 1 sends to partition 2
NO_IN = (5, 6, 1002, 1023, 1024, 1859, V - 1)
NO_OUT = (1033, 1034, 1890, 1891, V - 2)


def make_graph(seed=7):
    """Edge list [E, 2] (src, dst) of a multigraph on V vertices.  In layout a:
    every vertex of partition 0 has an edge into partition 1 (rank 1 reads all of rank 0's rows in order: copy-engine
    push); partition 2 -> 1 carries a third of partition 2's rows (kernel push); 1 -> 0 carries one row and 1 -> 2
    five (the push kernel's tails of fewer than 4 rows); 2 -> 0 carries nothing (a flag-only push); HUB has more than
    20 000 in-edges from all three partitions.  Self loops, multi-edges, vertices without in-edges (NO_IN) and
    without out-edges (NO_OUT) are included."""
    rng = np.random.default_rng(seed)
    a, b = PO["a"][1], PO["a"][2]
    part = [np.arange(PO["a"][i], PO["a"][i + 1]) for i in range(3)]

    def dsts(i, n):
        return rng.choice(np.setdiff1d(part[i], NO_IN), n)

    def srcs(i, n):
        return rng.choice(np.setdiff1d(part[i], NO_OUT), n)

    sub2 = np.setdiff1d(part[2][::3], NO_OUT)
    pairs = [
        (part[0], dsts(1, a)),                                    # 0 -> 1: every row of partition 0
        (srcs(0, 1500), dsts(1, 1500)),
        (rng.choice(part[0][::4], 900), dsts(2, 900)),            # 0 -> 2: a quarter of partition 0
        (np.repeat(SRC_1_TO_0, 6), dsts(0, 6)),                   # 1 -> 0: one row
        (np.repeat(SRC_1_TO_2, 3), dsts(2, 15)),                  # 1 -> 2: five rows
        (rng.choice(sub2, 1200), dsts(1, 1200)),                  # 2 -> 1: a subset
        (rng.choice(part[0], 8000), np.full(8000, HUB)),         # the hub, from every partition
        (srcs(1, 6500), np.full(6500, HUB)),
        (rng.choice(sub2, 6500), np.full(6500, HUB)),
    ]
    for i in range(3):                                            # local edges
        pairs.append((srcs(i, 2500), dsts(i, 2500)))
    loops = rng.choice(np.setdiff1d(np.arange(V), np.union1d(NO_IN, NO_OUT)), 40, replace=False)
    pairs.append((loops, loops))                                  # self loops
    e = np.concatenate([np.stack([s, d], 1) for s, d in pairs]).astype(np.int64)
    e = np.concatenate([e, e[rng.choice(e.shape[0], 400)]])       # multi-edges
    e = e[rng.permutation(e.shape[0])]
    return np.ascontiguousarray(e.astype(np.uint32))


class Topology:
    """What the engine is built from, derived from the edge list alone: per rank r and partition i the rows of i
    that r reads (global ids, ascending), the edge count of chunk i on rank r, and who pushes what to whom."""

    def __init__(self, edges, po):
        self.po = tuple(int(v) for v in po)
        src, dst = edges[:, 0].astype(np.int64), edges[:, 1].astype(np.int64)
        ps = np.searchsorted(self.po, src, side="right") - 1
        pd = np.searchsorted(self.po, dst, side="right") - 1
        self.P = len(po) - 1
        P = self.P
        self.owned = [self.po[r + 1] - self.po[r] for r in range(P)]
        self.edges = [[int(np.count_nonzero((pd == r) & (ps == i))) for i in range(P)] for r in range(P)]
        self.need = [[np.unique(src[(pd == r) & (ps == i)]) for i in range(P)] for r in range(P)]
        self.need_count = [[len(self.need[r][i]) if i != r else 0 for i in range(P)] for r in range(P)]
        # rank p sends to rank j what j reads from partition p; all of it, in order, goes by the copy engines
        self.send_count = [[len(self.need[j][p]) if j != p else 0 for j in range(P)] for p in range(P)]
        self.send_all = [[j != p and self.owned[p] > 0 and
                          np.array_equal(self.need[j][p] - self.po[p], np.arange(self.owned[p]))
                          for j in range(P)] for p in range(P)]

    def mirror_ids(self, r):
        return np.concatenate([self.need[r][i] for i in range(self.P)])

    def n_remote(self, p):
        return sum(1 for i in range(self.P) if i != p and self.edges[p][i] and self.need_count[p][i])


# ---- engine configurations and the call sequence ----------------------------------------------------------------------
CONFIGS = {
    # name: (layout, exact, environment)
    "defaults": ("a", True, {}),
    "merged_plans": ("a", True, {"NTS_EXCHANGE_MODE": "merged", "NTS_EXCHANGE_PLAN_MIN_EDGES": "1"}),
    "pipeline_nodma_1buf_1cta": ("a", True, {"NTS_EXCHANGE_MODE": "pipeline", "NTS_EXCHANGE_NO_DMA": "1",
                                             "NTS_EXCHANGE_BUFFERS": "1", "NTS_EXCHANGE_PUSH_CTAS": "1"}),
    "merged_1buf_512cta": ("a", True, {"NTS_EXCHANGE_MODE": "merged", "NTS_EXCHANGE_BUFFERS": "1",
                                       "NTS_EXCHANGE_PUSH_CTAS": "512"}),
    "empty_rank": ("b", True, {}),
    "random_weights": ("a", False, {}),
}
GROUPS = [("defaults", "merged_plans"), ("pipeline_nodma_1buf_1cta", "merged_1buf_512cta"),
          ("empty_rank", "random_weights")]

# (kind, F, variant); variant: "bf16" = BF16 gathers of an FP32 operand, "bf16in" = BF16 gathers of a BF16 operand,
# "off1" = an FP32 operand one float off 16-byte alignment.  Widths grow (the window is re-reserved between checked
# calls) and shrink again; every kind runs at least 3 times, more often than there are window buffers.
CALLS = [
    ("fwd", 6, None), ("bwd", 6, None), ("fetch", 3, None), ("ret", 3, None), ("fwd", 1, None),
    ("fwd", 64, None), ("fwd", 64, "off1"), ("fwd", 64, "bf16in"), ("fwd", 64, None), ("bwd", 64, None),
    ("fetch", 131, None), ("ret", 131, None), ("fwd", 131, None),
    ("fwd", 260, None), ("bwd", 260, "bf16"), ("fetch", 260, None),
    ("fwd", 602, None), ("bwd", 602, None), ("fwd", 602, "bf16"), ("ret", 602, None),
    ("fetch", 6, None), ("ret", 1, None), ("bwd", 3, None), ("fwd", 3, "bf16"),
]
KIND = {"fwd": 1, "bwd": 2, "fetch": 3, "ret": 4}


def engine_settings(env):
    return {"forced": {"pipeline": 1, "merged": 2}.get(env.get("NTS_EXCHANGE_MODE"), 0),
            "plan_min": int(env.get("NTS_EXCHANGE_PLAN_MIN_EDGES", 1 << 20)),
            "dma": "NTS_EXCHANGE_NO_DMA" not in env,
            "buffers": int(env.get("NTS_EXCHANGE_BUFFERS", 2))}


def push_vec(width, src_ptr):
    """The push kernel's VEC: the window rows of every buffer start 256-byte aligned, so only the width and the
    operand's alignment decide it."""
    if width % 4 == 0 and src_ptr % 16 == 0:
        return 4
    if width % 2 == 0 and src_ptr % 8 == 0:
        return 2
    return 1


def predict_paths(topo, p, settings, k, kind, F, var, src_ptr):
    """The path record of call k (0-based) on rank p.  mode None = measured (either is right)."""
    bf16 = var in ("bf16", "bf16in")
    P, owned = topo.P, topo.owned[p]
    out = {"kind": KIND[kind], "epoch": k + 1, "buffer": (k + 1) % settings["buffers"], "mode": 0,
           "kernel_peers": 0, "dma_peers": 0, "vec": 0, "plan_chunks": 0, "staging": 0}
    peers = [j for j in range(P) if j != p]
    if bf16 and owned:
        out["staging"] = 2 if (var == "bf16in" and F % 8 == 0 and src_ptr % 16 == 0) else 1
    if kind in ("fwd", "fetch"):
        for j in peers:
            if settings["dma"] and topo.send_all[p][j]:
                out["dma_peers"] |= 1 << j
            else:
                out["kernel_peers"] |= 1 << j
        if out["kernel_peers"]:   # BF16 rows of ld = ceil(F/8)*8 values travel as ld/2 floats
            width = (F + 7) // 8 * 4 if bf16 else F
            out["vec"] = push_vec(width, 0 if out["staging"] == 1 else src_ptr)
    else:
        out["dma_peers"] = sum(1 << j for j in peers)
    if kind in ("fwd", "bwd"):
        if settings["forced"] == 1 or topo.n_remote(p) < 2 or not owned or not sum(topo.need_count[p]):
            mode = 1
        else:
            mode = 2 if settings["forced"] == 2 else None
        out["mode"] = mode

        def planned(i, rows):
            e = topo.edges[p][i]
            return bool(e and rows and (e >= settings["plan_min"] or bf16))

        bits = 1 << p if planned(p, owned) else 0
        for i in peers:
            if not topo.need_count[p][i]:
                continue
            if mode == 2:
                bits |= (1 << i) if topo.edges[p][i] else 0
            elif planned(i, owned if kind == "fwd" else topo.need_count[p][i]):
                bits |= 1 << i
        out["plan_chunks"] = bits if mode is not None else None   # measured: depends on the mode taken
    return out


def paths_mismatch(got, want, topo, p, settings, kind, var):
    """None when the record matches the prediction (a measured mode may be either, and then decides the plan mask)."""
    want = dict(want)
    if want["mode"] is None:
        if got["mode"] not in (1, 2):
            return "measured mode %r" % got["mode"]
        want["mode"] = got["mode"]
        forced = dict(settings, forced=got["mode"])
        want["plan_chunks"] = predict_paths(topo, p, forced, 0, kind, 1, var, 0)["plan_chunks"]
    diff = {key: (got[key], want[key]) for key in want if got[key] != want[key]}
    return None if not diff else "paths (got, want): %r" % diff


# ---- float64 reference -------------------------------------------------------------------------------------------------
def exact_weight(src, dst):
    """q(src, dst) / 4 with q in 1..8: the same for both directions of an edge."""
    s, d = src.long(), dst.long()
    return (1 + (s * 5 + d * 3 + (s * d) % 7) % 8).to(torch.float32) / 4


def feature(ids, F, call, salt, device):
    """Integers in [-8, 8] that depend on (global id, column, call, salt)."""
    v = torch.as_tensor(ids, device=device).long()[:, None]
    c = torch.arange(F, device=device)[None, :]
    return (((v * 131 + c * 29 + call * 977 + salt * 7919 + (v * (c + 1)) % 13) % 17) - 8).double()


def uniform(n, F, call, salt, device):
    gen = torch.Generator().manual_seed(call * 1009 + salt)
    return (torch.rand((n, F), generator=gen, dtype=torch.float32) * 2 - 1).double().to(device)


class Truth:
    """Y = A X, dX = A^T G and the summed mirror gradients of the whole graph in float64, with |A| |X| beside them."""

    def __init__(self, fwd, bwd, topo, device):
        to = lambda a: torch.as_tensor(np.asarray(a), device=device)   # noqa: E731
        self.fs, self.fd, self.fw = to(fwd[0]).long(), to(fwd[1]).long(), to(fwd[2]).double()
        self.bs, self.bd, self.bw = to(bwd[0]).long(), to(bwd[1]).long(), to(bwd[2]).double()
        self.topo, self.device = topo, device
        self.mirror = [to(topo.mirror_ids(r)).long() for r in range(topo.P)]

    @staticmethod
    def exact(edges, topo, device):
        s, d = torch.as_tensor(edges[:, 0].astype(np.int64)), torch.as_tensor(edges[:, 1].astype(np.int64))
        w = exact_weight(s, d)
        return Truth((s, d, w), (s, d, w), topo, device)

    def forward(self, X):
        y = torch.zeros((V, X.shape[1]), dtype=torch.float64, device=self.device)
        return (y.index_add_(0, self.fd, X[self.fs] * self.fw[:, None]),
                torch.zeros_like(y).index_add_(0, self.fd, X[self.fs].abs() * self.fw.abs()[:, None]))

    def backward(self, G):
        dx = torch.zeros((V, G.shape[1]), dtype=torch.float64, device=self.device)
        return (dx.index_add_(0, self.bs, G[self.bd] * self.bw[:, None]),
                torch.zeros_like(dx).index_add_(0, self.bs, G[self.bd].abs() * self.bw.abs()[:, None]))

    def returned(self, grads):
        """grads[q] = rank q's mirror gradient rows (in its mirror order): their sum per owned vertex."""
        F = grads[0].shape[1]
        out = torch.zeros((V, F), dtype=torch.float64, device=self.device)
        mag = torch.zeros_like(out)
        for q in range(self.topo.P):
            out.index_add_(0, self.mirror[q], grads[q])
            mag.index_add_(0, self.mirror[q], grads[q].abs())
        return out, mag


def exact_mismatch(got, ref):
    """None when `got` equals the float64 reference exactly, else what differs."""
    g = got.double()
    if g.shape != ref.shape:
        return "shape %s, want %s" % (tuple(g.shape), tuple(ref.shape))
    if torch.equal(g, ref):
        return None
    bad = torch.nonzero(g != ref)
    r, c = bad[0].tolist()
    return "%d of %d elements differ, first (%d, %d): got %r, want %r" % (bad.shape[0], g.numel(), r, c,
                                                                          g[r, c].item(), ref[r, c].item())


def bound_mismatch(got, ref, mag):
    """None when every element is within 1e-4 of its |A| |X| of the float64 reference."""
    g = got.double()
    if g.shape != ref.shape:
        return "shape %s, want %s" % (tuple(g.shape), tuple(ref.shape))
    err = (g - ref).abs()
    bad = torch.nonzero(~(err <= 1e-4 * mag + 1e-30))
    if not bad.shape[0]:
        return None
    r, c = bad[0].tolist()
    return "%d elements out of bound, first (%d, %d): err %r, bound %r" % (bad.shape[0], r, c, err[r, c].item(),
                                                                         1e-4 * mag[r, c].item())


def exact_premise(mag):
    """Every partial sum of an exact-mode result is a multiple of 1/4 below 2^22, hence exact in FP32."""
    return None if not mag.numel() or mag.max().item() < 2.0 ** 22 else "|A| |X| reaches %r" % mag.max().item()


class Inputs:
    """The operands of call k: integer features (exact) or uniform ones, the same on every rank."""

    def __init__(self, exact, device):
        self.exact, self.device = exact, device

    def rows(self, ids, F, call, salt):
        if self.exact:
            return feature(ids, F, call, salt, self.device)
        return uniform(V, F, call, salt, self.device)[torch.as_tensor(ids, device=self.device).long()]

    def mirror_grad(self, truth, q, F, call):
        return self.rows(truth.mirror[q].cpu().numpy(), F, call, 10 + q)


def reference(truth, inputs, rank, k, kind, F, var):
    """(operand of this rank as float32, float64 result of this rank, |.| magnitudes) of call k."""
    lo, hi = truth.topo.po[rank], truth.topo.po[rank + 1]
    if kind in ("fwd", "bwd", "fetch"):
        full = inputs.rows(np.arange(V), F, k, {"fwd": 0, "bwd": 1, "fetch": 2}[kind]).float()
        used = full.to(torch.bfloat16).double() if var in ("bf16", "bf16in") else full.double()
        if kind == "fwd":
            ref, mag = truth.forward(used)
        elif kind == "bwd":
            ref, mag = truth.backward(used)
        else:
            m = used[truth.mirror[rank]]
            return full[lo:hi].contiguous(), m, m.abs()
        return full[lo:hi].contiguous(), ref[lo:hi], mag[lo:hi]
    grads = [inputs.mirror_grad(truth, q, F, k).float() for q in range(truth.topo.P)]
    ref, mag = truth.returned([g.double() for g in grads])
    return grads[rank].contiguous(), ref[lo:hi], mag[lo:hi]


# ---- the ranks ---------------------------------------------------------------------------------------------------------
def last_paths(handle):
    from neutronstarlite_b200 import _lib
    i = [C.c_int(-1) for _ in range(6)]
    u = [C.c_uint32(0xFFFFFFFF) for _ in range(3)]
    _lib.call("nts_exchange_last_paths", handle, C.byref(i[0]), C.byref(i[1]), C.byref(i[2]), C.byref(i[3]),
              C.byref(u[0]), C.byref(u[1]), C.byref(i[4]), C.byref(u[2]), C.byref(i[5]))
    return {"kind": i[0].value, "epoch": i[1].value, "buffer": i[2].value, "mode": i[3].value,
            "kernel_peers": u[0].value, "dma_peers": u[1].value, "vec": i[4].value, "plan_chunks": u[2].value,
            "staging": i[5].value}


def _chunk_edges(c, forward):
    """Global (src, dst) of every edge of a device chunk, in the order of its forward CSC or backward CSR."""
    if forward:
        off = c.column_offset_gpu.long()
        dst = c.dst_range[0] + torch.repeat_interleave(torch.arange(off.numel() - 1, device=off.device), off.diff())
        return c.row_indices_gpu.long(), dst
    off = c.row_offset_gpu.long()
    src = c.src_range[0] + torch.repeat_interleave(torch.arange(off.numel() - 1, device=off.device), off.diff())
    return src, c.column_indices_gpu.long()


def set_weights(pg, exact):
    """Exact mode: every chunk's weights become q(src, dst) / 4 in place; otherwise the GCN weights come back."""
    for c in pg.graph_chunks:
        if not c.edge_size:
            continue
        if not hasattr(c, "gcn_weights"):
            c.gcn_weights = (c.edge_weight_forward_gpu.clone(), c.edge_weight_backward_gpu.clone())
        if exact:
            c.edge_weight_forward_gpu.copy_(exact_weight(*_chunk_edges(c, True)))
            c.edge_weight_backward_gpu.copy_(exact_weight(*_chunk_edges(c, False)))
        else:
            c.edge_weight_forward_gpu.copy_(c.gcn_weights[0])
            c.edge_weight_backward_gpu.copy_(c.gcn_weights[1])
    torch.cuda.synchronize()


def gcn_truth(host, topo, device):
    """The reference at the real GCN weights: the single-partition chunk's CSC and CSR."""
    from neutronstarlite_b200.graph import PartitionedGraph
    c = PartitionedGraph(host, 1, 0).generate_all().graph_chunks[0]
    fd = np.repeat(np.arange(V), np.diff(c.column_offset.astype(np.int64)))
    bs = np.repeat(np.arange(V), np.diff(c.row_offset.astype(np.int64)))
    return Truth((c.row_indices.astype(np.int64), fd, c.edge_weight_forward),
                 (bs, c.column_indices.astype(np.int64), c.edge_weight_backward), topo, device)


def run_config(name, rank, host, edges, pgs, dev):
    """Every call of CALLS on a fresh engine; returns (failures, notes).  A mismatch is recorded, not raised, so every
    rank keeps taking part in the protocol to the end."""
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.exchange import GpuExchange
    from neutronstarlite_b200.graph import PartitionedGraph
    layout, exact, env = CONFIGS[name]
    po = PO[layout]
    if layout not in pgs:
        pgs[layout] = (PartitionedGraph(host, 3, rank, np.array(po, dtype=np.uint32)).generate_all(device=dev,
                                                                                                   dist=True),
                       Topology(edges, po))
    pg, topo = pgs[layout]
    set_weights(pg, exact)
    truth = Truth.exact(edges, topo, dev) if exact else gcn_truth(host, topo, dev)
    inputs = Inputs(exact, dev)
    settings = engine_settings(env)
    os.environ.update(env)
    try:
        ex = GpuExchange(pg, transport="p2p")
    finally:
        for key in env:
            del os.environ[key]
    L = _lib.load()
    fails, notes, grown = [], [], 0
    try:
        handle = ex._p2p.handle
        assert L.nts_exchange_last_paths(handle, *([None] * 9)) == 0
        for k, (kind, F, var) in enumerate(CALLS):
            operand, ref, mag = reference(truth, inputs, rank, k, kind, F, var)
            cap = L.nts_exchange_capacity_floats(handle)
            gd = torch.bfloat16 if var in ("bf16", "bf16in") else None
            x = operand
            if var == "off1":
                raw = torch.zeros(operand.numel() + 1, dtype=torch.float32, device=dev)
                raw[1:].copy_(operand.view(-1))
                x = raw[1:].view(operand.shape)
            elif var == "bf16in":
                x = operand.to(torch.bfloat16)
            if kind == "fwd":
                got = ex.forward(x, gather_dtype=gd)
            elif kind == "bwd":
                got = ex.backward(x, gather_dtype=gd)
            elif kind == "fetch":
                got = ex.fetch_mirrors(x)
            else:
                got = ex.return_mirror_grads(x)
            torch.cuda.synchronize()
            grown += k > 0 and L.nts_exchange_capacity_floats(handle) > cap
            where = "%s call %d (%s F=%d %s)" % (name, k, kind, F, var)
            if exact or kind == "fetch":   # a fetch copies rows: exact at any input
                bad = exact_mismatch(got, ref) or exact_premise(mag)
            else:
                bad = bound_mismatch(got, ref, mag)
            if bad:
                fails.append("%s: %s" % (where, bad))
            rec = last_paths(handle)
            want = predict_paths(topo, rank, settings, k, kind, F, var, x.data_ptr())
            bad = paths_mismatch(rec, want, topo, rank, settings, kind, var)
            if bad:
                fails.append("%s: %s" % (where, bad))
            if kind in ("fwd", "bwd") and want["mode"] is None:
                notes.append("%s rank %d %s F=%d %s: measured mode %d" % (name, rank, kind, F, var, rec["mode"]))
        if not grown:
            fails.append("%s: the window was never re-reserved between checked calls" % name)
    finally:
        dist.barrier()
        ex.close()
        dist.barrier()
    return fails, notes


def _worker(rank, world, port, group, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["NTS_EXCHANGE_TIMEOUT_MS"] = "120000"   # ranks time-slice one GPU: waits are long but bounded
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from neutronstarlite_b200.graph import HostGraph
        edges = make_graph()
        host = HostGraph(edges, V)
        pgs, fails, notes = {}, [], []
        for name in group:
            f, n = run_config(name, rank, host, edges, pgs, dev)
            fails += f
            notes += n
        q.put((rank, "ok" if not fails else "FAIL:\n" + "\n".join(fails[:12]), notes))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), []))
    finally:
        dist.destroy_process_group()


def _launch(target, world, args, timeout):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(r, world) + args + (q,)) for r in range(world)]
    for p in procs:
        p.start()
    results = []
    try:
        for _ in range(world):
            results.append(q.get(timeout=timeout))
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    for rank, msg, notes in sorted(results):
        for line in notes:
            print(line)
    for rank, msg, _ in sorted(results):
        assert msg == "ok", "rank %d: %s" % (rank, msg)


@pytest.mark.gpu
@pytest.mark.parametrize("group", GROUPS, ids=["+".join(g) for g in GROUPS])
def test_exchange_matches_float64_at_every_branch(group):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    _launch(_worker, 3, (30200 + GROUPS.index(group), group), 420)


# ---- CPU: the graph, the prediction and the comparator -----------------------------------------------------------------
@pytest.fixture(scope="module")
def graph():
    return make_graph()


def test_graph_has_the_properties_the_branches_need(graph):
    src, dst = graph[:, 0].astype(np.int64), graph[:, 1].astype(np.int64)
    t = Topology(graph, PO["a"])
    assert PO["a"][1] % 4 != 0
    assert t.need_count[1][0] == t.owned[0] and t.send_all[0][1]               # copy-engine push 0 -> 1
    assert 0 < t.need_count[1][2] < t.owned[2] and not t.send_all[2][1]       # kernel push 2 -> 1
    assert t.need[0][1].tolist() == list(SRC_1_TO_0) and t.need[2][1].tolist() == list(SRC_1_TO_2)
    assert t.edges[0][2] == 0 and t.send_count[2][0] == 0                     # flag-only push 2 -> 0
    assert [t.n_remote(p) for p in range(3)] == [1, 2, 2]
    hub = dst == HUB
    assert hub.sum() >= 20000 and len(set(np.searchsorted(PO["a"], src[hub], side="right") - 1)) == 3
    assert (src == dst).sum() >= 40
    assert len(np.unique(graph, axis=0)) < len(graph)                         # multi-edges
    assert not np.isin(NO_IN, dst).any() and not np.isin(NO_OUT, src).any()
    b = Topology(graph, PO["b"])
    assert b.owned[1] == 0 and b.send_all[0][2] and [b.n_remote(p) for p in range(3)] == [1, 0, 1]


class _ThreadSplit:
    """The collectives ExchangePlan uses, for P ranks run as threads of one process."""

    def __init__(self, P):
        self.P, self.bar, self.slots, self.local = P, threading.Barrier(P), [None] * P, threading.local()

    def get_backend(self, group=None):
        return "gloo"

    def all_to_all_single(self, out, inp, output_split_sizes=None, input_split_sizes=None, group=None):
        r = self.local.rank
        split = input_split_sizes or [inp.shape[0] // self.P] * self.P
        self.slots[r] = list(torch.split(inp, split))
        self.bar.wait()
        out.copy_(torch.cat([self.slots[j][r] for j in range(self.P)]))
        self.bar.wait()


@pytest.mark.parametrize("layout", sorted(PO))
def test_predicted_paths_agree_with_exchange_plan(graph, layout, monkeypatch):
    """ExchangePlan for all three ranks (threads sharing one fake split) has the need and send lists the prediction is
    built from, so the masks predicted from either are the same."""
    from neutronstarlite_b200 import exchange
    from neutronstarlite_b200.graph import HostGraph, PartitionedGraph
    host = HostGraph(graph, V)
    po = np.array(PO[layout], dtype=np.uint32)
    pgs = [PartitionedGraph(host, 3, r, po).generate_all(dist=True) for r in range(3)]
    split = _ThreadSplit(3)
    monkeypatch.setattr(exchange, "dist", split)
    plans, errors = [None] * 3, []

    def build(r):
        split.local.rank = r
        try:
            plans[r] = exchange.ExchangePlan(pgs[r], merged=False)
        except Exception as exc:  # pragma: no cover
            errors.append(exc)
            split.bar.abort()

    threads = [threading.Thread(target=build, args=(r,)) for r in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    topo = Topology(graph, PO[layout])
    for p, plan in enumerate(plans):
        assert plan.need_count[:p] + plan.need_count[p + 1:] == topo.need_count[p][:p] + topo.need_count[p][p + 1:]
        assert [int(pgs[p].graph_chunks[i].edge_size) for i in range(3)] == topo.edges[p]
        for i in range(3):
            assert np.array_equal(plan.need[i].numpy() + PO[layout][i], topo.need[p][i])
        for j in range(3):
            if j == p:
                continue
            assert plan.send_count[j] == topo.send_count[p][j]
            rows = plan.send_rows[j].numpy()
            send_all = pgs[p].owned_vertices > 0 and np.array_equal(rows, np.arange(pgs[p].owned_vertices))
            assert send_all == topo.send_all[p][j]


def test_prediction_covers_every_branch(graph):
    """Across the configurations the asserted records include every branch the file is meant to reach."""
    seen = set()
    for name, (layout, exact, env) in CONFIGS.items():
        topo, settings = Topology(graph, PO[layout]), engine_settings(env)
        seen.add(("buffers", settings["buffers"]))
        for p in range(3):
            seen.add(("owned", topo.owned[p] > 0))
            for k, (kind, F, var) in enumerate(CALLS):
                ptr = 4 if var == "off1" else 0
                w = predict_paths(topo, p, settings, k, kind, F, var, ptr)
                bf16 = var in ("bf16", "bf16in")
                seen.add(("vec", w["vec"]))
                seen.add(("staging", w["staging"]))
                if w["kernel_peers"]:
                    seen.add("kernel push")
                    if any(w["kernel_peers"] >> j & 1 and not topo.send_count[p][j] for j in range(3)):
                        seen.add("flag-only push")
                if w["dma_peers"] and kind in ("fwd", "fetch"):
                    seen.add("copy-engine push")
                if w["mode"]:
                    seen.add(("mode", w["mode"], bf16))
                if w["plan_chunks"]:
                    seen.add("planned chunk")
                if w["plan_chunks"] is not None and kind in ("fwd", "bwd") and topo.edges[p][p] and \
                        topo.owned[p] and not w["plan_chunks"] >> p & 1:
                    seen.add("K1 chunk")   # the local chunk
    for item in [("vec", 1), ("vec", 2), ("vec", 4), "kernel push", "copy-engine push", "flag-only push",
                 ("mode", 1, False), ("mode", 2, False), ("mode", 1, True), ("mode", 2, True), "planned chunk",
                 "K1 chunk", ("buffers", 1), ("buffers", 2), ("owned", False), ("staging", 2)]:
        assert item in seen, item


@pytest.fixture(scope="module")
def truth(graph):
    return Truth.exact(graph, Topology(graph, PO["a"]), torch.device("cpu"))


def test_exact_inputs_stay_exact_in_fp32(truth):
    """The widest call's |A| |X|, |A^T| |G| and summed mirror magnitudes stay below 2^22 on every rank."""
    inputs = Inputs(True, torch.device("cpu"))
    for kind in ("fwd", "bwd", "ret"):
        for rank in range(3):
            _, ref, mag = reference(truth, inputs, rank, 3, kind, 602, None)
            assert exact_premise(mag) is None
            assert torch.equal(ref, ref.float().double())


@pytest.mark.parametrize("kind", ["fwd", "bwd", "fetch", "ret"])
def test_exact_comparator_rejects_a_stale_epoch(truth, kind):
    """The result of call k computed from the operands of call k-1 (what a reader of the other buffer would see)."""
    inputs = Inputs(True, torch.device("cpu"))
    for rank in range(3):
        _, ref, _ = reference(truth, inputs, rank, 7, kind, 6, None)
        _, stale, _ = reference(truth, inputs, rank, 6, kind, 6, None)
        assert exact_mismatch(ref.float(), ref) is None
        assert exact_mismatch(stale.float(), ref) is not None


def test_exact_comparator_rejects_a_mirror_row_in_the_wrong_slot(truth):
    inputs = Inputs(True, torch.device("cpu"))
    _, ref, _ = reference(truth, inputs, 1, 2, "fetch", 3, None)
    for a in (0, ref.shape[0] // 2, ref.shape[0] - 2):
        assert not torch.equal(ref[a], ref[a + 1])
        moved = ref.clone()
        moved[a], moved[a + 1] = ref[a + 1], ref[a]
        assert exact_mismatch(moved.float(), ref) is not None


def test_exact_comparator_rejects_a_dropped_edge(graph, truth):
    """One edge into the hub, and one into a low-degree row, left out of the graph."""
    inputs = Inputs(True, torch.device("cpu"))
    hub_edge = int(np.nonzero(graph[:, 1] == HUB)[0][0])
    low = int(np.nonzero(graph[:, 0] == SRC_1_TO_0[0])[0][0])
    for drop in (hub_edge, low):
        rank = int(np.searchsorted(PO["a"], graph[drop, 1], side="right") - 1)
        short = Truth.exact(np.delete(graph, drop, axis=0), truth.topo, torch.device("cpu"))
        for kind in ("fwd", "bwd"):
            r = int(np.searchsorted(PO["a"], graph[drop, 0], side="right") - 1) if kind == "bwd" else rank
            _, ref, _ = reference(truth, inputs, r, 4, kind, 6, None)
            _, got, _ = reference(short, inputs, r, 4, kind, 6, None)
            assert exact_mismatch(got.float(), ref) is not None


def test_bound_rejects_a_stale_epoch_at_gcn_weights(graph):
    from neutronstarlite_b200.graph import HostGraph
    topo = Topology(graph, PO["a"])
    t = gcn_truth(HostGraph(graph, V), topo, torch.device("cpu"))
    inputs = Inputs(False, torch.device("cpu"))
    for kind in ("fwd", "bwd", "ret"):
        _, ref, mag = reference(t, inputs, 1, 5, kind, 6, None)
        _, stale, _ = reference(t, inputs, 1, 4, kind, 6, None)
        assert bound_mismatch(ref.float(), ref, mag) is None
        assert bound_mismatch(stale.float(), ref, mag) is not None
