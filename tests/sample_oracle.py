"""numpy restatement of the neighbour sampler (K8, nts_sampler of include/nts_b200.h), bit-exact: the same splitmix64
counter hash, Floyd's k-subset, ascending slot order, distinct sources ascending by global id and the transposed block
stable by edge position.  Used by the sampler tests as the oracle of the GPU kernels."""
import numpy as np

_M = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(z):
    """splitmix64 finaliser on uint64 scalars or arrays (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        z = np.asarray(z, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def step_key(seed, step):
    return splitmix64(splitmix64(np.uint64(seed)) ^ np.uint64(step))


def dst_keys(skey, hop, dst):
    return splitmix64(skey ^ ((np.uint64(hop) << np.uint64(32)) | np.asarray(dst, dtype=np.uint64)))


def floyd(keys, deg, k):
    """Chosen slots [n, k] (ascending per row) of destinations with deg > k, keys = dst_keys of each."""
    n = keys.shape[0]
    chosen = np.zeros((n, k), dtype=np.int64)
    deg = deg.astype(np.uint64)
    for i in range(k):
        j = deg - np.uint64(k) + np.uint64(i)
        h = splitmix64(keys ^ j) >> np.uint64(32)
        t = (h * (j + np.uint64(1))) >> np.uint64(32)
        t = t.astype(np.int64)
        hit = (chosen[:, :i] == t[:, None]).any(1) if i else np.zeros(n, dtype=bool)
        chosen[:, i] = np.where(hit, j.astype(np.int64), t)
    return np.sort(chosen, axis=1)


def sample_hop(col, row, w, dst, k, skey, hop):
    """One hop: the block of destinations `dst` (global ids) of the CSC (col, row, w)."""
    dst = np.asarray(dst, dtype=np.int64)
    deg = (col[dst + 1].astype(np.int64) - col[dst]) if dst.size else np.zeros(0, np.int64)
    cnt = np.minimum(deg, k)
    c_o = np.zeros(dst.size + 1, dtype=np.uint32)
    np.cumsum(cnt, out=c_o[1:])
    # absolute CSC positions of the kept slots: every slot of a destination with deg <= k, Floyd's subset otherwise
    edge_dst = np.repeat(np.arange(dst.size, dtype=np.int64), cnt)
    slots = col[dst[edge_dst]].astype(np.int64) + np.arange(int(c_o[-1])) - c_o[edge_dst]
    big = np.nonzero(deg > k)[0]
    if big.size:
        ch = floyd(dst_keys(skey, hop, dst[big]), deg[big], k)
        base = col[dst[big]].astype(np.int64)
        pos = c_o[big].astype(np.int64)[:, None] + np.arange(k)[None, :]
        slots[pos.reshape(-1)] = (base[:, None] + ch).reshape(-1)
    row_global = row[slots].astype(np.uint32)
    weight = w[slots].astype(np.float32)
    src, row_local = np.unique(row_global, return_inverse=True)
    order = np.argsort(row_local, kind="stable")
    r_o = np.zeros(src.size + 1, dtype=np.uint32)
    np.cumsum(np.bincount(row_local, minlength=src.size), out=r_o[1:])
    return {
        "dst": dst.astype(np.uint32), "column_offset": c_o, "row_indices": row_local.astype(np.uint32),
        "row_global": row_global, "weight": weight, "src": src.astype(np.uint32), "row_offset": r_o,
        "column_indices": edge_dst[order].astype(np.uint32), "weight_backward": weight[order],
    }


def sample(col, row, w, seeds, fanout, seed, step):
    """Every hop of one sample: list of dicts as sample_hop returns; hop h+1's destinations are hop h's sources."""
    col = np.asarray(col, dtype=np.uint32)
    row = np.asarray(row, dtype=np.uint32)
    w = np.asarray(w, dtype=np.float32)
    skey = step_key(seed, step)
    hops, dst = [], np.asarray(seeds, dtype=np.int64)
    for h, k in enumerate(fanout):
        b = sample_hop(col, row, w, dst, int(k), skey, h)
        hops.append(b)
        dst = b["src"].astype(np.int64)
    return hops
