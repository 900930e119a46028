"""Synthetic inputs of the shapes BASELINE.json names (SURVEY.md 8d): power-law multigraphs generated on the GPU.

Edges: both endpoints drawn from a Zipf(s) law over a random permutation of the vertices (hubs on both sides,
duplicates kept - they count in degrees like in the reference), plus one self loop per vertex.  Features U(-1,1),
labels U{0..C-1}, mask v % 3 (the reference's `random_generate`, core/ntsDataloador.hpp:63-71, uses all-ones
features which would hide index bugs)."""
from __future__ import annotations

import torch

WORKLOADS = {
    # name: (V, E_random, layers)            SURVEY.md 8 preamble / 8d
    "reddit": (232965, 114615892, [602, 128, 41]),
    "products": (2449029, 61859140, [100, 128, 47]),
    # config E: ogbn-papers100M's degree and widths at half its vertices and edges, so that one partition of 8 fits an
    # 80 GB H100 next to its receive window (tools/plan_memory.py); generated per partition (zipf_edges_owned)
    "papers100m": (55529978, 807842936, [128, 128, 172]),
    "papers_eighth": (6941247, 100980367, [128, 128, 172]),   # one GPU's share of config E as a stand-alone graph
    "cora_sized": (2708, 10858, [1433, 128, 7]),
    "tiny": (20000, 400000, [602, 128, 41]),
}

SEED_GRAPH = 0x5EED0001
SEED_FEATURES = 0x5EED0002


def _zipf_stream(V, E, device, s, seed, chunk):
    """Yields (src, dst) int64 chunks of the E random edges; the sequence is a function of (V, E, s, seed, chunk) and
    the GPU architecture only, so every rank - and the one-shot and the streaming consumers - see the same graph."""
    gen = torch.Generator(device=device).manual_seed(seed)
    w = torch.arange(1, V + 1, device=device, dtype=torch.float64).pow_(-s)
    cdf = torch.cumsum(w / w.sum(), 0)
    del w
    perm_s = torch.randperm(V, generator=gen, device=device)
    perm_d = torch.randperm(V, generator=gen, device=device)
    done = 0
    while done < E:
        n = min(chunk, E - done)
        u = torch.rand(n, generator=gen, device=device, dtype=torch.float64)
        src = perm_s[torch.searchsorted(cdf, u).clamp_(max=V - 1)]
        u = torch.rand(n, generator=gen, device=device, dtype=torch.float64)
        dst = perm_d[torch.searchsorted(cdf, u).clamp_(max=V - 1)]
        del u
        yield src, dst
        done += n


def zipf_edges(V, E, device, s=1.0, seed=SEED_GRAPH, self_loops=True, chunk=1 << 26):
    """int64 (src, dst) on `device`; deterministic for a given (V, E, s, seed) and GPU architecture."""
    src_parts, dst_parts = [], []
    for src, dst in _zipf_stream(V, E, device, s, seed, chunk):
        src_parts.append(src)
        dst_parts.append(dst)
    if self_loops:
        loops = torch.arange(V, device=device, dtype=torch.int64)
        src_parts.append(loops)
        dst_parts.append(loops)
    return torch.cat(src_parts), torch.cat(dst_parts)


def zipf_degrees(V, E, device, s=1.0, seed=SEED_GRAPH, self_loops=True, chunk=1 << 26):
    """(out_degree, in_degree) int64 [V] of the same graph WITHOUT materialising its edge list (pass 1 of the
    streaming generation of graphs that do not fit one GPU next to their features: papers100M-shaped, SURVEY 8d)."""
    out_d = torch.zeros(V, dtype=torch.int64, device=device)
    in_d = torch.zeros(V, dtype=torch.int64, device=device)
    for src, dst in _zipf_stream(V, E, device, s, seed, chunk):
        out_d += torch.bincount(src, minlength=V)
        in_d += torch.bincount(dst, minlength=V)
    if self_loops:
        out_d += 1
        in_d += 1
    return out_d, in_d


def zipf_edges_owned(V, E, device, v0, v1, s=1.0, seed=SEED_GRAPH, self_loops=True, chunk=1 << 26):
    """The edges of the same graph whose DESTINATION lies in [v0, v1) (pass 2: what rank p of a partitioned run
    keeps), in stream order, self loops of the owned vertices last."""
    src_parts, dst_parts = [], []
    for src, dst in _zipf_stream(V, E, device, s, seed, chunk):
        keep = (dst >= v0) & (dst < v1)
        src_parts.append(src[keep])
        dst_parts.append(dst[keep])
    if self_loops:
        loops = torch.arange(v0, v1, device=device, dtype=torch.int64)
        src_parts.append(loops)
        dst_parts.append(loops)
    return torch.cat(src_parts), torch.cat(dst_parts)


def features_labels_mask(V, F, classes, device, seed=SEED_FEATURES, rows=None):
    """Features of rows [rows[0], rows[1]) (default all), generated per row block so every rank of a partitioned
    run sees the same global matrix."""
    lo, hi = (0, V) if rows is None else rows
    gen = torch.Generator(device=device).manual_seed(seed)
    block = 1 << 15
    out = torch.empty((hi - lo, F), dtype=torch.float32, device=device)
    labels = torch.empty(hi - lo, dtype=torch.int64, device=device)
    # generate whole blocks and keep the overlap: deterministic per global row id
    b0 = (lo // block) * block
    gen_state_skip = b0 // block
    for _ in range(gen_state_skip):
        torch.rand((block, F), generator=gen, device=device)
        torch.randint(0, classes, (block,), generator=gen, device=device)
    pos = b0
    while pos < hi:
        x = torch.rand((block, F), generator=gen, device=device) * 2 - 1
        y = torch.randint(0, classes, (block,), generator=gen, device=device)
        a, b = max(pos, lo), min(pos + block, hi)
        if b > a:
            out[a - lo:b - lo] = x[a - pos:b - pos]
            labels[a - lo:b - lo] = y[a - pos:b - pos]
        pos += block
    mask = (torch.arange(lo, hi, device=device) % 3).to(torch.int64)
    return out, labels, mask
