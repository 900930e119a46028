#!/usr/bin/env python3
"""Small driver for `compute-sanitizer --tool memcheck|racecheck|synccheck python tools/sanitizer_smoke.py`:
every kernel family of libnts_b200 once on small inputs (both aggregation variants, odd widths, hubs, empty rows)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from neutronstarlite_b200 import _lib, ops
from neutronstarlite_b200.exchange import GpuExchange
from neutronstarlite_b200.graph import HostGraph, PartitionedGraph

dev = torch.device("cuda:0")
rng = np.random.default_rng(0)
V, E = 700, 9000
edges = np.stack([rng.integers(0, V, E), rng.integers(0, V, E)], 1).astype(np.uint32)
edges[:1500, 1] = 3
pg = PartitionedGraph(HostGraph(edges, V), 1, 0).generate_all(device=dev, dist=True)
for variant in (1, 2):
    _lib.call("nts_aggregate_set_variant", variant, 0)
    for F in (602, 128, 41, 7, 172):
        x = torch.rand((V, F), device=dev)
        op = ops.ForwardSingleGPUfuseOp(pg)
        y = op.forward(x)
        dx = op.backward(y)
_lib.call("nts_aggregate_set_variant", 0, 0)
# preprocessed aggregation (nts_gather_plan): slab counts, both staging variants, virtual warps (F <= 64), padded rows
c = pg.graph_chunks[0]
for variant in (0, 1):
    _lib.call("nts_gather_plan_set_variant", variant)
    for slabs in (1, 3):
        ops.set_plan_mode("on", slabs)
        for F in (602, 128, 64, 41, 7):
            x = torch.rand((V, F), device=dev)
            ops.gather_by_dst_from_src(c, torch.zeros_like(x), x)
            ops.gather_by_src_from_dst(c, torch.zeros_like(x), x)
        c.__dict__.pop("_gather_plans", None)
_lib.call("nts_gather_plan_set_variant", 0)
ops.set_plan_mode("on", 0)                      # measured slab count (nts_gather_plan_create_tuned_ex)
x = torch.rand((V, 128), device=dev)
ops.gather_by_dst_from_src(c, torch.zeros_like(x), x)
ops.set_plan_mode("auto")
# fused Adam
W, M, Vv, G = (torch.rand(1000, device=dev) for _ in range(4))
_lib.call("nts_adam_update", W.data_ptr(), M.data_ptr(), Vv.data_ptr(), G.data_ptr(), 1000, 1e-4, 0.9, 0.999, 0.01, 1e-9,
          torch.cuda.current_stream().cuda_stream)
ex = GpuExchange(pg)
dep = ops.DistGPUGetDepNbrOp(pg, None, exchange=ex)
for H, D in ((1, 16), (4, 8)):
    x = torch.rand((V, H * D), device=dev)
    mirror = dep.forward(x)
    e_src = ops.DistGPUScatterSrc(pg).forward(mirror[:, :H].contiguous())
    e_dst = ops.DistGPUScatterDst(pg).forward(x[:, :H].contiguous())
    sm = ops.DistGPUEdgeSoftMax(pg)
    a = sm.forward(e_src + e_dst)
    fw = ops.DistGPUAggregateDstFuseWeight(pg)
    y = fw.forward(mirror, a)
    dm = fw.backward(y)
    da = fw.get_additional_grad()
    g_in = sm.backward(da)
    ops.DistGPUScatterSrc(pg).backward(g_in)
    ops.DistGPUScatterDst(pg).backward(g_in)
    ops.DistGPUAggregateDst(pg).forward(torch.rand((pg.owned_edges, D), device=dev))
    dep.backward(dm)
    fused = ops.DistGPUFusedGATOp(pg)
    out = fused.forward(mirror, mirror[:, :H].contiguous(), x[:, :H].contiguous())
    fused.backward(out)
    single = ops.DistGPUFusedGATOp(pg, two_pass_backward=False)   # the single-pass (atomic) backward as well
    single.forward(mirror, mirror[:, :H].contiguous(), x[:, :H].contiguous())
    single.backward(out)
# neighbour sampling (K8): Floyd and keep-all destinations, a hub, an empty sample, the device transpose
from neutronstarlite_b200.sample import NeighborSampler, SampledSubgraph
sampler = NeighborSampler(pg, [5, 64, 3], 128)
sg = sampler.sample(np.arange(0, V, 6)[:128], 1, 0)
sampler.sample(np.zeros(0, dtype=np.int64), 1, 1)
sg = sampler.sample(np.array([3, 0, 1]), 1, 2)
b = sg.blocks[1]
SampledSubgraph.from_blocks([{"dst": b.dst, "column_offset": b.column_offset, "row_indices": b.row_indices,
                              "weight": b.weight, "src": b.src}])
op = ops.MiniBatchFuseOp(sg, 1)
op.backward(op.forward(torch.rand((b.n_src, 41), device=dev)))
torch.cuda.synchronize()
print("sanitizer smoke done, launches:", _lib.load().nts_kernel_launch_count())
