"""Time the K8 sampler on a sharded topology against the whole-graph sampler (one H100).

    python tools/sharded_topology_time.py [--batch 1024] [--epochs 3] [--warmup 1] [--out DIR]

Workload: bench.py's config B graph (synth.WORKLOADS["reddit"], synth.zipf_edges, self loops included), train ids
mask == 0, and the samplers of the two sampled toolkits: GCN (fanout 25-10) and GAT (fanout 10-10-5, include_dst).
Three variants, alternated epoch by epoch (an epoch samples every train batch once, steps as GCNSampleImpl numbers
them):
  * whole:    NeighborSampler on the single-partition PartitionedGraph;
  * shards_1: NeighborSampler on ShardedTopology.from_partitioned_graph (one shard, merged by nts_merge_chunk_csc);
  * shards_8: ShardedTopology.split into 8 shards in this process, at the reference partitioner's offsets (what 8
              ranks' samplers read, minus the NVLink hops).
Sampler time per step is a host clock around sample() (which synchronises the stream once per hop) and a device
synchronise.  Before timing, every batch of one epoch is sampled by all three and the blocks compared bit for bit.
Also reported: topology bytes per rank (allocated at world 1, computed for world 8 and for config E), slots each step
would read from other ranks' shards at world 8 (rank = batch mod 8, as in toolkits._SampledRounds), and the card's name
and power limit, read in the same run.  It runs on one GPU: multi-GPU epoch times need one process per GPU and are
reported as not measured.
One JSON object on stdout (and in DIR/sharded_topology_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from neutronstarlite_b200 import synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402
from neutronstarlite_b200.sample import NeighborSampler  # noqa: E402
from neutronstarlite_b200.topology import ShardedTopology, _sections  # noqa: E402
from sample_train_time import card  # noqa: E402

SAMPLERS = {"gcn": ([25, 10], False), "gat": ([10, 10, 5], True)}
WORLD = 8


def batches(ids, batch):
    return [ids[i:i + batch] for i in range(0, ids.numel(), batch)]


def epoch(sampler, seeds, step0):
    times = []
    for b, s in enumerate(seeds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sampler.sample(s, 0, step0 + b)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return times


def same_blocks(a, b):
    for x, y in zip(a.blocks, b.blocks):
        for k in ("dst", "column_offset", "row_indices", "row_global", "weight", "src", "row_offset",
                  "column_indices", "weight_backward", "dst_pos"):
            tx, ty = getattr(x, k), getattr(y, k)
            if (tx is None) != (ty is None) or (tx is not None and not torch.equal(tx.view(torch.int32),
                                                                                 ty.view(torch.int32))):
                return False
    return True


def remote_slots(sg, off, rank):
    """Slots a step on `rank` reads from other ranks' shards: every kept edge of a destination it does not own."""
    lo, hi = int(off[rank]), int(off[rank + 1])
    n = 0
    for b in sg.blocks:
        deg = b.column_offset[1:].long() - b.column_offset[:-1].long()
        dst = b.dst.long() & 0xFFFFFFFF
        n += int(deg[(dst < lo) | (dst >= hi)].sum())
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sharded_topology_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, E_rand, _ = synth.WORKLOADS["reddit"]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_raw = torch.bincount(src, minlength=V)
    in_raw = torch.bincount(dst, minlength=V)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_raw.clamp(min=1), in_raw.clamp(min=1))
    E = int(pg.owned_edges)
    del src, dst
    _, _, mask = synth.features_labels_mask(V, 8, 2, dev)
    train = (mask.cpu() == 0).nonzero().view(-1)
    seeds = batches(train, args.batch)
    off8 = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E, WORLD).astype(np.int64)
    col = pg.graph_chunks[0].column_offset_gpu.long().cpu().numpy()
    edges8 = [int(col[off8[r + 1]] - col[off8[r]]) for r in range(WORLD)]
    topo1 = ShardedTopology.from_partitioned_graph(pg)
    c = pg.graph_chunks[0]
    topo8 = ShardedTopology.split(c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, off8)
    Ve, Ee, _ = synth.WORKLOADS["papers100m"]
    res = {"card": card(), "workload": "reddit (config B)", "V": V, "E": E, "batch": args.batch,
           "steps_per_epoch": len(seeds), "world8_offsets": off8.tolist(),
           "topology_bytes_per_rank": {
               "replicated_partitioned_graph_16B_per_edge": 16 * E,
               "world1_allocated": topo1.local_bytes,
               "world8_computed_max": max(_sections(int(off8[r + 1] - off8[r]), edges8[r])[1] for r in range(WORLD)),
               "configE_half_scale_replicated_computed": 16 * Ee,
               "configE_half_scale_world8_computed_balanced": (4 * (Ve + WORLD) + 8 * Ee) // WORLD,
               "configE_full_shape_world8_computed_balanced": (4 * (Ve + WORLD) + 8 * 2 * Ee) // WORLD},
           "multi_gpu_epoch_ms": "not measured (needs one process per GPU)"}
    graphs = {"whole": pg, "shards_1": topo1, "shards_8": topo8}
    for kind, (fanout, inc) in SAMPLERS.items():
        smp = {v: NeighborSampler(g, fanout, args.batch, include_dst=inc) for v, g in graphs.items()}
        identical, remote = True, []
        for b, s in enumerate(seeds):
            ref = smp["whole"].sample(s, 0, b).clone()
            for v in ("shards_1", "shards_8"):
                identical &= same_blocks(smp[v].sample(s, 0, b), ref)
            remote.append(remote_slots(ref, off8, b % WORLD))
        for _ in range(args.warmup):
            for v in smp:
                epoch(smp[v], seeds, 0)
        times = {v: [] for v in smp}
        for e in range(args.epochs):
            for v in smp:                  # alternated
                times[v] += epoch(smp[v], seeds, (e + 1) * len(seeds))
        res[kind] = {"fanout": fanout, "include_dst": inc, "blocks_bit_identical": bool(identical),
                     "world8_remote_slots_per_step_mean": statistics.mean(remote),
                     "sampler_ms_per_step": {v: {"median": statistics.median(t), "min": min(t), "max": max(t)}
                                             for v, t in times.items()}}
        del smp
    topo1.close()
    topo8.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sharded_topology_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
