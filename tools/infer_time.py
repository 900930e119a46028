"""Time full-neighbour inference of sampled GCN (GCNSampleImpl.infer) against sampled evaluation, on config B.

    python tools/infer_time.py [--gpus N] [--repeats 5] [--epochs 3] [--reps 20] [--out DIR]

Workload: bench.py's config B graph (synth.WORKLOADS["reddit"], synth.zipf_edges, self loops included), layers
602-128-41, fanout 25-10, batch 1024, FP32, GCNSampleImpl on a ShardedFeatureTable and a ShardedTopology over N ranks
(one process per GPU, NCCL; rank r owns the reference partitioner's range r).  Reports, with the card's name and power
limit read in the same run:
  1. infer() wall time (host clock, ended by a device synchronise), and the per-layer split of one more call in which
     every part ends in a device synchronise: GEMM, table build, aggregation, scale and relu, close;
  2. evaluate(1) + evaluate(2) wall time on the same model, alternated with (1) over --repeats repeats;
  3. at N = 1, the time of nts_segment_gather_sum_sharded (K9, a one-shard FP32 table) on config B's whole CSC at
     F = 128 and F = 41, CUDA events over --reps launches, alternated round by round with K1
     (nts_segment_gather_sum) and K1P (ops.GatherPlan, tuned for F) on the same arrays, with the algorithmic bytes
     E*F*4 + 8*E over time and the largest difference of K9's and K1P's outputs from K1's;
  4. validation and test accuracy from evaluate_full and from evaluate after --epochs training epochs.
One JSON object on stdout from rank 0 (and in DIR/infer_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from neutronstarlite_b200 import _lib, ops, synth, toolkits  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402
from neutronstarlite_b200.topology import ShardedTopology  # noqa: E402
from sample_train_time import card  # noqa: E402

LAYERS, FANOUT, BATCH = [602, 128, 41], [25, 10], 1024


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


class Split:
    """Wraps the parts infer() calls so that each ends in a device synchronise and its host time is added to its
    part; restores them on exit."""

    PARTS = ("gemm", "table_build", "aggregate", "scale_relu", "close")

    def __init__(self):
        self.ms = dict.fromkeys(self.PARTS, 0.0)
        T = ShardedFeatureTable
        self.saved = [(T, "__init__", T.__init__), (T, "aggregate", T.aggregate), (T, "close", T.close),
                      (torch.Tensor, "mm", torch.Tensor.mm), (torch.Tensor, "mul_", torch.Tensor.mul_),
                      (toolkits.torch, "relu", torch.relu)]

    def __enter__(self):
        parts = {"__init__": "table_build", "aggregate": "aggregate", "close": "close", "mm": "gemm",
                 "mul_": "scale_relu", "relu": "scale_relu"}
        for owner, name, fn in self.saved:
            setattr(owner, name, self._timed(fn, parts[name]))
        return self

    def _timed(self, fn, part):
        def run(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize()
            self.ms[part] += (time.perf_counter() - t0) * 1e3
            return r
        return run

    def __exit__(self, *exc):
        for owner, name, fn in self.saved:
            setattr(owner, name, fn)


def kernels(pg, reps, dev):
    """K9 vs K1 vs K1P on the whole CSC of pg at F = 128 and 41 (world 1)."""
    c = pg.graph_chunks[0]
    V, E = int(pg.global_vertices), int(c.edge_size)
    col, row, w = c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu
    stream = torch.cuda.current_stream().cuda_stream
    res = {}
    for F in (128, 41):
        x = torch.rand((V, F), generator=torch.Generator().manual_seed(F)).to(dev)
        table = ShardedFeatureTable(x, [0, V])
        plan = ops.GatherPlan(col, row, w, 0, V, E, V, 0, tune_for=F, tune_accumulate=False)
        outs = {k: torch.zeros((V, F), device=dev) for k in ("K9", "K1", "K1P")}
        run = {"K9": lambda: table.aggregate(outs["K9"], col, row, w, 0, E),
               "K1": lambda: _lib.call("nts_segment_gather_sum", x.data_ptr(), outs["K1"].data_ptr(), w.data_ptr(),
                                       row.data_ptr(), col.data_ptr(), 0, V, E, F, stream),
               "K1P": lambda: plan.run(x, outs["K1P"], accumulate=False)}
        for k in run:                       # one call each into zeroed outputs, compared; then warm-up
            run[k]()
        torch.cuda.synchronize()
        ref = outs["K1"].clone()
        scale = ref.abs().max().item()
        diff = {k: (outs[k] - ref).abs().max().item() / scale for k in ("K9", "K1P")}
        for k in run:
            run[k]()
        times = {k: [] for k in run}
        for _ in range(3):                 # alternated rounds of `reps` launches each
            for k in run:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    run[k]()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / reps)
        nbytes = E * F * 4 + 8 * E
        res["F%d" % F] = {k: {"ms_median": statistics.median(t), "ms_min": min(t), "ms_max": max(t),
                              "GB_per_s": nbytes / statistics.median(t) / 1e6} for k, t in times.items()}
        res["F%d" % F]["K9_over_K1"] = statistics.median(times["K9"]) / statistics.median(times["K1"])
        res["F%d" % F]["max_rel_diff_vs_K1"] = diff
        res["F%d" % F]["algorithmic_bytes"] = nbytes
        table.close()
        del plan
    return res


def worker(rank, world, args, port):
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    V, E_rand, _ = synth.WORKLOADS["reddit"]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_raw = torch.bincount(src, minlength=V)
    in_raw = torch.bincount(dst, minlength=V)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_raw.clamp(min=1), in_raw.clamp(min=1))
    E = int(pg.owned_edges)
    del src, dst
    off = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E, world).astype(np.int64)
    lo, hi = int(off[rank]), int(off[rank + 1])
    feats, labels, mask = synth.features_labels_mask(V, LAYERS[0], LAYERS[-1], dev)
    table = ShardedFeatureTable(feats[lo:hi].contiguous(), off)
    c = pg.graph_chunks[0]
    colh = c.column_offset_gpu.long()
    e0, e1 = int(colh[lo]), int(colh[hi])
    topo = ShardedTopology((colh[lo:hi + 1] - e0).to(torch.int32), c.row_indices_gpu[e0:e1].clone(),
                           c.edge_weight_forward_gpu[e0:e1].clone(), off)
    res = {"card": card(), "workload": "reddit (config B)", "V": V, "E": E, "layers": LAYERS, "fanout": FANOUT,
           "batch": BATCH, "gpus": world}
    if world == 1:
        res["kernel_whole_csc"] = kernels(pg, args.reps, dev)
    del feats, pg, colh
    torch.cuda.empty_cache()
    m = toolkits.GCNSampleImpl(topo, LAYERS, table, labels, mask.cpu(), fanout=FANOUT, batch_size=BATCH, seed=0,
                               sample_seed=0)
    for _ in range(args.epochs):
        m.run_epoch(test=False)
    res["accuracy_after_epochs"] = {"epochs": args.epochs,
                                    "evaluate_full": [m.evaluate_full(1), m.evaluate_full(2)],
                                    "evaluate_sampled": [m.evaluate(1), m.evaluate(2)]}
    wall(m.infer)                                          # warm-up of both arms
    wall(lambda: (m.evaluate(1), m.evaluate(2)))
    t_inf, t_eval = [], []
    for _ in range(args.repeats):                          # alternated
        t_inf.append(wall(m.infer)[0])
        t_eval.append(wall(lambda: (m.evaluate(1), m.evaluate(2)))[0])
    with Split() as sp:
        wall(m.infer)
    res["infer_ms"] = {"median": statistics.median(t_inf), "min": min(t_inf), "max": max(t_inf)}
    res["evaluate_1_plus_2_ms"] = {"median": statistics.median(t_eval), "min": min(t_eval), "max": max(t_eval)}
    res["evaluate_over_infer"] = statistics.median(t_eval) / statistics.median(t_inf)
    res["infer_split_ms_synchronised"] = sp.ms
    table.close()
    topo.close()
    if rank == 0:
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "infer_time.json"), "w") as f:
                f.write(line + "\n")
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < args.gpus:
        raise SystemExit("infer_time.py needs %d CUDA devices" % args.gpus)
    if args.gpus == 1:
        worker(0, 1, args, 0)
    else:
        torch.multiprocessing.spawn(worker, args=(args.gpus, args, 29770), nprocs=args.gpus, join=True)


if __name__ == "__main__":
    main()
