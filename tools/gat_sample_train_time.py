"""Time neighbour-sampled mini-batch GAT training (toolkits.GATSampleImpl) on one GPU.

    python tools/gat_sample_train_time.py [--workload reddit] [--fanout 10 10 5] [--batch 1024] [--heads 8]
                                          [--epochs 3] [--warmup 1] [--out DIR]

Workload: bench.py's graph for the workload (synth.zipf_edges, self loops included) with config D's model on it
(602-64-64-41 for reddit: two hidden layers of 8 heads x 8 and a single-head output layer), train ids mask == 0 (every
third vertex).  Three hops at fanout 10 reach nearly all of the config B graph's vertices, so the default fanout
narrows the deeper hops; the per-hop block sizes of the chosen fanout are reported.  Reports:
  * median and spread of the training-epoch time over --epochs timed epochs after --warmup (host clock around an epoch
    that ends in a device synchronise), FP32 and BF16 gathers alternated epoch by epoch, and the per-step time;
  * a per-step CUDA-event breakdown of one more epoch of each arm: sampling (nts_sampler), the K7 launches
    (statistics, forward, BF16 rounding, two-pass backward through ops.KernelTimer) and the rest of the step (feature
    gather, dense GEMMs, scores, loss, tape, Adam);
  * the sampler alone with and without include_dst on the same seeds and (seed, step), alternated;
  * mean n_dst / n_src / n_edges of every hop over the breakdown epoch;
  * the card's name and power limit, read in the same run.
One JSON object on stdout (and in DIR/gat_sample_train_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph  # noqa: E402
from neutronstarlite_b200.sample import NeighborSampler  # noqa: E402
from neutronstarlite_b200.toolkits import GATSampleImpl  # noqa: E402
from sample_train_time import TimedSampler, card  # noqa: E402

ARMS = {"fp32": None, "bf16": torch.bfloat16}


def epoch(model):
    ids = model.nids[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, ids.numel(), model.batch_size):
        model.train_step(ids[b:b + model.batch_size])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def breakdown(model, n_hops):
    """One epoch with CUDA events around every step, every sample() and every K7 launch."""
    ts = TimedSampler(model.sampler)
    model.sampler = ts
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    ids = model.nids[0]
    steps, sizes = [], [[0, 0, 0] for _ in range(n_hops)]
    for b in range(0, ids.numel(), model.batch_size):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        model.train_step(ids[b:b + model.batch_size])
        e1.record()
        steps.append((e0, e1))
        for h, blk in enumerate(model.subgraph.blocks):
            sizes[h][0] += blk.n_dst
            sizes[h][1] += blk.n_src
            sizes[h][2] += blk.n_edges
    ops.set_kernel_timer(None)
    model.sampler = ts.inner
    k7 = timer.summary()
    torch.cuda.synchronize()
    n = len(steps)
    total = sum(a.elapsed_time(b) for a, b in steps) / n
    sampling = sum(a.elapsed_time(b) for a, b in ts.events) / n
    k7_ms = sum(d["ms"] for d in k7.values()) / n
    per_tag = {}
    for (tag, F), d in k7.items():
        per_tag[tag] = per_tag.get(tag, 0.0) + d["ms"] / n
    return ({"total": total, "sampling": sampling, "k7": k7_ms, "rest": total - sampling - k7_ms, "k7_by_kind": per_tag,
             "k7_calls": {"%s F=%d" % k: {"calls": d["calls"], "ms": d["ms"]} for k, d in k7.items()}},
            [{"n_dst": s[0] / n, "n_src": s[1] / n, "n_edges": s[2] / n} for s in sizes])


def sampler_cost(pg, fanout, batch, ids, rounds):
    """Median per-epoch time of the sampler alone, default vs include_dst, on the same seeds and (seed, step)."""
    samplers = {"default": NeighborSampler(pg, fanout, batch), "include_dst": NeighborSampler(pg, fanout, batch,
                                                                                            include_dst=True)}
    times = {k: [] for k in samplers}
    for r in range(rounds + 1):
        for k, s in samplers.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i, b in enumerate(range(0, ids.numel(), batch)):
                s.sample(ids[b:b + batch], 0, i)
            torch.cuda.synchronize()
            if r:                                        # round 0 warms up
                times[k].append((time.perf_counter() - t0) * 1e3)
    steps = (ids.numel() + batch - 1) // batch
    return {k: {"epoch_ms_median": statistics.median(t), "per_step_ms": statistics.median(t) / steps,
                "bytes": samplers[k].bytes()} for k, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--fanout", type=int, nargs="+", default=[10, 10, 5])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--layers", type=int, nargs="+", default=None, help="default: 602-64-64-41 (config D)")
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gat_sample_train_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, E_rand, wl_layers = synth.WORKLOADS[args.workload]
    layers = args.layers or [wl_layers[0], 64, 64, wl_layers[-1]]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_deg = torch.bincount(src, minlength=V).clamp(min=1)
    in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_deg, in_deg)
    del src, dst
    feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev)
    res = {"card": card(), "workload": args.workload, "V": V, "E": int(pg.owned_edges), "layers": layers,
           "heads": args.heads, "fanout": args.fanout, "batch": args.batch}
    models = {arm: GATSampleImpl(pg, layers, feats, labels, mask.cpu(), fanout=args.fanout, batch_size=args.batch,
                                 heads=args.heads, seed=0, sample_seed=0, gather_dtype=g) for arm, g in ARMS.items()}
    steps = (models["fp32"].nids[0].numel() + args.batch - 1) // args.batch
    res["steps_per_epoch"] = steps
    for _ in range(args.warmup):
        for arm in ARMS:
            epoch(models[arm])
    times = {arm: [] for arm in ARMS}
    for _ in range(args.epochs):
        for arm in ARMS:                       # alternated
            times[arm].append(epoch(models[arm]))
    for arm in ARMS:
        t = times[arm]
        res["epoch_ms_" + arm] = {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t,
                                  "per_step": statistics.median(t) / steps}
    for arm in ARMS:
        res["per_step_ms_" + arm], hops = breakdown(models[arm], len(args.fanout))
    res["hops"] = hops
    res["sampler"] = sampler_cost(pg, args.fanout, args.batch, models["fp32"].nids[0], max(args.epochs, 3))
    res["loss_last_epoch"] = {arm: float(models[arm].loss.detach()) for arm in ARMS}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gat_sample_train_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
