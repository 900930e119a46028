"""Time neighbour-sampled mini-batch GCN training (toolkits.GCNSampleImpl) on one GPU.

    python tools/sample_train_time.py [--workload reddit] [--fanout 25 10] [--batch 1024] [--epochs 5] [--warmup 2]
                                      [--out DIR]

Workload: bench.py's graph for the workload (synth.zipf_edges, self loops included), layers of the workload
(602-128-41 for reddit), train ids mask == 0 (every third vertex), FP32.  Reports:
  * median and spread of the training-epoch time over --epochs timed epochs after --warmup (host clock around an epoch
    that ends in a device synchronise);
  * a per-step CUDA-event breakdown of one more epoch: sampling (nts_sampler), aggregation (the MiniBatchFuseOp K1
    launches, forward and backward) and the rest of the step (dense GEMMs, loss, tape, Adam);
  * the algorithmic gather bytes of the deepest hop's table gather (K1's B_alg on that block) per step;
  * a torch-only arm of the same step, alternated with ours epoch by epoch: the same sampled edges, deduplicated with
    torch.unique, aggregated with index_select + index_add_ (autograd for the backward), the same dense layers and
    Adam kernel;
  * the card's name and power limit, read in the same run.
One JSON object on stdout (and in DIR/sample_train_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph  # noqa: E402
from neutronstarlite_b200.toolkits import GCNSampleImpl  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


class TimedSampler:
    """Records CUDA events around every sample() of the wrapped sampler."""

    def __init__(self, inner):
        self.inner, self.events = inner, []

    def sample(self, *a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sg = self.inner.sample(*a)
        e1.record()
        self.events.append((e0, e1))
        return sg


def torch_step(model, seeds):
    """The same step with torch doing the dedupe and the aggregation (sampling selection by nts_sampler)."""
    for p in model.P:
        p.zero_grad()
    sg = model.sampler.sample(seeds, model.sample_seed, model.step)
    model.step += 1
    L = len(model.layers) - 1
    x = model.features
    for l in range(L):
        b = sg.blocks[L - 1 - l]
        n = b.n_dst
        e_dst = torch.repeat_interleave(torch.arange(n, device=x.device), b.column_offset.diff())
        if l == 0:
            rows = x.index_select(0, b.row_global.long())
        else:
            _, inv = torch.unique(b.row_global, return_inverse=True)
            rows = x.index_select(0, inv)
        y = torch.zeros((n, x.shape[1]), dtype=x.dtype, device=x.device).index_add_(0, e_dst, rows * b.weight[:, None])
        x = model.P[l].forward(y)
        if l < L - 1:
            x = torch.relu(x)
    loss = torch.nn.functional.nll_loss(x.log_softmax(1), model.L_GT.index_select(0, sg.seeds().long()))
    loss.backward()
    model.Update()
    return loss.detach()


def epoch(model, arm):
    ids = model.nids[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, ids.numel(), model.batch_size):
        if arm == "nts":
            model.train_step(ids[b:b + model.batch_size])
        else:
            torch_step(model, ids[b:b + model.batch_size])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--fanout", type=int, nargs="+", default=[25, 10])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_train_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, E_rand, layers = synth.WORKLOADS[args.workload]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_deg = torch.bincount(src, minlength=V).clamp(min=1)
    in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_deg, in_deg)
    del src, dst
    feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev)
    res = {"card": card(), "workload": args.workload, "V": V, "E": int(pg.owned_edges), "layers": layers,
           "fanout": args.fanout, "batch": args.batch}

    models = {arm: GCNSampleImpl(pg, layers, feats, labels, mask.cpu(), fanout=args.fanout, batch_size=args.batch,
                                 drop_rate=0.0, seed=0, sample_seed=0) for arm in ("nts", "torch")}
    res["steps_per_epoch"] = (models["nts"].nids[0].numel() + args.batch - 1) // args.batch
    res["sampler_bytes"] = models["nts"].sampler.bytes()
    for _ in range(args.warmup):
        for arm in ("nts", "torch"):
            epoch(models[arm], arm)
    times = {"nts": [], "torch": []}
    for _ in range(args.epochs):
        for arm in ("nts", "torch"):           # alternated
            times[arm].append(epoch(models[arm], arm))
    for arm in ("nts", "torch"):
        t = times[arm]
        res["epoch_ms_" + arm] = {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t}

    # breakdown epoch (ours): events around the sampler and every aggregation launch
    m = models["nts"]
    ts = TimedSampler(m.sampler)
    m.sampler = ts
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    deep_bytes, deep_edges, step_ms = [], [], []
    ids = m.nids[0]
    L = len(layers) - 1
    F0 = layers[0]
    for b in range(0, ids.numel(), m.batch_size):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.train_step(ids[b:b + m.batch_size])
        e1.record()
        step_ms.append((e0, e1))
        blk = m.subgraph.blocks[L - 1]
        deep_edges.append(blk.n_edges)
        deep_bytes.append(blk.n_edges * (4 + 4 + 4 * F0) + blk.n_dst * 4 * F0 + 4 * (blk.n_dst + 1))
    ops.set_kernel_timer(None)
    agg = timer.summary()
    torch.cuda.synchronize()
    n = len(step_ms)
    total = sum(a.elapsed_time(b) for a, b in step_ms) / n
    sampling = sum(a.elapsed_time(b) for a, b in ts.events) / n
    aggregation = sum(d["ms"] for d in agg.values()) / n
    res["per_step_ms"] = {"total": total, "sampling": sampling, "aggregation": aggregation,
                          "dense_loss_tape_adam": total - sampling - aggregation,
                          "aggregation_calls": {"%s F=%d" % k: d for k, d in agg.items()}}
    res["deepest_hop"] = {"edges_per_step": sum(deep_edges) / n, "gather_bytes_per_step": sum(deep_bytes) / n}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sample_train_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
