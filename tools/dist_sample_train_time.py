"""Time data-parallel sampled training over a ShardedFeatureTable (one rank per GPU of one node).

    python tools/dist_sample_train_time.py --gpus N [--model gcn|gat] [--batch 1024] [--epochs 5] [--warmup 2]
                                           [--gather-reps 50] [--out DIR]

Workload: bench.py's config B graph (synth.WORKLOADS["reddit"], synth.zipf_edges, self loops included), replicated on
every rank as a single partition; the [V, 602] features split over the ranks by the reference's partitioner
(HostGraph-equivalent partition_offsets_from_out_degree); train ids mask == 0 (every third vertex), dropout 0, FP32.
--model gcn: layers 602-128-41, fanout 25-10 (GCNSampleImpl); --model gat: config D's model 602-64-64-41 with 8 heads,
fanout 10-10-5 (GATSampleImpl).  Rank 0 reports:
  * median and spread of the training-epoch time over --epochs timed epochs after --warmup (host clock around an epoch
    that ends in a device synchronise and a barrier);
  * a per-step CUDA-event split of one more epoch: sampling (nts_sampler), feature gather (nts_gather_rows_sharded),
    aggregation (the MiniBatchFuseOp / MiniBatchGATOp launches) and the rest (dense GEMMs, loss, tape, gradient
    all-reduce, Adam); and the gathered and remote (other ranks' shards) bytes per step;
  * with --gpus 1, a second arm alternated with the first epoch by epoch: the same toolkit with the feature tensor
    (GCN: the first layer's K1 reads the table rows in place, MiniBatchFuseOp(table=True));
  * with --gpus 1, the gather kernel against torch.index_select on the same ids (the deepest hop's src of one config B
    batch, F = 602), CUDA events over --gather-reps calls of each, alternated;
  * the card's name and power limit, read in the same run.
One JSON object on stdout (and in DIR/dist_sample_train_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402
from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl  # noqa: E402
from sample_train_time import TimedSampler, card  # noqa: E402

MODELS = {"gcn": ([602, 128, 41], [25, 10]), "gat": ([602, 64, 64, 41], [10, 10, 5])}


class TimedTable:
    """Records CUDA events around every _gather() of the wrapped table, and the rows it gathers from other ranks."""

    def __init__(self, inner):
        self.inner, self.events, self.rows, self.remote = inner, [], 0, []
        lo, hi = int(inner.offsets[inner.rank]), int(inner.offsets[inner.rank + 1])
        self.own = (lo, hi)

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def _gather(self, ids):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.inner._gather(ids)
        e1.record()
        self.events.append((e0, e1))
        self.rows += ids.numel()
        self.remote.append(((ids < self.own[0]) | (ids >= self.own[1])).sum())
        return out


def make_model(kind, pg, features, labels, mask, batch):
    layers, fanout = MODELS[kind]
    if kind == "gcn":
        return GCNSampleImpl(pg, layers, features, labels, mask, fanout=fanout, batch_size=batch, drop_rate=0.0,
                             seed=0, sample_seed=0)
    return GATSampleImpl(pg, layers, features, labels, mask, fanout=fanout, batch_size=batch, heads=8, seed=0,
                         sample_seed=0)


def epoch_ms(model, world):
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    model.run_epoch(test=False)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    return (time.perf_counter() - t0) * 1e3


def spread(t):
    return {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t}


def breakdown(model, F0):
    """One more training epoch with events around every step, sample() and table gather, and the aggregation
    launches through ops.KernelTimer."""
    ts, tt = TimedSampler(model.sampler), TimedTable(model.table)
    model.sampler, model.table = ts, tt
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    steps = []
    real = model.train_step

    def timed_step(seeds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = real(seeds)
        e1.record()
        steps.append((e0, e1))
        return r

    model.train_step = timed_step
    model.run_epoch(test=False)
    ops.set_kernel_timer(None)
    model.train_step, model.sampler, model.table = real, ts.inner, tt.inner
    torch.cuda.synchronize()
    n = max(len(steps), 1)
    ms = lambda ev: sum(a.elapsed_time(b) for a, b in ev) / n
    agg = timer.summary()
    total, sampling, gather = ms(steps), ms(ts.events), ms(tt.events)
    aggregation = sum(d["ms"] for d in agg.values()) / n
    return {"steps": len(steps), "total": total, "sampling": sampling, "feature_gather": gather,
            "aggregation": aggregation, "rest": total - sampling - gather - aggregation,
            "gathered_bytes_per_step": tt.rows * F0 * 4 / n,
            "remote_bytes_per_step": int(sum(int(r) for r in tt.remote)) * F0 * 4 / n,
            "aggregation_calls": {"%s F=%d" % k: d for k, d in agg.items()}}


def gather_vs_index_select(table, feats, src, reps):
    """CUDA-event time of nts_gather_rows_sharded and torch.index_select on the same ids, alternated."""
    idx = src.long()
    assert torch.equal(table._gather(src), feats.index_select(0, idx))
    arms = {"nts_gather_rows_sharded": lambda: table._gather(src), "torch_index_select": lambda: feats.index_select(0, idx)}
    for f in arms.values():
        for _ in range(5):
            f()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    res = {"rows": int(src.numel()), "F": int(feats.shape[1]), "reps": reps}
    for k, ev in times.items():
        t = [a.elapsed_time(b) for a, b in ev]
        res[k] = {"median_ms": statistics.median(t), "min_ms": min(t),
                  "GB_per_s_at_median": 2 * src.numel() * feats.shape[1] * 4 / statistics.median(t) / 1e6}
    return res


def run(rank, world, port, args, q):
    try:
        if world > 1:
            os.environ["MASTER_ADDR"] = "127.0.0.1"
            os.environ["MASTER_PORT"] = str(port)
            torch.cuda.set_device(rank)
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        dev = torch.device("cuda", rank)
        V, E_rand, _ = synth.WORKLOADS["reddit"]
        layers, fanout = MODELS[args.model]
        src, dst = synth.zipf_edges(V, E_rand, dev)
        out_raw = torch.bincount(src, minlength=V)
        out_deg = out_raw.clamp(min=1)
        in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
        pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_deg, in_deg)
        del src, dst
        offsets = partition_offsets_from_out_degree(out_raw.cpu().numpy(), int(pg.owned_edges), world)
        feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev)
        lo, hi = int(offsets[rank]), int(offsets[rank + 1])
        table = ShardedFeatureTable(feats[lo:hi].contiguous(), offsets)
        res = {"card": card(), "gpus": world, "model": args.model, "workload": "reddit", "V": V,
               "E": int(pg.owned_edges), "layers": layers, "fanout": fanout, "batch": args.batch,
               "table_offsets": [int(o) for o in offsets]}
        arms = {"table": make_model(args.model, pg, table, labels, mask.cpu(), args.batch)}
        if world == 1:
            arms["tensor"] = make_model(args.model, pg, feats, labels, mask.cpu(), args.batch)
        else:
            del feats
        n_batches = -(-arms["table"].nids[0].numel() // args.batch)
        res["steps_per_epoch_per_rank"] = -(-n_batches // world)
        for _ in range(args.warmup):
            for m in arms.values():
                epoch_ms(m, world)
        times = {k: [] for k in arms}
        for _ in range(args.epochs):
            for k, m in arms.items():          # alternated
                times[k].append(epoch_ms(m, world))
        for k, t in times.items():
            res["epoch_ms_" + k] = spread(t)
        res["per_step_ms_table"] = breakdown(arms["table"], layers[0])
        if world == 1:
            m = arms["table"]
            sg = m.sampler.sample(m.nids[0][:args.batch], m.sample_seed, 0)
            deep = sg.blocks[-1].src.clone()
            res["gather_kernel"] = gather_vs_index_select(table, feats, deep, args.gather_reps)
        arms.clear()
        table.close()
        q.put((rank, "ok", res))
    except Exception as exc:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL: %r\n%s" % (exc, traceback.format_exc()), None))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--model", choices=sorted(MODELS), default="gcn")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gather-reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or torch.cuda.device_count() < args.gpus:
        raise SystemExit("dist_sample_train_time.py needs %d CUDA devices" % args.gpus)
    if args.gpus == 1:
        import queue
        q = queue.Queue()
        run(0, 1, 0, args, q)
        results = [q.get()]
    else:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = 29500 + os.getpid() % 400
        procs = [ctx.Process(target=run, args=(r, args.gpus, port, args, q)) for r in range(args.gpus)]
        for p in procs:
            p.start()
        results = [q.get(timeout=3600) for _ in procs]
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    bad = [r for r in results if r[1] != "ok"]
    if bad:
        raise SystemExit("\n".join("rank %d: %s" % (r[0], r[1]) for r in bad))
    res = next(r[2] for r in results if r[0] == 0)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dist_sample_train_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
