"""Time sampled GCN training on a learnable vertex embedding (feature_table.ShardedEmbedding) against the same model
on a frozen table (feature_table.ShardedFeatureTable) of the same width and initial rows, on one GPU.

    python tools/embedding_train_time.py [--workload reddit] [--width 128] [--fanout 25 10] [--batch 1024]
                                         [--epochs 5] [--warmup 2] [--reps 50] [--out DIR]

Workload: tools/sample_train_time.py's graph and labels for the workload (config B: reddit), GCNSampleImpl with layers
[width, 128, classes], drop_rate 0, train ids mask == 0.  The two arms alternate epoch by epoch in one run.  Reports:
  * median and spread of the training-epoch time of each arm (host clock around an epoch that ends in a device
    synchronise);
  * the embedding step per round (ShardedEmbedding._step: outbox write, fences, K11) from CUDA events over one more
    epoch, and the touched rows per round;
  * K11 alone (nts_embedding_step) replayed --reps times on the last round's outbox, with its achieved bytes/s from
    (6 + contributors) * 4 * width bytes per touched row (read and write the row, M and V; read each contributor's
    gradient row; one contributor at one rank) against the H100 SXM data sheet's 3.35 TB/s;
  * the card's name and power limit, read in the same run.
One JSON object on stdout (and in DIR/embedding_train_time.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from neutronstarlite_b200 import _lib, synth  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedEmbedding, ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph  # noqa: E402
from neutronstarlite_b200.toolkits import GCNSampleImpl  # noqa: E402
from sample_train_time import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def epoch(model):
    ids = model.nids[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, ids.numel(), model.batch_size):
        model.train_step(ids[b:b + model.batch_size])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def k11_replay(t, reps):
    """ms per nts_embedding_step call on the outbox as the last step left it (it updates the rows each time)."""
    lo, hi = (int(o) for o in t.offsets[t.rank:t.rank + 2])

    def run():
        _lib.call("nts_embedding_step", t._buf, t.M.data_ptr(), t.V.data_ptr(), t._mask.data_ptr(),
                  t._positions.data_ptr(), t._touched.data_ptr(), t._outboxes.data_ptr(), t.world, t.capacity, lo,
                  hi, t.pitch, t.F, float(t.weight_decay), float(t.beta1), float(t.beta2), float(t.alpha),
                  float(t.epsilon), _lib.stream())
    for _ in range(3):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--fanout", type=int, nargs="+", default=[25, 10])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("embedding_train_time.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, E_rand, layers = synth.WORKLOADS[args.workload]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_deg = torch.bincount(src, minlength=V).clamp(min=1)
    in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_deg, in_deg)
    del src, dst
    layers = [args.width] + list(layers[1:])
    init, labels, mask = synth.features_labels_mask(V, args.width, layers[-1], dev)
    res = {"card": card(), "workload": args.workload, "V": V, "E": int(pg.owned_edges), "layers": layers,
           "fanout": args.fanout, "batch": args.batch}
    tables = {"learnable": ShardedEmbedding(init, [0, V]), "frozen": ShardedFeatureTable(init, [0, V])}
    models = {arm: GCNSampleImpl(pg, layers, tables[arm], labels, mask.cpu(), fanout=args.fanout,
                                 batch_size=args.batch, drop_rate=0.0, seed=0, sample_seed=0) for arm in tables}
    res["steps_per_epoch"] = (models["frozen"].nids[0].numel() + args.batch - 1) // args.batch
    for _ in range(args.warmup):
        for arm in models:
            epoch(models[arm])
    times = {arm: [] for arm in models}
    for _ in range(args.epochs):
        for arm in models:                      # alternated
            times[arm].append(epoch(models[arm]))
    for arm, t in times.items():
        res["epoch_ms_" + arm] = {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t}

    # one more epoch of the learnable arm: CUDA events around every embedding step, and the rows it touched
    t = tables["learnable"]
    events, rows = [], []
    step = t._step

    def timed_step(ids, grad):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(ids, grad)
        e1.record()
        events.append((e0, e1))
        rows.append(int(ids.numel()))
    t._step = timed_step
    epoch(models["learnable"])
    t._step = step
    ms = [a.elapsed_time(b) for a, b in events]
    res["embedding_step_ms_per_round"] = {"median": statistics.median(ms), "mean": sum(ms) / len(ms),
                                          "min": min(ms), "max": max(ms)}
    res["touched_rows_per_round"] = {"mean": sum(rows) / len(rows), "min": min(rows), "max": max(rows)}
    last = rows[-1]
    k11_ms = k11_replay(t, args.reps)
    k11_bytes = (6 + 1) * 4 * args.width * last
    res["k11_replay"] = {"touched_rows": last, "ms": k11_ms, "bytes": k11_bytes,
                         "bytes_per_s": k11_bytes / (k11_ms * 1e-3),
                         "share_of_3_35_TBps": k11_bytes / (k11_ms * 1e-3) / HBM_BYTES_PER_S}
    res["card_after"] = card()
    for tab in tables.values():
        tab.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "embedding_train_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
