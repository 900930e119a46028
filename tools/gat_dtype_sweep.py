#!/usr/bin/env python3
"""FP32 vs BF16 gathers of the fused GAT layer (K7) on config D, in one run on one GPU: the Reddit-shaped graph with
the 3-layer 8-head GAT of `bench.py --toolkit gat` (602-64-64-41, fused kernel, two-pass backward).

Both arms are built in one process from the same seed.  Their last-layer outputs of the first forward (same weights)
give the largest and median per-row difference.  Then the arms are alternated --rounds times; each round times
--epochs `run_epoch` calls per arm with CUDA events (after --warmup) and keeps the median.  One more epoch per arm
under ops.KernelTimer splits the epoch into per-call times of the softmax statistics (gat_stats), the forward
(gat_fwd), the two backward passes (gat_bwd) and, in the BF16 arm, the rounding passes (gat_bf16_round), per layer
width.  --tune adds (U, virtual warps) points of the BF16 forward (NTS_GAT_BF16_TUNE) on the one-chunk rows of the
64- and 41-wide layers.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/gat_dtype_sweep.py [--rounds 3] [--epochs 5] [--tune] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gather_dtype_sweep import card, row_rel  # noqa: E402
from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.exchange import GpuExchange  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402
from neutronstarlite_b200.toolkits import GATImpl  # noqa: E402

BF16 = torch.bfloat16
ARMS = ((None, "fp32"), (BF16, "bf16"))
TUNE_POINTS = [(u, g) for g in (1, 2, 4) for u in (2, 4, 8)]   # (U, virtual warps) of the one-chunk BF16 rows


def config_d(dev, heads):
    """The graph, widths and inputs of `bench.py --toolkit gat` on one GPU."""
    V, E, layers = synth.WORKLOADS["reddit"]
    layers = [layers[0], 64, 64, layers[-1]]
    src, dst = synth.zipf_edges(V, E, dev)
    out_raw = torch.bincount(src, minlength=V)
    po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E + V, 1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, po, out_raw.clamp(min=1),
                                            torch.bincount(dst, minlength=V).clamp_(min=1))
    del src, dst
    c0 = pg.graph_chunks[0]
    pg.owned_vertices, pg.owned_edges = V, c0.edge_size
    pg.column_offset_gpu, pg.row_indices_gpu = c0.column_offset_gpu, c0.row_indices_gpu
    has_src = torch.zeros(V + 1, dtype=torch.int32, device=dev)
    ro = c0.row_offset_gpu.long()
    has_src[1:] = (ro[1:] > ro[:-1]).to(torch.int32)
    pg.mirror_index_gpu = torch.cumsum(has_src, 0).to(torch.int32)
    pg.owned_mirrors = int(pg.mirror_index_gpu[-1].item())
    feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev, rows=(0, V))
    torch.cuda.empty_cache()
    return pg, layers, feats, labels, mask


def epoch_ms(model, n):
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        model.run_epoch()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def per_call(model, epochs=1):
    """ms per call by (tag, width) over `epochs` epochs under ops.KernelTimer."""
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    try:
        for _ in range(epochs):
            model.run_epoch()
        s = timer.summary()
    finally:
        ops.set_kernel_timer(None)
    return {"%s_F%d" % (tag, F): d["ms"] / d["calls"] for (tag, F), d in sorted(s.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the FP32 and BF16 arms (>= 3)")
    ap.add_argument("--epochs", type=int, default=5, help="timed epochs per arm and round (median)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--tune", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gat_dtype_sweep needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(card(), workload="config D: reddit-shaped graph, GAT %s, %d heads, fused K7, two-pass backward")
    pg, layers, feats, labels, mask = config_d(dev, args.heads)
    res["workload"] %= ("-".join(map(str, layers)), args.heads)
    res["edges"] = int(pg.owned_edges)
    models, first = {}, {}
    for t, tag in ARMS:
        torch.manual_seed(0)
        m = GATImpl(pg, layers, feats, labels, mask, heads=args.heads, exchange=GpuExchange(pg), seed=0,
                    fused_kernel=True, two_pass_backward=True, gather_dtype=t)
        m.Forward()                               # first forward, same weights in both arms: outputs compared
        first[tag] = m.X[-1].detach().clone()
        m.ctx.tape = []
        for _ in range(args.warmup):
            m.run_epoch()
        models[tag] = m
    torch.cuda.synchronize()
    d = row_rel(first["bf16"], first["fp32"])
    res["last_layer_row_rel_diff"] = {"max": d[0], "median": d[1]}
    ms = {tag: [] for _, tag in ARMS}
    for _ in range(args.rounds):
        for _, tag in ARMS:
            ms[tag].append(epoch_ms(models[tag], args.epochs))
    for _, tag in ARMS:
        res[tag] = {"epoch_ms": float(np.median(ms[tag])), "epoch_ms_rounds": ms[tag],
                    "per_call_ms": per_call(models[tag])}
    res["epoch_ratio_bf16_vs_fp32"] = res["bf16"]["epoch_ms"] / res["fp32"]["epoch_ms"]
    if args.tune:
        tune = []
        for u, g in TUNE_POINTS:
            os.environ["NTS_GAT_BF16_TUNE"] = "%d,%d" % (u, g)
            try:
                models["bf16"].run_epoch()
                calls = per_call(models["bf16"], epochs=3)
            finally:
                del os.environ["NTS_GAT_BF16_TUNE"]
            tune.append({"u": u, "g": g, **{k: v for k, v in calls.items() if k.startswith("gat_fwd")}})
        res["tune_bf16_forward"] = tune
    s = json.dumps(res)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
