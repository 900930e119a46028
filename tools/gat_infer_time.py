"""Time full-neighbour inference of sampled GAT (GATSampleImpl.infer) against sampled evaluation, on config B.

    python tools/gat_infer_time.py [--repeats 5] [--reps 20] [--out DIR]

Workload: bench.py's config B graph (synth.WORKLOADS["reddit"], synth.zipf_edges, self loops included) with config
D's model (602-64-64-41, 8 heads), the sampled-GAT fanout 10-10-5 and batch 1024, on one GPU (a tensor of features,
the replicated graph).  Reports, with the card's name and power limit read in the same run:
  1. infer() and evaluate(1) + evaluate(2) wall times (host clock ended by a device synchronise), alternated over
     --repeats repeats, for FP32 and BF16 gathers;
  2. K10 (nts_gat_softmax_stats_sharded + nts_gat_aggregate_sharded on a one-shard table) against K7
     (nts_gat_softmax_stats + nts_gat_fused_aggregate_forward[_bf16]) on the whole CSC, at 8 heads x 8 and 1 head x
     41, FP32 and BF16 rows: CUDA events over --reps calls, alternated round by round, and the largest difference of
     K10's output from K7's.
One JSON object on stdout (and in DIR/gat_infer_time.json with --out).  Multi-GPU times are not measured here."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from neutronstarlite_b200 import _lib, synth, toolkits  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph  # noqa: E402
from infer_time import wall  # noqa: E402
from sample_train_time import card  # noqa: E402

LAYERS, HEADS, FANOUT, BATCH = [602, 64, 64, 41], 8, [10, 10, 5], 1024


def spread(t):
    return {"median": statistics.median(t), "min": min(t), "max": max(t)}


def kernels(pg, reps, dev):
    """K10 vs K7 on the whole CSC of pg."""
    c = pg.graph_chunks[0]
    V, E = int(pg.global_vertices), int(c.edge_size)
    col, row = c.column_offset_gpu, c.row_indices_gpu
    st = torch.cuda.current_stream().cuda_stream
    res = {}
    for H, D in ((8, 8), (1, 41)):
        F = H * D
        gen = torch.Generator().manual_seed(F)
        x = (torch.rand((V, F), generator=gen) * 2 - 1).to(dev)
        s = (torch.rand((V, H), generator=gen) * 4 - 2).to(dev)
        d = (torch.rand((V, H), generator=gen) * 4 - 2).to(dev)
        scores = ShardedFeatureTable(s, [0, V])
        for dtype in (torch.float32, torch.bfloat16):
            name = "%dx%d_%s" % (H, D, "bf16" if dtype == torch.bfloat16 else "f32")
            table = ShardedFeatureTable(x, [0, V], dtype=dtype)
            ld = (F + 7) // 8 * 8
            x16 = torch.zeros((V, ld), dtype=torch.bfloat16, device=dev)
            x16[:, :F] = x.to(torch.bfloat16)
            seg = torch.empty((2, V, H), device=dev)
            # K7's BF16 forward writes rows of stride ld
            outs = {"K10": torch.zeros((V, F), device=dev),
                    "K7": torch.zeros((V, ld if dtype == torch.bfloat16 else F), device=dev)}

            def k7():
                _lib.call("nts_gat_softmax_stats", seg[0].data_ptr(), seg[1].data_ptr(), s.data_ptr(), d.data_ptr(),
                          row.data_ptr(), col.data_ptr(), None, V, H, 0.2, st)
                outs["K7"].zero_()
                if dtype == torch.bfloat16:
                    _lib.call("nts_gat_fused_aggregate_forward_bf16", x16.data_ptr(), outs["K7"].data_ptr(),
                              s.data_ptr(), d.data_ptr(), seg[0].data_ptr(), seg[1].data_ptr(), row.data_ptr(),
                              col.data_ptr(), None, V, E, F, ld, H, 0.2, st)
                else:
                    _lib.call("nts_gat_fused_aggregate_forward", x.data_ptr(), outs["K7"].data_ptr(), s.data_ptr(),
                              d.data_ptr(), seg[0].data_ptr(), seg[1].data_ptr(), row.data_ptr(), col.data_ptr(),
                              None, V, E, F, H, 0.2, st)

            def k10():
                outs["K10"].zero_()
                table.gat_aggregate(outs["K10"], scores, d, col, row, 0, E, H)

            run = {"K10": k10, "K7": k7}
            for k in run:                                   # compared once, then warmed up
                run[k]()
            torch.cuda.synchronize()
            k7 = outs["K7"][:, :F]
            scale = k7.abs().max().item()
            diff = (outs["K10"] - k7).abs().max().item() / scale
            times = {k: [] for k in run}
            for _ in range(3):                              # alternated rounds of `reps` calls each
                for k in run:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        run[k]()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) / reps)
            res[name] = {k: spread(t) for k, t in times.items()}
            res[name]["K10_over_K7"] = statistics.median(times["K10"]) / statistics.median(times["K7"])
            res[name]["max_rel_diff_vs_K7"] = diff
            table.close()
        scores.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gat_infer_time.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, E_rand, _ = synth.WORKLOADS["reddit"]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_raw = torch.bincount(src, minlength=V)
    in_raw = torch.bincount(dst, minlength=V)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_raw.clamp(min=1), in_raw.clamp(min=1))
    del src, dst
    res = {"card": card(), "workload": "reddit (config B)", "V": V, "E": int(pg.owned_edges), "layers": LAYERS,
           "heads": HEADS, "fanout": FANOUT, "batch": BATCH, "gpus": 1}
    res["kernel_whole_csc"] = kernels(pg, args.reps, dev)
    feats, labels, mask = synth.features_labels_mask(V, LAYERS[0], LAYERS[-1], dev)
    for name, gd in (("f32", None), ("bf16", torch.bfloat16)):
        m = toolkits.GATSampleImpl(pg, LAYERS, feats, labels, mask.cpu(), fanout=FANOUT, batch_size=BATCH,
                                   heads=HEADS, seed=0, sample_seed=0, gather_dtype=gd)
        wall(m.infer)                                       # warm-up of both arms
        wall(lambda: (m.evaluate(1), m.evaluate(2)))
        t_inf, t_eval = [], []
        for _ in range(args.repeats):                       # alternated
            t_inf.append(wall(m.infer)[0])
            t_eval.append(wall(lambda: (m.evaluate(1), m.evaluate(2)))[0])
        res[name] = {"infer_ms": spread(t_inf), "evaluate_1_plus_2_ms": spread(t_eval),
                     "evaluate_over_infer": statistics.median(t_eval) / statistics.median(t_inf)}
        del m
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gat_infer_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
