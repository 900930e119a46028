#!/usr/bin/env python3
"""The two schedules of the hub-row block on the Reddit-shaped graph (config B) on one GPU: sequential (the row block
as its own launch before the slab launches) against fused (its tiles inside the slab launches, planned_slab_hub_kernel),
forward F = 602 / 128 and backward F = 128.  Per width and direction the plan is measured as the aggregation measures
it (slab and hub counts, then the schedule), then both schedules run on that plan alternately in one process: --rounds
rounds of the CUDA-event median of 5 calls each, then one torch.profiler pass per schedule that splits the call into
the hub blocks, the residual slab launches, the fused slab launches and the row padding.  One JSON line per width and
direction, with the card name and power limit read in the same run.

    python tools/hub_overlap_sweep.py [--rounds 3] [--out hub_overlap.jsonl]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from hub_sweep import card, timed  # noqa: E402
from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402


def breakdown(fn, reps=3):
    """ms per call by kernel family from one profiled run."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"hub_ms": 0.0, "residual_ms": 0.0, "fused_ms": 0.0, "pad_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3 / reps
        if "hub_block_gemm_kernel" in ev.key:
            out["hub_ms"] += t
        elif "planned_slab_hub_kernel" in ev.key:
            out["fused_ms"] += t
        elif "planned_gather_sum" in ev.key:
            out["residual_ms"] += t
        elif "pad_rows_kernel" in ev.key:
            out["pad_ms"] += t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    V, E_rand, layers = synth.WORKLOADS["reddit"]
    info = card()
    out = open(args.out, "w") if args.out else None

    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_raw = torch.bincount(src, minlength=V)
    po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E_rand + V, 1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, po, out_raw.clamp(min=1),
                                            torch.bincount(dst, minlength=V).clamp_(min=1))
    del src, dst
    c = pg.graph_chunks[0]
    for direction, F in (("fwd", layers[0]), ("fwd", layers[1]), ("bwd", layers[1])):
        if direction == "fwd":
            arrays = (c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, c.src_range[0])
        else:
            arrays = (c.row_offset_gpu, c.column_indices_gpu, c.edge_weight_backward_gpu, c.dst_range[0])
        x = torch.rand((V, F), device=dev) * 2 - 1
        y = torch.zeros((V, F), device=dev)
        plan = ops.GatherPlan(*arrays, V, c.edge_size, V, 0, tune_for=F)
        chosen = plan.overlap
        res = {"dir": direction, "F": F, "slabs": plan.slabs, "hub_cols": plan.hub_cols, "hub_rows": plan.hub_rows,
               "tuned_overlap": chosen, "build_s": plan.build_s}
        if plan.hub_rows:
            ms = {"sequential": [], "fused": []}
            for _ in range(args.rounds):
                for name, ov in (("sequential", False), ("fused", True)):
                    plan.set_overlap(ov)
                    ms[name].append(timed(lambda: plan.run(x, y)))
            for name, ov in (("sequential", False), ("fused", True)):
                plan.set_overlap(ov)
                res[name] = {"ms_rounds": ms[name], "ms_median": statistics.median(ms[name]),
                             **breakdown(lambda: plan.run(x, y))}
            plan.set_overlap(chosen)
        else:
            res["sequential"] = {"ms_median": timed(lambda: plan.run(x, y)), **breakdown(lambda: plan.run(x, y))}
        s = json.dumps(dict(res, **info))
        print(s, flush=True)
        if out:
            out.write(s + "\n")
            out.flush()
        del plan, x, y
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
