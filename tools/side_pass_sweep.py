#!/usr/bin/env python3
"""What the passes around the planned gather cost on the Reddit-shaped graph (config B) on one GPU, forward F = 602 /
128 and backward F = 128.  Four arms of the same call, alternated in one process (--rounds rounds of the CUDA-event
median of 5 calls each):

    accumulate / contiguous   zero fill of the output, out += A x on a contiguous x (F = 602: the row padding copy)
    overwrite  / contiguous   out = A x (the column block stores, or the run zeroes the output), contiguous x
    accumulate / pitched      zero fill, out += A x on x[:, :F] of a [V, 4 ceil(F/4)] tensor, gathered in place
    overwrite  / pitched      what ForwardSingleGPUfuseOp runs on GCNImpl's X[0]

At F = 128 the pitched input is the contiguous one.  The plan is measured in overwrite mode (as the single-GPU op
measures it); the counts an accumulate-mode measurement picks are reported beside it.  Then one torch.profiler pass
per arm splits the call into the hub blocks, the slab launches, the row padding and the zero fill.  One JSON line per
width and direction, with the card name and power limit read in the same run.

    python tools/side_pass_sweep.py [--rounds 3] [--out side_pass.jsonl]
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

ARMS = (("accumulate_contiguous", True, False), ("overwrite_contiguous", False, False),
        ("accumulate_pitched", True, True), ("overwrite_pitched", False, True))


def breakdown(fn, reps=3):
    """ms per call by kernel family from one profiled run."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"hub_ms": 0.0, "slab_ms": 0.0, "pad_ms": 0.0, "fill_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3 / reps
        if "hub_block_gemm_kernel" in ev.key:
            out["hub_ms"] += t
        elif "planned_slab_hub_kernel" in ev.key or "planned_gather_sum" in ev.key:
            out["slab_ms"] += t
        elif "pad_rows_kernel" in ev.key:
            out["pad_ms"] += t
        elif "fill" in ev.key.lower() or "memset" in ev.key.lower():
            out["fill_ms"] += t
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
        ld = (F + 3) // 4 * 4
        xp = torch.zeros((V, ld), device=dev)
        xp[:, :F] = x
        xp = xp[:, :F]
        y = torch.empty((V, F), device=dev)
        acc_plan = ops.GatherPlan(*arrays, V, c.edge_size, V, 0, tune_for=F)
        acc_counts = {"slabs": acc_plan.slabs, "hub_cols": acc_plan.hub_cols, "hub_rows": acc_plan.hub_rows,
                      "overlap": acc_plan.overlap}
        del acc_plan
        plan = ops.GatherPlan(*arrays, V, c.edge_size, V, 0, tune_for=F, tune_accumulate=False)
        res = {"dir": direction, "F": F, "pitch": ld, "slabs": plan.slabs, "hub_cols": plan.hub_cols,
               "hub_rows": plan.hub_rows, "overlap": plan.overlap, "build_s": plan.build_s,
               "accumulate_tuned": acc_counts}

        def call(accumulate, pitched):
            if accumulate:
                y.zero_()
            plan.run(xp if pitched else x, y, accumulate=accumulate)

        ms = {name: [] for name, _, _ in ARMS}
        for _ in range(args.rounds):
            for name, accumulate, pitched in ARMS:
                ms[name].append(timed(lambda: call(accumulate, pitched)))
        results = {}
        for name, accumulate, pitched in ARMS:
            call(accumulate, pitched)
            torch.cuda.synchronize()
            results[name] = y.clone()
            res[name] = {"ms_rounds": ms[name], "ms_median": statistics.median(ms[name]),
                         **breakdown(lambda: call(accumulate, pitched))}
        ref = results["accumulate_contiguous"]
        scale = ref.abs().amax(dim=1).clamp(min=1e-30)
        res["max_row_rel_diff"] = max(float(((r - ref).abs().amax(dim=1) / scale).max()) for r in results.values())
        s = json.dumps(dict(res, **info))
        print(s, flush=True)
        if out:
            out.write(s + "\n")
            out.flush()
        del plan, x, xp, y, results
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
