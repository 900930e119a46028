#!/usr/bin/env python3
"""Sweep of the planned aggregation with dense hub blocks on the Reddit-shaped graph (config B) on one GPU: forced
(slabs, hub columns, hub rows) points and the measured pick, forward F = 602 / 128 and backward F = 128.  Per point:
the call's CUDA-event time (median of 5 after 2 warm launches), then one torch.profiler pass that splits it into the
dense blocks (hub_block_gemm_kernel: achieved TFLOP/s from 2 * rows * K * ld flops against the 67 TFLOP/s FP32 data
sheet figure of the H100 SXM), the residual slab launches and the row padding.  One JSON line per point, each with
the card name and power limit.

    python tools/hub_sweep.py [--points 4:0:0,4:128:128,...] [--out hub_sweep.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from neutronstarlite_b200 import ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402

FP32_PEAK_TFLOPS = 67.0
DEFAULT_POINTS = "4:0:0,4:64:0,4:128:0,4:256:0,4:128:64,4:128:128,4:128:256,2:128:128,1:128:128,tuned"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception:  # noqa: BLE001 - the card name from torch is still worth reporting
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def timed(fn, warm=2, reps=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def breakdown(fn, reps=3):
    """ms per call by kernel family from one profiled run."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"dense_ms": 0.0, "residual_ms": 0.0, "pad_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3 / reps
        if "hub_block_gemm_kernel" in ev.key:
            out["dense_ms"] += t
        elif "planned_gather_sum" in ev.key:
            out["residual_ms"] += t
        elif "pad_rows_kernel" in ev.key:
            out["pad_ms"] += t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", default=DEFAULT_POINTS, help="comma list of slabs:hub_cols:hub_rows, or 'tuned'")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    V, E_rand, layers = synth.WORKLOADS["reddit"]
    info = card()
    out = open(args.out, "w") if args.out else None

    def emit(d):
        s = json.dumps(dict(d, **info))
        print(s, flush=True)
        if out:
            out.write(s + "\n")
            out.flush()

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
        ld = (F + 3) // 4 * 4
        for p in args.points.split(","):
            if p == "tuned":
                plan = ops.GatherPlan(*arrays, V, c.edge_size, V, 0, tune_for=F)
            else:
                s, hc, hr = (int(v) for v in p.split(":"))
                plan = ops.GatherPlan(*arrays, V, c.edge_size, V, s, hubs=(hc, hr))
            ms = timed(lambda: plan.run(x, y))
            parts = breakdown(lambda: plan.run(x, y))
            flops = 2.0 * ld * (V * plan.hub_cols + plan.hub_rows * V)
            tflops = flops / (parts["dense_ms"] * 1e-3) / 1e12 if parts["dense_ms"] > 0 else None
            emit({"dir": direction, "F": F, "point": p, "slabs": plan.slabs, "hub_cols": plan.hub_cols,
                  "hub_rows": plan.hub_rows, "ms": ms, "build_s": plan.build_s, "plan_bytes": plan.bytes(),
                  "dense_tflops": tflops, "dense_frac_of_fp32_peak": tflops / FP32_PEAK_TFLOPS if tflops else None,
                  **parts})
            del plan
            torch.cuda.empty_cache()
        del x, y


if __name__ == "__main__":
    main()
