#!/usr/bin/env python3
"""FP32 vs BF16 gathers of the planned aggregation on one GPU, in one run: the Reddit-shaped graph (config B), the
products-shaped graph and the uniform graph (config B's sizes, Zipf exponent 0).

Per graph and call (forward at the first layer width, forward and backward at 128): a plan tuned per (width, type)
for each arm, then per-call CUDA-event medians (5 calls after 2 warm ones) with the two arms alternated --rounds times,
then one torch.profiler pass per arm that splits a call into conversion / padding (bf16_rows_kernel, pad_rows_kernel),
dense hub blocks (hub_block_gemm_kernel) and the residual slab launches (planned_gather_sum_kernel).  On config B also
one GCN epoch per arm (GCNImpl, single-GPU operator, median of --epochs timed epochs) and the per-row relative
difference of the last layer's output between the arms (same weights, first forward).  --tune adds (U, min CTAs/SM)
points of the BF16 kernel.  One JSON line per point, each with the card name and power limit read in this run.

    python tools/gather_dtype_sweep.py [--graphs reddit,products,uniform] [--rounds 3] [--tune] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from neutronstarlite_b200 import _lib, ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402

BF16 = torch.bfloat16
TUNE_POINTS = {602: [(4, 2), (2, 3), (6, 1)], 128: [(4, 4), (8, 2)]}   # (U, min CTAs/SM) with BF16 rows


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
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"convert_ms": 0.0, "hub_ms": 0.0, "residual_ms": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3 / reps
        if "hub_block_gemm_kernel" in ev.key:
            out["hub_ms"] += t
        elif "planned_gather_sum" in ev.key:
            out["residual_ms"] += t
        elif "bf16_rows_kernel" in ev.key or "pad_rows_kernel" in ev.key:
            out["convert_ms"] += t
    return out


def build_graph(name, dev):
    V, E, layers = synth.WORKLOADS["reddit" if name == "uniform" else name]
    src, dst = synth.zipf_edges(V, E, dev, s=0.0 if name == "uniform" else 1.0)
    out_raw = torch.bincount(src, minlength=V)
    po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E + V, 1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, po, out_raw.clamp(min=1),
                                            torch.bincount(dst, minlength=V).clamp_(min=1))
    return pg, V, layers


def sweep_calls(name, pg, V, layers, args, emit, dev):
    c = pg.graph_chunks[0]
    for direction, F in (("fwd", layers[0]), ("fwd", 128), ("bwd", 128)):
        if direction == "fwd":
            arrays = (c.column_offset_gpu, c.row_indices_gpu, c.edge_weight_forward_gpu, c.src_range[0])
        else:
            arrays = (c.row_offset_gpu, c.column_indices_gpu, c.edge_weight_backward_gpu, c.dst_range[0])
        x = torch.rand((V, F), device=dev) * 2 - 1
        y = {None: torch.zeros((V, F), device=dev), BF16: torch.zeros((V, F), device=dev)}
        plans = {t: ops.GatherPlan(*arrays, V, c.edge_size, V, 0, tune_for=F, gather_dtype=t) for t in (None, BF16)}
        calls = {t: (lambda t=t: plans[t].run(x, y[t], gather_dtype=t)) for t in (None, BF16)}
        ms = {None: [], BF16: []}
        for _ in range(args.rounds):
            for t in (None, BF16):
                ms[t].append(timed(calls[t]))
        # the same call on a BF16-stored input (no conversion pass, gathered in place when F % 8 == 0)
        xb = x.to(BF16)
        ms_bf16_in = timed(lambda: plans[BF16].run(xb, y[BF16], gather_dtype=BF16))
        parts = {t: breakdown(calls[t]) for t in (None, BF16)}
        diff = None
        y32 = plans[None].run(x, torch.zeros((V, F), device=dev))
        y16 = plans[BF16].run(x, torch.zeros((V, F), device=dev), gather_dtype=BF16)
        diff = row_rel(y16, y32)
        med = {t: float(np.median(ms[t])) for t in ms}
        for t, tag in ((None, "fp32"), (BF16, "bf16")):
            p = plans[t]
            emit({"graph": name, "dir": direction, "F": F, "gather": tag, "ms": med[t], "ms_rounds": ms[t],
                  "slabs": p.slabs, "hub_cols": p.hub_cols, "hub_rows": p.hub_rows, "build_s": p.build_s,
                  **parts[t]})
        emit({"graph": name, "dir": direction, "F": F, "gather": "bf16_vs_fp32", "ratio": med[BF16] / med[None],
              "ms_bf16_input": ms_bf16_in, "row_rel_diff_max": diff[0], "row_rel_diff_median": diff[1]})
        if args.tune and name == "reddit" and F in TUNE_POINTS:
            for u, b in TUNE_POINTS[F]:
                _lib.call("nts_gather_plan_set_tuning", u, b, 0)
                try:
                    t_ms = timed(calls[BF16])
                finally:
                    _lib.call("nts_gather_plan_set_tuning", 0, 0, 0)
                emit({"graph": name, "dir": direction, "F": F, "gather": "bf16", "tune_u": u, "tune_minb": b,
                      "ms": t_ms})
        del plans, calls, x, xb, y
        torch.cuda.empty_cache()


def row_rel(a, b):
    """max over columns of |a - b| per row over max |b| of that row: (max, median) over the rows with b != 0."""
    err = (a - b).abs().amax(1).double()
    scale = b.abs().amax(1).double()
    r = (err[scale > 0] / scale[scale > 0]).cpu().numpy()
    return (float(r.max()), float(np.median(r))) if r.size else (0.0, 0.0)


def gcn_epochs(pg, V, layers, args, emit, dev):
    from neutronstarlite_b200.toolkits import GCNImpl
    gen = torch.Generator(device=dev).manual_seed(0)
    feats = torch.rand((V, layers[0]), device=dev, generator=gen) * 2 - 1
    labels = torch.randint(0, layers[-1], (V,), device=dev, generator=gen)
    mask = torch.arange(V, device=dev) % 3
    outs = {}
    for t, tag in ((None, "fp32"), (BF16, "bf16")):
        torch.manual_seed(0)
        model = GCNImpl(pg, layers, feats.clone(), labels, mask, seed=0, gather_dtype=t)
        model.Forward()                                    # first forward with the initial weights: output compared
        outs[tag] = model.X[-1].detach().clone()
        model.ctx.tape = []
        for _ in range(args.warmup):
            model.run_epoch()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.epochs):
            t0 = time.perf_counter()
            model.run_epoch()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        emit({"graph": "reddit", "gcn_epoch": tag, "ms": float(np.median(ts)), "ms_all": ts,
              "x0_bytes": model.X[0].numel() * model.X[0].element_size()})
        del model
        torch.cuda.empty_cache()
    d = row_rel(outs["bf16"], outs["fp32"])
    emit({"graph": "reddit", "gcn_last_layer": "bf16_vs_fp32", "row_rel_diff_max": d[0], "row_rel_diff_median": d[1]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", default="reddit,products,uniform")
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the FP32 and BF16 arms (>= 3)")
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tune", action="store_true")
    ap.add_argument("--no-gcn", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gather_dtype_sweep needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    out = open(args.out, "w") if args.out else None

    def emit(d):
        s = json.dumps(dict(d, **info))
        print(s, flush=True)
        if out:
            out.write(s + "\n")
            out.flush()

    for name in args.graphs.split(","):
        pg, V, layers = build_graph(name, dev)
        sweep_calls(name, pg, V, layers, args, emit, dev)
        if name == "reddit" and not args.no_gcn:
            gcn_epochs(pg, V, layers, args, emit, dev)
        del pg
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
