#!/usr/bin/env python3
"""Sweep of the aggregation kernels on the Reddit-shaped graph (config B) on one GPU: the plain kernel on the reference
layout vs nts_gather_plan at several slab counts and (U, min CTAs/SM) points, Zipf and uniform endpoints, forward
(F = 602, 128) and backward (F = 128).  CUDA events, 2 warm + 5 timed launches each (inputs >> L2).  One JSON line
per point on stdout / --out.

    python tools/k1_sweep.py [--quick] [--out k1_sweep.jsonl]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from neutronstarlite_b200 import _lib, ops, synth  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402


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
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--tma", action="store_true", help="also time variant 1 (TMA row staging)")
    ap.add_argument("--slabs", default=None, help="comma list of slab counts to try (default: 1, auto, 2, 4, 8, 16, 24)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    L = _lib.load()
    V, E_rand, layers = synth.WORKLOADS[args.workload]
    out = open(args.out, "w") if args.out else None

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        if out:
            out.write(s + "\n")
            out.flush()

    for zipf in ((1.0,) if args.quick else (1.0, 0.0)):
        src, dst = synth.zipf_edges(V, E_rand, dev, s=zipf)
        out_raw = torch.bincount(src, minlength=V)
        po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E_rand + V, 1)
        pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, po, out_raw.clamp(min=1),
                                                torch.bincount(dst, minlength=V).clamp_(min=1))
        del src, dst
        c = pg.graph_chunks[0]
        for direction, F in (("fwd", layers[0]), ("fwd", layers[1]), ("bwd", layers[1])):
            x = torch.rand((V, F), device=dev) * 2 - 1
            y = torch.zeros((V, F), device=dev)
            call = ops.gather_by_dst_from_src if direction == "fwd" else ops.gather_by_src_from_dst
            ops.set_plan_mode("off")
            med, best = timed(lambda: call(c, y, x))
            ref = torch.zeros_like(y)
            call(c, ref, x)
            emit({"zipf": zipf, "dir": direction, "F": F, "kernel": "plain", "ms": med, "ms_best": best})
            auto = int(L.nts_gather_plan_pick_slabs(V, c.edge_size, V, F, 0))
            c.__dict__.pop("_gather_plan_for", None)
            slab_list = sorted(set([1, auto] + ([] if args.quick else [2, 4, 8, 16, 24])))
            if args.slabs:
                slab_list = sorted(set(int(v) for v in args.slabs.split(",")))
                auto = slab_list[-1]
            for S in slab_list:
                ops.set_plan_mode("on", S)
                pts = [(0, 0)]
                if not args.quick and S in (1, auto):
                    pts += [(1, 3), (2, 3), (4, 2), (4, 1)] if F > 512 else [(8, 4), (8, 3), (16, 2)]
                for (u, b) in pts:
                    _lib.call("nts_gather_plan_set_tuning", u, b, 0)
                    try:
                        med, best = timed(lambda: call(c, y, x))
                    except Exception as exc:  # no instantiation for this point
                        emit({"zipf": zipf, "dir": direction, "F": F, "kernel": "plan", "slabs": S, "u": u, "minb": b,
                              "error": str(exc)[:80]})
                        continue
                    chk = torch.zeros_like(y)
                    call(c, chk, x)
                    torch.cuda.synchronize()
                    err = float(((chk - ref).abs().max(dim=1).values /
                                 ref.abs().max(dim=1).values.clamp(min=1e-30)).max().item())
                    emit({"zipf": zipf, "dir": direction, "F": F, "kernel": "plan", "slabs": S, "u": u, "minb": b,
                          "ms": med, "ms_best": best, "max_row_rel_diff_vs_plain": err})
                _lib.call("nts_gather_plan_set_tuning", 0, 0, 0)
                if args.tma and S in (1, auto):   # variant 1: rows staged in shared memory by per-row TMA copies
                    _lib.call("nts_gather_plan_set_variant", 1)
                    for (u, b) in ([(2, 2), (4, 2), (4, 1), (8, 1)] if F > 512 else [(4, 4), (8, 4), (8, 3)]):
                        _lib.call("nts_gather_plan_set_tuning", u, b, 0)
                        try:
                            med, best = timed(lambda: call(c, y, x))
                            chk = torch.zeros_like(y)
                            call(c, chk, x)
                            torch.cuda.synchronize()
                            err = float(((chk - ref).abs().max(dim=1).values /
                                         ref.abs().max(dim=1).values.clamp(min=1e-30)).max().item())
                            emit({"zipf": zipf, "dir": direction, "F": F, "kernel": "plan_tma_rows", "slabs": S,
                                  "stages": u, "minb": b, "ms": med, "ms_best": best,
                                  "max_row_rel_diff_vs_plain": err})
                        except Exception as exc:
                            emit({"zipf": zipf, "dir": direction, "F": F, "kernel": "plan_tma_rows", "slabs": S,
                                  "stages": u, "minb": b, "error": str(exc)[:80]})
                    _lib.call("nts_gather_plan_set_variant", 0)
                    _lib.call("nts_gather_plan_set_tuning", 0, 0, 0)
                c.__dict__.pop("_gather_plans", None)   # free this slab count's arrays before the next
                torch.cuda.empty_cache()
            ops.set_plan_mode("auto")
            del x, y, ref
        del pg, c
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
