"""Time the three chunk builders on one GPU for one rank of the bench.py workload.

    python tools/graph_build_time.py --out DIR [--workload reddit] [--partitions 1 8] [--rank 0]
                                     [--block-edges 67108864] [--host-budget-edges 2e9]

Writes the workload's edges (bench.py's generator, same seeds, self loops included) as a packed {u32 src, u32 dst}
file under DIR, then times, for rank r of each P:
  * PartitionedGraph.from_edge_file (streaming reader + device kernels), after one warm-up build;
  * PartitionedGraph.from_device_edges on the same edges as int64 device tensors (the call bench.py makes), after one
    warm-up build;
  * the host builder (HostGraph + generate_all(dist=True)) once, when edges x P stays under --host-budget-edges.
Reports per-pass seconds, the builder's peak device scratch and its bytes per owned edge, the torch allocator peak,
the cudaMemGetInfo drop across the build, and the card name and power limit read in the same run.  The file has
just been written, so its reads come from the page cache; a cold read from storage is not measured.  The edge file is
removed at the end; the report lands in DIR/graph_build_time.json.
`--workload papers100m --partitions 8 --rank 0` models one GPU's share of config E (a 6.5 GB file)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neutronstarlite_b200 import synth  # noqa: E402
from neutronstarlite_b200.graph import HostGraph, PartitionedGraph, partition_offsets_from_out_degree  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def write_edge_file(path, V, E_rand, dev):
    """bench.py's edges in bench.py's order (synth.zipf_edges: the random stream, then one self loop per vertex)."""
    with open(path, "wb") as f:
        for src, dst in synth._zipf_stream(V, E_rand, dev, 1.0, synth.SEED_GRAPH, 1 << 26):
            np.stack([src.to(torch.int32).cpu().numpy(), dst.to(torch.int32).cpu().numpy()], 1).astype(np.uint32).tofile(f)
        loops = np.arange(V, dtype=np.uint32)
        np.stack([loops, loops], 1).tofile(f)


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    pg = fn()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    free1 = torch.cuda.mem_get_info()[0]
    st = getattr(pg, "build_stats", None) or {}
    owned = max(pg.owned_edges, 1)
    res = {"seconds": dt, "owned_edges": pg.owned_edges, "owned_vertices": pg.owned_vertices,
           "torch_peak_allocated_bytes": torch.cuda.max_memory_allocated(),
           "mem_get_info_drop_bytes": free0 - free1}
    if st:
        res["pass_seconds"] = st["seconds"]
        res["scratch_peak_bytes"] = st["scratch_peak_bytes"]
        res["scratch_bytes_per_owned_edge"] = st["scratch_peak_bytes"] / owned
        res["scratch_bound_bytes"] = 40 * pg.owned_edges + 16 * pg.global_vertices
    return pg, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--partitions", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--rank", type=int, default=0)
    ap.add_argument("--block-edges", type=int, default=1 << 26)
    ap.add_argument("--host-budget-edges", type=float, default=2e9,
                    help="run the host builder only when edges x partitions stays below this")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_build_time.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    V, E_rand, _ = synth.WORKLOADS[args.workload]
    E = E_rand + V
    path = os.path.join(args.out, "%s.edges" % args.workload)
    t0 = time.perf_counter()
    write_edge_file(path, V, E_rand, dev)
    torch.cuda.empty_cache()
    report = {"workload": args.workload, "vertices": V, "edges": E, "file_bytes": os.path.getsize(path),
              "write_seconds": time.perf_counter() - t0, "block_edges": args.block_edges, "card": card(),
              "note": "the edge file was just written: its reads come from the page cache (cold reads not measured)",
              "runs": []}
    for P in args.partitions:
        r = args.rank
        run = {"partitions": P, "rank": r}
        build = lambda: PartitionedGraph.from_edge_file(path, V, P, r, device=dev, block_edges=args.block_edges)
        build()
        torch.cuda.empty_cache()
        pg, run["from_edge_file"] = timed(build)
        po = pg.partition_offset
        del pg
        torch.cuda.empty_cache()
        # bench.py's call: all edges as int64 device tensors, int64 clamped degrees, given offsets
        raw = np.fromfile(path, dtype=np.uint32).reshape(-1, 2)
        src = torch.from_numpy(raw[:, 0].astype(np.int64)).to(dev)
        dst = torch.from_numpy(raw[:, 1].astype(np.int64)).to(dev)
        out_raw = torch.bincount(src, minlength=V)
        in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
        assert np.array_equal(partition_offsets_from_out_degree(out_raw.cpu().numpy(), E, P), po)
        out_deg = out_raw.clamp(min=1)
        dbuild = lambda: PartitionedGraph.from_device_edges(src, dst, V, P, r, po, out_deg, in_deg)
        dbuild()
        torch.cuda.empty_cache()
        pg, run["from_device_edges"] = timed(dbuild)
        del pg, src, dst, out_raw, out_deg, in_deg
        torch.cuda.empty_cache()
        if E * P <= args.host_budget_edges:
            t0 = time.perf_counter()
            hg = HostGraph(raw, V)
            hpg = PartitionedGraph(hg, P, r).generate_all(dist=True)
            run["host_builder"] = {"seconds": time.perf_counter() - t0, "owned_edges": hpg.owned_edges,
                                   "runs": "one run, no warm-up"}
            del hg, hpg
        else:
            run["host_builder"] = "not measured (edges x partitions over --host-budget-edges)"
        del raw
        report["runs"].append(run)
        print(json.dumps(run), flush=True)
    with open(os.path.join(args.out, "graph_build_time.json"), "w") as f:
        json.dump(report, f, indent=1)
    os.remove(path)
    print(json.dumps({k: report[k] for k in ("workload", "vertices", "edges", "file_bytes", "card", "note")}))


if __name__ == "__main__":
    main()
