#!/usr/bin/env python3
"""Per-GPU HBM budget of the distributed aggregation path for a graph shape (no GPU needed): which arrays live on a
rank, how large they are, and whether the shape fits an 80 GB H100.  Upper bounds where the exact number depends on the graph
(distinct remote sources of a rank <= V - V_p).

    python tools/plan_memory.py --V 111059956 --E 1616000000 --layers 128-128-172 --gpus 8
"""
import argparse
import json


def plan(V, E, layers, P, hbm_gb=80.0, slabs=1, n_buffers=2):
    Vp = -(-V // P)                      # vertices of a rank (balanced by the partitioner up to 1024-alignment)
    Ep = -(-(E + V) // P)                # in-edges of a rank incl. self loops (mean; skew adds up to ~1.25x at P=8)
    local = Ep // P                      # edges whose source is local (uniform estimate)
    remote = Ep - local
    Fmax = -(-max(layers[:-1]) // slabs)  # widest AGGREGATED width (GCN.hpp aggregates before the GEMM), per column slab
    mirrors = min(V - Vp, remote)        # distinct remote sources: at most all other vertices
    b = {}
    b["chunks_csc_csr"] = Ep * (4 + 4 + 4 + 4) + (Vp + 1) * 4 * (P + 1) + (V + P) * 4   # idx+w both directions, offsets
    b["per_chunk_slots_and_compact_offsets"] = remote * 4 + (mirrors + P) * 4      # what the push engine adds per chunk
    b["gather_plans_pairs_and_offsets"] = 2 * Ep * 8 + 2 * (Vp + mirrors + 2 * P) * 4   # nts_gather_plan, both directions
    b["need_and_send_lists"] = 2 * mirrors * 4
    b["features_X0"] = Vp * layers[0] * 4
    b["activations_and_grads"] = sum(Vp * f * 4 * 4 for f in layers[1:])   # Y, relu(Y W), and their gradients
    b["receive_window_per_epoch_buffer"] = mirrors * Fmax * 4     # rows pushed by the peers (x n_buffers below)
    b["backward_partials_staging"] = mirrors * Fmax * 4          # local, read by the push kernel
    b["receive_window_second_buffer"] = (n_buffers - 1) * mirrors * Fmax * 4
    total = sum(b.values())
    return {"V": V, "E": E, "layers": layers, "gpus": P, "n_buffers": n_buffers, "vertices_per_gpu": Vp, "edges_per_gpu": Ep,
            "remote_source_rows_upper_bound": mirrors, "bytes": b, "total_gb": total / 1e9,
            "fits_%dGB" % int(hbm_gb): total / 1e9 < hbm_gb * 0.9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, required=True)
    ap.add_argument("--E", type=int, required=True)
    ap.add_argument("--layers", default="128-128-172")
    ap.add_argument("--gpus", type=int, default=8)
    ap.add_argument("--slabs", type=int, default=1, help="exchange the feature columns in this many passes")
    ap.add_argument("--buffers", type=int, default=2, help="epoch buffers of the receive window (NTS_EXCHANGE_BUFFERS)")
    a = ap.parse_args()
    r = plan(a.V, a.E, [int(x) for x in a.layers.split("-")], a.gpus, slabs=a.slabs, n_buffers=a.buffers)
    r["gb"] = {k: round(v / 1e9, 2) for k, v in r.pop("bytes").items()}
    print(json.dumps(r, indent=1))


if __name__ == "__main__":
    main()
