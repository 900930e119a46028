"""FP32 against BF16 gathers in sampled training (GCNSampleImpl(gather_dtype=...), ShardedFeatureTable(dtype=...)),
in one run on one GPU.

    python tools/sample_dtype_sweep.py [--workload reddit] [--fanout 25 10] [--batch 1024] [--epochs 5] [--warmup 2]
                                       [--gpus 1] [--out DIR]

Reports, with the card's name, power limit and SM clock read in the same run:
  * GCN epoch times on the workload's graph (602-128-41 for reddit), dropout 0, tensor features: the FP32 and the BF16
    arm alternated epoch by epoch, --warmup then --epochs timed epochs each (host clock around an epoch that ends in a
    device synchronise): median, min, max;
  * a per-step CUDA-event breakdown of one more epoch of each arm: sampling, aggregation launches by label and width
    (the BF16 arm's rounding passes included), and the rest of the step.  With tensor features the first layer reads
    the table by global id inside K1, so there is no separate table gather in the step;
  * K1 on the same sampled block, FP32 and BF16, CUDA events, median of 50 launches: the table-mode forward at the
    input width, the hidden-width forward and backward; algorithmic bytes (indices, weights, gathered rows in the
    operand's type, output read and write, offsets) and the rate derived from them; and every BF16 instantiation
    reachable at each width through NTS_K1_BF16_TUNE;
  * the deepest hop's table gather (its src) from one-shard tables: FP32 -> FP32, BF16 -> BF16, BF16 -> FP32;
  * table bytes per rank for the workload and for papers100m (config E), computed from the shapes;
  * GAT: config D's model (602-64-64-41, 8 heads, fanout 10-10-5) with an FP32 table against a BF16 table, 3 epochs
    each after one warm-up epoch;
  * accuracy: on one batch with the same weights, the per-row relative difference ||y16 - y32|| / ||y32|| of the
    last layer's output, median and max.
--gpus N > 1 would report remote bytes per step of the data-parallel rounds; that needs a multi-GPU node and is not
implemented here ("not measured").  One JSON object on stdout (and in DIR/sample_dtype_sweep.json with --out)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neutronstarlite_b200 import _lib, ops, synth  # noqa: E402
from neutronstarlite_b200.feature_table import ShardedFeatureTable  # noqa: E402
from neutronstarlite_b200.graph import PartitionedGraph  # noqa: E402
from neutronstarlite_b200.toolkits import GATSampleImpl, GCNSampleImpl  # noqa: E402

ARMS = {"fp32": None, "bf16": torch.bfloat16}
# every NTS_BF16_CASE point per chunk count (U, MINB, G); G applies to one-chunk rows only
TUNE_POINTS = {1: [(4, 2, 2), (4, 2, 1), (4, 4, 4), (4, 4, 2), (4, 4, 1), (2, 4, 4), (8, 2, 4), (4, 2, 4), (2, 4, 2), (8, 2, 2)],
               3: [(4, 2, 1), (2, 2, 1), (2, 1, 1), (4, 1, 1)]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi_name_power_sm_clock_max_sm_clock":
            q.stdout.strip().splitlines()[:1]}


class TimedSampler:
    def __init__(self, inner):
        self.inner, self.events = inner, []

    def sample(self, *a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        sg = self.inner.sample(*a)
        e1.record()
        self.events.append((e0, e1))
        return sg


def epoch(model):
    ids = model.nids[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(0, ids.numel(), model.batch_size):
        model.train_step(ids[b:b + model.batch_size])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def spread(t):
    return {"median": statistics.median(t), "min": min(t), "max": max(t), "all": t}


def events_ms(fn, n=50):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        ts.append((a, b))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ts)


def breakdown(m):
    ts = TimedSampler(m.sampler)
    m.sampler = ts
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    ids, steps = m.nids[0], []
    for b in range(0, ids.numel(), m.batch_size):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.train_step(ids[b:b + m.batch_size])
        e1.record()
        steps.append((e0, e1))
    ops.set_kernel_timer(None)
    agg = timer.summary()
    m.sampler = ts.inner
    n = len(steps)
    total = sum(a.elapsed_time(b) for a, b in steps) / n
    sampling = sum(a.elapsed_time(b) for a, b in ts.events) / n
    aggregation = sum(d["ms"] for d in agg.values()) / n
    return {"total": total, "sampling": sampling, "table_gather": 0.0, "aggregation": aggregation,
            "rest": total - sampling - aggregation,
            "aggregation_calls": {"%s F=%d" % k: {"calls_per_step": d["calls"] / n, "ms_per_step": d["ms"] / n}
                                  for k, d in agg.items()}}


def k1_bytes(n_edges, n_rows, F, esize):
    return n_edges * (4 + 4 + F * esize) + 2 * n_rows * F * 4 + 4 * (n_rows + 1)


def k1_times(sg, feats, hidden):
    """FP32 and BF16 K1 on the same blocks: table-mode forward (deepest hop), hidden forward and backward (hop 0), and a
    41-wide forward on hop 0."""
    d = feats.device
    L = len(sg.blocks)
    deep, top = sg.blocks[L - 1], sg.blocks[0]
    F0 = feats.shape[1]
    ld0 = (F0 + 7) // 8 * 8
    t16 = torch.zeros((feats.shape[0], ld0), dtype=torch.bfloat16, device=d)
    t16[:, :F0] = feats.to(torch.bfloat16)
    xh = torch.rand((top.n_src, hidden), device=d)
    gh = torch.rand((top.n_dst, hidden), device=d)
    x16 = xh.to(torch.bfloat16)            # hidden width a multiple of 8: contiguous rows are already pitched
    g16 = gh.to(torch.bfloat16)
    x41 = torch.rand((top.n_src, 41), device=d)
    x41p = torch.zeros((top.n_src, 48), dtype=torch.bfloat16, device=d)
    x41p[:, :41] = x41.to(torch.bfloat16)
    cases = {
        "fwd_table F=%d" % F0: (deep.row_global, deep.column_offset, deep.weight, deep.n_dst, deep.n_edges, F0,
                                feats, (t16, ld0)),
        "fwd F=%d" % hidden: (top.row_indices, top.column_offset, top.weight, top.n_dst, top.n_edges, hidden, xh,
                              (x16, hidden)),
        "bwd F=%d" % hidden: (top.column_indices, top.row_offset, top.weight_backward, top.n_src, top.n_edges, hidden,
                              gh, (g16, hidden)),
        "fwd F=41": (top.row_indices, top.column_offset, top.weight, top.n_dst, top.n_edges, 41, x41, (x41p, 48)),
    }
    out = {}
    for name, (idx, off, w, n_rows, n_edges, F, x32, rows16) in cases.items():
        y = torch.zeros((n_rows, F), device=d)
        r = {}
        ms32 = events_ms(lambda: ops.segment_gather_sum(y, x32, w, idx, off, 0, n_rows, n_edges))
        ms16 = events_ms(lambda: ops.segment_gather_sum_bf16(y, rows16, w, idx, off, n_rows, n_edges))
        for arm, ms, es in (("fp32", ms32, 4), ("bf16", ms16, 2)):
            b = k1_bytes(n_edges, n_rows, F, es)
            r[arm] = {"ms": ms, "alg_bytes": b, "alg_GBps": b / ms / 1e6}
        # every BF16 point reachable at this width
        k = ((F + 7) // 8 + 31) // 32
        tuned = {}
        for tp in TUNE_POINTS.get(k, []):
            os.environ["NTS_K1_BF16_TUNE"] = "%d,%d,%d" % tp
            try:
                tuned["u%d_b%d_g%d" % tp] = events_ms(
                    lambda: ops.segment_gather_sum_bf16(y, rows16, w, idx, off, n_rows, n_edges))
            except _lib.NtsError as exc:
                tuned["u%d_b%d_g%d" % tp] = str(exc)[:80]
            finally:
                del os.environ["NTS_K1_BF16_TUNE"]
        r["bf16_points_ms"] = tuned
        r["edges"], r["rows"] = int(n_edges), int(n_rows)
        out[name] = r
    return out


def table_bytes(V, F):
    return {"fp32": V * ((F + 3) // 4 * 4) * 4, "bf16": V * ((F + 7) // 8 * 8) * 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--fanout", type=int, nargs="+", default=[25, 10])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_dtype_sweep.py needs a CUDA device")
    dev = torch.device("cuda:0")
    V, E_rand, layers = synth.WORKLOADS[args.workload]
    src, dst = synth.zipf_edges(V, E_rand, dev)
    out_deg = torch.bincount(src, minlength=V).clamp(min=1)
    in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
    pg = PartitionedGraph.from_device_edges(src, dst, V, 1, 0, None, out_deg, in_deg)
    del src, dst
    feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev)
    res = {"card": card(), "workload": args.workload, "V": V, "E": int(pg.owned_edges), "layers": layers,
           "fanout": args.fanout, "batch": args.batch}

    # GCN epochs, alternated
    models = {arm: GCNSampleImpl(pg, layers, feats, labels, mask.cpu(), fanout=args.fanout, batch_size=args.batch,
                                 drop_rate=0.0, seed=0, sample_seed=0, gather_dtype=gd) for arm, gd in ARMS.items()}
    res["steps_per_epoch"] = (models["fp32"].nids[0].numel() + args.batch - 1) // args.batch
    for _ in range(args.warmup):
        for arm in ARMS:
            epoch(models[arm])
    times = {arm: [] for arm in ARMS}
    for _ in range(args.epochs):
        for arm in ARMS:
            times[arm].append(epoch(models[arm]))
    res["gcn_epoch_ms"] = {arm: spread(t) for arm, t in times.items()}
    res["gcn_per_step_ms"] = {arm: breakdown(models[arm]) for arm in ARMS}

    # accuracy on one batch with the same weights
    m32, m16 = models["fp32"], models["bf16"]
    with torch.no_grad():
        for a, b in zip(m16.P, m32.P):
            a.W.copy_(b.W)
        seeds = m32.nids[0][:args.batch]
        m32.step = m16.step = 10 ** 6
        y32, y16 = m32.Forward(seeds, False), m16.Forward(seeds, False)
        rel = (y16 - y32).norm(dim=1) / y32.norm(dim=1).clamp_min(1e-30)
    res["last_layer_rel_diff_per_row"] = {"median": float(rel.median()), "max": float(rel.max())}

    # K1 on the same sampled blocks
    sg = m32.sampler.sample(m32.nids[0][:args.batch], 0, 0)
    res["k1"] = k1_times(sg, feats, layers[1])

    # the deepest hop's table gather from one-shard tables
    t32 = ShardedFeatureTable(feats, [0, V])
    t16 = ShardedFeatureTable(feats, [0, V], dtype=torch.bfloat16)
    srcs = sg.blocks[len(sg.blocks) - 1].src
    F0 = layers[0]
    gat = {}
    for name, fn, es_in, es_out in (("fp32_to_fp32", lambda: t32._gather(srcs), 4, 4),
                                    ("bf16_to_bf16", lambda: t16._gather(srcs, torch.bfloat16), 2, 2),
                                    ("bf16_to_fp32", lambda: t16._gather(srcs, torch.float32), 2, 4)):
        ms = events_ms(fn)
        b = srcs.numel() * (F0 * (es_in + es_out) + 4)
        gat[name] = {"ms": ms, "alg_bytes": b, "alg_GBps": b / ms / 1e6}
    res["table_gather"] = dict(gat, rows=int(srcs.numel()))
    Ve, _, le = synth.WORKLOADS["papers100m"]
    res["table_bytes_per_rank"] = {args.workload + "_allocated": {"fp32": t32.local_bytes, "bf16": t16.local_bytes},
                                   args.workload + "_computed": table_bytes(V, F0),
                                   "papers100m_computed_world_1": table_bytes(Ve, le[0])}
    t32.close()
    t16.close()
    del models, m32, m16

    # GAT, config D's model, FP32 table against BF16 table
    gl = [layers[0], 64, 64, layers[-1]]
    tables = {"fp32_table": ShardedFeatureTable(feats, [0, V]),
              "bf16_table": ShardedFeatureTable(feats, [0, V], dtype=torch.bfloat16)}
    gmods = {k: GATSampleImpl(pg, gl, t, labels, mask.cpu(), fanout=[10, 10, 5], batch_size=args.batch, heads=8,
                              seed=0, sample_seed=0) for k, t in tables.items()}
    for k in gmods:
        epoch(gmods[k])
    gt = {k: [] for k in gmods}
    for _ in range(3):
        for k in gmods:
            gt[k].append(epoch(gmods[k]))
    res["gat_epoch_ms"] = {k: spread(t) for k, t in gt.items()}
    for t in tables.values():
        t.close()
    res["multi_gpu_remote_bytes_per_step"] = "not measured" if args.gpus <= 1 else "not implemented"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sample_dtype_sweep.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
