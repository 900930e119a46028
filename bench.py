#!/usr/bin/env python3
"""bench.py - the headline benchmark of BASELINE.json: GCN epochs/s and aggregated-edges/s on the Reddit-shaped
synthetic graph (232 965 V, 114.6 M power-law edges + self loops, LAYERS 602-128-41, fp32), N GPUs of one node.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference]
                    [--workload reddit|products|papers100m|tiny] [--toolkit gcn|gcn_eager|gat] [--dump-outputs DIR]
    torchrun --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...        (N > 1: one rank per GPU, NCCL)

One step = one training epoch through the reference-shaped API (toolkits.GCNImpl <-> toolkits/GCN.hpp):
3 aggregation calls (fwd 602, fwd 128, bwd 128) + the dense GEMMs, loss, tape backward, gradient all-reduce (N > 1),
fused Adam.  N > 1 partitions the SAME graph with the reference's partitioner (strong scaling) and exchanges rows
through the peer-memory engine (csrc/nts_exchange.cu).  `--workload products` / `papers100m` are configs C / E,
`--toolkit gat` is config D (3-layer 8-head GAT on the fused attention aggregation, 1 GPU).

Prints ONE JSON line (rank 0).  `value` = aggregated edges per second over the whole job (3*E / epoch time) with
inputs resident in HBM; `e2e` = the same with the feature matrix coming from pinned host memory every step and the
loss read back; `roofline` = the layer-0 forward aggregation kernel timed live with CUDA events (`frac` algorithmic
bytes, `frac_min` compulsory bytes);
`parity` (N > 1) = the benchmarked distributed operator against a float64 reference on this box; `exchange_timeline`
(N > 1) = per-phase device time of one forward exchange; `cpu_baseline` / `--impl reference` = the UNMODIFIED
reference CPU GCN (toolkits/GCN_CPU.hpp via oracle/_ref, built from the reference sources by oracle/Makefile) on the
host's usable threads - on the workload itself when it fits the time budget, else on a stated 1/div scale model;
null when oracle/_ref was not built.

`--dump-outputs DIR` writes what the last timed step computed: the loss `run_epoch` returns (`loss.npy`) and the last
layer's output rows it was computed from (`output.npy`; float32, a fixed seeded sample of rows with their ids in
`output_rows.npy` when the matrix would exceed 64 MB); ranks > 0 of a multi-GPU run add `_rank<r>` to each name.
The weights are left out: Adam turns last-bit differences of near-zero gradients into steps of the learning rate.  Inputs are generated
from fixed seeds, so two builds run with the same arguments can be compared file by file.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="reddit")
    ap.add_argument("--transport", default=os.environ.get("NTS_TRANSPORT", "auto"), choices=["auto", "nccl", "p2p"],
                    help="partition-boundary exchange: p2p = CUDA-IPC peer-memory pull over NVLink, nccl = all-to-all; "
                         "auto = p2p, falling back to nccl if peer mappings cannot be set up")
    ap.add_argument("--variant", type=int, default=0, help="aggregation kernel variant (0 auto, 1 shuffle, 2 bulk)")
    ap.add_argument("--edges-per-warp", type=int, default=0)
    ap.add_argument("--drop-rate", type=float, default=0.0,
                    help="both arms run DROP_RATE 0: the reference's in-place dropout trips libtorch 2.11's autograd "
                         "version check (SURVEY 8c), so its CPU arm cannot run with dropout")
    ap.add_argument("--toolkit", default="gcn", choices=["gcn", "gcn_eager", "gat"],
                    help="gcn = toolkits/GCN.hpp order (aggregate, then GEMM: the headline config); gcn_eager = "
                         "toolkits/GCN_EAGER*.hpp order (GEMM, then aggregate the narrow result) - opt-in; gat = config D "
                         "of BASELINE.json: 3-layer 8-head GAT on the fused attention aggregation (K7), 1 GPU")
    ap.add_argument("--layers", default=None, help="override LAYERS, e.g. 602-64-64-41 (the gat default on reddit)")
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--cpu-sample-div", type=int, default=0,
                    help="CPU arm runs a 1/div scale model of the workload (V/div vertices, E/div edges, same degree "
                         "law, mean degree and widths); 0 = pick div from a probe so the run fits --cpu-budget-s")
    ap.add_argument("--cpu-budget-s", type=float, default=150.0)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-ref-gpu", action="store_true", help="skip timing the reference's own CUDA kernels")
    ap.add_argument("--zipf-s", type=float, default=1.0, help="endpoint skew (1.0 = SURVEY 8d power law, 0 = uniform)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the outputs of the last timed step to DIR/<name>.npy")
    return ap.parse_args()


# ---------------------------------------------------------------------------------------------------------------
# clocks sampler (nvidia-smi during the timed region)
# ---------------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, device_index=0):
        self.proc = None
        self.lines = []
        self.idx = device_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._pump, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, power = [], [], set(), []
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
                power.append(float(f[3]))
            except ValueError:
                continue
            for k, nm in enumerate(names):
                if f[5 + k].lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(power) if power else None, "samples": len(sm), "reasons": sorted(reasons)}


# ---------------------------------------------------------------------------------------------------------------
# reference CPU arm (oracle/_ref/nts_ref_main = the reference's stock main.cpp + GCN_CPU.hpp, unmodified)
# ---------------------------------------------------------------------------------------------------------------
def usable_cores():
    """Host threads this process may actually use: the scheduler affinity mask clipped by the cgroup CPU quota
    (os.cpu_count() reports the machine, not the lease: round 1's CPU arm ran 128 OpenMP threads on a fraction of
    that and moved 4.6x between two boxes)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    quota = None
    try:  # cgroup v2
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        try:  # cgroup v1
            q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    if quota:
        n = max(1, min(n, int(quota + 0.5)))
    return n


def reference_cpu_epochs(V, layers, edges_u32, steps, warmup, threads=None):
    """Run ALGORITHM:GCNCPU of the unmodified reference on `edges_u32` ([E,2] numpy) for warmup+steps epochs and
    time epochs from its own per-epoch log lines.  Returns dict(value edges/s, s_per_epoch, cores, kind)."""
    import numpy as np
    binary = os.path.join(ROOT, "oracle", "_ref", "nts_ref_main")
    cores = threads or usable_cores()
    E = int(edges_u32.shape[0])
    if not os.path.exists(binary):
        # never substitute the port silently: a "port" number must not be mistaken for the reference
        raise SystemExit("bench.py: oracle/_ref/nts_ref_main is missing - build it with `make -C oracle ref` "
                         "(needs the reference sources)")
    work = tempfile.mkdtemp(prefix="nts_bench_ref_")
    try:
        efile = os.path.join(work, "g.edge")
        edges_u32.astype(np.uint32).tofile(efile)
        cfg = os.path.join(work, "g.cfg")
        with open(cfg, "w") as f:
            f.write("ALGORITHM:GCNCPU\nVERTICES:%d\nLAYERS:%s\nEPOCHS:%d\nEDGE_FILE:%s\nFEATURE_FILE:random\n"
                    "LABEL_FILE:random\nMASK_FILE:random\nPROC_OVERLAP:0\nPROC_LOCAL:0\nPROC_CUDA:0\nPROC_REP:0\n"
                    "LOCK_FREE:1\nLEARN_RATE:0.01\nWEIGHT_DECAY:0.0001\nDECAY_RATE:0.97\nDECAY_EPOCH:100\n"
                    "DROP_RATE:0.0\n" % (V, "-".join(str(x) for x in layers), warmup + steps, efile))
        env = dict(os.environ)
        env["NTS_THREADS"] = str(cores)
        env["OMP_NUM_THREADS"] = str(cores)
        proc = subprocess.Popen([binary, cfg], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
        stamps = []
        for line in proc.stdout:
            if "Running.Epoch[" in line:
                stamps.append(time.perf_counter())
        proc.wait()
        if proc.returncode != 0 or len(stamps) < warmup + steps:
            raise SystemExit("bench.py: the reference CPU binary failed (rc %s, %d of %d epochs logged)" % (
                proc.returncode, len(stamps), warmup + steps))
        # epoch k ends at stamps[k]; timed region = epochs warmup .. warmup+steps-1
        t = stamps[warmup + steps - 1] - stamps[warmup - 1] if warmup >= 1 else None
        if t is None:
            t = (stamps[-1] - stamps[0]) * steps / max(1, len(stamps) - 1)
        s_per_epoch = t / steps
        return {"value": 3.0 * E / s_per_epoch, "unit": "edges/s", "s_per_epoch": s_per_epoch, "cores": cores,
                "kind": "reference"}
    finally:
        import shutil
        shutil.rmtree(work, ignore_errors=True)


def reference_cpu_op_level(V, layers, edges_u32, threads=None):
    """Op-level CPU numbers (BASELINE.md plan 3a): ForwardCPUfuseOp::forward / backward of the unmodified reference,
    bracketed with its own get_time() by oracle/_ref/nts_ref_driver in `time` mode, one warm call + 1 timed call per
    width.  Returns {"F602": {"forward_s":..., "backward_s":..., "gedges_per_s_fwd":...}, ...} or None."""
    import numpy as np
    binary = os.path.join(ROOT, "oracle", "_ref", "nts_ref_driver")
    if not os.path.exists(binary):
        return None
    cores = threads or usable_cores()
    work = tempfile.mkdtemp(prefix="nts_bench_refop_")
    out = {}
    try:
        efile = os.path.join(work, "g.edge")
        edges_u32.astype(np.uint32).tofile(efile)
        cfg = os.path.join(work, "g.cfg")
        with open(cfg, "w") as f:
            f.write("ALGORITHM:GCNCPU\nVERTICES:%d\nLAYERS:%s\nEPOCHS:1\nEDGE_FILE:%s\nFEATURE_FILE:random\n"
                    "LABEL_FILE:random\nMASK_FILE:random\nPROC_OVERLAP:0\nPROC_LOCAL:0\nPROC_CUDA:0\nPROC_REP:0\n"
                    "LOCK_FREE:1\nLEARN_RATE:0.01\nWEIGHT_DECAY:0.0001\nDECAY_RATE:0.97\nDECAY_EPOCH:100\n"
                    "DROP_RATE:0.0\n" % (V, "-".join(str(x) for x in layers), efile))
        env = dict(os.environ)
        env["NTS_THREADS"] = str(cores)
        env["OMP_NUM_THREADS"] = str(cores)
        for F in layers[:-1]:
            try:
                p = subprocess.run([binary, cfg, work, "time", str(F), "1"], stdout=subprocess.PIPE,
                                   stderr=subprocess.DEVNULL, text=True, env=env, timeout=600)
                line = [ln for ln in p.stdout.splitlines() if ln.startswith("{\"ref_cpu\"")]
                if line:
                    r = json.loads(line[-1])
                    E = int(edges_u32.shape[0])
                    out["F%d" % F] = {"forward_s": r["forward_s"], "backward_s": r["backward_s"],
                                      "gedges_per_s_forward": E / r["forward_s"] / 1e9, "threads": r["threads"]}
            except Exception:
                pass
        return out or None
    finally:
        import shutil
        shutil.rmtree(work, ignore_errors=True)


# ---------------------------------------------------------------------------------------------------------------
def main():
    args = parse_args()
    # stdout carries exactly one JSON line: keep NCCL's own banner / debug output (NCCL_DEBUG=VERSION|INFO) off it
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    import numpy as np
    import torch
    import torch.distributed as dist

    from neutronstarlite_b200 import synth

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    V, E_rand, layers = synth.WORKLOADS[args.workload]
    if args.toolkit == "gat" and args.layers is None:
        layers = [layers[0], 64, 64, layers[-1]]           # config D: hidden layers of 8 heads x 8
    if args.layers:
        layers = [int(x) for x in args.layers.split("-")]
    E_total = E_rand + V

    # ------------------------------------------------------------------ reference arm: CPU only, rank 0 only
    if args.impl == "reference":
        if rank != 0:
            return 0
        cores = usable_cores()
        div, probe = pick_cpu_sample(V, E_rand, layers, args.cpu_sample_div, args.cpu_budget_s,
                                     args.steps + args.warmup, cores)
        Vs, edges = _scale_model(V, E_rand, div)
        res = reference_cpu_epochs(Vs, layers, edges, args.steps, args.warmup, threads=cores)
        sample = _sample_text(div, Vs, edges.shape[0], probe)
        line = {
            "impl": "reference", "metric": "gcn_aggregated_edges_per_sec", "value": res["value"], "unit": "edges/s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": res["s_per_epoch"] * 1e3, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "epochs_per_sec": 1.0 / res["s_per_epoch"],
            "config": _config(args, V, E_total, layers),
            "run": {"parallelism": "unmodified reference ALGORITHM:GCNCPU, one process, %d host threads" % res["cores"]},
            "cpu_baseline": {"value": res["value"], "unit": "edges/s", "cores": res["cores"], "kind": res["kind"],
                             "sample": sample},
            "e2e": {"value": res["value"], "unit": "edges/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0,
        }
        print(json.dumps(line))
        return 0

    # ------------------------------------------------------------------ our arm
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device - libnts_b200 has no CPU fallback (use --impl reference for the CPU arm)")
    from neutronstarlite_b200 import _lib, ops
    from neutronstarlite_b200.exchange import GpuExchange
    from neutronstarlite_b200.graph import PartitionedGraph, partition_offsets_from_out_degree
    from neutronstarlite_b200.toolkits import GATImpl, GCNImpl, GCNEagerImpl

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    lib = _lib.load()
    _lib.call("nts_aggregate_set_variant", args.variant, args.edges_per_warp)

    # graph: every rank generates the same edge list (same seed), keeps only what it owns
    if E_total > (1 << 29):
        # too big to hold next to its features: two streaming passes over the same deterministic edge stream
        # (degrees -> the reference's partition offsets -> only the edges this rank owns), SURVEY 8d config E
        out_raw, in_raw = synth.zipf_degrees(V, E_rand, dev, s=args.zipf_s)
        # (every vertex has its self loop, so no degree is 0; the partitioner wants the degrees with multiplicity)
        po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E_total, world)
        src, dst = synth.zipf_edges_owned(V, E_rand, dev, int(po[rank]), int(po[rank + 1]), s=args.zipf_s)
        pg = PartitionedGraph.from_device_edges(src, dst, V, world, rank, po, out_raw.clamp(min=1), in_raw.clamp(min=1))
        del src, dst, out_raw, in_raw
    else:
        src, dst = synth.zipf_edges(V, E_rand, dev, s=args.zipf_s)
        out_raw = torch.bincount(src, minlength=V)
        out_deg = out_raw.clamp(min=1)
        in_deg = torch.bincount(dst, minlength=V).clamp_(min=1)
        po = partition_offsets_from_out_degree(out_raw.cpu().numpy(), E_total, world)
        pg = PartitionedGraph.from_device_edges(src, dst, V, world, rank, po, out_deg, in_deg)
        del src, dst
    torch.cuda.empty_cache()
    v0, v1 = int(po[rank]), int(po[rank + 1])
    feats, labels, mask = synth.features_labels_mask(V, layers[0], layers[-1], dev, rows=(v0, v1))
    op_kwargs = {}
    transport = args.transport
    if world > 1:
        if transport == "auto":
            # every rank must take the same branch: agree on whether the IPC windows could be set up
            try:
                ex = GpuExchange(pg, transport="p2p")
                ok = torch.ones(1, device=dev)
            except Exception as exc:  # noqa: BLE001 - any failure means "no peer access here"
                sys.stderr.write("bench.py: p2p exchange unavailable (%r), using nccl\n" % (exc,))
                ex, ok = None, torch.zeros(1, device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
            if ok.item() < 1:
                ex = GpuExchange(pg, transport="nccl")
                transport = "nccl"
            else:
                transport = "p2p"
        else:
            ex = GpuExchange(pg, transport=transport)
        op_kwargs["exchange"] = ex
    eager = args.toolkit == "gcn_eager"
    gat = args.toolkit == "gat"
    n_layers = len(layers) - 1
    if gat:
        if world != 1:
            raise SystemExit("bench.py: --toolkit gat is config D (1 GPU)")
        # whole-partition CSC + MirrorIndex of the edge operators (P = 1: chunk 0 is the whole partition,
        # core/PartitionedGraph.hpp:105-143,295-305)
        c0 = pg.graph_chunks[0]
        pg.owned_vertices, pg.owned_edges = V, c0.edge_size
        pg.column_offset_gpu, pg.row_indices_gpu = c0.column_offset_gpu, c0.row_indices_gpu
        has_src = torch.zeros(V + 1, dtype=torch.int32, device=dev)
        ro = c0.row_offset_gpu.long()
        has_src[1:] = (ro[1:] > ro[:-1]).to(torch.int32)
        pg.mirror_index_gpu = torch.cumsum(has_src, 0).to(torch.int32)
        pg.owned_mirrors = int(pg.mirror_index_gpu[-1].item())
        del has_src, ro
        gat_model = GATImpl(pg, layers, feats, labels, mask, heads=args.heads, exchange=GpuExchange(pg),
                            fused_kernel=True, two_pass_backward=True)

        class _AsGcn:                      # same (loss, acc) return and X[0] slot as the GCN toolkits
            X = gat_model.X
            gat = gat_model

            @staticmethod
            def run_epoch():
                return gat_model.run_epoch(), None
        model = _AsGcn
    else:
        model = (GCNEagerImpl if eager else GCNImpl)(pg, layers, feats, labels, mask, drop_rate=args.drop_rate,
                                                      op_kwargs=op_kwargs)
    # aggregation calls per epoch: GCN.hpp never back-propagates its first graph op (SURVEY 8 note) -> L + (L-1);
    # the eager order and GAT start with an NN op, so all L graph ops have a backward -> 2L
    agg_calls = float(2 * n_layers if (eager or gat) else 2 * n_layers - 1)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- warm-up
    for _ in range(max(3, args.warmup)):
        model.run_epoch()
    barrier()

    # ---- timed region A: inputs resident in HBM
    timer = ops.KernelTimer()
    ops.set_kernel_timer(timer)
    launches0 = lib.nts_kernel_launch_count()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ev0 = torch.cuda.Event(enable_timing=True)
    ev1 = torch.cuda.Event(enable_timing=True)
    barrier()
    torch.cuda.nvtx.range_push("nts_timed")
    ev0.record()
    for _ in range(args.steps):
        model.run_epoch()
    ev1.record()
    barrier()
    torch.cuda.nvtx.range_pop()
    ms_total = ev0.elapsed_time(ev1)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, model, rank, world)
    launches = lib.nts_kernel_launch_count() - launches0
    ops.set_kernel_timer(None)
    ksum = timer.summary()
    t = torch.tensor([ms_total], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total = float(t.item())
    ms_step = ms_total / args.steps
    value = agg_calls * E_total / (ms_step * 1e-3)

    # ---- timed region B: end to end through the public API with HOST buffers
    e2e = None
    if not args.no_e2e:
        host_feats = torch.empty(feats.shape, dtype=torch.float32).pin_memory()
        host_feats.copy_(feats.detach())      # (a copy from a requires-grad tensor would tie host_feats into autograd)
        host_loss = torch.empty((), dtype=torch.float32).pin_memory()
        # every step copies ITS input from pinned host memory and reads ITS loss back; the copy of step k+1 is
        # issued on a copy stream while step k computes (two device buffers), the way a host-fed trainer would
        dev_in = [torch.empty_like(feats), torch.empty_like(feats)]
        copy_stream = torch.cuda.Stream(device=dev)
        ready = [torch.cuda.Event(), torch.cuda.Event()]
        consumed = [torch.cuda.Event(), torch.cuda.Event()]

        def prefetch(k):
            b = k & 1
            with torch.no_grad(), torch.cuda.stream(copy_stream):
                copy_stream.wait_event(consumed[b])          # the step that used this buffer has finished with it
                dev_in[b].copy_(host_feats, non_blocking=True)
                ready[b].record(copy_stream)

        def e2e_step(k):
            b = k & 1
            cur = torch.cuda.current_stream()
            cur.wait_event(ready[b])
            model.X[0] = dev_in[b] if eager else dev_in[b].requires_grad_(True)
            prefetch(k + 1)
            loss, _ = model.run_epoch()
            consumed[b].record(cur)
            host_loss.copy_(loss.detach(), non_blocking=True)

        for b in (0, 1):
            consumed[b].record(torch.cuda.current_stream())
        prefetch(0)
        for k in range(2):
            e2e_step(k)
        barrier()
        ev0.record()
        for k in range(2, 2 + args.steps):
            e2e_step(k)
        ev1.record()
        barrier()
        t = torch.tensor([ev0.elapsed_time(ev1)], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_e2e = float(t.item()) / args.steps
        hb = torch.tensor([feats.numel() * 4], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(hb)
        e2e = {"value": agg_calls * E_total / (ms_e2e * 1e-3), "unit": "edges/s", "ms_per_step": ms_e2e,
               "h2d_bytes_per_step": int(hb.item()), "d2h_bytes_per_step": 4 * world}

    # ---- roofline of the dominant kernel: layer-0 forward aggregation (widest F), this rank's launches
    F0 = layers[1] if (eager or gat) else layers[0]
    k = ksum.get(("gat_fwd" if gat else "fwd", F0))
    roof = None
    if gat and k and k["ms"] > 0:
        roof = _gat_roofline(k, ksum, F0, args.heads)
    elif k and k["ms"] > 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", 3350.0))
        which = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "H100 SXM data sheet 3.35 TB/s"
        # algorithmic bytes (SURVEY 8d): E*(4 idx + 4 w + 4F row) + V_out*4F + (V_out+1)*4, summed over launches
        b_alg = k["edges"] * (8 + 4 * F0) + k["rows"] * 4 * F0 + (k["rows"] + k["calls"]) * 4
        achieved = b_alg / (k["ms"] * 1e-3) / 1e9
        t_launch = k["ms"] / k["calls"] * 1e-3
        # compulsory traffic (SURVEY 8d): every feature row once in, every output row once out, the graph arrays once
        b_min = (k["rows"] * 4 * F0 * 2 + k["edges"] * 8 + (k["rows"] + k["calls"]) * 4) / k["calls"]
        roof = {"bound": "hbm",
                "kernel": ("planned_gather_sum_kernel" if ops._plan_mode != "off" else "segment_gather_sum_kernel") +
                          " (fwd, F=%d)" % F0,
                "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": which,
                "frac_note": "achieved = ALGORITHMIC bytes / time (SURVEY 8d: every gathered row counted as if it "
                             "came from HBM); > 1 means L1/L2 reuse, it is NOT a physical HBM fraction - see "
                             "frac_min (compulsory bytes)",
                "frac_min": b_min / t_launch / 1e9 / peak,
                "launches": k["calls"], "avg_ms_per_launch": k["ms"] / k["calls"],
                "algorithmic_bytes_per_launch": b_alg / k["calls"], "compulsory_bytes_per_launch": b_min}
    kernels = {"%s_F%d" % (tag, F): {"calls": d["calls"], "avg_ms": d["ms"] / d["calls"],
                                      "gedges_per_s": d["edges"] / (d["ms"] * 1e-3) / 1e9}
               for (tag, F), d in ksum.items()}

    ref_gpu = None
    if world == 1 and not args.no_ref_gpu and not gat:
        try:
            ref_gpu = reference_gpu_kernels(pg, feats, layers, torch)
        except Exception as exc:  # baseline only: never fail the bench because of it
            ref_gpu = {"error": repr(exc)}
    # ---- N > 1: parity of the distributed operator on THIS box, outside the timed regions
    parity = multi_gpu_parity(pg, op_kwargs["exchange"], feats.detach(), layers, rank, world, dev) if world > 1 else None
    timeline = exchange_timeline(op_kwargs["exchange"], feats.detach(), layers, world, dev) if world > 1 else None
    agg_ms = sum(d["ms"] for d in ksum.values()) / args.steps   # this rank's aggregation launches per step
    agg_only = {"ms_per_step": agg_ms, "edges_per_s": agg_calls * E_total / (agg_ms * 1e-3) if agg_ms > 0 else None,
                "note": "CUDA-event time of the aggregation launches only (rank 0), SURVEY 8d"}
    if rank == 0:
        cpu = None
        ref_built = os.path.exists(os.path.join(ROOT, "oracle", "_ref", "nts_ref_main"))
        if not args.no_cpu_baseline and world == 1 and not eager and not gat and ref_built:   # ALGORITHM:GCNCPU
            cores = usable_cores()
            div, probe = pick_cpu_sample(V, E_rand, layers, args.cpu_sample_div, min(args.cpu_budget_s, 25.0), 3, cores)
            Vs, edges = _scale_model(V, E_rand, div)
            r = reference_cpu_epochs(Vs, layers, edges, 2, 1, threads=cores)
            cpu = {"value": r["value"], "unit": "edges/s", "cores": r["cores"], "kind": r["kind"],
                   "s_per_epoch": r["s_per_epoch"], "op_level": reference_cpu_op_level(Vs, layers, edges, threads=cores),
                   "sample": _sample_text(div, Vs, edges.shape[0], probe) +
                             "; unmodified reference ALGORITHM:GCNCPU, 1 warm-up + 2 timed epochs"}
        line = {
            "metric": "gcn_aggregated_edges_per_sec", "value": value, "unit": "edges/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms_step, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "epochs_per_sec": 1e3 / ms_step,
            "config": _config(args, V, E_total, layers),
            "run": {"parallelism": "graph-partition x%d (reference partitioner), %s exchange" % (world, transport)
                    if world > 1 else "single GPU",
                    "per_rank": "features %.0f MB, graph arrays %.0f MB" % (feats.numel() * 4 / 1e6,
                                                                           pg.owned_edges * 16 / 1e6),
                    "aggregation": "nts_gather_plan (measured slab count) for chunks >= 2^20 edges, plain kernel below"
                    if ops._plan_mode != "off" else "plain kernel on the reference layout",
                    "tape_note": "like the reference (core/ntsContext.hpp:283) the first graph op gets no backward "
                                 "aggregation; unlike it, the dead input-layer dY = dH W^T GEMM is skipped too "
                                 "(<2% of the epoch)"},
            "parity": parity, "exchange_timeline": timeline,
            "e2e": e2e, "gpu_launches": int(launches), "roofline": roof, "cpu_baseline": cpu,
            "kernels": kernels, "aggregation_only": agg_only, "reference_gpu_kernels": ref_gpu, "clocks": clocks,
        }
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def multi_gpu_parity(pg, ex, feats, layers, rank, world, dev):
    """ForwardGPUfuseOp forward + backward through the exchange engine actually benchmarked, against an fp64 reference
    that shares nothing with it: 8 feature columns, the reference-layout chunk arrays (global ids), plain torch
    index_add in float64, all-gather / all-reduce over NCCL for the rows other ranks own.  Per-ROW relative error
    (max |err| of a row / max |truth| of that row); pass = 1e-4 (north_star).  The check the reference makes in
    toolkits/test_getdepneighbor_gpu.hpp:184-328 (same inputs to both paths, forward and backward)."""
    import torch
    import torch.distributed as dist
    from neutronstarlite_b200 import ops
    C = 8
    V = int(pg.partition_offset[-1])
    lo, hi = int(pg.partition_offset[rank]), int(pg.partition_offset[rank + 1])
    Vp = hi - lo
    gen = torch.Generator(device=dev).manual_seed(0x5EED0003 + rank)
    g = torch.rand((Vp, layers[1]), generator=gen, device=dev) * 2 - 1
    op = ops.ForwardGPUfuseOp(pg, None, exchange=ex)
    y = op.forward(feats.contiguous())
    dx = op.backward(g)
    # global 8-column copies of X and (zero-padded) G
    x8 = torch.zeros((V, C), dtype=torch.float64, device=dev)
    x8[lo:hi] = feats[:, :C].double()
    dist.all_reduce(x8)
    y64 = torch.zeros((Vp, C), dtype=torch.float64, device=dev)
    yabs = torch.zeros((Vp, C), dtype=torch.float64, device=dev)       # sum of |terms|: the conditioning of the row
    contrib = torch.zeros((V, 2 * C), dtype=torch.float64, device=dev)  # [:, :C] sums, [:, C:] sums of |terms|
    g8 = g[:, :C].double()
    rows = torch.arange(Vp, device=dev)
    for c in pg.graph_chunks:
        if not c.edge_size:
            continue
        co = c.column_offset_gpu.long()
        dst = torch.repeat_interleave(rows, co[1:] - co[:-1])
        src = c.row_indices_gpu.long()
        t = x8[src] * c.edge_weight_forward_gpu.double()[:, None]
        y64.index_add_(0, dst, t)
        yabs.index_add_(0, dst, t.abs_())
        del t, dst, src
        ro = c.row_offset_gpu.long()
        srcs = torch.repeat_interleave(torch.arange(c.src_range[0], c.src_range[1], device=dev), ro[1:] - ro[:-1])
        dl = c.column_indices_gpu.long() - lo
        t = g8[dl] * c.edge_weight_backward_gpu.double()[:, None]
        contrib[:, :C].index_add_(0, srcs, t)
        contrib[:, C:].index_add_(0, srcs, t.abs_())
        del t, srcs, dl
    dist.all_reduce(contrib)
    dx64, dxabs = contrib[lo:hi, :C], contrib[lo:hi, C:]

    def row_rel(a, t, tabs):
        """(max per-row error relative to the row's largest |truth|, the same restricted to WELL-CONDITIONED rows,
        max per-row error relative to the row's sum of |terms|).  A hub row that sums tens of millions of +/- terms
        is ill-conditioned (sum|t| / |sum t| ~ sqrt(n)): no fp32 summation order, the reference's included, can
        hold 1e-4 of the RESULT there, only a small multiple of eps of sum|t|."""
        if not t.numel():
            return 0.0, 0.0, 0.0
        err = (a.double() - t).abs().amax(dim=1)
        scale = t.abs().amax(dim=1).clamp(min=1e-30)
        backward_err = err / tabs.amax(dim=1).clamp(min=1e-30)
        cond = tabs.amax(dim=1) / scale
        rel = err / scale
        well = cond <= 100.0
        return (float(rel.max().item()), float(rel[well].max().item()) if bool(well.any()) else 0.0,
                float(backward_err.max().item()))

    f_all, f_well, f_bwd = row_rel(y[:, :C], y64, yabs)
    b_all, b_well, b_bwd = row_rel(dx[:, :C], dx64, dxabs)
    worst = torch.tensor([f_all, f_well, f_bwd, b_all, b_well, b_bwd], dtype=torch.float64, device=dev)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    f_all, f_well, f_bwd, b_all, b_well, b_bwd = (float(v) for v in worst.tolist())
    # pass: every well-conditioned row within 1e-4 of its own magnitude (north_star), and EVERY row within 1e-6 of
    # its sum of |terms| (about 16 eps: what any fp32 summation of that row can promise)
    ok = max(f_well, b_well) <= 1e-4 and max(f_bwd, b_bwd) <= 1e-6
    return {"op": "ForwardGPUfuseOp forward (F=%d) + backward (F=%d) through the benchmarked exchange" % (
                layers[0], layers[1]),
            "reference": "float64 torch index_add on the reference-layout chunk arrays, %d columns, all %d ranks" % (C, world),
            "max_row_rel_forward": f_all, "max_row_rel_backward": b_all,
            "max_row_rel_forward_well_conditioned": f_well, "max_row_rel_backward_well_conditioned": b_well,
            "max_row_err_over_sum_abs_terms_forward": f_bwd, "max_row_err_over_sum_abs_terms_backward": b_bwd,
            "max_rel": max(f_well, b_well), "tolerance": 1e-4,
            "rule": "rows with sum|terms| <= 100 * |result| (well conditioned) within 1e-4 of the row's largest "
                    "|result|; every row within 1e-6 of its sum|terms|",
            "ok": bool(ok)}


def exchange_timeline(ex, feats, layers, world, dev):
    """Per-phase device time of ONE forward exchange per width on the engine (outside the timed regions): push kernel
    (side stream), local chunk, and per ring step the wait for the rows of partition (p+s) and the aggregation of
    chunk (p+s).  Rank 0's numbers plus the max over ranks of the whole call and of the summed waits."""
    import ctypes as C
    import torch
    import torch.distributed as dist
    from neutronstarlite_b200 import _lib, ops
    if getattr(ex, "_p2p", None) is None:
        return None
    L = _lib.load()
    h = ex._p2p.handle
    op = ops.ForwardGPUfuseOp(ex.pg, None, exchange=ex)
    out = {}
    n = 2 * world + 1
    buf = (C.c_float * n)()
    _lib.call("nts_exchange_set_trace", h, 1)
    try:
        for F in sorted(set(layers[:-1]), reverse=True):
            x = feats if F == feats.shape[1] else torch.rand((feats.shape[0], F), device=dev)
            op.forward(x.contiguous())          # warm (plans exist from the timed epochs)
            dist.barrier()
            op.forward(x.contiguous())
            _lib.call("nts_exchange_last_timeline", h, buf, n)
            ms = [float(v) for v in buf]
            waits = sum(ms[2 * s] for s in range(1, world))
            worst = torch.tensor([ms[2 * world], waits, ms[0]], dtype=torch.float64, device=dev)
            dist.all_reduce(worst, op=dist.ReduceOp.MAX)
            out["F%d" % F] = {"rank0_ms": {"push_kernel": ms[0], "local_chunk": ms[1],
                                           "wait_for_partition": [ms[2 * s] for s in range(1, world)],
                                           "aggregate_chunk": [ms[2 * s + 1] for s in range(1, world)],
                                           "whole_call": ms[2 * world]},
                            "max_over_ranks_ms": {"whole_call": float(worst[0].item()),
                                                  "sum_of_waits": float(worst[1].item()),
                                                  "push_kernel": float(worst[2].item())}}
    finally:
        _lib.call("nts_exchange_set_trace", h, 0)
    return out


def reference_gpu_kernels(pg, feats, layers, torch):
    """Time the UNMODIFIED reference CUDA kernels (cuda/ntsCUDAFuseKernel.cuh, compiled for sm_90a into
    oracle/_ref/libnts_refcuda.so) on the same chunk and inputs: 1 warm-up + 2 timed launches per width, CUDA events
    on the reference's own stream.  Also cross-checks their output against ours.  Bench-only baseline."""
    import ctypes as C
    so = os.path.join(ROOT, "oracle", "_ref", "libnts_refcuda.so")
    if not os.path.exists(so):
        return None
    from neutronstarlite_b200 import ops
    ref = C.CDLL(so)
    ref.refcuda_stream_create.restype = C.c_void_p
    ref.refcuda_stream_handle.restype = C.c_void_p
    ref.refcuda_stream_handle.argtypes = [C.c_void_p]
    ref.refcuda_stream_sync.argtypes = [C.c_void_p]
    ref.refcuda_gather_by_dst_from_src.argtypes = [C.c_void_p] * 6 + [C.c_uint] * 7 + [C.c_int, C.c_int]
    ref.refcuda_gather_by_dst_from_src.restype = None
    cs = ref.refcuda_stream_create()
    ext = torch.cuda.ExternalStream(ref.refcuda_stream_handle(cs))
    c = pg.graph_chunks[0]
    out = {}
    for F, optim in ((layers[0], 0), (layers[1], 0), (layers[1], 1)):
        x = feats[:, :F].contiguous() if F <= feats.shape[1] else torch.rand((feats.shape[0], F), device=feats.device)
        y = torch.zeros((c.batch_size_forward, F), device=feats.device)
        torch.cuda.synchronize()
        times = []
        for it in range(3):
            y.zero_()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(ext)
            ref.refcuda_gather_by_dst_from_src(cs, x.data_ptr(), y.data_ptr(), c.edge_weight_forward_gpu.data_ptr(),
                                               c.row_indices_gpu.data_ptr(), c.column_offset_gpu.data_ptr(),
                                               c.src_range[0], c.src_range[1], c.dst_range[0], c.dst_range[1],
                                               c.edge_size, c.batch_size_forward, F, 1, optim)
            b.record(ext)
            ref.refcuda_stream_sync(cs)
            torch.cuda.synchronize()
            ms = a.elapsed_time(b)
            if it > 0 or ms > 2000.0:   # keep the baseline bounded: a launch slower than 2 s is measured once
                times.append(ms)
            if ms > 2000.0:
                break
        mine = torch.zeros_like(y)
        ops.gather_by_dst_from_src(c, mine, x)
        torch.cuda.synchronize()
        err = float(((mine - y).abs().max() / y.abs().max().clamp(min=1e-30)).item())
        # who is right where they differ?  float64 truth for the highest-degree destination (8 columns): the
        # reference accumulates that row's millions of edges sequentially in fp32
        co = c.column_offset_gpu.long()
        hub = int(torch.argmax(co[1:] - co[:-1]).item())
        e0, e1 = int(co[hub].item()), int(co[hub + 1].item())
        srcs = c.row_indices_gpu[e0:e1].long() - c.src_range[0]
        truth = (x[srcs, :8].double() * c.edge_weight_forward_gpu[e0:e1].double()[:, None]).sum(0)
        scale = truth.abs().max().clamp(min=1e-30)
        key = "F%d_%s" % (F, "optim_nts" if optim else "plain")
        out[key] = {"avg_ms": sum(times) / len(times), "max_rel_diff_vs_ours": err,
                    "hub_row_degree": e1 - e0,
                    "hub_row_rel_err_vs_f64": {"ours": float(((mine[hub, :8].double() - truth).abs().max() / scale).item()),
                                               "reference": float(((y[hub, :8].double() - truth).abs().max() / scale).item())},
                    "gedges_per_s": c.edge_size / (sum(times) / len(times) * 1e-3) / 1e9}
    return out


DUMP_BYTES = 64 << 20


def dump_outputs(d, model, rank, world):
    """What the last timed step computed: its loss and the last layer's output rows (float32).  An output matrix too
    large for this rank's share of DUMP_BYTES is cut to a fixed seeded sample of rows (their ids in output_rows.npy)."""
    import numpy as np
    import torch
    os.makedirs(d, exist_ok=True)
    sfx = "_rank%d" % rank if rank else ""
    loss = model.loss if hasattr(model, "loss") else model.gat.loss
    arrays = {"loss": np.array([float(loss.detach().item())], dtype=np.float32)}
    out = model.X[-1].detach().float()
    room = DUMP_BYTES // world - 4096   # (4 KB: the .npy headers and the loss)
    if out.numel() * 4 > room:
        n = room // (out.shape[1] * 4 + 8)
        rows = np.sort(np.random.default_rng(0x5EED0004).choice(out.shape[0], size=n, replace=False))
        arrays["output_rows"] = rows.astype(np.float64)
        out = out[torch.from_numpy(rows).to(out.device)]
    arrays["output"] = out.cpu().numpy()
    for name, a in arrays.items():
        np.save(os.path.join(d, name + sfx + ".npy"), a)


def _gat_roofline(k, ksum, F, H):
    """K7 forward (segment_gather_sum_kernel in head mode 2): per edge one slot index, one [H] source-score row and
    one F-wide mirror row; per destination its F-wide output and three [H] rows (score, max, sum)."""
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))
    b_alg = k["edges"] * (4 + 4 * H + 4 * F) + k["rows"] * (4 * F + 12 * H) + (k["rows"] + k["calls"]) * 4
    achieved = b_alg / (k["ms"] * 1e-3) / 1e9
    out = {"bound": "hbm", "kernel": "segment_gather_sum_kernel<HM=2> (fused GAT attention forward, F=%d, %d heads)" % (F, H),
           "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
           "peak_source": "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "H100 SXM data sheet 3.35 TB/s",
           "frac_note": "algorithmic bytes / time; > 1 means L1/L2 reuse of the gathered rows", "traffic": None,
           "launches": k["calls"], "avg_ms_per_launch": k["ms"] / k["calls"],
           "algorithmic_bytes_per_launch": b_alg / k["calls"]}
    kb = ksum.get(("gat_bwd", F))
    if kb and kb["ms"] > 0:   # two edge passes: mirror rows once, gradient rows once, 16-byte records per (dst, head)
        bb = kb["edges"] * (4 + 4 * F) + kb["edges"] // 2 * 16 * H
        out["backward"] = {"kernel": "gat_backward_pass_kernel x2 (dst-major + src-major)",
                           "avg_ms_per_call": kb["ms"] / kb["calls"], "achieved": bb / (kb["ms"] * 1e-3) / 1e9,
                           "frac": bb / (kb["ms"] * 1e-3) / 1e9 / peak}
    return out


def _config(args, V, E_total, layers):
    """The workload as both arms see it (identical dict in `ours` and `--impl reference`)."""
    eager = args.toolkit in ("gcn_eager", "gat")
    n_layers = len(layers) - 1
    return {"workload": _workload_name(args.workload, V, E_total, layers, args), "toolkit": args.toolkit,
            "aggregations_per_epoch": 2 * n_layers if eager else 2 * n_layers - 1, "drop_rate": args.drop_rate,
            "zipf_s": args.zipf_s,
            "l2": "%s: features %.0f MB + graph arrays %.0f MB (all ranks), no flush between steps" % (
                "inputs larger than L2" if V * layers[0] * 4 + E_total * 16 > 2 * 50e6 else
                "inputs NOT larger than the 50 MB L2 (a test workload, not a bench line)",
                V * layers[0] * 4 / 1e6, E_total * 16 / 1e6)}


def _scale_model(V, E_rand, div):
    """1/div scale model of the workload for the CPU arm: V/div vertices, E/div random edges of the same Zipf law
    (so the mean degree, the skew and the feature widths are the workload's) + self loops.  [E,2] uint32."""
    import numpy as np
    import torch
    from neutronstarlite_b200 import synth
    Vs = max(1024, V // div)
    src, dst = synth.zipf_edges(Vs, max(1, E_rand // div), torch.device("cpu"))
    return Vs, torch.stack([src, dst], 1).numpy().astype(np.uint32)


def pick_cpu_sample(V, E_rand, layers, div, budget_s, epochs, cores):
    """div such that `epochs` epochs of the reference CPU GCN fit budget_s, from a probe at 1/64 scale (epoch time is
    close to linear in the scale: aggregation ~ E, GEMMs ~ V).  div = 1 is the workload itself."""
    if div and div > 0:
        return int(div), None
    pdiv = 64
    Vp, edges = _scale_model(V, E_rand, pdiv)
    r = reference_cpu_epochs(Vp, layers, edges, 1, 1, threads=cores)
    full = r["s_per_epoch"] * pdiv
    div = 1
    while div < pdiv and full / div * epochs > budget_s:
        div *= 2
    return div, {"probe_div": pdiv, "probe_s_per_epoch": r["s_per_epoch"], "estimated_full_s_per_epoch": full}


def _sample_text(div, Vs, Es, probe):
    t = ("the workload itself (div 1)" if div == 1 else
         "1/%d scale model of the workload: %d vertices, %d edges (same Zipf law, mean degree and widths)" % (div, Vs, Es))
    if probe:
        t += "; div chosen from a 1/%d probe (%.2f s/epoch -> %.0f s/epoch estimated at full size)" % (
            probe["probe_div"], probe["probe_s_per_epoch"], probe["estimated_full_s_per_epoch"])
    return t


def _workload_name(name, V, E, layers, args=None):
    model = "%d-layer GCN" % (len(layers) - 1)
    if args is not None and args.toolkit == "gat":
        model = "%d-layer GAT, %d heads" % (len(layers) - 1, args.heads)
    return "%s-shaped synthetic power-law graph: %d V, %d E (incl. self loops), %s %s fp32" % (
        name, V, E, model, "-".join(str(x) for x in layers))


if __name__ == "__main__":
    sys.exit(main())
