#!/usr/bin/env python3
"""TEST INFRASTRUCTURE ONLY - regenerate the golden vectors under tests/golden/ from the UNMODIFIED reference.

Runs oracle/_ref/nts_ref_driver (built by `make -C oracle ref` from the reference sources) on
  * the reference's own Cora fixture (data/cora.2708.edge.self) at P = 1, 2, 4 ranks and
  * a small synthetic multigraph (hubs, duplicates, self loops, isolated vertices) at P = 1, 2, 3, 4, 8
and packs every dumped artefact into tests/golden/<case>/, split over a few .npz parts (save_case) so that no
stored file exceeds 1 MB.  Needs the reference sources (oracle/Makefile REF); the outputs are committed, so the
tests never do.

    python oracle/make_golden.py            # all cases
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DRIVER = os.path.join(HERE, "_ref", "nts_ref_driver")
GOLD = os.path.join(ROOT, "tests", "golden")

INT_U32 = {"partition_offset", "out_degree", "in_degree", "mirror_index", "whole_column_offset",
           "whole_row_indices", "whole_compressed_row_offset", "whole_column_indices",
           "column_offset", "row_indices", "row_offset", "column_indices"}
U8 = {"source_active", "has_mirror_at"}
COPY_ONLY = {"scatter_src_msg", "scatter_dst_msg", "aggregate_dst_dmsg"}
INPUTS = {"X", "G", "dep_Gm", "Ge", "softmax_in", "softmax_gout"}


def _part(key):
    base = key.split("/")[-1]
    base = base.split("_", 1)[1] if base.startswith("chunk") else base
    if key in ("edges", "case") or base in INT_U32 or base in U8 or base == "meta" or base.startswith("edge_weight"):
        return "topology"
    if base in INPUTS:
        return "inputs"
    return "copies" if base in COPY_ONLY else "outputs"


def save_case(name, data):
    """tests/golden/<name>/{topology,inputs,outputs,copies}.npz (tests/golden_store.py reads them back)."""
    d = os.path.join(GOLD, name)
    os.makedirs(d, exist_ok=True)
    for f in os.listdir(d):
        if f.endswith(".npz"):
            os.remove(os.path.join(d, f))
    parts = {}
    for k, v in data.items():
        parts.setdefault(_part(k), {})[k] = v
    for part, arrays in parts.items():
        dst = os.path.join(d, part + ".npz")
        np.savez_compressed(dst, **arrays)
        print("wrote", dst, "%.1f KB" % (os.path.getsize(dst) / 1024))


def synth_edges(V=9216, E=20000, seed=0x5EED0001):
    """Small adversarial multigraph: Zipf-ish endpoints, one destination hub, one source hub,
    duplicate edges, self loops on a subset, a block of isolated vertices."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, V + 1) ** 0.9
    perm = rng.permutation(V)
    p = np.empty(V)
    p[perm] = w / w.sum()
    src = rng.choice(V, size=E, p=p)
    dst = rng.choice(V, size=E, p=p[::-1] / p[::-1].sum())
    hub_d = int(perm[3])
    hub_s = int(perm[5])
    src = np.concatenate([src, rng.integers(0, V, 1500), np.full(700, hub_s)])
    dst = np.concatenate([dst, np.full(1500, hub_d), rng.integers(0, V, 700)])
    # duplicates
    dup = rng.integers(0, src.shape[0], 400)
    src = np.concatenate([src, src[dup], src[dup[:50]]])
    dst = np.concatenate([dst, dst[dup], dst[dup[:50]]])
    # self loops on every other vertex of the first half
    sl = np.arange(0, V // 2, 2)
    src = np.concatenate([src, sl])
    dst = np.concatenate([dst, sl])
    # isolate a block of vertices entirely
    iso = (src >= 4096) & (src < 4300) | (dst >= 4096) & (dst < 4300)
    src, dst = src[~iso], dst[~iso]
    order = rng.permutation(src.shape[0])
    return np.stack([src[order], dst[order]], axis=1).astype(np.uint32)


def write_cfg(path, edge_file, V, lock_free=1):
    with open(path, "w") as f:
        f.write("ALGORITHM:GCNCPU\nVERTICES:%d\nLAYERS:4-4-2\nEPOCHS:1\nEDGE_FILE:%s\n"
                "FEATURE_FILE:random\nLABEL_FILE:random\nMASK_FILE:random\nPROC_OVERLAP:0\n"
                "PROC_LOCAL:0\nPROC_CUDA:0\nPROC_REP:0\nLOCK_FREE:%d\nLEARN_RATE:0.01\n"
                "WEIGHT_DECAY:0.0001\nDECAY_RATE:0.97\nDECAY_EPOCH:100\nDROP_RATE:0.0\n"
                % (V, edge_file, lock_free))


def parse_dump(outdir, P, F, keep_copy_only):
    data = {}
    for name in sorted(os.listdir(outdir)):
        if not name.endswith(".bin"):
            continue
        stem = name[:-4]
        rank_s, key = stem.split("_", 1)
        rank = int(rank_s[1:])
        base = key.split("_", 1)[1] if key.startswith("chunk") else key
        path = os.path.join(outdir, name)
        if base == "meta":
            arr = np.fromfile(path, dtype=np.int64 if not key.startswith("chunk") else np.int32)
        elif base in INT_U32:
            arr = np.fromfile(path, dtype=np.uint32)
        elif base in U8:
            arr = np.fromfile(path, dtype=np.uint8)
        else:
            if base in COPY_ONLY and not keep_copy_only:
                continue
            arr = np.fromfile(path, dtype=np.float32)
        if base in ("out_degree", "in_degree", "partition_offset") and rank != 0:
            ref = data["r0/" + key]
            assert np.array_equal(ref, arr), "rank-replicated artefact differs: " + key
            continue
        data["r%d/%s" % (rank, key)] = arr
    return data


def run_case(name, edges, V, P, F, keep_copy_only, threads):
    sys.path.insert(0, HERE)
    from run_ref import launch
    work = tempfile.mkdtemp(prefix="nts_gold_")
    try:
        efile = os.path.join(work, "graph.edge")
        edges.astype(np.uint32).tofile(efile)
        cfg = os.path.join(work, "case.cfg")
        write_cfg(cfg, efile, V)
        out = os.path.join(work, "out")
        os.makedirs(out)
        rc = launch(P, [DRIVER, cfg, out, "dump", str(F)], threads=threads, quiet=True)
        if rc != 0:
            raise RuntimeError("reference driver failed rc=%d for %s" % (rc, name))
        data = parse_dump(out, P, F, keep_copy_only)
        data["edges"] = edges.astype(np.uint32)
        data["case"] = np.array([V, edges.shape[0], P, F], dtype=np.int64)
        save_case("%s_P%d_F%d" % (name, P, F), data)
    finally:
        shutil.rmtree(work, ignore_errors=True)


def run_adam(steps=8):
    """Parameter / Adam golden vectors (core/NtsScheduler.hpp:639-791 driven as toolkits/GCN.hpp:209-215 does):
    tests/golden/adam/adam_ref.npz - kept in a sub-directory, the top-level *.npz files are graph cases."""
    sys.path.insert(0, HERE)
    from run_ref import launch
    work = tempfile.mkdtemp(prefix="nts_gold_adam_")
    try:
        cfg = os.path.join(work, "case.cfg")
        write_cfg(cfg, os.path.join(work, "none.edge"), 16)
        out = os.path.join(work, "out")
        os.makedirs(out)
        rc = launch(1, [DRIVER, cfg, out, "adam", str(steps)], threads=1, quiet=True)
        if rc != 0:
            raise RuntimeError("reference driver (adam) failed rc=%d" % rc)
        w, h, n = (int(x) for x in np.fromfile(os.path.join(out, "r0_adam_meta.bin"), dtype=np.int64))
        data = {"meta": np.array([w, h, n], dtype=np.int64),
                "hyper": np.array([0.01, 0.9, 0.999, 1e-9, 0.0001, 0.97, 4], dtype=np.float64),
                "W0": np.fromfile(os.path.join(out, "r0_adam_W0.bin"), dtype=np.float32).reshape(w, h)}
        for k in ("grads", "W", "M", "V"):
            data[k] = np.fromfile(os.path.join(out, "r0_adam_%s.bin" % k), dtype=np.float32).reshape(n, w, h)
        os.makedirs(os.path.join(GOLD, "adam"), exist_ok=True)
        dst = os.path.join(GOLD, "adam", "adam_ref.npz")
        np.savez_compressed(dst, **data)
        print("wrote", dst, "%.1f KB" % (os.path.getsize(dst) / 1024))
    finally:
        shutil.rmtree(work, ignore_errors=True)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--adam":         # python oracle/make_golden.py --adam
        run_adam()
        return
    if len(sys.argv) > 1 and sys.argv[1] == "--synth-only":   # python oracle/make_golden.py --synth-only 3 5
        os.makedirs(GOLD, exist_ok=True)
        syn = synth_edges()
        for P in (int(x) for x in sys.argv[2:]):
            run_case("synth9k", syn, 9216, P, 2, False, max(1, 4 // P))
        return
    if not os.path.exists(DRIVER):
        subprocess.check_call(["make", "-C", HERE, "ref"])
    os.makedirs(GOLD, exist_ok=True)
    cora = np.fromfile(os.path.join(HERE, "_ref", "data", "cora.2708.edge.self"), dtype=np.uint32).reshape(-1, 2)
    run_case("cora_self", cora, 2708, 1, 8, True, 4)
    run_case("cora_self", cora, 2708, 2, 4, True, 2)
    run_case("cora_self", cora, 2708, 4, 2, False, 1)   # two EMPTY partitions (1024-vertex page rounding)
    syn = synth_edges()
    for P in (1, 2, 3, 4, 8):                            # 3: a ring that is not a power of two
        run_case("synth9k", syn, 9216, P, 2, False, max(1, 4 // P))
    run_adam()


if __name__ == "__main__":
    main()
