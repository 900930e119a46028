#!/usr/bin/env python3
"""TEST INFRASTRUCTURE ONLY - regenerate tests/golden/cora_sample_B64_F8/ from the UNMODIFIED reference sampler.

Builds oracle/_ref/nts_ref_sample_driver (`make -C oracle -f Makefile -f sample.mk sample`, reference sources needed)
and runs it with NTS_THREADS=1 on the reference's Cora fixture (data/cora.2708.edge.self, its feature / label / mask
tables) as gcn_cora_sample.cfg configures GCNSAMPLESINGLE, with LAYERS 1433-128-7, FANOUT 5-10 and BATCH_SIZE 64:
the first train batch's blocks (dst, c_o, r_i, src in the reference's first-appearance order, per-edge weights) and
MiniBatchFuseOp forward / backward on the driver's deterministic inputs (F = 8), per hop.  The arrays go to
tests/golden/cora_sample_B64_F8/blocks.npz (data only; the tests never need the reference).

    python oracle/make_sample_golden.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DRIVER = os.path.join(HERE, "_ref", "nts_ref_sample_driver")
DATA = os.path.join(HERE, "_ref", "data")
OUT = os.path.join(ROOT, "tests", "golden", "cora_sample_B64_F8")
F = 8


def main():
    subprocess.check_call(["make", "-s", "-C", HERE, "-f", "Makefile", "-f", "sample.mk", "sample"])
    sys.path.insert(0, HERE)
    from run_ref import launch
    work = tempfile.mkdtemp(prefix="nts_gold_sample_")
    try:
        cfg = os.path.join(work, "sample.cfg")
        with open(cfg, "w") as f:
            f.write("ALGORITHM:GCNSAMPLESINGLE\nVERTICES:2708\nLAYERS:1433-128-7\nFANOUT:5-10\nBATCH_SIZE:64\n"
                    "EPOCHS:1\nEDGE_FILE:%s\nFEATURE_FILE:%s\nLABEL_FILE:%s\nMASK_FILE:%s\nPROC_OVERLAP:0\n"
                    "PROC_LOCAL:0\nPROC_CUDA:0\nPROC_REP:0\nLOCK_FREE:1\nLEARN_RATE:0.01\nWEIGHT_DECAY:0.0001\n"
                    "DECAY_RATE:0.97\nDECAY_EPOCH:100\nDROP_RATE:0.0\n"
                    % tuple(os.path.join(DATA, n) for n in ("cora.2708.edge.self", "cora.featuretable",
                                                            "cora.labeltable", "cora.mask")))
        out = os.path.join(work, "out")
        os.makedirs(out)
        rc = launch(1, [DRIVER, cfg, out, str(F)], threads=1, quiet=True)
        if rc != 0:
            raise RuntimeError("reference sampling driver failed rc=%d" % rc)
        meta = np.fromfile(os.path.join(out, "meta.bin"), dtype=np.int64)
        data = {"meta": meta}
        for h in range(int(meta[0])):
            for k in ("dst", "c_o", "r_i", "src"):
                data["h%d/%s" % (h, k)] = np.fromfile(os.path.join(out, "h%d_%s.bin" % (h, k)), dtype=np.uint32)
            for k in ("w", "X", "Y", "G", "dX"):
                a = np.fromfile(os.path.join(out, "h%d_%s.bin" % (h, k)), dtype=np.float32)
                data["h%d/%s" % (h, k)] = a if k == "w" else a.reshape(-1, F)
        os.makedirs(OUT, exist_ok=True)
        dst = os.path.join(OUT, "blocks.npz")
        np.savez_compressed(dst, **data)
        print("wrote", dst, "%.1f KB" % (os.path.getsize(dst) / 1024))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
