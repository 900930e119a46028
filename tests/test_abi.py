"""CPU-only checks of the drop-in boundary: the shared object loads and exports every symbol that
include/nts_b200.h declares, the ctypes table covers the header, and the product has no CPU fallback."""
import os

import pytest

from neutronstarlite_b200 import _lib


def test_library_loads_and_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _lib.header_symbols()
    assert len(declared) >= 50
    for name in declared:
        assert hasattr(lib, name), "libnts_b200.so does not export %s" % name
    assert lib.nts_version() == 1


def test_ctypes_table_matches_header():
    assert sorted(_lib.SIGNATURES) == _lib.header_symbols()


def test_product_does_not_import_the_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "neutronstarlite_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert "nts_oracle" not in text, "%s references the oracle" % f
                assert "oracle/" not in text, "%s references the oracle directory" % f


def test_ops_refuse_cpu_tensors():
    import torch
    from neutronstarlite_b200 import ops
    with pytest.raises(_lib.NtsError):
        ops._check_input(torch.zeros(4, 4))


def test_argument_errors_are_reported_not_swallowed():
    lib = _lib.load()
    rc = lib.nts_aggregate_set_variant(7, 0)
    assert rc != 0
    assert b"variant" in lib.nts_last_error()
    assert lib.nts_aggregate_set_variant(0, 0) == 0


def test_aggregate_launch_record_takes_null_outputs():
    """nts_aggregate_last_shape fills what it is given and skips null pointers; before any launch it reports zeros."""
    import ctypes as C
    lib = _lib.load()
    assert lib.nts_aggregate_last_shape(None, None, None, None, None) == 0
    vals = [C.c_int(-1) for _ in range(5)]
    assert lib.nts_aggregate_last_shape(*[C.byref(v) for v in vals]) == 0
    assert all(v.value >= 0 for v in vals)


def test_exchange_path_record_refuses_a_null_engine():
    lib = _lib.load()
    assert lib.nts_exchange_last_paths(None, *([None] * 9)) != 0
    assert b"null engine" in lib.nts_last_error()


def test_empty_chunks_are_a_no_op_before_any_pointer_is_looked_at():
    """A rank that owns no vertices (or a chunk without edges) hands the aggregation entries empty tensors, whose data
    pointers are NULL: the entries must return success without touching CUDA or complaining about the pointers."""
    lib = _lib.load()
    for name in ("nts_gather_by_dst_from_src", "nts_gather_by_src_from_dst"):
        fn = getattr(lib, name)
        assert fn(None, None, None, None, None, 0, 0, 0, 0, 0, 0, 16, 1, None) == 0      # no rows
        assert fn(None, None, None, None, None, 0, 8, 0, 8, 0, 8, 16, 1, None) == 0      # rows but no edges
    assert lib.nts_segment_gather_sum(None, None, None, None, None, 0, 0, 0, 16, None) == 0


@pytest.mark.skipif(not os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                   "oracle", "_ref", "nts_ref_main")),
                    reason="oracle/_ref/nts_ref_main not built (make -C oracle ref needs the reference sources)")
def test_bench_reference_arm_prints_the_contract_keys():
    """`bench.py --impl reference` (CPU only: the unmodified reference GCNCPU built under oracle/_ref) on the tiny
    workload: one JSON line with the keys a caller reads."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--workload", "tiny",
                          "--steps", "1", "--warmup", "1"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-800:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "config", "cpu_baseline", "e2e"):
        assert key in line
    assert line["impl"] == "reference" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] in ("reference", "port") and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0
