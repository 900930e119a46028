"""GNNDatum host loader (SURVEY 8 f3) on the reference's own Cora tables (stored gzipped under tests/golden/cora_tables,
unpacked into a temporary directory): the parallel parser must give exactly what a record-by-record read of the
text tables gives (the contract of core/ntsDataloador.hpp:156-221), for the whole graph and for a partition's rows; a
packed binary table must round-trip."""
import gzip
import os
import shutil

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES = os.path.join(ROOT, "tests", "golden", "cora_tables")


@pytest.fixture(scope="module")
def cora_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("cora")
    for name in ("cora.featuretable", "cora.labeltable", "cora.mask"):
        with gzip.open(os.path.join(TABLES, name + ".gz"), "rb") as src, open(d / name, "wb") as dst:
            shutil.copyfileobj(src, dst)
    return str(d)


def _reference_read(DATA, V, F):
    """Record by record, like the reference's three istreams."""
    feats = np.zeros((V, F), dtype=np.float32)
    labels = np.zeros(V, dtype=np.int64)
    masks = np.zeros(V, dtype=np.int32)
    names = {"train": 0, "eval": 1, "val": 1, "test": 2}
    with open(os.path.join(DATA, "cora.featuretable")) as ff, open(os.path.join(DATA, "cora.labeltable")) as fl, \
            open(os.path.join(DATA, "cora.mask")) as fm:
        for lf, ll, lm in zip(ff, fl, fm):
            tok = lf.split()
            if not tok:
                continue
            vid = int(tok[0])
            feats[vid] = np.array(tok[1:1 + F], dtype=np.float32)
            labels[vid] = int(ll.split()[1])
            masks[vid] = names.get(lm.split()[1], 3)
    return feats, labels, masks


def test_text_tables_match_a_record_by_record_read(cora_dir):
    from neutronstarlite_b200.dataloader import GNNDatum
    DATA = cora_dir
    V, F = 2708, 1433
    feats, labels, masks = _reference_read(DATA, V, F)
    d = GNNDatum(F, 7, 0, V).readFeature_Label_Mask(os.path.join(DATA, "cora.featuretable"),
                                                    os.path.join(DATA, "cora.labeltable"),
                                                    os.path.join(DATA, "cora.mask"))
    assert np.array_equal(d.local_feature.view(np.uint32), feats.view(np.uint32))
    assert np.array_equal(d.local_label, labels) and np.array_equal(d.local_mask, masks)
    assert set(np.unique(masks)) <= {0, 1, 2, 3} and feats.sum() > 0
    # a partition's rows only (the reference skips foreign ids but still consumes their label / mask records)
    lo, hi = 1024, 2048
    p = GNNDatum(F, 7, lo, hi).readFeature_Label_Mask(os.path.join(DATA, "cora.featuretable"),
                                                      os.path.join(DATA, "cora.labeltable"),
                                                      os.path.join(DATA, "cora.mask"))
    assert np.array_equal(p.local_feature, feats[lo:hi]) and np.array_equal(p.local_label, labels[lo:hi])
    assert np.array_equal(p.local_mask, masks[lo:hi])


def test_binary_table_round_trip_and_errors(tmp_path):
    from neutronstarlite_b200 import _lib
    from neutronstarlite_b200.dataloader import GNNDatum
    rng = np.random.default_rng(3)
    V, F = 1000, 37
    table = rng.standard_normal((V, F)).astype(np.float32)
    path = tmp_path / "features.bin"
    table.tofile(path)
    d = GNNDatum(F, 5, 200, 777).read_feature_binary(path)
    assert np.array_equal(d.local_feature, table[200:777])
    with pytest.raises(_lib.NtsError):
        GNNDatum(F, 5, 900, 1100).read_feature_binary(path)          # rows past the end of the file
    with pytest.raises(_lib.NtsError):
        GNNDatum(F, 5, 0, 10).readFeature_Label_Mask(tmp_path / "missing", None, None)
    # text table with a short line is rejected, a well-formed one is parsed (ids in any order, exponents, negatives)
    good = tmp_path / "good.ftr"
    good.write_text("2 1e-3 -2.5 3\n0 0 0.125 7\n1 4 5 6\n")
    g = GNNDatum(3, 2, 0, 3).readFeature_Label_Mask(good, None, None)
    assert np.array_equal(g.local_feature, np.array([[0, 0.125, 7], [4, 5, 6], [1e-3, -2.5, 3]], dtype=np.float32))
    bad = tmp_path / "bad.ftr"
    bad.write_text("0 1 2\n")
    with pytest.raises(_lib.NtsError):
        GNNDatum(3, 2, 0, 1).readFeature_Label_Mask(bad, None, None)
    r = GNNDatum(4, 3, 0, 9)
    r.random_generate()
    assert r.local_feature.min() == 1.0 and set(r.local_mask) == {0, 1, 2} and r.local_label.max() < 3
