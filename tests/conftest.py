"""pytest configuration: markers, import path, golden-vector loader."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
ORACLE_DIR = os.path.join(ROOT, "oracle")
if ORACLE_DIR not in sys.path:
    sys.path.insert(0, ORACLE_DIR)

import golden_store  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


class Golden:
    """One reference run: integer artefacts and operator results of P ranks (oracle/make_golden.py)."""

    def __init__(self, name):
        z = golden_store.load(name)
        self.name = z.name
        self._z = z
        self.V, self.E, self.P, self.F = (int(x) for x in z["case"])
        self.edges = z["edges"]

    def has(self, rank, key):
        return ("r%d/%s" % (rank, key)) in self._z

    def get(self, rank, key):
        return self._z["r%d/%s" % (rank, key)]

    def mat(self, rank, key, cols=None):
        a = self.get(rank, key)
        return a.reshape(-1, cols if cols is not None else self.F)

    @property
    def partition_offset(self):
        return self.get(0, "partition_offset")


@pytest.fixture(params=golden_store.case_names())
def golden(request):
    return Golden(request.param)
