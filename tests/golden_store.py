"""Golden vectors of one reference run (oracle/make_golden.py): tests/golden/<case>/ holds the arrays split over a few
.npz parts (graph artefacts, operator inputs, operator results, pure-copy results) so that no stored file grows past
1 MB.  load() merges the parts back into one read-only mapping keyed like the dump ("edges", "r0/X", ...)."""
import glob
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class GoldenCase:
    def __init__(self, name):
        name = os.path.basename(name)
        self.name = name[:-4] if name.endswith(".npz") else name
        parts = sorted(glob.glob(os.path.join(GOLDEN_DIR, self.name, "*.npz")))
        if not parts:
            raise FileNotFoundError("no golden case %s under %s" % (self.name, GOLDEN_DIR))
        self._where = {}
        for p in parts:
            z = np.load(p)
            for k in z.files:
                self._where[k] = z
        self.files = sorted(self._where)

    def __contains__(self, key):
        return key in self._where

    def __getitem__(self, key):
        return self._where[key][key]


def load(name):
    """`name` is a case ("synth9k_P2_F2"), optionally with the historical ".npz" suffix, or its directory."""
    return GoldenCase(name)


def case_names():
    return sorted(os.path.basename(os.path.dirname(p)) for p in glob.glob(os.path.join(GOLDEN_DIR, "*", "topology.npz")))
