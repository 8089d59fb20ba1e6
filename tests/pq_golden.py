"""Loaders for the heap A* goldens (tests/golden/pq/, written by tests/golden/make_golden_pq.py) and for the staged
reference's `solve_single` with tests/pqdict_shim.py as its `pqdict`."""
from __future__ import annotations

import glob
import importlib
import os
import sys
import types

import numpy as np

from golden_util import GOLDEN_DIR, Golden

REF_PLANNER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                           "neural_astar", "planner")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "pq", "*.npz")))


class PqGolden(Golden):
    def __init__(self, name: str):
        super().__init__(os.path.join("pq", name))

    @property
    def expected(self):
        """histories f32, paths i64 (each [B,1,H,W]), status i32 [B], expansions i32 [B] (meaningful where solved)"""
        return (self.bits("hist_bits").astype(np.float32), self.bits("path_bits").astype(np.int64),
                self.z["status"], self.z["expansions"])


def staged_solve_single():
    """The staged reference's solve_single, imported under a private package name so that it does not meet this
    project's `neural_astar`, with the shim as `pqdict`; None where oracle/_ref/ is not staged."""
    if not os.path.isfile(os.path.join(REF_PLANNER, "pq_astar.py")):
        return None
    import pqdict_shim

    if "_ref_planner" not in sys.modules:
        pkg = types.ModuleType("_ref_planner")
        pkg.__path__ = [REF_PLANNER]
        sys.modules["_ref_planner"] = pkg
    saved = sys.modules.get("pqdict")
    shim = types.ModuleType("pqdict")
    shim.pqdict = pqdict_shim.pqdict
    sys.modules["pqdict"] = shim
    try:
        mod = importlib.import_module("_ref_planner.pq_astar")
    finally:
        if saved is None:
            sys.modules.pop("pqdict", None)
        else:
            sys.modules["pqdict"] = saved
    return mod.solve_single
