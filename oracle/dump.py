"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checkers of the MetOp X-band dump decoder (metop_dump_decoder):

  impl "ref"   oracle/_ref/libsatref_dump.so: the unmodified reference translation units + oracle/dump_harness.cpp (oracle/Makefile)
  impl "port"  oracle/libdump_port.so: our own C restatement (oracle/dump_port.c), pinned to "ref" by tests/test_metop_dump_oracle.py

Both export the same C ABI (prefix ref_ / orc_). impl=None means "ref". Where "ref" was not built (the reference is absent) the tests read
tests/golden/metop_dump_pins.json.
"""
import ctypes as C
import os

import numpy as np

from . import _checker
from ._checker import HERE, Handle, Library, ref_path

F = 8192
CADU = 1024
REC = ("offset", "pos", "corr", "phase", "swap", "rs0", "rs1", "rs2", "rs3")

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("dump"), "ref_"), "port": (os.path.join(HERE, "libdump_port.so"), "orc_")},
              [("dump_create", vp, []), ("dump_destroy", None, [vp]), ("dump_run", cl, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl])])
available = lib.available


class Dump(Handle):
    """The module loop over a soft stream; run() may be called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, impl="ref"):
        super().__init__(lib(impl), "dump")

    def run(self, soft):
        """Returns cadu (uint8 [frames, 1024], every frame) and recs (int64 [n, 9], columns REC)."""
        soft = np.ascontiguousarray(soft, np.int8)
        cap = soft.size // F + 4
        out = np.zeros(cap * CADU, np.uint8)
        recs = np.zeros((cap, 9), np.int64)
        nb = C.c_long(0)
        n = self.L["dump_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, C.byref(nb), recs.ctypes.data, cap)
        assert n >= 0
        return dict(cadu=out[:nb.value].reshape(-1, CADU).copy(), recs=recs[:n].copy())


def run_pieces(soft, cuts=(), impl="ref"):
    """One decoder over soft pushed in the pieces cut at `cuts`; the concatenated results."""
    return _checker.run_pieces(Dump(impl), soft, cuts)
