"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the METEOR-M LRPT decoder (meteor_lrpt_decoder):

  oracle/_ref/libsatref_meteor.so: the unmodified reference translation units + oracle/meteor_harness.cpp (oracle/Makefile)

Where it was not built (the reference is absent) the tests read tests/golden/meteor_lrpt_pins.json.
"""
import ctypes as C

import numpy as np

from . import _checker
from ._checker import Handle, Library, ref_path

F = 16384
CADU = 1024
REC = ("offset", "pos", "corr", "phase", "swap", "rs0", "rs1", "rs2", "rs3", "ber")
STATS = ("correlator_lock", "viterbi_ber", "rs_avg")
M2X_STATS = ("deframer_state", "viterbi_ber", "viterbi_lock", "rs_avg")

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("meteor"), "ref_")},
              [("meteor_create", vp, [C.c_int]), ("meteor_destroy", None, [vp]), ("meteor_run", cl, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl, vp]),
               ("meteor_m2x_create", vp, [C.c_int, C.c_float, C.c_int]), ("meteor_m2x_destroy", None, [vp]),
               ("meteor_m2x_run", cl, [vp, vp, cl, vp, cl, vp])])
available = lib.available


def _f32(bits):
    return float(np.array([bits], np.uint32).view(np.float32)[0])


class Meteor(Handle):
    """m2x_mode false: the module loop over a soft stream; run() may be called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, diff_decode=False):
        super().__init__(lib(), "meteor", int(diff_decode))

    def run(self, soft):
        """Returns cadu (uint8 [frames written, 1024]), recs (int64 [n, 10], columns REC, ber as float32 bits) and stats (STATS; viterbi_ber
        as float32 bits)."""
        soft = np.ascontiguousarray(soft, np.int8)
        cap = soft.size // F + 4
        out = np.zeros(cap * CADU, np.uint8)
        recs = np.zeros((cap, 10), np.int64)
        st = np.zeros(3, np.int64)
        nb = C.c_long(0)
        n = self.L["meteor_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, C.byref(nb), recs.ctypes.data, cap, st.ctypes.data)
        assert n >= 0
        return dict(cadu=out[:nb.value].reshape(-1, CADU).copy(), recs=recs[:n].copy(), stats=dict(zip(STATS, st.tolist())))


class MeteorM2x(Handle):
    """m2x_mode without "interleaved": the module loop over 8192-byte calls."""

    def __init__(self, diff_decode, ber_thresold, outsync_after):
        super().__init__(lib(), "meteor_m2x", int(diff_decode), ber_thresold, outsync_after)

    def run(self, soft):
        soft = np.ascontiguousarray(soft, np.int8)
        cap = (soft.size // 8192 + 4) * 2 * CADU + 65536
        out = np.zeros(cap, np.uint8)
        st = np.zeros(5, np.int64)
        n = self.L["meteor_m2x_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, st.ctypes.data)
        assert n >= 0
        return dict(cadu=out[:n * CADU].reshape(-1, CADU).copy(), stats=dict(zip(M2X_STATS, st[:4].tolist())))


def run_pieces(soft, cuts=(), diff_decode=False):
    """One decoder over soft pushed in the pieces cut at `cuts`; the concatenated results and the stats after every piece."""
    return _checker.run_pieces(Meteor(diff_decode), soft, cuts)
