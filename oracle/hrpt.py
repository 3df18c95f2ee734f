"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the NOAA and METEOR HRPT decoders (noaa_hrpt_decoder,
meteor_hrpt_decoder):

  oracle/_ref/libsatref_hrpt.so: the unmodified reference deframers + oracle/hrpt_harness.cpp (oracle/Makefile)

Where it was not built (the reference is absent) the tests read tests/golden/hrpt_pins.json.
"""
import ctypes as C

import numpy as np

from . import _checker
from ._checker import Handle, Library, ref_path

NOAA_WORDS = 11090
CADU = 1024

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("hrpt"), "ref_")}, [("hrpt_create", vp, [C.c_int, C.c_int]), ("hrpt_destroy", None, [vp]),
                                                   ("hrpt_run", cl, [vp, vp, cl, vp, cl, C.POINTER(cl), C.c_int, vp, cl, vp])])
available = lib.available


class Hrpt(Handle):
    """The module loop of noaa_hrpt_decoder (meteor False, deframer_thresold thr) or meteor_hrpt_decoder (meteor True); run() may be
    called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, meteor, thr=0):
        self.meteor = bool(meteor)
        super().__init__(lib(), "hrpt", int(self.meteor), int(thr))

    def run(self, soft, records=True):
        """Returns out (NOAA: uint16 words; METEOR: uint8 [frames, 1024]), recs (int64 [n, 3] = stream bit of the sync's last bit,
        inverted, accepting state; empty without `records`) and stats (units = words / frames written so far, state)."""
        soft = np.ascontiguousarray(soft, np.int8)
        cap = 2 * soft.size + 8 * CADU
        out = np.zeros(cap, np.uint8)
        rcap = soft.size // 8000 + 8
        recs = np.zeros((rcap, 3), np.int64)
        st = np.zeros(2, np.int64)
        nb = C.c_long(0)
        n = self.L["hrpt_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), int(records), recs.ctypes.data, rcap,
                               st.ctypes.data)
        assert n >= 0
        o = out[:nb.value].copy()
        o = o.reshape(-1, CADU) if self.meteor else o.view(np.uint16)
        return dict(out=o, recs=recs[:n].copy(), stats=dict(units=int(st[0]), state=int(st[1])))


def run_pieces(soft, cuts=(), meteor=False, thr=0):
    """One decoder over soft pushed in the pieces cut at `cuts`: the concatenated output and records, and the stats after every piece."""
    return _checker.run_pieces(Hrpt(meteor, thr), soft, cuts)
