"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the NOAA and METEOR HRPT decoders (noaa_hrpt_decoder,
meteor_hrpt_decoder):

  oracle/_ref/libsatref_hrpt.so: the unmodified reference deframers + oracle/hrpt_harness.cpp (oracle/hrpt.mk)

Where it was not built (the reference is absent) the tests read tests/golden/hrpt_pins.json.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_ref", "libsatref_hrpt.so")
NOAA_WORDS = 11090
CADU = 1024


def available():
    return os.path.exists(PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        vp, cl = C.c_void_p, C.c_long
        for name, res, args in [("ref_hrpt_create", vp, [C.c_int, C.c_int]), ("ref_hrpt_destroy", None, [vp]),
                                ("ref_hrpt_run", cl, [vp, vp, cl, vp, cl, C.POINTER(cl), C.c_int, vp, cl, vp])]:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


class Hrpt:
    """The module loop of noaa_hrpt_decoder (meteor False, deframer_thresold thr) or meteor_hrpt_decoder (meteor True); run() may be
    called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, meteor, thr=0):
        self.meteor = bool(meteor)
        self.h = lib().ref_hrpt_create(int(self.meteor), int(thr))

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_hrpt_destroy(self.h)
            self.h = None

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
        n = lib().ref_hrpt_run(self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), int(records), recs.ctypes.data, rcap,
                               st.ctypes.data)
        assert n >= 0
        o = out[:nb.value].copy()
        o = o.reshape(-1, CADU) if self.meteor else o.view(np.uint16)
        return dict(out=o, recs=recs[:n].copy(), stats=dict(units=int(st[0]), state=int(st[1])))


def run_pieces(soft, cuts=(), meteor=False, thr=0):
    """One decoder over soft pushed in the pieces cut at `cuts`: the concatenated output and records, and the stats after every piece."""
    d = Hrpt(meteor, thr)
    out, recs, stats = [], [], []
    for a, b in zip([0, *cuts], [*cuts, soft.size]):
        r = d.run(soft[a:b])
        out.append(r["out"])
        recs.append(r["recs"])
        stats.append(r["stats"])
    return dict(out=np.concatenate(out), recs=np.concatenate(recs), stats=stats)
