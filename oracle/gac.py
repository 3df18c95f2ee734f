"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the NOAA GAC and DMSP RTD decoders (noaa_gac_decoder, dmsp_rtd_decoder):

  oracle/_ref/libsatref_gac.so: the unmodified reference deframers + oracle/gac_harness.cpp (oracle/Makefile)

Where it was not built (the reference is absent) the tests read tests/golden/gac_pins.json.
"""
import ctypes as C

import numpy as np

from . import _checker
from ._checker import Handle, Library, ref_path

GAC_BYTES, DMSP_BYTES = 4159, 19

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("gac"), "ref_")},
              [("gac_pn_table", None, [vp]), ("gac_create", vp, [C.c_int, C.c_int, C.c_double]), ("gac_destroy", None, [vp]),
               ("gac_run", C.c_int, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl, C.POINTER(cl), vp])])
available = lib.available


def pn_table():
    """the reference's gac_rand_bits (1023 entries, 0 / 1)"""
    out = np.zeros(1023, np.uint8)
    lib()["gac_pn_table"](out.ctypes.data)
    return out


class Ref(Handle):
    """The module loop of noaa_gac_decoder (dmsp False, `backward`) or dmsp_rtd_decoder (dmsp True, start_timestamp, -1: none); run() may
    be called repeatedly (the stream continues; only whole 8192-byte reads from the stream's start are decoded)."""

    def __init__(self, dmsp, backward=False, start_timestamp=-1.0):
        self.dmsp = bool(dmsp)
        super().__init__(lib(), "gac", int(self.dmsp), int(bool(backward)), float(start_timestamp))

    def run(self, soft):
        """frames uint8 [n, 4159 | 19] in decode order, ts (DMSP timestamps, float64) and stats (frames so far, state)"""
        soft = np.ascontiguousarray(soft, np.int8)
        nbytes = GAC_BYTES if not self.dmsp else DMSP_BYTES
        cap = (soft.size + 8192) // 100 * nbytes + 8 * GAC_BYTES
        out = np.zeros(cap, np.uint8)
        ts = np.zeros(soft.size // 100 + 128, np.float64)
        st = np.zeros(2, np.int64)
        nb, nt = C.c_long(0), C.c_long(0)
        rc = self.L["gac_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), ts.ctypes.data, ts.size, C.byref(nt),
                               st.ctypes.data)
        assert rc == 0
        return dict(out=out[:nb.value].reshape(-1, nbytes).copy(), ts=ts[:nt.value].copy(), stats=dict(frames=int(st[0]), state=int(st[1])))


def run_pieces(soft, cuts=(), dmsp=False, backward=False, start_timestamp=-1.0):
    """One decoder over soft pushed in the pieces cut at `cuts`: the concatenated frames and timestamps, and the stats after every piece."""
    return _checker.run_pieces(Ref(dmsp, backward, start_timestamp), soft, cuts)
