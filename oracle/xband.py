"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the METEOR-M X-band dump decoder (meteor_xband_decoder):

  oracle/_ref/libsatref_xband.so: the unmodified reference record deframers, NRZMDiff, RepackBitsByte and SimpleDeframer +
  oracle/xband_harness.cpp (oracle/xband.mk)

Where it was not built (the reference is absent) the tests read tests/golden/meteor_xband_pins.json.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_ref", "libsatref_xband.so")
FRAME_BYTES = {0: 380, 1: 60160}  # by instrument_type: mtvza, kmss_bpsk


def available():
    return os.path.exists(PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        vp, cl = C.c_void_p, C.c_long
        for name, res, args in [("ref_xb_create", vp, [C.c_int]), ("ref_xb_destroy", None, [vp]),
                                ("ref_xb_run", C.c_int, [vp, vp, cl, vp, cl, C.POINTER(cl), vp])]:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


class Ref:
    """The module loop of meteor_xband_decoder (instrument_type 0 mtvza, 1 kmss_bpsk); run() may be called repeatedly (the stream
    continues; only whole 8192-byte reads from the stream's start are decoded)."""

    def __init__(self, instrument_type):
        self.kind = int(instrument_type)
        self.h = lib().ref_xb_create(self.kind)

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_xb_destroy(self.h)
            self.h = None

    def run(self, soft):
        """frames uint8 [n, 380 | 60160] in the order the module writes them, and stats (frame_count so far)"""
        soft = np.ascontiguousarray(soft, np.int8)
        nb_frame = FRAME_BYTES[self.kind]
        cap = (soft.size + 16384) // 256 * nb_frame + 8 * nb_frame
        out = np.zeros(cap, np.uint8)
        st = np.zeros(2, np.int64)
        nb = C.c_long(0)
        assert lib().ref_xb_run(self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), st.ctypes.data) == 0
        return dict(out=out[:nb.value].reshape(-1, nb_frame).copy(), frame_count=int(st[0]))
