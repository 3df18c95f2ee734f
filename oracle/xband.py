"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the METEOR-M X-band dump decoder (meteor_xband_decoder):

  oracle/_ref/libsatref_xband.so: the unmodified reference record deframers, NRZMDiff, RepackBitsByte and SimpleDeframer +
  oracle/xband_harness.cpp (oracle/Makefile)

Where it was not built (the reference is absent) the tests read tests/golden/meteor_xband_pins.json.
"""
import ctypes as C

import numpy as np

from ._checker import Handle, Library, ref_path

FRAME_BYTES = {0: 380, 1: 60160}  # by instrument_type: mtvza, kmss_bpsk

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("xband"), "ref_")}, [("xb_create", vp, [C.c_int]), ("xb_destroy", None, [vp]),
                                                    ("xb_run", C.c_int, [vp, vp, cl, vp, cl, C.POINTER(cl), vp])])
available = lib.available


class Ref(Handle):
    """The module loop of meteor_xband_decoder (instrument_type 0 mtvza, 1 kmss_bpsk); run() may be called repeatedly (the stream
    continues; only whole 8192-byte reads from the stream's start are decoded)."""

    def __init__(self, instrument_type):
        self.kind = int(instrument_type)
        super().__init__(lib(), "xb", self.kind)

    def run(self, soft):
        """frames uint8 [n, 380 | 60160] in the order the module writes them, and stats (frame_count so far)"""
        soft = np.ascontiguousarray(soft, np.int8)
        nb_frame = FRAME_BYTES[self.kind]
        cap = (soft.size + 16384) // 256 * nb_frame + 8 * nb_frame
        out = np.zeros(cap, np.uint8)
        st = np.zeros(2, np.int64)
        nb = C.c_long(0)
        assert self.L["xb_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), st.ctypes.data) == 0
        return dict(out=out[:nb.value].reshape(-1, nb_frame).copy(), frame_count=int(st[0]))
