"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the Aqua / Aura DB decoder (aqua_db_decoder):

  oracle/_ref/libsatref_eos.so: the unmodified reference blocks + oracle/eos_harness.cpp (oracle/Makefile)

Where it was not built (the reference is absent) the tests read tests/golden/eos_pins.json.
"""
import ctypes as C

import numpy as np

from . import _checker
from ._checker import Handle, Library, ref_path

CADU = 1024
READ = 65536

vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("eos"), "ref_")}, [("aqua_create", vp, []), ("aqua_destroy", None, [vp]),
                                                  ("aqua_run", C.c_int, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl, vp])])
available = lib.available


class Aqua(Handle):
    """The module loop of aqua_db_decoder over 65 536-byte reads; run() may be called repeatedly (the stream continues, and bytes short of
    a whole read wait for the next call)."""

    def __init__(self):
        super().__init__(lib(), "aqua")

    def run(self, soft):
        """Returns cadu (uint8 [frames, 1024]), rs (int32 [frames, 4]: decode_interlaved's errors[]) and stats (frames written so far,
        deframer state, bytes corrected and codewords failed so far, bytes waiting for the next read)."""
        soft = np.ascontiguousarray(soft, np.int8)
        nf = (soft.size + READ) // 8192 + 8
        out = np.zeros(nf * CADU, np.uint8)
        rs = np.zeros(nf * 4, np.int32)
        st = np.zeros(5, np.int64)
        nb = C.c_long(0)
        assert self.L["aqua_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, C.byref(nb), rs.ctypes.data, rs.size,
                                  st.ctypes.data) == 0
        k = nb.value // CADU
        return dict(cadu=out[:nb.value].reshape(-1, CADU).copy(), rs=rs[:4 * k].reshape(-1, 4).copy(),
                    stats=dict(frames=int(st[0]), state=int(st[1]), corrected=int(st[2]), failed=int(st[3]), pending=int(st[4])))


def run_pieces(soft, cuts=()):
    """One decoder over soft pushed in the pieces cut at `cuts`: the concatenated CADUs and RS results, and the stats after every piece."""
    return _checker.run_pieces(Aqua(), soft, cuts)
