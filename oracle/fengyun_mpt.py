"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the FengYun-3 MPT decoder (fengyun_mpt_decoder):

  oracle/_ref/libsatref_fengyun_mpt.so: the unmodified reference Viterbi1_2, rotate_soft, FengyunDiff, BPSK_CCSDS_Deframer, the
  derandomiser and Reed-Solomon + oracle/fengyun_mpt_harness.cpp (oracle/fengyun_mpt.mk)

Where it was not built (the reference is absent) the tests read tests/golden/fengyun_mpt_pins.json.
"""
import ctypes as C

import numpy as np

from ._checker import Handle, Library, ref_path

READ = 16384
vp, cl = C.c_void_p, C.c_long
lib = Library({"ref": (ref_path("fengyun_mpt"), "ref_")}, [("mpt_create", vp, [C.c_float, C.c_int]), ("mpt_destroy", None, [vp]),
                                                          ("mpt_run", C.c_int, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl, C.POINTER(cl), vp])])
available = lib.available


class RefMpt(Handle):
    """The module loop of fengyun_mpt_decoder; run() may be called repeatedly (the stream continues; only whole 16384-byte reads from
    the stream's start are decoded)."""

    def __init__(self, viterbi_outsync_after, viterbi_ber_thresold):
        super().__init__(lib(), "mpt", float(viterbi_ber_thresold), int(viterbi_outsync_after))

    def run(self, soft):
        """as oracle.fengyun.Ref.run: frames uint8 [n, 1024]; recs float64 [reads, 9] (shift, invert_branches, v1, v2, viterbi1 state,
        viterbi2 state, viterbi1 ber, viterbi2 ber, deframer state after the read); rs (errors[0] of the read's last frame, -2 without
        one); the stats after the call (rs_avg, deframer_lock, reads)"""
        soft = np.ascontiguousarray(soft, np.int8)
        nreads = (soft.size + READ) // READ + 1
        cap = nreads * 2 * 1024 + 4096
        out = np.zeros(cap, np.uint8)
        recs = np.zeros((nreads, 10), np.float32)
        st = np.zeros(3, np.int64)
        nb, nr = C.c_long(0), C.c_long(0)
        assert self.L["mpt_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, cap, C.byref(nb), recs.ctypes.data, nreads, C.byref(nr),
                                 st.ctypes.data) == 0
        r = recs[:nr.value].astype(np.float64)
        return dict(out=out[:nb.value].reshape(-1, 1024).copy(), recs=r[:, :9], rs=r[:, 9], rs_avg=int(st[0]), deframer_lock=int(st[1]),
                    reads=int(st[2]))
