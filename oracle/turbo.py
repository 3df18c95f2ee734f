"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checkers of the CCSDS turbo decoder (ccsds_turbo_decoder):

  impl "ref"   oracle/_ref/libsatref_turbo.so: the unmodified reference translation units + oracle/turbo_harness.cpp (oracle/Makefile)
  impl "port"  oracle/libturbo_port.so: our own C restatement (oracle/turbo_port.c), pinned to "ref" by tests/test_turbo_oracle.py

Both export the same C ABI (prefix ref_ / orc_; the encoder only in "ref"). impl=None means "ref". Where "ref" was not built (the reference
is absent) the tests read tests/golden/turbo_pins.json.
"""
import ctypes as C
import os

import numpy as np

from ._checker import HERE, Handle, Library, ref_path

RATES = {"1/2": 2, "1/3": 3, "1/4": 4, "1/6": 6}
REC = ("offset", "pos", "cor_bits", "swapped", "crc_ok", "locked")

vp, ci, cl = C.c_void_p, C.c_int, C.c_long
lib = Library({"ref": (ref_path("turbo"), "ref_"), "port": (os.path.join(HERE, "libturbo_port.so"), "orc_")},
              [("turbo_create", vp, [ci, ci, ci]), ("turbo_destroy", None, [vp]), ("turbo_frame_size", ci, [vp]),
               ("turbo_run", cl, [vp, vp, cl, vp, cl, C.POINTER(cl), vp, cl]), ("turbo_encode", ci, [ci, ci, vp, vp]),
               ("turbo_perm", ci, [ci, vp]), ("turbo_half", None, [ci, ci, ci, vp, vp, vp, ci, vp])], optional=("turbo_encode",))
available = lib.available


class Turbo(Handle):
    """The module loop over a soft stream; run() may be called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, rate, base, iters, impl="ref"):
        self.rate, self.base, self.iters = RATES[rate], int(base), int(iters)
        super().__init__(lib(impl), "turbo", self.rate, self.base, self.iters)
        self.F = self.L["turbo_frame_size"](self.h)

    def run(self, soft):
        """Returns cadu (uint8 [frames, base + 4], the frames whose CRC passes) and recs (int64 [n, 6], columns REC) of every frame."""
        soft = np.ascontiguousarray(soft, np.int8)
        cap = soft.size // self.F + 4
        out = np.zeros(cap * (self.base + 4), np.uint8)
        recs = np.zeros((cap, 6), np.int64)
        nb = C.c_long(0)
        n = self.L["turbo_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, C.byref(nb), recs.ctypes.data, cap)
        assert n >= 0
        return dict(cadu=out[:nb.value].reshape(-1, self.base + 4).copy(), recs=recs[:n].copy())


def perm(base, impl="ref"):
    p = np.zeros(8 * base, np.int32)
    lib(impl)["turbo_perm"](base, p.ctypes.data)
    return p


def encode(rate, base, info):
    """CCSDSTurbo::encode of base information bytes: the codeword bits (the last partial byte unpacked from its low bits)."""
    nbits = {2: 2, 3: 3, 4: 4, 6: 6}[RATES[rate]] * (8 * base + 4)
    out = np.zeros(nbits // 8 + 1, np.uint8)
    n = lib()["turbo_encode"](RATES[rate], base, np.ascontiguousarray(info, np.uint8).ctypes.data, out.ctypes.data)
    bits = np.unpackbits(out[:n])
    tail = nbits - 8 * n
    if tail:
        bits = np.concatenate([bits, np.unpackbits(out[n:n + 1])[8 - tail:]])
    return bits


def half(rate, base, lower, stream, app0, app1, decision=False, impl="ref"):
    """One convcode_extrinsic call: returns the new a-priori arrays and (decision) the decisions."""
    stream = np.ascontiguousarray(stream, np.float64)
    a0, a1 = np.array(app0, np.float64), np.array(app1, np.float64)
    dec = np.zeros(8 * base, np.int32)
    lib(impl)["turbo_half"](RATES[rate], base, int(lower), stream.ctypes.data, a0.ctypes.data, a1.ctypes.data, int(decision), dec.ctypes.data)
    return a0, a1, (dec if decision else None)


def cor_of(recs):
    return np.asarray(recs)[:, 2].astype(np.uint32).view(np.float32)
