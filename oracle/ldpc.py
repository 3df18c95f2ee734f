"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checkers of the CCSDS LDPC decoder (ccsds_ldpc_decoder, rate 7/8 C2 code):

  impl "ref"   oracle/_ref/libsatref_ldpc.so: the unmodified reference translation units + oracle/ldpc_harness.cpp (oracle/Makefile)
  impl "port"  oracle/libldpc_port.so: our own C restatement (oracle/ldpc_port.c), pinned to "ref" by tests/test_ldpc_oracle.py

Both export the same C ABI (prefix ref_ / orc_). impl=None picks "ref" when it was built, else "port" — like tests.common.oracle().
"""
import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

from ._checker import HERE, Handle, Library, ref_path

CONST = {"bpsk": 0, "qpsk": 1, "oqpsk": 2}
F = 8192      # soft bytes per frame: 32-bit ASM + 8160 code bits
CW = 8160     # code bits sent per frame (8176 minus the 18 shortened positions, plus 2 fill bits)
REC = ("offset", "pos", "cor_bits", "phase", "swap", "ldpc_corr", "locked", "deframer_state")


_lib = Library({"ref": (ref_path("ldpc"), "ref_"), "port": (os.path.join(HERE, "libldpc_port.so"), "orc_")},
               [("ldpc_create", C.c_void_p, [C.c_int] * 4 + [C.c_uint]), ("ldpc_destroy", None, [C.c_void_p]),
                ("ldpc_run", C.c_long, [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.POINTER(C.c_long), C.c_void_p, C.c_long]),
                ("ldpc_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]), ("ldpc_matrix", C.c_int, [C.c_void_p, C.c_int])])
available = _lib.available


def default_impl():
    return "ref" if available("ref") else "port"


def lib(impl=None):
    """{name without prefix: function}"""
    return _lib(impl or default_impl())


@dataclass(frozen=True)
class LdpcCfg:
    constellation: str
    iterations: int = 10
    derandomize: bool = True
    internal_cadu_size: int = 0      # > 0: "internal_stream" with this "internal_cadu_size" (bits)
    internal_asm: int = 0x1ACFFC1D   # "internal_asm"


def ldpc_cfg(constellation, iterations=10, derandomize=True, internal_cadu_size=0, internal_asm=0x1ACFFC1D):
    """CCSDSLDPCDecoderModule's parameters for ldpc_rate "7/8" (module_ccsds_ldpc_decoder.cpp:19-124)."""
    if constellation not in CONST:
        raise ValueError(f"CCSDS LDPC Decoder : invalid constellation type {constellation!r}")
    return LdpcCfg(constellation, int(iterations), bool(derandomize), int(internal_cadu_size), int(internal_asm))


class Fec(Handle):
    """The module loop over a soft stream; run() may be called repeatedly (the stream continues, like ragged pushes)."""

    def __init__(self, cfg, impl=None):
        self.cfg, self.impl = cfg, impl or default_impl()
        self.cadu_bytes = cfg.internal_cadu_size // 8 if cfg.internal_cadu_size else 1024
        super().__init__(lib(self.impl), "ldpc", CONST[cfg.constellation], cfg.iterations, int(cfg.derandomize), cfg.internal_cadu_size,
                         cfg.internal_asm)

    def run(self, soft):
        """Returns cadu (uint8 [frames, cadu_bytes]: the CADUs, or with internal_stream the inner frames) and recs (int64 [n, 8], columns
        REC + the deframer state) of the LDPC frames the soft bytes complete."""
        soft = np.ascontiguousarray(soft, np.int8)
        cap = soft.size // F + 4
        out = np.zeros(cap * 1024 + 4 * self.cadu_bytes, np.uint8)
        recs = np.zeros((cap, 8), np.int64)
        nb = C.c_long(0)
        n = self.L["ldpc_run"](self.h, soft.ctypes.data, soft.size, out.ctypes.data, out.size, C.byref(nb), recs.ctypes.data, cap)
        assert n >= 0
        return dict(cadu=out[:nb.value].reshape(-1, self.cadu_bytes).copy(), recs=recs[:n].copy())

    def decode(self, codeword, iterations=None):
        """CCSDSLDPC::decode alone: 8158 soft bytes of one codeword (after the 18 zero positions) -> (8158 hard bits, ldpc_corr)."""
        cw = np.zeros(CW, np.int8)
        cw[:8158] = np.asarray(codeword, np.int8)[:8158]
        out = np.zeros(CW, np.uint8)
        corr = self.L["ldpc_decode"](self.h, cw.ctypes.data, out.ctypes.data, self.cfg.iterations if iterations is None else iterations)
        return out[:8158].copy(), corr


def matrix(impl=None):
    """Column indices of H's 1022 rows, 32 per row, ascending: int32 [1022, 32]."""
    cols = np.zeros((1022, 32), np.int32)
    n = lib(impl)["ldpc_matrix"](cols.ctypes.data, 1022)
    assert n == 1022, n
    return cols


def cor_of(recs):
    """correlator_corr of each record as float32."""
    return np.asarray(recs)[:, 2].astype(np.uint32).view(np.float32)
