"""TEST INFRASTRUCTURE ONLY — ctypes bindings of the checker of the FSK demodulator (fsk_demod):

  oracle/_ref/libsatref_fsk.so: the unmodified reference blocks + oracle/fsk_harness.cpp (oracle/Makefile)

QuadratureDemodBlock's atan2f is glibc's (atan2_mode(0)) or the correctly rounded one (atan2_mode(1), the default: what the GPU computes).
"""
import ctypes as C

import numpy as np

from ._checker import Handle, Library, ref_path

STREAM_BUFFER_SIZE = 1000000  # dsp::STREAM_BUFFER_SIZE (common/dsp/buffer.cpp)

vp, cl, ci, cf = C.c_void_p, C.c_long, C.c_int, C.c_float
lib = Library({"ref": (ref_path("fsk"), "ref_")},
              [("fsk_atan2_mode", None, [ci]), ("fsk_atan2f", cf, [cf, cf]), ("fsk_create", vp, [cf, ci, cf, ci, cf, cf, cf, cf, cf, ci]),
               ("fsk_destroy", None, [vp]), ("fsk_run", ci, [vp, vp, cl, vp, vp, vp, vp, vp, cl, vp, vp, cl, vp, cl, vp, vp]),
               ("fsk_run_stage", cl, [vp, ci, vp, cl, vp, cl]), ("fsk_taps", ci, [vp, vp, ci, vp]), ("fsk_snr", None, [vp, vp, ci, vp])])
available = lib.available


def atan2_mode(correctly_rounded):
    lib()["fsk_atan2_mode"](1 if correctly_rounded else 0)


def atan2f(y, x):
    """QuadratureDemodBlock's atan2f as the harness currently resolves it."""
    f = lib()["fsk_atan2f"]
    return np.array([f(float(a), float(b)) for a, b in zip(np.ravel(y), np.ravel(x))], np.float32)


def snr(blocks):
    """The reference's M2M4SNREstimator over float symbol blocks, each one update of its complex pairs (an odd last symbol dropped), as
    FSKDemodModule feeds it per read: the snr after every block."""
    sym = np.ascontiguousarray(np.concatenate(blocks), np.float32)
    sizes = np.array([b.size for b in blocks], np.int64)
    out = np.zeros(len(blocks), np.float32)
    lib()["fsk_snr"](sym.ctypes.data, sizes.ctypes.data, len(blocks), out.ctypes.data)
    return out


def buffer_size_for(samplerate):
    """BaseDemodModule's read size (module_demod_base.cpp:25)."""
    return min(STREAM_BUFFER_SIZE, max(8192 + 1, int(samplerate) // 200))


class Fsk(Handle):
    """FSKDemodModule's chain behind BaseDemodModule's AGC, from the cfg of satdump_b200.capi.fsk_demod_cfg; run() may be called repeatedly
    (the stream continues)."""

    def __init__(self, cfg, buffer_size=None):
        fs = cfg.final_samplerate if cfg.final_samplerate > 0 else cfg.samplerate
        super().__init__(lib(), "fsk", float(np.float32(fs)), int(cfg.symbolrate), cfg.rrc_alpha, cfg.rrc_taps, cfg.agc_rate, cfg.clock_gain_omega,
                         cfg.clock_mu, cfg.clock_gain_mu, cfg.clock_omega_limit, buffer_size or buffer_size_for(cfg.samplerate))

    def run(self, iq):
        """iq: complex64 samples as the reader hands them on. Returns the stage outputs (agc complex64; quad, dc2, agc2, fir float32), the
        symbols (float32), the soft bytes, the snr after every read and (snr, peak_snr) after the call."""
        iq = np.ascontiguousarray(iq, np.complex64)
        n = iq.size
        agc = np.zeros(n, np.complex64)
        st = {k: np.zeros(n, np.float32) for k in ("quad", "dc2", "agc2", "fir")}
        cap_sym = n + 1024
        sym, soft = np.zeros(cap_sym, np.float32), np.zeros(cap_sym, np.int8)
        snr = np.zeros(n // 8192 + 16, np.float32)
        counts, stats = np.zeros(7, np.int64), np.zeros(2, np.float32)
        rc = self.L["fsk_run"](self.h, iq.ctypes.data, n, agc.ctypes.data, st["quad"].ctypes.data, st["dc2"].ctypes.data, st["agc2"].ctypes.data,
                               st["fir"].ctypes.data, n, sym.ctypes.data, soft.ctypes.data, cap_sym, snr.ctypes.data, snr.size, counts.ctypes.data,
                               stats.ctypes.data)
        assert rc == 0
        ns, reads = int(counts[5]), int(counts[6])
        return dict(agc=agc, **st, sym=sym[:ns].copy(), soft=soft[:ns].copy(), snr_reads=snr[:reads].copy(), snr=float(stats[0]),
                    peak_snr=float(stats[1]))

    def run_stage(self, which, x):
        """ONE block of this (fresh) chain: "quad" (complex64 input), "dc2", "agc2", "fir", "mm" (float32 input)."""
        stage = {"quad": 8, "dc2": 9, "agc2": 10, "fir": 1, "mm": 5}[which]
        x = np.ascontiguousarray(x, np.complex64 if which == "quad" else np.float32)
        out = np.zeros(x.size + 1024, np.float32)
        n = self.L["fsk_run_stage"](self.h, stage, x.ctypes.data, x.size, out.ctypes.data, out.size)
        assert n >= 0
        return out[:n].copy()

    def taps(self):
        out, om = np.zeros(64, np.float32), C.c_float(0)
        nt = self.L["fsk_taps"](self.h, out.ctypes.data, 64, C.byref(om))
        return out[:nt].copy(), om.value
