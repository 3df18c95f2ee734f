"""TEST INFRASTRUCTURE ONLY — ctypes binding of oracle/_ref/libsatref.so (the unmodified reference
translation units + oracle/ref_harness.cpp).  See oracle/__init__.py."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "_ref", "libsatref.so")
_PFX = "ref_"

CONST = {"bpsk": 0, "qpsk": 1, "oqpsk": 2, "8psk": 3, "none": 4, "bpsk_90": 5}
FMT = {"cf32": 0, "cs16": 1, "cs8": 2}
CONV_RATE = {"1/2": 0, "2/3": 2, "3/4": 3, "5/6": 5, "7/8": 7}


class DemodCfg(C.Structure):
    _fields_ = [("samplerate", C.c_double), ("symbolrate", C.c_double), ("constellation", C.c_int),
                ("rrc_alpha", C.c_float), ("rrc_taps", C.c_int), ("pll_bw", C.c_float), ("agc_rate", C.c_float),
                ("clock_gain_omega", C.c_float), ("clock_mu", C.c_float), ("clock_gain_mu", C.c_float),
                ("clock_omega_limit", C.c_float), ("costas_max_offset", C.c_float), ("format", C.c_int),
                ("buffer_size", C.c_int), ("iq_swap", C.c_int), ("final_samplerate", C.c_double), ("dc_block", C.c_int), ("post_costas_dc", C.c_int),
                ("clock_recovery", C.c_int),
                # pm_demod (module_pm_demod.cpp) and the freq_shift option of BaseDemodModule
                ("pm", C.c_int), ("pm_pll_bw", C.c_float), ("pm_pll_max_offset", C.c_float), ("pm_resample_after_pll", C.c_int),
                ("pm_subcarrier_offset", C.c_double), ("freq_shift", C.c_double),
                ("has_carrier", C.c_int), ("carrier_pll_bw", C.c_float), ("carrier_pll_max_offset", C.c_float)]


class FecCfg(C.Structure):
    _fields_ = [("kind", C.c_int), ("constellation", C.c_int), ("cadu_size", C.c_int), ("outsync_after", C.c_int),
                ("ber_thresold", C.c_float), ("nrzm", C.c_int), ("derandomize", C.c_int), ("derand_after_rs", C.c_int),
                ("derand_start", C.c_int), ("rs_i", C.c_int), ("rs_dualbasis", C.c_int), ("rs_fill_bytes", C.c_int),
                ("rs_usecheck", C.c_int), ("rs_type", C.c_int), ("iq_invert", C.c_int), ("asm_sync", C.c_uint),
                ("qpsk_swap_iq", C.c_int), ("qpsk_swap_diff", C.c_int), ("oqpsk_delay", C.c_int), ("conv_rate", C.c_int)]


class _Prefixed:
    """Resolve ref_xxx names against a library exporting <prefix>xxx (shared by oracle.ref and oracle.port)."""

    def __init__(self, cdll, prefix):
        self._l, self._p = cdll, prefix

    def __getattr__(self, name):
        if name.startswith("ref_"):
            try:
                f = getattr(self._l, self._p + name[4:])
            except AttributeError:
                raise AttributeError(name)
            setattr(self, name, f)
            return f
        raise AttributeError(name)


def available():
    return os.path.exists(_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = _Prefixed(C.CDLL(_PATH), _PFX)
        L.ref_demod_create.restype = C.c_void_p
        L.ref_demod_create.argtypes = [C.POINTER(DemodCfg)]
        L.ref_demod_destroy.argtypes = [C.c_void_p]
        L.ref_demod_buffer_size.argtypes = [C.c_void_p]
        L.ref_demod_sps.argtypes = [C.c_void_p]
        L.ref_demod_sps.restype = C.c_float
        L.ref_demod_rrc_taps.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_mm_taps.argtypes = [C.c_void_p]
        L.ref_rrc_design.argtypes = [C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_void_p]
        L.ref_demod_run.restype = C.c_long
        L.ref_demod_run.argtypes = [C.c_void_p, C.c_void_p, C.c_long] + [C.c_void_p] * 5 + [C.c_long]
        L.ref_demod_state.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_demod_run_stage.restype = C.c_long
        L.ref_demod_run_stage.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_long, C.c_void_p, C.c_long]
        L.ref_demod_last_front.restype = C.c_long
        L.ref_demod_last_front.argtypes = [C.c_void_p]
        L.ref_demod_pm_dumps.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_demod_pm_state.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_fast_atan2f.restype = C.c_float
        L.ref_fast_atan2f.argtypes = [C.c_float, C.c_float]
        L.ref_fast_cos.restype = C.c_float
        L.ref_fast_cos.argtypes = [C.c_float]
        L.ref_fast_sin.restype = C.c_float
        L.ref_fast_sin.argtypes = [C.c_float]
        L.ref_rotator.argtypes = [C.c_void_p, C.c_long, C.c_long, C.c_double, C.c_double, C.c_void_p]
        L.ref_demux_create.restype = C.c_void_p
        L.ref_demux_create.argtypes = [C.c_int] * 4
        L.ref_demux_destroy.argtypes = [C.c_void_p]
        L.ref_demux_run.restype = C.c_long
        L.ref_demux_run.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_ulonglong, C.c_long, C.c_void_p, C.c_long, C.POINTER(C.c_long), C.c_void_p, C.c_long]
        L.ref_resample.restype = C.c_long
        L.ref_resample.argtypes = [C.POINTER(DemodCfg), C.c_void_p, C.c_long, C.c_void_p, C.c_long]
        L.ref_resampler_taps.argtypes = [C.c_uint, C.c_uint, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.ref_fec_create.restype = C.c_void_p
        L.ref_fec_create.argtypes = [C.POINTER(FecCfg)]
        L.ref_fec_destroy.argtypes = [C.c_void_p]
        L.ref_fec_chunk_size.argtypes = [C.c_void_p]
        L.ref_fec_cadu_bytes.argtypes = [C.c_void_p]
        L.ref_fec_run.restype = C.c_long
        L.ref_fec_run.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_long] + [C.c_void_p] * 7
        L.ref_rs_encode_interleaved.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.ref_rs_decode_interleaved.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.ref_derand.argtypes = [C.c_void_p, C.c_int]
        L.ref_cc_encode.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.ref_cc_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.ref_rotate_soft.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.ref_deframe.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.ref_pipeline_timed.restype = C.c_double
        L.ref_pipeline_timed.argtypes = [C.POINTER(DemodCfg), C.POINTER(FecCfg), C.c_void_p, C.c_long, C.c_void_p, C.c_long,
                                         C.POINTER(C.c_long), C.POINTER(C.c_int)]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def demod_cfg(samplerate, symbolrate, constellation, rrc_alpha, pll_bw=0.003, fmt="cs16", rrc_taps=31, agc_rate=1e-2,
              clock_alpha=None, clock_gain_omega=None, clock_mu=0.5, clock_gain_mu=8.7e-3, clock_omega_limit=0.005,
              costas_max_offset=1.0, buffer_size=0, iq_swap=False, final_samplerate=None, min_sps=None, max_sps=None, dc_block=False, post_costas_dc=False,
              clock_recovery="mm", pm=False, pm_pll_bw=0.01, pm_pll_max_offset=0.5, resample_after_pll=False, subcarrier_offset=0, freq_shift=0.0,
              has_carrier=False, carrier_pll_bw=0.001, carrier_pll_max_offset=3.14):
    """Defaults follow module_psk_demod.h:31-39 and module_demod_base.h:54. pm=True: PMDemodModule's chain (module_pm_demod.cpp:61-88; pll_bw is
    then its "costas_bw", pm_pll_bw its "pll_bw"; MAX_SPS = 10 unless max_sps is given). final_samplerate=None applies BaseDemodModule::initb's
    rule (resample when samplerate/symbolrate is outside [min_sps, max_sps]); 0 = no resampler."""
    if pm and max_sps is None:
        max_sps = 10.0  # module_pm_demod.cpp:56
    if final_samplerate is None:
        final_samplerate = final_samplerate_of(samplerate, symbolrate, constellation, min_sps, max_sps)
        if final_samplerate == float(int(samplerate)):
            final_samplerate = 0.0
    if clock_alpha is not None:  # module_psk_demod.cpp:36-41 ; DVB-S2 REC_ALPHA module_dvbs2_demod.h:49-53
        clock_gain_omega = np.float32(clock_alpha) ** 2 / 4.0
        clock_gain_mu = clock_alpha
    if clock_gain_omega is None:
        clock_gain_omega = float(np.float32(pow(8.7e-3, 2) / 4.0))
    if has_carrier and costas_max_offset == 1.0:
        costas_max_offset = 0.2  # module_psk_demod.cpp:116
    return DemodCfg(float(samplerate), float(symbolrate), CONST[constellation], rrc_alpha, rrc_taps, pll_bw, agc_rate,
                    float(clock_gain_omega), clock_mu, float(clock_gain_mu), clock_omega_limit, costas_max_offset, FMT[fmt],
                    buffer_size, int(iq_swap), float(final_samplerate), int(dc_block), int(post_costas_dc), {"mm": 0, "gardner": 1}[clock_recovery],
                    int(pm), pm_pll_bw, pm_pll_max_offset, int(resample_after_pll), float(subcarrier_offset), float(freq_shift),
                    int(has_carrier), carrier_pll_bw, carrier_pll_max_offset)


def final_samplerate_of(samplerate, symbolrate, constellation, min_sps=None, max_sps=None, custom=None):
    """BaseDemodModule::initb (module_demod_base.cpp:59-80) with its types: long d_samplerate, int d_symbolrate, float MIN_SPS /
    MAX_SPS / final_samplerate; psk_demod's OQPSK window module_psk_demod.cpp:65-70."""
    f32 = np.float32
    d_samplerate, d_symbolrate = int(samplerate), int(symbolrate)
    MIN_SPS = f32(1.6 if constellation == "oqpsk" else 1.1) if not min_sps else f32(min_sps)
    MAX_SPS = f32(2.4 if constellation == "oqpsk" else 4.0) if not max_sps else f32(max_sps)
    input_sps = f32(d_samplerate) / f32(d_symbolrate)
    resample = input_sps > MAX_SPS or input_sps < MIN_SPS
    rng = int(pow(10, len(str(d_symbolrate)) - 1))
    final = f32(d_samplerate)
    if custom:
        final = f32(int(custom))
    elif MAX_SPS == MIN_SPS:
        final = f32(d_symbolrate) * MAX_SPS
    elif input_sps > MAX_SPS:
        final = f32(float(round(d_symbolrate // rng) * rng) * float(MAX_SPS)) if resample else f32(d_samplerate)
    elif input_sps < MIN_SPS:
        final = f32(d_symbolrate) * MIN_SPS if resample else f32(d_samplerate)
    return float(final)


def metop_cfg(ber_thresold=0.28, outsync_after=10):
    return FecCfg(0, 1, 8192, outsync_after, ber_thresold, 0, 1, 0, 4, 4, 1, -1, 0, 0, 0, 0x1ACFFC1D, 0, 0, 0, 0)


def simple_cfg(constellation, cadu_size, rs_i, nrzm=False, derandomize=True, rs_usecheck=False, rs_dualbasis=True, rs_fill_bytes=-1,
               derand_after_rs=False, derand_start=4, rs_type=0, asm_sync=0x1ACFFC1D, qpsk_swap_iq=False, qpsk_swap_diff=True, oqpsk_delay=False):
    """ccsds_simple_psk_decoder (module_ccsds_simple_psk_decoder.cpp:19-44 defaults): no convolutional code."""
    return FecCfg(2, CONST[constellation], cadu_size, 0, 0.0, int(nrzm), int(derandomize), int(derand_after_rs), derand_start, rs_i,
                  int(rs_dualbasis), rs_fill_bytes, int(rs_usecheck), rs_type, 0, asm_sync, int(qpsk_swap_iq), int(qpsk_swap_diff), int(oqpsk_delay), 0)


def ccsds_cfg(constellation, cadu_size, ber_thresold, outsync_after, rs_i, nrzm=False, derandomize=True, rs_usecheck=False,
              rs_dualbasis=True, rs_fill_bytes=-1, derand_after_rs=False, derand_start=4, iq_invert=False, rs_type=0,
              asm_sync=0x1ACFFC1D, conv_rate="1/2"):
    return FecCfg(1, CONST[constellation], cadu_size, outsync_after, ber_thresold, int(nrzm), int(derandomize),
                  int(derand_after_rs), derand_start, rs_i, int(rs_dualbasis), rs_fill_bytes, int(rs_usecheck), rs_type,
                  int(iq_invert), asm_sync, 0, 0, 0, CONV_RATE[conv_rate])


class Demod:
    def __init__(self, cfg):
        self.cfg = cfg
        self.h = lib().ref_demod_create(C.byref(cfg))

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_demod_destroy(self.h)
            self.h = None

    @property
    def buffer_size(self):
        return lib().ref_demod_buffer_size(self.h)

    @property
    def sps(self):
        return lib().ref_demod_sps(self.h)

    def rrc_taps(self):
        out = np.zeros(256, np.float32)
        n = lib().ref_demod_rrc_taps(self.h, _p(out))
        return out[:n].copy()

    def state(self):
        out = np.zeros(8, np.float32)
        lib().ref_demod_state(self.h, _p(out))
        return dict(gain=out[0], phase=out[1], freq=out[2], mu=out[3], omega=out[4], inc=int(out[5]), alpha=out[6], beta=out[7])

    def run(self, raw, stages=True):
        """raw: cf32 (complex64) / cs16 (int16 pairs) / cs8 (int8 pairs) array. Returns dict of stage dumps."""
        raw = np.ascontiguousarray(raw)
        n = raw.size if self.cfg.format == 0 and np.iscomplexobj(raw) else raw.size // 2
        bps = 1 if self.cfg.constellation == 0 else 2
        ratio = self.cfg.final_samplerate / self.cfg.samplerate if self.cfg.final_samplerate > 0 else 1.0
        nf = int(n * ratio) + 64  # samples after the front-end resampler (upper bound)
        cap = int(nf / max(1.0, self.sps) * 1.1) + 64
        pm_after = bool(self.cfg.pm and self.cfg.pm_resample_after_pll)
        na = n + 64 if pm_after else nf  # pm_demod with resample_after_pll: AGC / PLL / PMToBPSK run at the input rate
        pll = pmo = None
        if self.cfg.has_carrier and stages:  # psk_demod's carrier mode: carrier PLL / DC blocker outputs (behind the RRC)
            pll, pmo = np.zeros(nf, np.complex64), np.zeros(nf, np.complex64)
            lib().ref_demod_pm_dumps(self.h, _p(pll), _p(pmo))
        if self.cfg.pm and stages:
            pll, pmo = np.zeros(na, np.complex64), np.zeros(na, np.complex64)
            lib().ref_demod_pm_dumps(self.h, _p(pll), _p(pmo))
        agc = np.zeros(na, np.complex64) if stages else None
        fir = np.zeros(nf, np.complex64) if stages else None
        cos = np.zeros(nf, np.complex64) if (stages and self.cfg.constellation != 4) else None
        mm = np.zeros(cap, np.complex64)
        soft = np.zeros(cap * bps, np.int8)
        ns = lib().ref_demod_run(self.h, _p(raw), n, _p(agc), _p(fir), _p(cos), _p(mm), _p(soft), cap)
        front = lib().ref_demod_last_front(self.h)
        cut = (lambda a: None if a is None else a[:front])
        if self.cfg.pm:
            lib().ref_demod_pm_dumps(self.h, None, None)
            cin = (lambda a: None if a is None else a[:n if pm_after else front])
            return dict(agc=cin(agc), pll=cin(pll), pm=cin(pmo), fir=cut(fir), costas=cut(cos), mm=mm[:ns].copy(), soft=soft[:ns].copy(), front=front)
        if self.cfg.has_carrier:
            lib().ref_demod_pm_dumps(self.h, None, None)
            return dict(agc=cut(agc), fir=cut(fir), pll=cut(pll), carrier_dc=cut(pmo), costas=cut(cos), mm=mm[:ns].copy(), soft=soft[:ns * bps].copy(), front=front)
        return dict(agc=cut(agc), fir=cut(fir), costas=cut(cos), mm=mm[:ns].copy(), soft=soft[:ns * bps].copy(), front=front)

    def pm_state(self):
        out = np.zeros(4, np.float32)
        lib().ref_demod_pm_state(self.h, _p(out))
        return dict(pll_phase=out[0], pll_freq=out[1], agc2_gain=out[2])


class Demux:
    """One ccsds_aos::Demuxer per virtual channel behind parseVCDU's channel id (module_metop_instruments.cpp:66-140)."""

    def __init__(self, mpdu_data_size=884, insert_zone=0, secondary_header_extends=False, vcid_mask=(1 << 63) - 1):
        self.h = lib().ref_demux_create(mpdu_data_size, int(insert_zone > 0), insert_zone, int(secondary_header_extends))
        self.mask, self.frame0 = vcid_mask, 0

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_demux_destroy(self.h)
            self.h = None

    def run(self, frames):
        """frames: uint8 [n, cadu_size]. Returns (bytes of all packets back to back: 6 header bytes + payload each, recs int32 [npackets, 4] =
        frame index, vcid, payload length, apid)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        n, size = frames.shape
        out = np.zeros(n * size + (1 << 20), np.uint8)
        recs = np.zeros((n * 130 + 16, 4), np.int32)
        nb = C.c_long(0)
        k = lib().ref_demux_run(self.h, _p(frames), n, size, self.mask, self.frame0, _p(out), out.size, C.byref(nb), _p(recs), recs.shape[0])
        if k < 0:
            raise RuntimeError("demux output capacity too small")
        self.frame0 += n
        return out[:nb.value].copy(), recs[:k].copy()


def rotator(x, inc, call=8192):
    """The VOLK rotator (oracle/shim restatement of the generic flavour) as FreqShiftBlock / PMToBPSK call it, in `call`-sample calls."""
    x = np.ascontiguousarray(x, np.complex64)
    out = np.zeros_like(x)
    lib().ref_rotator(_p(x), x.size, call, float(np.real(inc)), float(np.imag(inc)), _p(out))
    return out


def run_stage(cfg, which, x):
    """ONE block ("fir" / "costas" incl. post-Costas DC blocker and OQPSK delay / "mm") of a FRESH chain on the cf32 stage input x."""
    x = np.ascontiguousarray(x, np.complex64)
    d = Demod(cfg)
    out = np.zeros(x.size + 64, np.complex64)
    n = lib().ref_demod_run_stage(d.h, {"agc": 0, "fir": 1, "costas": 2, "mm": 5}[which], _p(x), x.size, _p(out), out.size)
    if n < 0:
        raise RuntimeError("this configuration has no such stage")
    return out[:n].copy()


class Fec:
    def __init__(self, cfg):
        self.cfg = cfg
        self.h = lib().ref_fec_create(C.byref(cfg))
        self.chunk = lib().ref_fec_chunk_size(self.h)
        self.cadu_bytes = lib().ref_fec_cadu_bytes(self.h)
        self.rate_num = 3 if cfg.kind == 0 else 1  # decoded bits per 2 soft (x rate)

    def __del__(self):
        if getattr(self, "h", None):
            lib().ref_fec_destroy(self.h)
            self.h = None

    def run(self, soft):
        soft = np.ascontiguousarray(soft, np.int8)
        nch = soft.size // self.chunk
        bits_per_chunk = self.chunk * 3 // 4 if self.cfg.kind == 0 else (self.chunk if (self.cfg.kind == 2 or self.cfg.conv_rate) else self.chunk // 2)
        cap = (nch * bits_per_chunk // max(1, self.cfg.cadu_size) + 2) * self.cadu_bytes
        cadu = np.zeros(cap, np.uint8)
        vs = np.zeros(nch, np.int32)
        vb = np.zeros(nch, np.float32)
        ds = np.zeros(nch, np.int32)
        bits = np.zeros(nch * bits_per_chunk + 8, np.uint8)
        rs_i = max(1, self.cfg.rs_i)
        rse = np.zeros((cap // self.cadu_bytes + 2) * rs_i, np.int32)
        nbits = C.c_long(0)
        nfr = C.c_long(0)
        w = lib().ref_fec_run(self.h, _p(soft), soft.size, _p(cadu), cap, _p(vs), _p(vb), _p(ds), _p(bits), C.byref(nbits),
                              _p(rse), C.byref(nfr))
        return dict(cadu=cadu[:w].copy(), vit_state=vs, vit_ber=vb, defr_state=ds, bits=bits[:nbits.value].copy(),
                    rs_err=rse[:nfr.value * rs_i].reshape(-1, rs_i).copy(), nframes=nfr.value)


def resample(cfg, raw):
    """Conversion (+ iq_swap) and the front-end SmartResamplerBlock alone, on a fresh resampler."""
    raw = np.ascontiguousarray(raw)
    n = raw.size if cfg.format == 0 and np.iscomplexobj(raw) else raw.size // 2
    ratio = cfg.final_samplerate / cfg.samplerate if cfg.final_samplerate > 0 else 1.0
    out = np.zeros(int(n * ratio) + 64, np.complex64)
    m = lib().ref_resample(C.byref(cfg), _p(raw), n, _p(out), out.size)
    if m < 0:
        raise RuntimeError("resampling ratio needs the power-of-two decimator (not restated)")
    return out[:m].copy()


def resampler_taps(interpolation, decimation):
    """Polyphase bank of RationalResamplerBlock(interpolation, decimation): array [arms, taps per arm]."""
    out = np.zeros(1 << 20, np.float32)
    nf = C.c_int(0)
    nt = lib().ref_resampler_taps(interpolation, decimation, _p(out), out.size, C.byref(nf))
    return out[:nf.value * nt].reshape(nf.value, nt).copy()


def rrc_design(gain, fs, rs, alpha, ntaps):
    out = np.zeros(ntaps + 2, np.float32)
    n = lib().ref_rrc_design(gain, fs, rs, alpha, ntaps, _p(out))
    return out[:n].copy()


def mm_taps():
    out = np.zeros(128 * 8, np.float32)
    lib().ref_mm_taps(_p(out))
    return out.reshape(128, 8)


def rs_encode_interleaved(data, dual=True, interleave=4, rs_type=0):
    d = np.ascontiguousarray(data, np.uint8).copy()
    lib().ref_rs_encode_interleaved(_p(d), int(dual), interleave, rs_type)
    return d


def rs_decode_interleaved(data, dual=True, interleave=4, rs_type=0, fill_bytes=-1):
    # with fill_bytes -1 ReedSolomon's (de)interleave loops run 256 rows (255 - fill_bytes): the decoder reads and writes one byte per
    # codeword past the 255 * interleave bytes, so the buffer gets that many spare bytes. They are dropped here: what comes back in them
    # (the corrected first message byte of each word that decodes, the byte as it was for one that does not) is tested through Fec with
    # CADUs longer than 4 + 255 * interleave
    d = np.zeros(np.asarray(data).size + interleave, np.uint8)
    d[:np.asarray(data).size] = np.ascontiguousarray(data, np.uint8).reshape(-1)
    err = np.zeros(interleave, np.int32)
    lib().ref_rs_decode_interleaved(_p(d), int(dual), interleave, rs_type, fill_bytes, _p(err))
    return d[:d.size - interleave].reshape(np.shape(data)), err


def derand(data):
    d = np.ascontiguousarray(data, np.uint8).copy()
    lib().ref_derand(_p(d), d.size)
    return d


def cc_encode(bits):
    b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros(2 * b.size, np.uint8)
    lib().ref_cc_encode(_p(b), b.size, _p(out))
    return out


def cc_decode(syms, frame, ncalls):
    s = np.ascontiguousarray(syms, np.uint8)
    assert s.size >= ncalls * 2 * frame + 12
    out = np.zeros(ncalls * frame, np.uint8)
    lib().ref_cc_decode(_p(s), frame, ncalls, _p(out))
    return out


def rotate_soft(soft, phase, iqswap=False):
    s = np.ascontiguousarray(soft, np.int8).copy()
    lib().ref_rotate_soft(_p(s), s.size, phase, int(iqswap))
    return s


def deframe(bits, cadu_size=8192, state_synced=12):
    b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros((b.size // cadu_size + 2) * (cadu_size // 8), np.uint8)
    n = lib().ref_deframe(_p(b), b.size, cadu_size, state_synced, _p(out))
    return out[:n * (cadu_size // 8)].reshape(n, cadu_size // 8).copy()


def pipeline_timed(dcfg, fcfg, raw):
    """The reference's own threaded execution model (one thread per block). Returns (seconds, cadu bytes, threads)."""
    raw = np.ascontiguousarray(raw)
    n = raw.size if dcfg.format == 0 and np.iscomplexobj(raw) else raw.size // 2
    cap = int(n * 0.2) + 65536
    cadu = np.zeros(cap, np.uint8)
    nb = C.c_long(0)
    nt = C.c_int(0)
    secs = lib().ref_pipeline_timed(C.byref(dcfg), C.byref(fcfg) if fcfg is not None else None, _p(raw), n, _p(cadu), cap, C.byref(nb), C.byref(nt))
    return secs, cadu[:nb.value].copy(), nt.value


def snr_m2m4(symbols, chunk=11667):
    """M2M4SNREstimator of the reference over complex64 symbols, updated every `chunk` symbols like PSKDemodModule::process; returns
    (snr after the last update, peak) in dB."""
    x = np.ascontiguousarray(symbols, np.complex64)
    out = np.zeros(4, np.float32)
    L = C.CDLL(_PATH)
    L.ref_snr_m2m4.argtypes = [C.c_void_p, C.c_long, C.c_long, C.c_void_p]
    L.ref_snr_m2m4(x.ctypes.data, x.size, chunk, out.ctypes.data)
    return float(out[0]), float(out[1])
