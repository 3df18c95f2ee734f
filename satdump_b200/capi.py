"""ctypes binding of the C ABI in include/b200dsp.h (libb200dsp.so, built in satdump_b200/csrc).

This is the same boundary a SatDump plugin links (see INTEGRATION.md); Python is only the test/bench driver.
There is no fallback of any kind: if the library is missing the import of `lib()` raises, and without an H100 every
create() fails with B200_ENODEV.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200dsp.so")

CONST = {"bpsk": 0, "qpsk": 1, "oqpsk": 2, "8psk": 3, "none": 4, "bpsk_90": 5}
FMT = {"cf32": 0, "cs16": 1, "cs8": 2}
FMT_BYTES = {0: 8, 1: 4, 2: 2}
CKPT = 512  # samples between the repair checkpoints of the loop kernels (demod.cuh)
E_NAMES = {0: "OK", -1: "EINVAL", -2: "ENODEV", -3: "ECUDA", -4: "ENOMEM", -5: "ESTATE", -6: "EUNSUPPORTED"}

# every symbol include/b200dsp.h declares (tests check the built library exports all of them)
SYMBOLS = [
    "b200_last_error", "b200_device_count", "b200_demod_final_samplerate", "b200_demod_resample_decision", "b200_demod_resampler_bank",
    "b200_demod_create", "b200_demod_destroy", "b200_demod_push_iq", "b200_demod_push_iq_device", "b200_demod_pull_soft",
    "b200_demod_pull_symbols", "b200_demod_debug_stage", "b200_demod_debug_convert", "b200_demod_debug_run_stage", "b200_demod_debug_junctions", "b200_demod_debug_repair_merge", "b200_demod_debug_shape", "b200_demod_debug_loop_cycles", "b200_demod_reset", "b200_demod_prefetch_iq", "b200_demod_last_timing", "b200_demod_get_stats", "b200_demod_get_taps",
    "b200_fec_create", "b200_fec_destroy", "b200_fec_push_soft", "b200_fec_push_soft_device", "b200_fec_pull_frames",
    "b200_fec_debug_bits", "b200_fec_get_stats", "b200_fec_cadu_bytes", "b200_fec_chunk_size", "b200_fec_debug_ldpc_frames", "b200_fec_ldpc_timing",
    "b200_fec_debug_turbo_frames", "b200_fec_debug_turbo_llr", "b200_fec_turbo_timing", "b200_fec_debug_dump_frames", "b200_fec_debug_meteor_frames",
    "b200_fec_debug_hrpt_frames", "b200_fec_frame_bits", "b200_fec_debug_fengyun_reads",
    "b200_chain_create", "b200_chain_destroy", "b200_chain_push_iq", "b200_chain_push_iq_device", "b200_chain_prefetch_iq", "b200_chain_pull_frames",
    "b200_chain_frames_device", "b200_chain_get_stats", "b200_chain_last_timing", "b200_chain_reset",
    "b200_chain_set_pipelined", "b200_chain_sync", "b200_chain_span_begin", "b200_chain_span_end",
    "b200_demux_create", "b200_demux_destroy", "b200_demux_push_frames", "b200_demux_push_frames_device", "b200_demux_pull", "b200_demux_reset",
    "b200_demux_get_stats",
]


class DemodCfg(C.Structure):
    _fields_ = [("samplerate", C.c_double), ("symbolrate", C.c_double), ("constellation", C.c_int), ("rrc_alpha", C.c_float),
                ("rrc_taps", C.c_int), ("pll_bw", C.c_float), ("agc_rate", C.c_float), ("clock_gain_omega", C.c_float),
                ("clock_mu", C.c_float), ("clock_gain_mu", C.c_float), ("clock_omega_limit", C.c_float),
                ("costas_max_offset", C.c_float), ("format", C.c_int), ("device", C.c_int), ("max_batch", C.c_long),
                ("keep_stages", C.c_int), ("iq_swap", C.c_int), ("final_samplerate", C.c_double), ("dc_block", C.c_int), ("post_costas_dc", C.c_int),
                ("front_resample", C.c_int), ("clock_recovery", C.c_int),
                ("pm_demod", C.c_int), ("pm_pll_bw", C.c_float), ("pm_pll_max_offset", C.c_float), ("pm_resample_after_pll", C.c_int),
                ("pm_subcarrier_offset", C.c_double), ("freq_shift", C.c_double),
                ("has_carrier", C.c_int), ("carrier_pll_bw", C.c_float), ("carrier_pll_max_offset", C.c_float), ("fsk_demod", C.c_int)]


class FecCfg(C.Structure):
    _fields_ = [("kind", C.c_int), ("constellation", C.c_int), ("cadu_size", C.c_int), ("outsync_after", C.c_int),
                ("ber_thresold", C.c_float), ("nrzm", C.c_int), ("derandomize", C.c_int), ("derand_after_rs", C.c_int),
                ("derand_start", C.c_int), ("rs_i", C.c_int), ("rs_dualbasis", C.c_int), ("rs_fill_bytes", C.c_int),
                ("rs_usecheck", C.c_int), ("rs_type", C.c_int), ("iq_invert", C.c_int), ("asm_sync", C.c_uint),
                ("device", C.c_int), ("max_soft", C.c_long), ("qpsk_swap_iq", C.c_int), ("qpsk_swap_diff", C.c_int), ("oqpsk_delay", C.c_int), ("conv_rate", C.c_int),
                ("ldpc_rate", C.c_int), ("ldpc_block_size", C.c_int), ("ldpc_iterations", C.c_int), ("ldpc2", C.c_int), ("internal_stream", C.c_int),
                ("internal_cadu_size", C.c_int), ("turbo_rate", C.c_int), ("turbo_base", C.c_int), ("turbo_iters", C.c_int),
                ("diff_decode", C.c_int), ("m2x_mode", C.c_int), ("interleaved", C.c_int), ("deframer_thresold", C.c_int),
                ("backward", C.c_int), ("instrument_type", C.c_int), ("invert_second_viterbi", C.c_int)]


class DemuxCfg(C.Structure):
    _fields_ = [("cadu_size", C.c_int), ("mpdu_data_size", C.c_int), ("has_insert_zone", C.c_int), ("insert_zone_size", C.c_int),
                ("secondary_header_extends", C.c_int), ("vcid_mask", C.c_ulonglong), ("device", C.c_int), ("max_frames", C.c_long), ("max_packets", C.c_long)]


class Packet(C.Structure):
    _fields_ = [("offset", C.c_long), ("payload_len", C.c_int), ("frame", C.c_int), ("vcid", C.c_short), ("apid", C.c_short)]


class DemuxStats(C.Structure):
    _fields_ = [("frames_in", C.c_long), ("packets_out", C.c_long), ("kernel_launches", C.c_long), ("redone_channels", C.c_long)]


class DemodStats(C.Structure):
    _fields_ = [("samples_in", C.c_long), ("symbols_out", C.c_long), ("agc_gain", C.c_float), ("costas_phase", C.c_float),
                ("costas_freq", C.c_float), ("mm_mu", C.c_float), ("mm_omega", C.c_float), ("costas_unconverged", C.c_long),
                ("mm_unconverged", C.c_long), ("agc_clamped", C.c_int), ("repairs", C.c_int), ("kernel_launches", C.c_long),
                ("agc_exact_passes", C.c_long), ("last_front_samples", C.c_long), ("snr", C.c_float), ("peak_snr", C.c_float),
                ("pll_freq", C.c_float), ("pll_unconverged", C.c_long), ("repair_merge_hist", C.c_int * 8),
                ("last_range_tiles", C.c_int)]


class FecStats(C.Structure):
    _fields_ = [("soft_in", C.c_long), ("chunks", C.c_long), ("bits_out", C.c_long), ("frames_out", C.c_long),
                ("viterbi_state", C.c_int), ("viterbi_ber", C.c_float), ("deframer_state", C.c_int), ("rs_corrected", C.c_long),
                ("rs_failed", C.c_long), ("replays", C.c_long), ("kernel_launches", C.c_long), ("start_redone", C.c_long), ("tb_serial", C.c_long),
                ("spec_steps", C.c_int), ("tb_overlap", C.c_int),
                ("correlator_lock", C.c_int), ("correlator_corr", C.c_float), ("ldpc_corr", C.c_int), ("ldpc_resyncs", C.c_long),
                ("crc_ok", C.c_long), ("crc_fail", C.c_long), ("turbo_near_ties", C.c_long), ("rs_avg", C.c_int),
                ("viterbi2_state", C.c_int), ("viterbi2_ber", C.c_float)]


class LdpcFrame(C.Structure):
    _fields_ = [("offset", C.c_long), ("pos", C.c_int), ("cor", C.c_float), ("phase", C.c_int), ("swap", C.c_int), ("ldpc_corr", C.c_int)]


class TurboFrame(C.Structure):
    _fields_ = [("offset", C.c_long), ("pos", C.c_int), ("cor", C.c_float), ("swapped", C.c_int), ("crc_ok", C.c_int)]


class DumpFrame(C.Structure):
    _fields_ = [("offset", C.c_long), ("pos", C.c_int), ("corr", C.c_int), ("phase", C.c_int), ("swap", C.c_int), ("rs", C.c_int * 4)]


class MeteorFrame(C.Structure):
    _fields_ = [("offset", C.c_long), ("pos", C.c_int), ("corr", C.c_int), ("phase", C.c_int), ("swap", C.c_int), ("rs", C.c_int * 4),
                ("ber", C.c_float)]


class HrptFrame(C.Structure):
    _fields_ = [("bit", C.c_long), ("inverted", C.c_int), ("state", C.c_int)]


class FengyunRead(C.Structure):
    _fields_ = [("read", C.c_long), ("shift", C.c_int), ("invert_branches", C.c_int), ("v1", C.c_int), ("v2", C.c_int), ("state1", C.c_int),
                ("state2", C.c_int), ("ber1", C.c_float), ("ber2", C.c_float), ("deframer_state", C.c_int), ("pad", C.c_int)]


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{E_NAMES.get(code, code)}: {msg}")
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no fallback exists)")
        L = C.CDLL(LIB_PATH)
        vp, ci, cl = C.c_void_p, C.c_int, C.c_long
        L.b200_last_error.restype = C.c_char_p
        L.b200_demod_create.restype = vp
        L.b200_demod_final_samplerate.restype = C.c_double
        L.b200_demod_final_samplerate.argtypes = [C.c_double, C.c_double, ci, C.c_float, C.c_float, C.c_double]
        L.b200_demod_resample_decision.argtypes = [C.c_double, C.c_double, ci, C.c_float, C.c_float]
        L.b200_demod_resampler_bank.argtypes = [C.c_double, C.c_double, vp, cl, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)]
        L.b200_demod_create.argtypes = [C.POINTER(DemodCfg)]
        L.b200_demod_destroy.argtypes = [vp]
        L.b200_demod_push_iq.argtypes = [vp, vp, cl]
        L.b200_demod_push_iq_device.argtypes = [vp, vp, cl]
        L.b200_demod_pull_soft.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_demod_pull_symbols.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_demod_debug_stage.argtypes = [vp, ci, vp, cl]
        L.b200_demod_debug_convert.argtypes = [vp, vp, cl, vp]
        L.b200_demod_debug_run_stage.argtypes = [vp, ci, vp, cl, ci, vp, cl, C.POINTER(cl)]
        L.b200_demod_debug_junctions.argtypes = [vp, vp, vp, cl, C.POINTER(cl), C.POINTER(cl)]
        L.b200_demod_get_stats.argtypes = [vp, C.POINTER(DemodStats)]
        L.b200_demod_debug_repair_merge.argtypes = [vp, ci]
        L.b200_demod_debug_shape.argtypes = [vp, ci, ci, ci]
        L.b200_demod_reset.argtypes = [vp]
        L.b200_demod_prefetch_iq.argtypes = [vp, vp, cl]
        L.b200_demod_last_timing.argtypes = [vp, vp, ci]
        L.b200_demod_get_taps.argtypes = [vp, vp, ci, vp]
        L.b200_fec_create.restype = vp
        L.b200_fec_create.argtypes = [C.POINTER(FecCfg)]
        L.b200_fec_destroy.argtypes = [vp]
        L.b200_fec_push_soft.argtypes = [vp, vp, cl]
        L.b200_fec_push_soft_device.argtypes = [vp, vp, cl]
        L.b200_fec_pull_frames.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_fec_debug_bits.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_fec_get_stats.argtypes = [vp, C.POINTER(FecStats)]
        L.b200_fec_cadu_bytes.argtypes = [vp]
        L.b200_fec_chunk_size.argtypes = [vp]
        L.b200_fec_debug_ldpc_frames.argtypes = [vp, C.POINTER(LdpcFrame), cl, C.POINTER(cl)]
        L.b200_fec_ldpc_timing.argtypes = [vp, vp, ci]
        L.b200_fec_debug_turbo_frames.argtypes = [vp, C.POINTER(TurboFrame), cl, C.POINTER(cl)]
        L.b200_fec_turbo_timing.argtypes = [vp, vp, ci]
        L.b200_fec_debug_turbo_llr.argtypes = [vp, cl, vp, vp, cl, C.POINTER(cl)]
        L.b200_fec_debug_dump_frames.argtypes = [vp, C.POINTER(DumpFrame), cl, C.POINTER(cl)]
        L.b200_fec_debug_meteor_frames.argtypes = [vp, C.POINTER(MeteorFrame), cl, C.POINTER(cl)]
        L.b200_fec_debug_hrpt_frames.argtypes = [vp, C.POINTER(HrptFrame), cl, C.POINTER(cl)]
        L.b200_fec_frame_bits.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_fec_debug_fengyun_reads.argtypes = [vp, C.POINTER(FengyunRead), cl, C.POINTER(cl)]
        L.b200_chain_create.restype = vp
        L.b200_chain_create.argtypes = [C.POINTER(DemodCfg), C.POINTER(FecCfg)]
        L.b200_chain_destroy.argtypes = [vp]
        L.b200_chain_push_iq.argtypes = [vp, vp, cl]
        L.b200_chain_push_iq_device.argtypes = [vp, vp, cl]
        L.b200_chain_prefetch_iq.argtypes = [vp, vp, cl]
        L.b200_chain_pull_frames.argtypes = [vp, vp, cl, C.POINTER(cl)]
        L.b200_chain_frames_device.argtypes = [vp, C.POINTER(vp), C.POINTER(cl)]
        L.b200_chain_get_stats.argtypes = [vp, C.POINTER(DemodStats), C.POINTER(FecStats)]
        L.b200_chain_last_timing.argtypes = [vp, vp, ci]
        L.b200_chain_reset.argtypes = [vp]
        L.b200_demux_create.restype = vp
        L.b200_demux_create.argtypes = [C.POINTER(DemuxCfg)]
        L.b200_demux_destroy.argtypes = [vp]
        L.b200_demux_push_frames.argtypes = [vp, vp, cl]
        L.b200_demux_push_frames_device.argtypes = [vp, vp, cl]
        L.b200_demux_pull.argtypes = [vp, vp, cl, C.POINTER(cl), vp, cl, C.POINTER(cl)]
        L.b200_demux_reset.argtypes = [vp]
        L.b200_demux_get_stats.argtypes = [vp, C.POINTER(DemuxStats)]
        L.b200_chain_set_pipelined.argtypes = [vp, ci]
        L.b200_chain_sync.argtypes = [vp]
        L.b200_chain_span_begin.argtypes = [vp]
        L.b200_chain_span_end.argtypes = [vp, C.POINTER(C.c_float)]
        _lib = L
    return _lib


def last_error():
    return lib().b200_last_error().decode()


def _chk(rc):
    if rc != 0:
        raise B200Error(rc, last_error())


def loop_cycles():
    """Cycle counters of the loop kernels' main passes since the previous call (a library built with -DB200_LOOP_CYCLES only):
    {"k_costas": [wait, loop, copy-out, tail, warps], "k_mm": [wait, fix-up, symbols, copy-out, warps]}, cycles summed over warps."""
    out = (C.c_ulonglong * 10)()
    f = lib().b200_demod_debug_loop_cycles  # (looked up here: tools/profile_loops.py --lib also loads builds that predate it)
    f.argtypes = [C.c_void_p, C.c_int]
    _chk(f(out, 10))
    return {"k_costas": list(out[0:5]), "k_mm": list(out[5:10])}


def demod_cfg(samplerate, symbolrate, constellation, rrc_alpha, pll_bw=0.003, fmt="cs16", rrc_taps=31, agc_rate=1e-2, clock_alpha=None,
              clock_gain_omega=None, clock_mu=0.5, clock_gain_mu=8.7e-3, clock_omega_limit=0.005, costas_max_offset=1.0, device=0,
              max_batch=1 << 24, keep_stages=False, iq_swap=False, final_samplerate=None, min_sps=0.0, max_sps=0.0, dc_block=False, post_costas_dc=False,
              front_resample=0, clock_recovery="mm", pm=False, pm_pll_bw=0.01, pm_pll_max_offset=0.5, resample_after_pll=False, subcarrier_offset=0,
              freq_shift=0.0, has_carrier=False, carrier_pll_bw=0.001, carrier_pll_max_offset=3.14, fsk_demod=False):
    """Parameter defaults = module_psk_demod.h:31-39, module_demod_base.h:54. final_samplerate=None applies BaseDemodModule::initb's
    rule (resample when samplerate/symbolrate is outside [min_sps, max_sps]); 0 forces "no resampler". pm=True: pm_demod's chain
    (module_pm_demod.cpp; pll_bw is then its "costas_bw", pm_pll_bw its "pll_bw", MAX_SPS = 10)."""
    if pm and not max_sps:
        max_sps = 10.0  # module_pm_demod.cpp:56
    if has_carrier and costas_max_offset == 1.0:
        costas_max_offset = 0.2  # module_psk_demod.cpp:116
    if final_samplerate is None:
        final_samplerate = final_samplerate_of(samplerate, symbolrate, constellation, min_sps, max_sps)
        if final_samplerate == float(int(samplerate)):
            final_samplerate = 0.0
    if clock_alpha is not None:
        clock_gain_omega = float(np.float32(clock_alpha) ** 2 / 4.0)
        clock_gain_mu = clock_alpha
    if clock_gain_omega is None:
        clock_gain_omega = float(np.float32(pow(8.7e-3, 2) / 4.0))
    return DemodCfg(float(samplerate), float(symbolrate), CONST[constellation], rrc_alpha, rrc_taps, pll_bw, agc_rate, clock_gain_omega,
                    clock_mu, clock_gain_mu, clock_omega_limit, costas_max_offset, FMT[fmt], device, max_batch, int(keep_stages), int(iq_swap),
                    float(final_samplerate), int(dc_block), int(post_costas_dc), int(front_resample), {"mm": 0, "gardner": 1}[clock_recovery],
                    int(pm), pm_pll_bw, pm_pll_max_offset, int(resample_after_pll), float(subcarrier_offset), float(freq_shift),
                    int(has_carrier), carrier_pll_bw, carrier_pll_max_offset, int(fsk_demod))


# FSKDemodModule's clock defaults (module_fsk_demod.h:28-31), as the module's float members hold them
FSK_CLOCK_GAIN_OMEGA = float(np.float32(pow(1.7e-2, 2) / 4.0))
FSK_CLOCK_GAIN_MU = float(np.float32(1.7e-2))


def fsk_demod_kwargs(samplerate, symbolrate, rrc_alpha, fmt="cs16", clock_alpha=None, clock_gain_omega=None, clock_mu=None, clock_gain_mu=None,
                     clock_omega_relative_limit=None, rrc_taps=31):
    """demod_cfg arguments of fsk_demod (module_fsk_demod.cpp:13-57): the module's defaults, "clock_alpha" setting gain_omega = alpha^2 / 4
    and gain_mu = alpha, then the explicit gains over it, in the constructor's order. The working rate is BaseDemodModule::initb's for the
    base window [1.1, 4.0] samples per symbol."""
    if rrc_alpha is None:
        raise ValueError("RRC Alpha parameter must be present!")
    gain_omega, gain_mu = FSK_CLOCK_GAIN_OMEGA, FSK_CLOCK_GAIN_MU
    if clock_alpha is not None:  # the module parses a float and squares it exactly in double before the float member rounds it
        a = np.float32(clock_alpha)
        gain_omega, gain_mu = float(np.float32(np.float64(a) ** 2 / 4.0)), float(a)
    if clock_gain_omega is not None:
        gain_omega = float(np.float32(clock_gain_omega))
    if clock_gain_mu is not None:
        gain_mu = float(np.float32(clock_gain_mu))
    return dict(samplerate=samplerate, symbolrate=symbolrate, constellation="bpsk", rrc_alpha=rrc_alpha, rrc_taps=rrc_taps, fmt=fmt,
                clock_gain_omega=gain_omega, clock_gain_mu=gain_mu, clock_mu=0.5 if clock_mu is None else clock_mu,
                clock_omega_limit=0.005 if clock_omega_relative_limit is None else clock_omega_relative_limit, fsk_demod=True)


def fsk_demod_cfg(samplerate, symbolrate, rrc_alpha, fmt="cs16", device=0, max_batch=1 << 24, clock_alpha=None, clock_gain_omega=None, clock_mu=None,
                  clock_gain_mu=None, clock_omega_relative_limit=None, rrc_taps=31, **kw):
    """fsk_demod's chain as a b200_demod_cfg (fsk_demod_kwargs); kw: the BaseDemodModule parameters of demod_cfg."""
    return demod_cfg(**fsk_demod_kwargs(samplerate, symbolrate, rrc_alpha, fmt, clock_alpha, clock_gain_omega, clock_mu, clock_gain_mu,
                                        clock_omega_relative_limit, rrc_taps), device=device, max_batch=max_batch, **kw)


def resampler_bank(samplerate, final_samplerate):
    """Polyphase bank of the front-end resampler for (samplerate -> final_samplerate): array [arms, taps per arm], reduced (I, D)."""
    out = np.zeros(1 << 20, np.float32)
    nt, i, d = C.c_int(0), C.c_int(0), C.c_int(0)
    _chk(lib().b200_demod_resampler_bank(float(samplerate), float(final_samplerate), out.ctypes.data, out.size, C.byref(nt), C.byref(i), C.byref(d)))
    return out[:i.value * nt.value].reshape(i.value, nt.value).copy(), i.value, d.value


def final_samplerate_of(samplerate, symbolrate, constellation, min_sps=0.0, max_sps=0.0, custom=0.0):
    """BaseDemodModule::initb's working sample rate (module_demod_base.cpp:59-87)."""
    return lib().b200_demod_final_samplerate(float(samplerate), float(symbolrate), CONST[constellation], min_sps, max_sps, custom)


def metop_cfg(ber_thresold=0.28, outsync_after=10, device=0, max_soft=1 << 24):
    return FecCfg(0, 1, 8192, outsync_after, ber_thresold, 0, 1, 0, 4, 4, 1, -1, 0, 0, 0, 0x1ACFFC1D, device, max_soft, 0, 0, 0)


def simple_cfg(constellation, cadu_size, rs_i, nrzm=False, derandomize=True, rs_usecheck=False, rs_dualbasis=True, rs_fill_bytes=-1,
               derand_after_rs=False, derand_start=4, rs_type=0, asm_sync=0x1ACFFC1D, qpsk_swap_iq=False, qpsk_swap_diff=True, oqpsk_delay=False,
               device=0, max_soft=1 << 24):
    """ccsds_simple_psk_decoder (module_ccsds_simple_psk_decoder.cpp:19-44 defaults): soft symbols -> deframer(s) -> RS, no convolutional code."""
    return FecCfg(2, CONST[constellation], cadu_size, 0, 0.0, int(nrzm), int(derandomize), int(derand_after_rs), derand_start, rs_i,
                  int(rs_dualbasis), rs_fill_bytes, int(rs_usecheck), rs_type, 0, asm_sync, device, max_soft, int(qpsk_swap_iq),
                  int(qpsk_swap_diff), int(oqpsk_delay))


def ccsds_cfg(constellation, cadu_size, ber_thresold, outsync_after, rs_i, nrzm=False, derandomize=True, rs_usecheck=False, rs_dualbasis=True,
              rs_fill_bytes=-1, derand_after_rs=False, derand_start=4, iq_invert=False, rs_type=0, asm_sync=0x1ACFFC1D, device=0,
              max_soft=1 << 24, conv_rate="1/2"):
    return FecCfg(1, CONST[constellation], cadu_size, outsync_after, ber_thresold, int(nrzm), int(derandomize), int(derand_after_rs),
                  derand_start, rs_i, int(rs_dualbasis), rs_fill_bytes, int(rs_usecheck), rs_type, int(iq_invert), asm_sync, device, max_soft,
                  0, 0, 0, {"1/2": 0, "2/3": 2, "3/4": 3, "5/6": 5, "7/8": 7}[conv_rate])


LDPC_RATES = {"1/2": 1, "2/3": 2, "4/5": 4, "7/8": 7}


def ldpc_cfg(constellation, ldpc_rate="7/8", ldpc_iterations=10, derandomize=True, internal_stream=False, internal_cadu_size=0,
             internal_asm=0x1ACFFC1D, ldpc_block_size=0, ldpc2=False, device=0, max_soft=1 << 24):
    """ccsds_ldpc_decoder (module_ccsds_ldpc_decoder.cpp:19-124). Built: ldpc_rate "7/8" (the C2 code) without internal_stream; the
    library refuses the other options by name."""
    if ldpc_rate not in LDPC_RATES:
        raise ValueError(f"Invalid LDPC code rate {ldpc_rate}")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.derandomize, cfg.asm_sync, cfg.device, cfg.max_soft = 3, CONST[constellation], int(derandomize), internal_asm, device, max_soft
    cfg.cadu_size = internal_cadu_size if internal_stream else 8192  # bits of one output frame
    cfg.ldpc_rate, cfg.ldpc_block_size, cfg.ldpc_iterations, cfg.ldpc2 = LDPC_RATES[ldpc_rate], ldpc_block_size, ldpc_iterations, int(ldpc2)
    cfg.internal_stream, cfg.internal_cadu_size = int(internal_stream), internal_cadu_size
    return cfg


TURBO_RATES = {"1/2": 2, "1/3": 3, "1/4": 4, "1/6": 6}


def turbo_cfg(turbo_rate=None, turbo_base=None, turbo_iters=None, device=0, max_soft=1 << 24):
    """ccsds_turbo_decoder (module_ccsds_turbo_decoder.cpp:17-135): all three parameters are required, as the module's constructor asks.
    The library refuses an unknown rate or base and turbo_iters < 1 by name."""
    if turbo_rate is None:
        raise ValueError("Turbo Rate is required!")
    if turbo_base is None:
        raise ValueError("Turbo Base is required!")
    if turbo_iters is None:
        raise ValueError("Turbo Iters is required!")
    cfg = FecCfg()
    cfg.kind, cfg.device, cfg.max_soft = 4, device, max_soft
    cfg.turbo_rate = TURBO_RATES.get(turbo_rate, -1) if isinstance(turbo_rate, str) else int(turbo_rate)
    cfg.turbo_base, cfg.turbo_iters = int(turbo_base), int(turbo_iters)
    return cfg


def dump_cfg(device=0, max_soft=1 << 24):
    """metop_dump_decoder (module_metop_dump_decoder.cpp): the module takes no parameters."""
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 5, CONST["qpsk"], 8192, device, max_soft
    return cfg


def meteor_lrpt_cfg(diff_decode=None, m2x_mode=False, viterbi_outsync_after=None, viterbi_ber_thresold=None, interleaved=False, device=0,
                    max_soft=1 << 24):
    """meteor_lrpt_decoder (module_meteor_lrpt_decoder.cpp:22-49): diff_decode is required; with m2x_mode, viterbi_outsync_after and
    viterbi_ber_thresold are required too, as the module's constructor asks. The library refuses interleaved (not built) by name."""
    if diff_decode is None:
        raise ValueError("meteor_lrpt_decoder: diff_decode is required")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 6, CONST["qpsk"], 8192, device, max_soft
    cfg.diff_decode, cfg.m2x_mode, cfg.interleaved = int(bool(diff_decode)), int(bool(m2x_mode)), int(bool(interleaved))
    if m2x_mode:
        if viterbi_outsync_after is None:
            raise ValueError("meteor_lrpt_decoder: viterbi_outsync_after is required with m2x_mode")
        if viterbi_ber_thresold is None:
            raise ValueError("meteor_lrpt_decoder: viterbi_ber_thresold is required with m2x_mode")
        cfg.outsync_after, cfg.ber_thresold = int(viterbi_outsync_after), float(viterbi_ber_thresold)
    return cfg


def noaa_hrpt_cfg(deframer_thresold=None, device=0, max_soft=1 << 24):
    """noaa_hrpt_decoder (module_noaa_hrpt_decoder.cpp:14-20): deframer_thresold is required, as the module reads it without a default.
    The output unit is one 10-bit word (cadu_bytes 2: the .raw16 file's little-endian uint16)."""
    if deframer_thresold is None:
        raise ValueError("noaa_hrpt_decoder: deframer_thresold is required")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 7, CONST["bpsk"], 16, device, max_soft
    cfg.deframer_thresold = int(deframer_thresold)
    return cfg


def meteor_hrpt_cfg(device=0, max_soft=1 << 24):
    """meteor_hrpt_decoder (module_meteor_hrpt_decoder.cpp): the module takes no parameters; 1024-byte CADUs."""
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 8, CONST["bpsk"], 8192, device, max_soft
    return cfg


def terra_db_demod_kwargs(samplerate, symbolrate, fmt="cs16"):
    """demod_cfg arguments of terra_db_demod (module_terra_db_demod.cpp:21-31): psk_demod's BPSK chain at twice the symbol rate (RRC alpha
    0.5, Costas bw 0.004 with a 1 MHz frequency limit, M&M gains pow(0.001, 2) / 4 and 0.001, mu 0.5, limit 1e-4; soft = clamp(real * 50)),
    at the working rate BaseDemodModule::initb picks for the real symbol rate. Raises ValueError, naming samplerate, when that rate gives
    fewer than 1.1 samples per half-symbol."""
    work = final_samplerate_of(samplerate, symbolrate, "bpsk")
    if np.float32(work) / np.float32(2 * int(symbolrate)) < np.float32(1.1):
        raise ValueError(f"terra_db_demod: samplerate {int(work)} gives fewer than 1.1 samples per half-symbol at symbolrate {int(symbolrate)}")
    return dict(samplerate=samplerate, symbolrate=2 * int(symbolrate), constellation="bpsk", rrc_alpha=0.5, pll_bw=0.004, fmt=fmt,
                clock_gain_omega=float(np.float32(pow(0.001, 2) / 4.0)), clock_mu=0.5, clock_gain_mu=0.001, clock_omega_limit=1e-4,
                costas_max_offset=float(np.float32(2.0 * np.pi * (1e6 / work))),
                final_samplerate=0.0 if work == float(int(samplerate)) else work)


def terra_db_demod_cfg(samplerate, symbolrate, fmt="cs16", device=0, max_batch=1 << 24, **kw):
    """terra_db_demod's chain as a b200_demod_cfg (terra_db_demod_kwargs)."""
    return demod_cfg(**terra_db_demod_kwargs(samplerate, symbolrate, fmt), device=device, max_batch=max_batch, **kw)


def aqua_db_cfg(device=0, max_soft=1 << 24):
    """aqua_db_decoder (module_aqua_db_decoder.cpp, Aqua and Aura DB): the module takes no parameters; 1024-byte CADUs, every frame
    written whatever RS returned."""
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 9, CONST["qpsk"], 8192, device, max_soft
    return cfg


def noaa_gac_cfg(backward=None, device=0, max_soft=1 << 24):
    """noaa_gac_decoder (module_noaa_gac_decoder.cpp:17): backward is required, as the module reads it without a default. 4159-byte
    frames; with backward each frame's bits come out reversed (the reversal of the frame order is the file writer's)."""
    if backward is None:
        raise ValueError("noaa_gac_decoder: backward is required")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 10, CONST["bpsk"], 33270, device, max_soft
    cfg.backward = int(bool(backward))
    return cfg


def dmsp_rtd_cfg(device=0, max_soft=1 << 24):
    """dmsp_rtd_decoder (module_dmsp_rtd_decoder.cpp): no decoder parameters (start_timestamp is the file writer's); 19-byte frames."""
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.cadu_size, cfg.device, cfg.max_soft = 11, CONST["bpsk"], 150, device, max_soft
    return cfg


METEOR_XBAND_TYPES = {"mtvza": 0, "kmss_bpsk": 1}


def meteor_xband_cfg(instrument_type=None, device=0, max_soft=1 << 24):
    """meteor_xband_decoder (module_meteor_xband_decoder.cpp, meteor_xband_types.h): instrument_type "mtvza" (380-byte frames) or
    "kmss_bpsk" (60160-byte frames: the four lanes of one frame) is required, as the module refuses anything else."""
    if instrument_type not in METEOR_XBAND_TYPES:
        raise ValueError("Invalid METEOR instrument type!")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.device, cfg.max_soft = 12, CONST["bpsk"], device, max_soft
    cfg.instrument_type = METEOR_XBAND_TYPES[instrument_type]
    return cfg


def fengyun_ahrpt_cfg(viterbi_outsync_after=None, viterbi_ber_thresold=None, invert_second_viterbi=None, device=0, max_soft=1 << 24):
    """fengyun_ahrpt_decoder (module_fengyun_ahrpt_decoder.cpp:17-20): viterbi_outsync_after, viterbi_ber_thresold and
    invert_second_viterbi are all required, as the module reads them with no default."""
    for name, v in (("viterbi_outsync_after", viterbi_outsync_after), ("viterbi_ber_thresold", viterbi_ber_thresold),
                    ("invert_second_viterbi", invert_second_viterbi)):
        if v is None:
            raise ValueError(f"fengyun_ahrpt_decoder: {name} is required")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.device, cfg.max_soft = 13, CONST["qpsk"], device, max_soft
    cfg.outsync_after, cfg.ber_thresold, cfg.invert_second_viterbi = int(viterbi_outsync_after), float(viterbi_ber_thresold), int(bool(invert_second_viterbi))
    return cfg


def fengyun_mpt_cfg(viterbi_outsync_after=None, viterbi_ber_thresold=None, device=0, max_soft=1 << 24):
    """fengyun_mpt_decoder (module_fengyun_mpt_decoder.cpp:17-20): viterbi_outsync_after and viterbi_ber_thresold are both required, as
    the module reads them with no default. The module has no invert_second_viterbi (its Q branch is always complemented)."""
    for name, v in (("viterbi_outsync_after", viterbi_outsync_after), ("viterbi_ber_thresold", viterbi_ber_thresold)):
        if v is None:
            raise ValueError(f"fengyun_mpt_decoder: {name} is required")
    cfg = FecCfg()
    cfg.kind, cfg.constellation, cfg.device, cfg.max_soft = 14, CONST["qpsk"], device, max_soft
    cfg.outsync_after, cfg.ber_thresold = int(viterbi_outsync_after), float(viterbi_ber_thresold)
    return cfg


def dmsp_timestamps(bits, start_timestamp, read_bits_seen=None):
    """dmsp_rtd_decoder's "_timestamps.txt" values for frames completed at stream bits `bits` (b200_fec_frame_bits): start +
    8192 * (reads of 8192 soft bytes from the stream's start that produced frames, up to the frame's) / 1.024e6. read_bits_seen carries
    the count and the last read across calls: a dict, updated."""
    st = read_bits_seen if read_bits_seen is not None else {}
    n, last = st.get("n", 0), st.get("last", -1)
    out = []
    for b in np.asarray(bits, np.int64).tolist():
        r = b // 8192
        if r != last:
            n, last = n + 1, r
        out.append(start_timestamp + float(n * 8192) / 1.024e6)
    st["n"], st["last"] = n, last
    return out


def fec_cfg_for(sig, max_soft, device=0):
    """The decoder configuration that goes with a satdump_b200.synth.SignalCfg (metop_ahrpt_decoder / ccsds_conv_concat_decoder /
    ccsds_simple_psk_decoder parameters of the shipped pipeline JSONs)."""
    if sig.decoder == "metop":
        return metop_cfg(sig.ber_thresold, sig.outsync_after, device=device, max_soft=max_soft)
    if sig.decoder == "dump":
        return dump_cfg(device=device, max_soft=max_soft)
    if sig.decoder == "meteor":
        return meteor_lrpt_cfg(sig.nrzm, device=device, max_soft=max_soft)
    if sig.decoder == "noaa_hrpt":
        return noaa_hrpt_cfg(sig.deframer_thresold, device=device, max_soft=max_soft)
    if sig.decoder == "meteor_hrpt":
        return meteor_hrpt_cfg(device=device, max_soft=max_soft)
    if sig.decoder == "aqua_db":
        return aqua_db_cfg(device=device, max_soft=max_soft)
    if sig.decoder == "noaa_gac":
        return noaa_gac_cfg(sig.backward, device=device, max_soft=max_soft)
    if sig.decoder == "dmsp_rtd":
        return dmsp_rtd_cfg(device=device, max_soft=max_soft)
    if sig.decoder == "fengyun_ahrpt":
        return fengyun_ahrpt_cfg(sig.outsync_after, sig.ber_thresold, sig.invert_second_viterbi, device=device, max_soft=max_soft)
    if sig.decoder == "fengyun_mpt":
        return fengyun_mpt_cfg(sig.outsync_after, sig.ber_thresold, device=device, max_soft=max_soft)
    if sig.decoder in ("meteor_mtvza", "meteor_kmss_bpsk"):
        return meteor_xband_cfg("mtvza" if sig.decoder == "meteor_mtvza" else "kmss_bpsk", device=device, max_soft=max_soft)
    if sig.decoder == "turbo":
        return turbo_cfg(sig.turbo_rate, sig.turbo_base, sig.turbo_iters, device=device, max_soft=max_soft)
    if sig.decoder == "ldpc":
        return ldpc_cfg(sig.constellation, internal_stream=bool(sig.internal_cadu_size), internal_cadu_size=sig.internal_cadu_size,
                        internal_asm=sig.internal_asm, device=device, max_soft=max_soft)
    if sig.decoder == "simple":
        return simple_cfg(sig.constellation, (4 + 255 * sig.interleave) * 8, sig.interleave, nrzm=sig.nrzm, qpsk_swap_iq=sig.constellation == "qpsk",
                          device=device, max_soft=max_soft)
    return ccsds_cfg(sig.constellation, (4 + 255 * sig.interleave) * 8, sig.ber_thresold, sig.outsync_after, sig.interleave, nrzm=sig.nrzm,
                     rs_usecheck=sig.rs_usecheck, device=device, max_soft=max_soft, conv_rate=sig.conv[1:] if sig.conv.startswith("p") else "1/2")


def demod_cfg_for(sig, max_batch, device=0, **kw):
    """psk_demod parameters of a satdump_b200.synth.SignalCfg (decoder "none": the Costas-less DVB-S2 front half)."""
    extra = dict(clock_alpha=sig.clock_alpha) if sig.clock_alpha else {}
    if sig.post_costas_dc:
        extra["post_costas_dc"] = True
    return demod_cfg(sig.samplerate, sig.symbolrate, sig.constellation if sig.decoder != "none" else "none", sig.rrc_alpha, sig.pll_bw, sig.fmt,
                     device=device, max_batch=max_batch, **extra, **kw)


def _nsamples(raw, fmt):
    raw = np.ascontiguousarray(raw)
    if fmt == 0:
        return raw, (raw.size if np.iscomplexobj(raw) else raw.size // 2)
    return raw, raw.size // 2


def _struct_dict(s):
    return {k: list(v) if isinstance(v, C.Array) else v for k, v in ((k, getattr(s, k)) for k, _ in s._fields_)}


STAGES = {"agc": 0, "fir": 1, "costas": 2, "resamp": 3, "dc": 4, "mm": 5, "pll": 6, "pm": 7, "quad": 8, "dc2": 9, "agc2": 10}


class Demod:
    """Host mirror of PSKDemodModule's DSP chain for one stream (module_psk_demod.cpp:86-236)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.h = lib().b200_demod_create(C.byref(cfg))
        if not self.h:
            raise B200Error(-1 if "device" not in last_error().lower() else -2, last_error())
        self.bps = 1 if cfg.constellation == 0 else 2
        self.pm = bool(cfg.pm_demod)
        self.fsk = bool(cfg.fsk_demod)

    def close(self):
        if getattr(self, "h", None):
            lib().b200_demod_destroy(self.h)
            self.h = None

    __del__ = close

    def push(self, raw):
        raw, n = _nsamples(raw, self.cfg.format)
        _chk(lib().b200_demod_push_iq(self.h, raw.ctypes.data, n))
        self._n = n
        return self

    def push_device(self, ptr, n):
        _chk(lib().b200_demod_push_iq_device(self.h, ptr, n))
        self._n = n
        return self

    def push_ptr(self, host_ptr, n):
        _chk(lib().b200_demod_push_iq(self.h, host_ptr, n))
        self._n = n
        return self

    def prefetch_ptr(self, host_ptr, n):
        _chk(lib().b200_demod_prefetch_iq(self.h, host_ptr, n))
        return self

    def reset(self):
        _chk(lib().b200_demod_reset(self.h))
        return self

    def repair_merge(self, enable):
        """Test hook: False makes every repair run its whole segment (tolerance 0 for meeting the stored run)."""
        _chk(lib().b200_demod_debug_repair_merge(self.h, 1 if enable else 0))
        return self

    def debug_shape(self, range_tiles=0, seg_len=0, keep_front=False):
        """Test hook: force the AGC + RRC kernel's range length (tiles) and the loop kernels' segment length (0: production rules);
        keep_front makes stage("fir") return the production front kernel's output. stats()["last_range_tiles"] and junctions()[2]
        report what the last push ran."""
        _chk(lib().b200_demod_debug_shape(self.h, int(range_tiles), int(seg_len), 1 if keep_front else 0))
        return self

    def timing(self):
        ms = np.zeros(4, np.float32)
        _chk(lib().b200_demod_last_timing(self.h, ms.ctypes.data, 4))
        return dict(zip(["stages_sum", "agc_fir", "costas", "mm"], ms.tolist()))

    def pull_symbols_into(self, host_ptr, cap_symbols):
        """Symbols of the last push straight into caller memory (complex64); returns the symbol count."""
        n = C.c_long(0)
        _chk(lib().b200_demod_pull_symbols(self.h, host_ptr, cap_symbols, C.byref(n)))
        return n.value

    def soft(self):
        cap = int(self._n * self.bps) + 1024
        out = np.zeros(cap, np.int8)
        n = C.c_long(0)
        _chk(lib().b200_demod_pull_soft(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def symbols(self):
        """complex64 symbols of the last push; fsk_demod: float32, one per symbol."""
        cap = int(self._n) + 1024
        out = np.zeros(cap, np.float32 if self.fsk else np.complex64)
        n = C.c_long(0)
        _chk(lib().b200_demod_pull_symbols(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def stage(self, which):
        """agc / fir / costas stage outputs, or resamp = what entered the AGC when the front-end resampler / iq_swap runs."""
        n = self._n if which == "dc" else self.stats()["last_front_samples"]
        if self.pm and self.cfg.pm_resample_after_pll and which in ("agc", "pll", "pm"):
            n = self._n  # pm_demod with resample_after_pll: the first AGC, the carrier PLL and PMToBPSK run at the input rate
        real = self.fsk and which in ("quad", "dc2", "agc2", "fir")
        out = np.zeros(n, np.float32 if real else np.complex64)
        _chk(lib().b200_demod_debug_stage(self.h, STAGES[which], out.ctypes.data, n))
        return out

    def run_stage(self, which, x, strict=False, sequential=False):
        """Stage-isolated parity hook: ONE stage ("fir" / "costas" / "mm") of a freshly reset demodulator on the cf32 stage input x.
        fsk_demod: "quad" (complex input), "dc2", "agc2", "fir", "mm" on float32 input, float32 output."""
        real_in = self.fsk and which != "quad"
        x = np.ascontiguousarray(x, np.float32 if real_in else np.complex64)
        out = np.zeros(x.size + 1024, np.float32 if self.fsk else np.complex64)
        n = C.c_long(0)
        _chk(lib().b200_demod_debug_run_stage(self.h, STAGES[which], x.ctypes.data, x.size,
                                              (1 if strict else 0) | (2 if sequential else 0), out.ctypes.data, out.size, C.byref(n)))
        return out[:n.value].copy()

    def junctions(self):
        """Junction residuals of the last push / run_stage: (costas [nseg, 2] phase / frequency, mm [nseg] sampling instant, segment length)."""
        cap = 1 << 22
        c, m = np.zeros(2 * cap), np.zeros(cap)
        ns, L = C.c_long(0), C.c_long(0)
        _chk(lib().b200_demod_debug_junctions(self.h, c.ctypes.data, m.ctypes.data, cap, C.byref(ns), C.byref(L)))
        return c[:2 * ns.value].reshape(-1, 2).copy(), m[:ns.value].copy(), L.value

    def convert(self, raw):
        raw, n = _nsamples(raw, self.cfg.format)
        out = np.zeros(n, np.complex64)
        _chk(lib().b200_demod_debug_convert(self.h, raw.ctypes.data, n, out.ctypes.data))
        return out

    def stats(self):
        s = DemodStats()
        _chk(lib().b200_demod_get_stats(self.h, C.byref(s)))
        return _struct_dict(s)

    def taps(self):
        rrc = np.zeros(64, np.float32)
        bank = np.zeros(128 * 8, np.float32)
        _chk(lib().b200_demod_get_taps(self.h, rrc.ctypes.data, 64, bank.ctypes.data))
        return rrc[:self.cfg.rrc_taps | 1].copy(), bank.reshape(128, 8)


class Fec:
    """Host mirror of MetOpAHRPTDecoderModule / CCSDSConvConcatDecoderModule for one stream."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.h = lib().b200_fec_create(C.byref(cfg))
        if not self.h:
            raise B200Error(-1 if "device" not in last_error().lower() else -2, last_error())
        self.cadu_bytes = lib().b200_fec_cadu_bytes(self.h)
        self.chunk = lib().b200_fec_chunk_size(self.h)

    def close(self):
        if getattr(self, "h", None):
            lib().b200_fec_destroy(self.h)
            self.h = None

    __del__ = close

    def push(self, soft):
        soft = np.ascontiguousarray(soft, np.int8)
        _chk(lib().b200_fec_push_soft(self.h, soft.ctypes.data, soft.size))
        self._n = soft.size
        return self

    def push_device(self, dev_ptr, n):
        """n soft bytes already in device memory of the decoder's device"""
        _chk(lib().b200_fec_push_soft_device(self.h, dev_ptr, n))
        self._n = n
        return self

    def frames(self):
        cap = int(self._n) + 65536 + 4 * self.cadu_bytes  # (meteor_xband_decoder: a byte that completes a read may release its frames)
        out = np.zeros(cap, np.uint8)
        n = C.c_long(0)
        _chk(lib().b200_fec_pull_frames(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].reshape(-1, self.cadu_bytes).copy()

    def bits(self):
        cap = int(self._n) + self.chunk
        out = np.zeros(cap, np.uint8)
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_bits(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def stats(self):
        s = FecStats()
        _chk(lib().b200_fec_get_stats(self.h, C.byref(s)))
        return _struct_dict(s)

    def ldpc_frames(self):
        """ccsds_ldpc_decoder: one record per frame of the last push (LdpcFrame fields) as int64 [n, 7] = offset, pos, cor (float32 bits),
        phase, swap, ldpc_corr, correlator_locked."""
        cap = int(self._n) // 8192 + 4
        recs = (LdpcFrame * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_ldpc_frames(self.h, recs, cap, C.byref(n)))
        out = np.zeros((n.value, 7), np.int64)
        for k in range(n.value):
            r = recs[k]
            out[k] = [r.offset, r.pos, int(np.float32(r.cor).view(np.uint32)), r.phase, r.swap, r.ldpc_corr, int(r.pos == 0)]
        return out

    def turbo_frames(self):
        """ccsds_turbo_decoder: one record per frame of the last push as int64 [n, 6] = offset, pos, cor (float32 bits), swapped, crc_ok,
        correlator_locked."""
        cap = int(self._n) // 1000 + 4
        recs = (TurboFrame * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_turbo_frames(self.h, recs, cap, C.byref(n)))
        out = np.zeros((n.value, 6), np.int64)
        for k in range(n.value):
            r = recs[k]
            out[k] = [r.offset, r.pos, int(np.float32(r.cor).view(np.uint32)), r.swapped, r.crc_ok, int(r.pos == 0)]
        return out

    def dump_frames(self):
        """metop_dump_decoder: one record per frame of the last push as int64 [n, 9] = offset, pos, corr, phase, swap, rs[0..3]
        (oracle.dump.REC)."""
        cap = int(self._n) // 8192 + 4
        recs = (DumpFrame * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_dump_frames(self.h, recs, cap, C.byref(n)))
        out = np.zeros((n.value, 9), np.int64)
        for k in range(n.value):
            r = recs[k]
            out[k] = [r.offset, r.pos, r.corr, r.phase, r.swap, *r.rs]
        return out

    def meteor_frames(self):
        """meteor_lrpt_decoder (m2x_mode false): one record per frame of the last push as int64 [n, 10] = offset, pos, corr, phase, swap,
        rs[0..3], ber (float32 bits) (oracle.meteor.REC)."""
        cap = int(self._n) // 16384 + 4
        recs = (MeteorFrame * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_meteor_frames(self.h, recs, cap, C.byref(n)))
        out = np.zeros((n.value, 10), np.int64)
        for k in range(n.value):
            r = recs[k]
            out[k] = [r.offset, r.pos, r.corr, r.phase, r.swap, *r.rs, int(np.float32(r.ber).view(np.uint32))]
        return out

    def hrpt_frames(self):
        """noaa_hrpt_decoder / meteor_hrpt_decoder: one record per sync accepted in the last push as int64 [n, 3] = stream bit of the
        sync's last bit, inverted, accepting state (oracle.hrpt)."""
        cap = int(self._n) // 8000 + 8
        recs = (HrptFrame * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_hrpt_frames(self.h, recs, cap, C.byref(n)))
        return np.array([[recs[k].bit, recs[k].inverted, recs[k].state] for k in range(n.value)], np.int64).reshape(-1, 3)

    def fengyun_reads(self):
        """fengyun_ahrpt_decoder / fengyun_mpt_decoder: one record per 16384-byte read the last push completed, as float64 [n, 9] = shift,
        invert_branches, v1, v2, viterbi1 state, viterbi2 state, viterbi1 ber, viterbi2 ber, deframer state after the read (the records of
        oracle.fengyun and oracle.fengyun_mpt)"""
        cap = int(self._n) // 16384 + 4
        recs = (FengyunRead * cap)()
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_fengyun_reads(self.h, recs, cap, C.byref(n)))
        f = ("shift", "invert_branches", "v1", "v2", "state1", "state2", "ber1", "ber2", "deframer_state")
        return np.array([[getattr(recs[k], x) for x in f] for k in range(n.value)], np.float64).reshape(-1, len(f))

    def frame_bits(self):
        """noaa_gac_decoder / dmsp_rtd_decoder: the stream bit that completed each frame of the last frames() pull, as int64"""
        cap = int(getattr(self, "_n", 0)) // 100 + 1024
        out = np.zeros(cap, np.int64)
        n = C.c_long(0)
        _chk(lib().b200_fec_frame_bits(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def turbo_llr(self, frame, K):
        """ccsds_turbo_decoder: the a-priori arrays (input 0, input 1) of a frame of the last push after its last iteration."""
        a0, a1 = np.zeros(K), np.zeros(K)
        n = C.c_long(0)
        _chk(lib().b200_fec_debug_turbo_llr(self.h, frame, a0.ctypes.data, a1.ctypes.data, K, C.byref(n)))
        return a0, a1

    def turbo_timing(self):
        """ccsds_turbo_decoder: device milliseconds of the last push: correlation, walk, gather, BCJR, pack + CRC + compaction, whole push."""
        ms = np.zeros(6, np.float32)
        _chk(lib().b200_fec_turbo_timing(self.h, ms.ctypes.data, 6))
        return dict(zip(["corr", "walk", "gather", "bcjr", "pack", "push"], ms.tolist()))

    def timing(self):
        """ccsds_ldpc_decoder: device milliseconds of the last push: correlation, walk, gather, decode (+ repack), whole push."""
        ms = np.zeros(5, np.float32)
        _chk(lib().b200_fec_ldpc_timing(self.h, ms.ctypes.data, 5))
        return dict(zip(["corr", "walk", "gather", "decode", "push"], ms.tolist()))


class Chain:
    """Demodulator + decoder of one stream on one GPU; the soft stream stays in HBM."""

    def __init__(self, dcfg, fcfg):
        self.dcfg, self.fcfg = dcfg, fcfg
        self.h = lib().b200_chain_create(C.byref(dcfg), C.byref(fcfg))
        if not self.h:
            raise B200Error(-1 if "device" not in last_error().lower() else -2, last_error())
        self.cadu_bytes = (fcfg.cadu_size + 7) // 8 if fcfg.kind in (1, 3, 7) else (fcfg.turbo_base + 4 if fcfg.kind == 4 else 1024)
        if fcfg.kind in (10, 11):  # noaa_gac_decoder, dmsp_rtd_decoder: (cadu_size + padding) / 8
            self.cadu_bytes = 4159 if fcfg.kind == 10 else 19
        if fcfg.kind == 12:  # meteor_xband_decoder
            self.cadu_bytes = 60160 if fcfg.instrument_type == 1 else 380

    def close(self):
        if getattr(self, "h", None):
            lib().b200_chain_destroy(self.h)
            self.h = None

    __del__ = close

    def push(self, raw):
        raw, n = _nsamples(raw, self.dcfg.format)
        _chk(lib().b200_chain_push_iq(self.h, raw.ctypes.data, n))
        self._n = n
        return self

    def push_ptr(self, host_ptr, n):
        _chk(lib().b200_chain_push_iq(self.h, host_ptr, n))
        self._n = n
        return self

    def push_device(self, dev_ptr, n):
        _chk(lib().b200_chain_push_iq_device(self.h, dev_ptr, n))
        self._n = n
        return self

    def prefetch_ptr(self, host_ptr, n):
        _chk(lib().b200_chain_prefetch_iq(self.h, host_ptr, n))
        return self

    def frames(self, cap=None):
        cap = cap or int(self._n) + 65536
        out = np.zeros(cap, np.uint8)
        n = C.c_long(0)
        _chk(lib().b200_chain_pull_frames(self.h, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].reshape(-1, self.cadu_bytes).copy()

    def pull_into(self, host_ptr, cap):
        """CADUs since the last pull straight into caller memory (no numpy temporaries); returns the byte count."""
        n = C.c_long(0)
        _chk(lib().b200_chain_pull_frames(self.h, host_ptr, cap, C.byref(n)))
        return n.value

    def frames_device(self):
        p = C.c_void_p(0)
        n = C.c_long(0)
        _chk(lib().b200_chain_frames_device(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def stats(self):
        d, f = DemodStats(), FecStats()
        _chk(lib().b200_chain_get_stats(self.h, C.byref(d), C.byref(f)))
        return _struct_dict(d), _struct_dict(f)

    def timing(self):
        ms = np.zeros(9, np.float32)
        _chk(lib().b200_chain_last_timing(self.h, ms.ctypes.data, 9))
        return dict(zip(["stages_sum", "agc_fir", "costas", "mm", "viterbi", "deframe_rs", "k_vit_acs", "vit_chunks", "push_events"], ms.tolist()))

    def set_pipelined(self, on=True):
        """Decoder on a worker thread / own stream, one batch behind the demodulator; frames of a push appear after the next one
        (or after sync())."""
        _chk(lib().b200_chain_set_pipelined(self.h, 1 if on else 0))
        return self

    def sync(self):
        _chk(lib().b200_chain_sync(self.h))

    def span_begin(self):
        _chk(lib().b200_chain_span_begin(self.h))

    def span_end(self):
        ms = C.c_float()
        _chk(lib().b200_chain_span_end(self.h, C.byref(ms)))
        return ms.value

    def reset(self):
        _chk(lib().b200_chain_reset(self.h))
        return self


class Demux:
    """CADUs -> CCSDS space packets: one ccsds_aos::Demuxer per selected virtual channel (module_metop_instruments.cpp:66-140)."""

    def __init__(self, cadu_size=1024, mpdu_data_size=884, insert_zone=0, secondary_header_extends=False, vcid_mask=(1 << 63) - 1, device=0,
                 max_frames=1 << 16, max_packets=0):
        self.cfg = DemuxCfg(cadu_size, mpdu_data_size, int(insert_zone > 0), insert_zone, int(secondary_header_extends), vcid_mask, device, max_frames,
                            max_packets)
        self.h = lib().b200_demux_create(C.byref(self.cfg))
        if not self.h:
            raise B200Error(-1 if "device" not in last_error().lower() else -2, last_error())

    def close(self):
        if getattr(self, "h", None):
            lib().b200_demux_destroy(self.h)
            self.h = None

    __del__ = close

    def _pull(self, nframes):
        cap_b = nframes * 2 * self.cfg.mpdu_data_size + (1 << 23) + (self.cfg.max_packets or 8 * self.cfg.max_frames + 1024) * 6
        cap_p = self.cfg.max_packets or 8 * self.cfg.max_frames + 1024
        out = np.zeros(cap_b, np.uint8)
        pk = (Packet * cap_p)()
        nb, npk = C.c_long(0), C.c_long(0)
        _chk(lib().b200_demux_pull(self.h, out.ctypes.data, cap_b, C.byref(nb), C.addressof(pk), cap_p, C.byref(npk)))
        a = np.frombuffer(pk, dtype=np.dtype([("offset", "<i8"), ("payload_len", "<i4"), ("frame", "<i4"), ("vcid", "<i2"), ("apid", "<i2"), ("pad", "<i4")]),
                          count=npk.value)
        recs = np.stack([a["frame"], a["vcid"], a["payload_len"], a["apid"], a["offset"]], axis=1).astype(np.int64)  # frame, vcid, payload length, apid, offset
        return out[:nb.value].copy(), recs

    def run(self, frames):
        """frames: uint8 [n, cadu_size] on the host. Returns (packet bytes back to back, recs int64 [npackets, 5] = frame, vcid, payload length,
        apid, offset) like oracle.ref.Demux.run (whose recs carry the first four columns)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        _chk(lib().b200_demux_push_frames(self.h, frames.ctypes.data, frames.shape[0]))
        return self._pull(frames.shape[0])

    def run_device(self, dev_ptr, nframes):
        _chk(lib().b200_demux_push_frames_device(self.h, dev_ptr, nframes))
        return self._pull(nframes)

    def reset(self):
        _chk(lib().b200_demux_reset(self.h))

    def stats(self):
        s = DemuxStats()
        _chk(lib().b200_demux_get_stats(self.h, C.byref(s)))
        return _struct_dict(s)
