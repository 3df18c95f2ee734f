"""Synthetic CCSDS transmitter + channel: the workload generator for tests, smoke() and bench.py.

NOT part of the receive hot path (nothing here is timed or shipped as the product): it manufactures
the baseband the hot path consumes, following SURVEY.md §8(d):

  payload -> CADU (ASM 1ACFFC1D | I x RS(255,223) dual-basis, byte interleaved) -> CCSDS randomiser from byte 4
          -> [NRZ-M] -> conv. code k=7 (polys 79,109 = the reference CCEncoder convention, cc_encoder.cpp:92-104)
          -> [puncture 3/4 in MetOp order: inverse of viterbi_3_4.cpp:84-104] -> BPSK/QPSK/OQPSK mapping
          -> RRC pulse shaping at a fractional samples-per-symbol -> carrier offset/phase, clock offset, AWGN
          -> cf32 / cs16 / cs8.

All coding is written from the CCSDS definitions (GF(256) poly 0x187, generator roots alpha^(11*(112+i)),
dual basis, PN h(x)=x^8+x^7+x^5+x^3+1); tests/test_synth.py cross-checks every encoder against the
reference's own encoders (oracle/_ref) and checks that the reference receiver recovers the payload.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

ASM = bytes([0x1A, 0xCF, 0xFC, 0x1D])

# ----------------------------------------------------------------------------- GF(256), RS(255,223)
_GF_POLY = 0x187


def _gf_tables():
    exp = np.zeros(512, np.int32)
    log = np.zeros(256, np.int32)
    x = 1
    for i in range(255):
        exp[i] = x
        log[x] = i
        x <<= 1
        if x & 0x100:
            x ^= _GF_POLY
    exp[255:510] = exp[0:255]
    return exp, log


GF_EXP, GF_LOG = _gf_tables()


def gf_mul(a, b):
    a = np.asarray(a, np.int32)
    b = np.asarray(b, np.int32)
    r = GF_EXP[(GF_LOG[a] + GF_LOG[b]) % 255]
    return np.where((a == 0) | (b == 0), 0, r)


def rs_generator(nroots=32, fcr=112, gap=11):
    """g(x) = prod_i (x - alpha^(gap*(fcr+i))), returned lowest order first, g[nroots] = 1."""
    g = np.array([1], np.int32)
    for i in range(nroots):
        root = GF_EXP[(gap * (fcr + i)) % 255]
        g = np.concatenate([[0], g]) ^ np.concatenate([gf_mul(g, root), [0]])
    return g


# CCSDS dual-basis map is GF(2)-linear: images of the 8 unit vectors of the conventional basis
_TO_DUAL_BASIS_IMAGES = [0x7B, 0xAF, 0x99, 0xFA, 0x86, 0xEC, 0xEF, 0x8D]


def _dual_tables():
    to = np.zeros(256, np.uint8)
    for v in range(256):
        r = 0
        for b in range(8):
            if v >> b & 1:
                r ^= _TO_DUAL_BASIS_IMAGES[b]
        to[v] = r
    frm = np.zeros(256, np.uint8)
    frm[to] = np.arange(256, dtype=np.uint8)
    return to, frm


TO_DUAL, FROM_DUAL = _dual_tables()


def rs_encode(msg, dual=True, nroots=32):
    """msg: (ncw, 255-nroots) uint8 -> (ncw, 255) codewords (message then parity, highest order first)."""
    msg = np.asarray(msg, np.uint8)
    m = FROM_DUAL[msg] if dual else msg
    g = rs_generator(nroots, 112 if nroots == 32 else 120)
    glog = GF_LOG[g[:nroots]][::-1].copy()  # reg[0] is the highest-order remainder coefficient
    gz = (g[:nroots][::-1] == 0)
    reg = np.zeros((m.shape[0], nroots), np.int32)
    for i in range(m.shape[1]):
        fb = m[:, i].astype(np.int32) ^ reg[:, 0]
        reg = np.concatenate([reg[:, 1:], np.zeros((reg.shape[0], 1), np.int32)], axis=1)
        prod = GF_EXP[(GF_LOG[fb][:, None] + glog[None, :]) % 255]
        prod[fb == 0, :] = 0
        prod[:, gz] = 0
        reg ^= prod
    cw = np.concatenate([m, reg.astype(np.uint8)], axis=1)
    return TO_DUAL[cw] if dual else cw


def ccsds_pn(n):
    """CCSDS pseudo-randomiser bytes (h(x)=x^8+x^7+x^5+x^3+1, all-ones start), period 255 bytes... tiled to n."""
    reg = [1] * 8
    bits = []
    for _ in range(255 * 8):
        bits.append(reg[0])
        nb = reg[0] ^ reg[3] ^ reg[5] ^ reg[7]
        reg = reg[1:] + [nb]
    pn = np.packbits(np.array(bits, np.uint8))
    return np.resize(pn, n)


def build_cadus(payload, interleave, dual=True, randomize=True, nroots=32):
    """payload: (nframes, interleave*(255-nroots)) -> (nframes, 4 + interleave*255) CADUs and the clear (pre-randomiser) frames.
    nroots 32 = RS(255,223), 16 = RS(255,239)."""
    nf, k = payload.shape[0], 255 - nroots
    msg = payload.reshape(nf, k, interleave).transpose(0, 2, 1).reshape(nf * interleave, k)
    cw = rs_encode(msg, dual, nroots).reshape(nf, interleave, 255).transpose(0, 2, 1).reshape(nf, 255 * interleave)
    clear = np.concatenate([np.tile(np.frombuffer(ASM, np.uint8), (nf, 1)), cw], axis=1)
    tx = clear.copy()
    if randomize:
        tx[:, 4:] ^= ccsds_pn(255 * interleave)[None, :]
    return tx, clear


# ----------------------------------------------------------------------------- convolutional code
def conv_encode(bits):
    """k=7, polys 79 (taps 0,1,2,3,6) and 109 (taps 0,2,3,5,6), register = (state<<1)|bit, start state 0."""
    b = np.concatenate([np.zeros(6, np.uint8), np.asarray(bits, np.uint8)])
    n = b.size - 6
    s = lambda k: b[6 - k:6 - k + n]
    o0 = s(0) ^ s(1) ^ s(2) ^ s(3) ^ s(6)
    o1 = s(0) ^ s(2) ^ s(3) ^ s(5) ^ s(6)
    return np.stack([o0, o1], axis=1).reshape(-1)


def puncture_34_metop(coded):
    """From each 6 coded symbols e0..e5 transmit e0,e1,e4,e3 (inverse of Viterbi3_4::depuncture, shift=0)."""
    n = coded.size // 6 * 6
    e = coded[:n].reshape(-1, 6)
    return e[:, [0, 1, 4, 3]].reshape(-1)


# Puncturing patterns that Viterbi_Depunc undoes (src-core/common/codings/viterbi/depunc.h): which of the mother code's symbols of one
# period (C1, C2 of consecutive bits) are transmitted = the positions where its depuncturers place data rather than an erasure.
PUNCTURE_KEEP = {"p2/3": (4, [0, 1, 3]), "p3/4": (6, [0, 1, 3, 4]), "p5/6": (10, [0, 1, 3, 4, 7, 8]), "p7/8": (14, [0, 1, 3, 5, 7, 8, 11, 12])}


def puncture_dvb(coded, conv):
    period, keep = PUNCTURE_KEEP[conv]
    n = coded.size // period * period
    return coded[:n].reshape(-1, period)[:, keep].reshape(-1)


def nrzm_encode(bits):
    return (np.cumsum(bits.astype(np.int64)) & 1).astype(np.uint8)


# ----------------------------------------------------------------------------- waveform
def rrc_pulse(t, alpha):
    """Unit-energy root-raised-cosine impulse response at times t (in symbols)."""
    t = np.asarray(t, np.float64)
    out = np.empty_like(t)
    eps = 1e-9
    z = np.abs(t) < eps
    s = np.abs(np.abs(t) - 1.0 / (4 * alpha)) < eps
    r = ~(z | s)
    tr = t[r]
    out[r] = (np.sin(np.pi * tr * (1 - alpha)) + 4 * alpha * tr * np.cos(np.pi * tr * (1 + alpha))) / (np.pi * tr * (1 - (4 * alpha * tr) ** 2))
    out[z] = 1 - alpha + 4 * alpha / np.pi
    out[s] = alpha / np.sqrt(2) * ((1 + 2 / np.pi) * np.sin(np.pi / (4 * alpha)) + (1 - 2 / np.pi) * np.cos(np.pi / (4 * alpha)))
    return out


@dataclass
class SignalCfg:
    """One of the BASELINE.json configurations (SURVEY.md §8.0)."""
    name: str = "metop_ahrpt"
    samplerate: float = 6e6
    symbolrate: float = 2333333
    constellation: str = "qpsk"     # bpsk | qpsk | oqpsk
    conv: str = "3/4"               # "1/2" | "3/4" (MetOp order) | "none" | "p2/3" "p3/4" "p5/6" "p7/8" (Viterbi_Depunc's patterns)
    interleave: int = 4             # RS interleaving depth I
    nrzm: bool = False
    rrc_alpha: float = 0.5
    pll_bw: float = 0.003
    fmt: str = "cs16"
    esn0_db: float = 10.0
    carrier_rad: float = 1e-3       # rad / sample
    phase0: float = 0.7
    clock_ppm: float = 20.0
    rms: float = 0.25
    clock_alpha: float = None       # M&M gains override (DVB-S2 front half uses 1.7e-3)
    # receiver-side decoder parameters (pipeline JSON values)
    decoder: str = "metop"          # metop | ccsds | none
    ber_thresold: float = 0.28
    outsync_after: int = 10
    rs_usecheck: bool = False
    # phase-modulated residual-carrier signal for pm_demod (module_pm_demod.cpp): carrier * exp(j * pm_index * d(t) * sin(2 pi f_sc t)) with
    # d(t) the pulse-shaped BPSK stream and f_sc the subcarrier (0 = the symbol rate, the module's default for "subcarrier_offset")
    pm_index: float = 0.0           # rad; 0 = not a PM signal
    subcarrier: float = 0.0
    pm_pll_bw: float = 0.01         # receiver: carrier PLL bandwidth ("pll_bw" of pm_demod; pll_bw above is its "costas_bw")
    pm_pll_max_offset: float = 3.14
    resample_after_pll: bool = False
    # psk_demod's carrier mode ("has_carrier", module_psk_demod.cpp:93-113): BPSK phase-modulated directly onto a residual carrier
    # (pm_index * d(t), no subcarrier): carrier PLL -> DC blocker -> Costas loop
    has_carrier: bool = False
    carrier_pll_bw: float = 0.001
    # ccsds_ldpc_decoder (decoder "ldpc", rate 7/8 C2 code): 0 = the decoder writes the LDPC frames' CADUs; > 0 = "internal_stream": the info
    # bits carry inner CADUs of this many bits that start with internal_asm
    internal_cadu_size: int = 0
    internal_asm: int = 0x1ACFFC1D
    # ccsds_turbo_decoder (decoder "turbo"): "turbo_rate" 2, 3, 4, 6 = 1/2 .. 1/6, "turbo_base", "turbo_iters"; psk_demod's "post_costas_dc"
    turbo_rate: int = 2
    turbo_base: int = 1115
    turbo_iters: int = 5
    post_costas_dc: bool = False
    # noaa_hrpt_decoder's "deframer_thresold" (NOAA.json: 10)
    deframer_thresold: int = 10
    # noaa_gac_decoder's "backward" (NOAA.json "noaa_gac": false)
    backward: bool = False
    # fengyun_ahrpt_decoder's "invert_second_viterbi" (FengYun-3.json: false for A/B and C, true from D on)
    invert_second_viterbi: bool = False

    @property
    def cadu_bytes(self):
        if self.decoder == "turbo":
            return self.turbo_base + 4
        if self.decoder == "ldpc":
            return self.internal_cadu_size // 8 if self.internal_cadu_size else 1024
        return 4 + 255 * self.interleave

    @property
    def sps(self):
        return float(np.float32(np.float32(self.samplerate) / np.float32(int(self.symbolrate))))


CONFIGS = {
    # C1/C3: resources/pipelines/MetOp.json:30-47
    "metop_ahrpt": SignalCfg(),
    # C2: BPSK + r=1/2 + RS I=4 (ccsds_conv_concat_decoder), cf32 @3 MS/s, symbolrate chosen so sps=2.5 (SURVEY §8.0 C2)
    "bpsk_half": SignalCfg(name="bpsk_half", samplerate=3e6, symbolrate=1200000, constellation="bpsk", conv="1/2", interleave=4,
                           fmt="cf32", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=7.0),
    # C4: JPSS-HRD-type OQPSK r=1/2 NRZ-M RS I=5, cs16 @30 MS/s, 15 Msym/s (sps 2.0) (resources/pipelines/JPSS.json npp_hrd/jpss_hrd)
    "jpss_hrd": SignalCfg(name="jpss_hrd", samplerate=30e6, symbolrate=15000000, constellation="oqpsk", conv="1/2", interleave=5,
                          nrzm=True, pll_bw=0.002, fmt="cs16", decoder="ccsds", ber_thresold=0.3, outsync_after=20, rs_usecheck=True,
                          esn0_db=7.0),
    # C2 at the real NOAA HRPT rate: 665.4 kbaud @ 3 MS/s = 4.51 samples/symbol > MAX_SPS, so BaseDemodModule's front-end resampler
    # runs first (module_demod_base.cpp:66-80,203-204): 3 MS/s -> 2.4 MS/s (4/5), 3.607 samples/symbol
    "hrpt_bpsk": SignalCfg(name="hrpt_bpsk", samplerate=3e6, symbolrate=665400, constellation="bpsk", conv="1/2", interleave=4,
                           fmt="cf32", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=7.0),
    # a narrow-roll-off QPSK stream recorded too slowly: 2.4 Msym/s @ 2.6 MS/s = 1.083 samples/symbol < MIN_SPS -> interpolated to
    # 2.64 MS/s (66/65). Exercises the interpolating branch of the resampler; too close to aliasing to be a decoding test
    "qpsk_undersampled": SignalCfg(name="qpsk_undersampled", samplerate=2.6e6, symbolrate=2400000, constellation="qpsk", conv="1/2",
                                   interleave=4, rrc_alpha=0.1, fmt="cs16", decoder="none", esn0_db=14.0),
    # psk_demod -> ccsds_simple_psk_decoder (no convolutional code; 50 shipped pipelines have this shape, e.g. FengYun-3.json:630-639):
    # BPSK + NRZ-M + RS I=4, and QPSK (I rail first on air, so the receiver runs with qpsk_swap_iq) + RS I=4
    "bpsk_simple": SignalCfg(name="bpsk_simple", samplerate=3e6, symbolrate=1200000, constellation="bpsk", conv="none", interleave=4, nrzm=True,
                             fmt="cs16", decoder="simple", esn0_db=9.0),
    "qpsk_simple": SignalCfg(name="qpsk_simple", samplerate=6e6, symbolrate=2400000, constellation="qpsk", conv="none", interleave=4, fmt="cs16",
                             decoder="simple", esn0_db=12.0),
    # 8PSK through psk_demod alone (order-8 Costas loop; no decoder of this path takes 8PSK): demodulator parity only
    "psk8": SignalCfg(name="psk8", samplerate=6e6, symbolrate=2400000, constellation="8psk", conv="none", interleave=4, fmt="cs16",
                      decoder="demod", esn0_db=18.0),
    # MetOp AHRPT recorded at 24 MS/s: 10.3 samples/symbol -> BaseDemodModule resamples to 8 MS/s (round(2333333 / 1e6) * 1e6 * MAX_SPS), a
    # ratio of 3, so SmartResamplerBlock runs its power-of-two decimator (x2: one 69-tap stage) and then the rational resampler 2/3
    "metop_oversampled": SignalCfg(name="metop_oversampled", samplerate=24e6),
    # BPSK r=1/2 at 1 Msym/s recorded at 32 MS/s in cs8: ratio 8 -> power-of-two decimator alone (stages /4 and /2), no rational part
    "bpsk_decim8": SignalCfg(name="bpsk_decim8", samplerate=32e6, symbolrate=1000000, constellation="bpsk", conv="1/2", interleave=4,
                             fmt="cs8", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=9.0),
    # ccsds_conv_concat_decoder with conv_rate 2/3 ... 7/8 (Viterbi_Depunc, viterbi_punc.cpp): QPSK + punctured k=7 code + RS I=4
    "qpsk_p23": SignalCfg(name="qpsk_p23", symbolrate=2400000, conv="p2/3", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=9.0),
    "qpsk_p34": SignalCfg(name="qpsk_p34", symbolrate=2400000, conv="p3/4", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=10.0),
    "qpsk_p56": SignalCfg(name="qpsk_p56", symbolrate=2400000, conv="p5/6", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=11.5),
    "qpsk_p78": SignalCfg(name="qpsk_p78", symbolrate=2400000, conv="p7/8", decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=12.5),
    # pm_demod -> ccsds_conv_concat_decoder (14 shipped pipelines have this shape): residual-carrier PM, BPSK r=1/2 on a subcarrier at the
    # symbol rate, 6 samples per symbol (inside pm_demod's [1.1, 10] window: no resampler), RS I=4
    "pm_bpsk": SignalCfg(name="pm_bpsk", samplerate=3e6, symbolrate=500000, constellation="bpsk", conv="1/2", interleave=4, fmt="cs16",
                         decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=20.0, pll_bw=0.005, carrier_rad=2e-2, pm_index=1.0),
    # the same at 24 samples per symbol with "resample_after_pll" (27 shipped pipelines set it): carrier PLL and PMToBPSK at the input
    # rate, then SmartResamplerBlock 6 MS/s -> 2 MS/s (decimator /2 + rational 2/3) and the second AGC, 8 samples per symbol
    "pm_bpsk_after": SignalCfg(name="pm_bpsk_after", samplerate=6e6, symbolrate=250000, constellation="bpsk", conv="1/2", interleave=4, fmt="cf32",
                               decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=26.0, pll_bw=0.005, carrier_rad=1e-2, pm_index=1.0,
                               resample_after_pll=True),
    # the same 24 samples per symbol WITHOUT resample_after_pll: BaseDemodModule resamples 6 MS/s -> 2 MS/s in front (decimator /2 + rational
    # 2/3), the carrier PLL and PMToBPSK run at the working rate
    "pm_bpsk_front": SignalCfg(name="pm_bpsk_front", samplerate=6e6, symbolrate=250000, constellation="bpsk", conv="1/2", interleave=4, fmt="cs16",
                               decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=26.0, pll_bw=0.005, carrier_rad=1e-2, pm_index=1.0),
    # psk_demod with "has_carrier" (ODIN.json:16-24): BPSK r=1/2 phase-modulated onto a residual carrier, 2.5 samples per symbol
    "bpsk_carrier": SignalCfg(name="bpsk_carrier", samplerate=6e6, symbolrate=2400000, constellation="bpsk", conv="1/2", interleave=4, fmt="cs16",
                              decoder="ccsds", ber_thresold=0.3, outsync_after=20, esn0_db=10.0, pll_bw=0.001, carrier_rad=5e-3, pm_index=1.2,
                              has_carrier=True, carrier_pll_bw=0.001, rrc_alpha=0.35),
    # C5: DVB-S2 front half AGC->RRC->M&M, cs8, 45 Msym/s @ 90 MS/s (sps 2.0), alpha 0.25 (DVB_Test.json:132-137), REC_ALPHA 1.7e-3
    "dvbs2_front": SignalCfg(name="dvbs2_front", samplerate=90e6, symbolrate=45000000, constellation="qpsk", conv="none", interleave=4,
                             rrc_alpha=0.25, fmt="cs8", decoder="none", clock_alpha=1.7e-3, carrier_rad=0.0, phase0=0.0, esn0_db=12.0),
    # psk_demod -> ccsds_ldpc_decoder (rate 7/8 C2 code, 10 iterations): QPSK at 2 samples per symbol in cs8 (FengYun-3 MERSI / GOES-R
    # raw-data shape, FengYun-3.json:530-548, GOES.json:532-560)
    "ldpc_qpsk": SignalCfg(name="ldpc_qpsk", samplerate=6e6, symbolrate=3000000, constellation="qpsk", conv="ldpc", rrc_alpha=0.35, fmt="cs8",
                           decoder="ldpc", esn0_db=12.0),
    # LandSat-like (LandSat.json:35-63): OQPSK, internal_stream with 8272-bit inner CADUs behind the ASM 0x352EF853; 3 samples per symbol,
    # above OQPSK's MAX_SPS 2.4, so the front-end resampler runs (6 -> 4.8 MS/s)
    "ldpc_landsat": SignalCfg(name="ldpc_landsat", samplerate=6e6, symbolrate=2000000, constellation="oqpsk", conv="ldpc", rrc_alpha=0.5, fmt="cs16",
                              decoder="ldpc", esn0_db=12.0, pll_bw=0.002, internal_cadu_size=8272, internal_asm=0x352EF853),
    # pm_demod -> ccsds_turbo_decoder, Juice-like (Juice.json): residual-carrier PM, BPSK on a subcarrier at the symbol rate, turbo rate 1/2
    # with base 1115 and 5 iterations; 526316 baud at 3 MS/s (5.7 samples per symbol, no resampler)
    "turbo_pm": SignalCfg(name="turbo_pm", samplerate=3e6, symbolrate=526316, constellation="bpsk", conv="turbo", rrc_alpha=0.35, fmt="cs16",
                          decoder="turbo", esn0_db=14.0, pll_bw=0.001, pm_pll_bw=0.002, carrier_rad=2e-2, pm_index=1.0, turbo_rate=2,
                          turbo_base=1115, turbo_iters=5),
    # psk_demod BPSK -> ccsds_turbo_decoder, Psyche-like (Psyche.json): rate 1/6, base 1115, 1 iteration, post_costas_dc; 368 kbaud at
    # 1 MS/s (2.7 samples per symbol)
    "turbo_bpsk": SignalCfg(name="turbo_bpsk", samplerate=1e6, symbolrate=368000, constellation="bpsk", conv="turbo", rrc_alpha=0.35, fmt="cs16",
                            decoder="turbo", esn0_db=6.0, pll_bw=0.002, post_costas_dc=True, turbo_rate=6, turbo_base=1115, turbo_iters=1),
    # psk_demod QPSK -> metop_dump_decoder, the MetOp X-band dump (MetOp.json "metop_dump"): 35 Msym/s at 45 MS/s (1.286 samples per
    # symbol), pll_bw 0.03, no convolutional code, randomised CADUs with RS(255,223) I=4 dual basis; cs16 (cs8: dataclasses.replace)
    "metop_dump": SignalCfg(name="metop_dump", samplerate=45e6, symbolrate=35000000, constellation="qpsk", conv="none", interleave=4,
                            rrc_alpha=0.5, pll_bw=0.03, fmt="cs16", decoder="dump", esn0_db=16.0),
    # psk_demod QPSK -> meteor_lrpt_decoder, METEOR M2 LRPT 72k (Meteor-M.json): 72 ksym/s, pll_bw 0.002, diff_decode false; r=1/2 k=7
    # continuous, randomised CADUs with RS(255,223) I=4 in the conventional basis. At 200 kS/s (2.78 samples per symbol, no resampling) and
    # at the pipeline's default 1 MS/s (13.9 samples per symbol: through the front-end resampler)
    "meteor_lrpt": SignalCfg(name="meteor_lrpt", samplerate=200e3, symbolrate=72000, constellation="qpsk", conv="1/2", interleave=4,
                             rrc_alpha=0.5, pll_bw=0.002, fmt="cs16", decoder="meteor", esn0_db=8.0, carrier_rad=2e-4),
    "meteor_lrpt_1m": SignalCfg(name="meteor_lrpt_1m", samplerate=1e6, symbolrate=72000, constellation="qpsk", conv="1/2", interleave=4,
                                rrc_alpha=0.5, pll_bw=0.002, fmt="cs16", decoder="meteor", esn0_db=8.0, carrier_rad=4e-5),
    # pm_demod -> noaa_hrpt_decoder / meteor_hrpt_decoder (NOAA.json "noaa_hrpt", Meteor-M.json "meteor_hrpt"): residual-carrier PM at
    # 665 400 sym/s recorded at 3 MS/s (4.5 samples per symbol, no resampler), carrier PLL bandwidth 0.01, rrc_alpha 0.6 | 0.5. The PM
    # model's sinusoidal subcarrier at the symbol rate stands in for the split-phase data; the decoders only see the soft bits' signs.
    "noaa_hrpt": SignalCfg(name="noaa_hrpt", samplerate=3e6, symbolrate=665400, constellation="bpsk", conv="none", rrc_alpha=0.6, fmt="cs16",
                           decoder="noaa_hrpt", esn0_db=20.0, pll_bw=0.005, pm_pll_bw=0.01, carrier_rad=2e-2, pm_index=1.0, deframer_thresold=10),
    "meteor_hrpt": SignalCfg(name="meteor_hrpt", samplerate=3e6, symbolrate=665400, constellation="bpsk", conv="none", rrc_alpha=0.5, fmt="cs16",
                             decoder="meteor_hrpt", esn0_db=20.0, pll_bw=0.005, pm_pll_bw=0.01, carrier_rad=2e-2, pm_index=1.0),
    # psk_demod OQPSK -> aqua_db_decoder, EOS Aqua / Aura DB (EOS.json "aqua_db", "aura_db"): 7.5 Msym/s recorded at 15 MS/s (2 samples per
    # symbol), two NRZ-M rails of randomised CADUs with RS(255,223) I=4 dual basis, no convolutional code. The receiver's clock and Costas
    # parameters are the pipeline's (tests/eos_cases.aqua_demod_cfg); the signal starts in the phase the Costas loop keeps.
    "aqua_db": SignalCfg(name="aqua_db", samplerate=15e6, symbolrate=7500000, constellation="oqpsk", conv="none", interleave=4, rrc_alpha=0.5,
                         pll_bw=0.006, fmt="cs16", decoder="aqua_db", esn0_db=20.0, carrier_rad=1e-4, phase0=0.1),
    # terra_db_demod -> ccsds_conv_concat_decoder, EOS Terra DB (EOS.json "terra_db"): 13.125 Msym/s recorded at 45 MS/s. The demodulator
    # runs BPSK loops at twice the symbol rate (1.714 samples per half-symbol), so the signal is BPSK at 26.25 Mbaud carrying the r=1/2 code
    # (terra_db_frames). The receiver's parameters are the module's (capi.terra_db_demod_kwargs); clock_alpha only stands in for them here.
    # psk_demod BPSK -> noaa_gac_decoder / dmsp_rtd_decoder (NOAA.json "noaa_gac", DMSP.json "dmsp_rtd"): bit streams without FEC at
    # 2.6616 Msym/s (6 MS/s, post_costas_dc) and 1.024 Msym/s (2 MS/s)
    "noaa_gac": SignalCfg(name="noaa_gac", samplerate=6e6, symbolrate=2661600, constellation="bpsk", conv="none", rrc_alpha=0.5, pll_bw=0.004,
                          fmt="cs16", decoder="noaa_gac", esn0_db=15.0, carrier_rad=1e-4, phase0=0.1, post_costas_dc=True),
    "dmsp_rtd": SignalCfg(name="dmsp_rtd", samplerate=2e6, symbolrate=1024000, constellation="bpsk", conv="none", rrc_alpha=0.5, pll_bw=0.005,
                          fmt="cs16", decoder="dmsp_rtd", esn0_db=15.0, carrier_rad=1e-4, phase0=0.1),
    # psk_demod QPSK -> fengyun_ahrpt_decoder (FengYun-3.json): "FengYun-3 A/B AHRPT" at 2.8 Msym/s, the D shape (30 Msym/s,
    # invert_second_viterbi) and the E / F / H shape (38.4 Msym/s), recorded at about two samples per symbol
    "fengyun_ahrpt": SignalCfg(name="fengyun_ahrpt", samplerate=6e6, symbolrate=2800000, constellation="qpsk", conv="3/4", rrc_alpha=0.5,
                               pll_bw=0.003, fmt="cs16", decoder="fengyun_ahrpt", esn0_db=12.0, carrier_rad=1e-4, phase0=0.1,
                               ber_thresold=0.26, outsync_after=20),
    "fengyun_ahrpt_d": SignalCfg(name="fengyun_ahrpt_d", samplerate=60e6, symbolrate=30000000, constellation="qpsk", conv="3/4", rrc_alpha=0.35,
                                 pll_bw=0.008, fmt="cs16", decoder="fengyun_ahrpt", esn0_db=12.0, carrier_rad=1e-4, phase0=0.1,
                                 ber_thresold=0.26, outsync_after=20, invert_second_viterbi=True),
    "fengyun_ahrpt_e": SignalCfg(name="fengyun_ahrpt_e", samplerate=76.8e6, symbolrate=38400000, constellation="qpsk", conv="3/4", rrc_alpha=0.35,
                                 pll_bw=0.008, fmt="cs16", decoder="fengyun_ahrpt", esn0_db=12.0, carrier_rad=1e-4, phase0=0.1,
                                 ber_thresold=0.26, outsync_after=20, invert_second_viterbi=True),
    # psk_demod QPSK -> fengyun_mpt_decoder (FengYun-3.json "fengyun3_abc_mpt"): "FengYun-3 A/B/C MPT" at 18.7 Msym/s, recorded at
    # 40 MS/s (2.14 samples per symbol)
    "fengyun_mpt": SignalCfg(name="fengyun_mpt", samplerate=40e6, symbolrate=18700000, constellation="qpsk", conv="1/2", rrc_alpha=0.5,
                             pll_bw=0.0063, fmt="cs16", decoder="fengyun_mpt", esn0_db=12.0, carrier_rad=1e-4, phase0=0.1,
                             ber_thresold=0.3, outsync_after=20),
    # psk_demod BPSK -> meteor_xband_decoder (Meteor-M.json "meteor_m_mtvza_dump", "meteor_m_kmss_bpsk_db"): NRZ-M record streams at
    # 15.36 and 61.44 Msym/s, recorded at two samples per symbol
    "meteor_mtvza": SignalCfg(name="meteor_mtvza", samplerate=30.72e6, symbolrate=15360000, constellation="bpsk", conv="none", rrc_alpha=0.6,
                              pll_bw=0.004, fmt="cs16", decoder="meteor_mtvza", esn0_db=15.0, carrier_rad=1e-4, phase0=0.1),
    "meteor_kmss_bpsk": SignalCfg(name="meteor_kmss_bpsk", samplerate=122.88e6, symbolrate=61440000, constellation="bpsk", conv="none",
                                  rrc_alpha=0.6, pll_bw=0.004, fmt="cs16", decoder="meteor_kmss_bpsk", esn0_db=15.0, carrier_rad=1e-4,
                                  phase0=0.1),
    "terra_db": SignalCfg(name="terra_db", samplerate=45e6, symbolrate=26250000, constellation="bpsk", conv="none", interleave=4, rrc_alpha=0.5,
                          pll_bw=0.004, fmt="cs16", decoder="terra_db", esn0_db=12.0, carrier_rad=1e-4, phase0=0.1, clock_alpha=0.001),
}


def qpsk_diff_encode(dibits, swap=True):
    """Transmit side of the reference's QPSKDiff decoder (src-core/common/codings/differential/qpsk_diff.cpp:5-53): hard symbols
    s = 2*X + Y (X on the Q rail, Y on the I rail, as constellation_t::soft_demod reads them) such that decoding the pair
    (s[i-1], s[i]) gives dibits[i]. Two leading symbols fill the decoder's buffer."""
    def dec(prev, cur):
        xin_1, yin_1, xin, yin = prev & 2, prev & 1, cur & 2, cur & 1
        if ((xin >> 1) ^ yin) == 1:
            ou = ((yin_1 ^ yin) << 1) + ((xin_1 ^ xin) >> 1)
        else:
            ou = (xin_1 ^ xin) + (yin_1 ^ yin)
        return ((ou & 1) << 1 | (ou >> 1)) if swap else ou  # value of the two output bits, first bit = MSB
    nxt = np.zeros((4, 4), np.int64)
    for prev in range(4):
        for cur in range(4):
            nxt[prev, dec(prev, cur)] = cur
    d = np.asarray(dibits, np.int64)
    out = np.zeros(d.size + 2, np.int64)
    cur = 0
    for i, v in enumerate(d.tolist()):
        cur = int(nxt[cur, v])
        out[i + 2] = cur
    return out


def make_bitstream(cfg: SignalCfg, nframes, seed):
    if cfg.decoder == "turbo":  # nframes turbo frames
        tx, clear = turbo_frames(nframes, cfg.turbo_rate, cfg.turbo_base, seed)
        return tx.reshape(-1), clear
    if cfg.decoder == "dump":  # nframes CADUs, sent as they are
        tx, clear = dump_frames(nframes, seed)
        return tx.reshape(-1), clear
    if cfg.decoder == "meteor":  # nframes LRPT CADUs, convolutionally encoded as one stream
        coded, written = lrpt_frames(nframes, seed, nrzm=cfg.nrzm)
        return coded, written
    if cfg.decoder == "noaa_hrpt":  # nframes NOAA HRPT minor frames (10-bit words, no FEC); clear: the words
        bits, words = noaa_hrpt_frames(nframes, seed)
        return bits.reshape(-1), words
    if cfg.decoder == "noaa_gac":  # nframes GAC frames (no FEC); clear: the frames the decoder writes
        bits, frames = gac_frames(nframes, seed, cfg.backward)
        return bits.reshape(-1), frames
    if cfg.decoder == "dmsp_rtd":  # nframes DMSP RTD frames (no FEC)
        bits, frames = dmsp_frames(nframes, seed)
        return bits.reshape(-1), frames
    if cfg.decoder == "meteor_hrpt":  # nframes METEOR HRPT CADUs (no FEC)
        bits, cadu = meteor_hrpt_frames(nframes, seed)
        return bits.reshape(-1), cadu
    if cfg.decoder == "aqua_db":  # nframes CADUs on two NRZ-M rails. psk_demod's OQPSK output pairs each Q symbol with the NEXT I
        # symbol (the half-symbol-delayed Q is read with the I that follows it), so the I rail goes on air one symbol later
        bits, clear = aqua_db_frames(nframes, seed)
        I, Q = aqua_db_rails(bits)
        coded = np.zeros(2 * I.size, np.uint8)
        coded[2::2], coded[1::2] = I[:-1], Q
        return coded, clear
    if cfg.decoder == "terra_db":  # nframes CADUs, NRZ-M, r=1/2: one BPSK symbol per code symbol
        return terra_db_frames(nframes, seed)
    if cfg.decoder == "fengyun_ahrpt":  # nframes CADUs on two punctured branches: the module swaps I and Q, so its I branch rides on Q
        i_bits, q_bits, clear = fengyun_frames(nframes, seed)
        n = min(i_bits.size, q_bits.size)
        coded = np.empty(2 * n, np.uint8)
        coded[0::2], coded[1::2] = (1 - q_bits[:n]) if cfg.invert_second_viterbi else q_bits[:n], i_bits[:n]
        return coded, clear
    if cfg.decoder == "fengyun_mpt":  # nframes CADUs on two r=1/2 branches, in the order of fengyun_mpt_pairs
        i_bits, q_bits, clear = fengyun_mpt_frames(nframes, seed)
        b0, b1 = fengyun_mpt_pairs(i_bits, q_bits)
        coded = np.empty(2 * b0.size, np.uint8)
        coded[0::2], coded[1::2] = b0, b1
        return coded, clear
    if cfg.decoder in ("meteor_mtvza", "meteor_kmss_bpsk"):  # nframes inner frames in records, NRZ-M
        return meteor_xband_frames(cfg.decoder == "meteor_kmss_bpsk", nframes, seed)
    if cfg.decoder == "ldpc":  # nframes LDPC frames
        if cfg.internal_cadu_size:
            info, clear = ldpc_inner_frames(nframes, cfg.internal_cadu_size, cfg.internal_asm, seed)
            tx, _, _ = ldpc_frames(nframes, seed, info=info)
        else:
            tx, _, clear = ldpc_frames(nframes, seed)
        return tx.reshape(-1), clear
    rng = np.random.default_rng(seed)
    payload = rng.integers(0, 256, size=(nframes, cfg.interleave * 223), dtype=np.uint8)
    tx, clear = build_cadus(payload, cfg.interleave)
    bits = np.unpackbits(tx.reshape(-1))
    if cfg.nrzm:
        bits = nrzm_encode(bits)
    if cfg.conv == "none":
        coded = bits
    else:
        coded = conv_encode(bits)
        if cfg.conv == "3/4":
            coded = puncture_34_metop(coded)
        elif cfg.conv in PUNCTURE_KEEP:
            coded = puncture_dvb(coded, cfg.conv)
    return coded, clear


def modulate(cfg: SignalCfg, coded, seed, nsamples=None, device="cpu"):
    """coded bits -> raw IQ in cfg.fmt. Heavy lifting in torch so bench-sized signals are made on the GPU."""
    import torch
    dev = torch.device(device)
    bps = 1 if cfg.constellation == "bpsk" else (3 if cfg.constellation == "8psk" else 2)
    nsym = coded.size // bps
    if bps == 3:  # 8PSK: points at pi/8 + k*pi/4, where the order-8 Costas detector (costas_loop.cpp) has its stable locks
        b = coded[:nsym * 3].reshape(-1, 3).astype(np.int64)
        ang = np.pi / 8 + (b[:, 0] * 4 + b[:, 1] * 2 + b[:, 2]) * (np.pi / 4)
        ai = torch.from_numpy(np.cos(ang).astype(np.float32)).to(dev)
        aq = torch.from_numpy(np.sin(ang).astype(np.float32)).to(dev)
    else:
        a = torch.from_numpy((coded[:nsym * bps].astype(np.float32) * 2 - 1)).to(dev)
        if bps == 2:
            ai, aq = a[0::2].contiguous(), a[1::2].contiguous()
        else:
            ai, aq = a, None
    sps = cfg.samplerate / cfg.symbolrate * (1.0 + cfg.clock_ppm * 1e-6)  # samples per symbol seen by the receiver
    span = 10
    total = int((nsym - 2 * span) * sps)
    if nsamples is None or nsamples > total:
        nsamples = total
    # pulse table, 1/2048-symbol grid, linear interpolation
    res = 2048
    tgrid = np.arange(-span * res, span * res + 2) / res
    tab = torch.from_numpy(rrc_pulse(tgrid, cfg.rrc_alpha).astype(np.float32)).to(dev)
    out_i = torch.empty(nsamples, dtype=torch.float32, device=dev)
    out_q = torch.empty(nsamples, dtype=torch.float32, device=dev)
    step = 1 << 20
    qoff = 0.5 if cfg.constellation == "oqpsk" else 0.0

    def shape(sym, t):  # t: symbol-time of each output sample (float64)
        k0 = torch.floor(t)
        d = (t - k0)  # [0,1)
        k0 = k0.to(torch.int64)
        pos = d * res
        pb = torch.floor(pos)
        fr = (pos - pb).to(torch.float32)
        pb = pb.to(torch.int64)
        acc = torch.zeros(t.shape, dtype=torch.float32, device=t.device)
        for j in range(-span + 1, span + 1):
            p0 = pb + (span - j) * res  # table index of (t - (k0 + j)) on the 1/res grid
            h = tab[p0] * (1 - fr) + tab[p0 + 1] * fr
            acc += sym[k0 + j] * h
        return acc

    for s in range(0, nsamples, step):
        e = min(nsamples, s + step)
        n = torch.arange(s, e, device=dev, dtype=torch.float64)
        t = n / sps + span + 0.37
        out_i[s:e] = shape(ai, t)
        if cfg.pm_index:
            if cfg.has_carrier:
                ph = cfg.pm_index * out_i[s:e]
            else:
                fsc = cfg.subcarrier if cfg.subcarrier else cfg.symbolrate
                sub = torch.sin((2 * np.pi * fsc / cfg.samplerate * n) % (2 * np.pi)).float()
                ph = cfg.pm_index * out_i[s:e] * sub
            out_i[s:e] = torch.cos(ph)
            out_q[s:e] = torch.sin(ph)
        elif aq is not None:
            out_q[s:e] = shape(aq, t - qoff)
        else:
            out_q[s:e] = 0
    x = torch.complex(out_i, out_q)
    p = float((x.real ** 2 + x.imag ** 2).mean())
    gen = torch.Generator(device=dev)
    gen.manual_seed(int(seed) + 7)
    sigma2 = p * (cfg.samplerate / cfg.symbolrate) / (10 ** (cfg.esn0_db / 10))
    for s in range(0, nsamples, step * 8):
        e = min(nsamples, s + step * 8)
        n = torch.arange(s, e, device=dev, dtype=torch.float64)
        ph = (cfg.carrier_rad * n + cfg.phase0) % (2 * np.pi)
        rot = torch.complex(torch.cos(ph).float(), torch.sin(ph).float())
        noise = torch.randn(e - s, 2, generator=gen, device=dev, dtype=torch.float32) * float(np.sqrt(sigma2 / 2))
        x[s:e] = x[s:e] * rot + torch.complex(noise[:, 0], noise[:, 1])
    scale = cfg.rms / float(np.sqrt(p + sigma2))
    x = x * scale
    v = torch.view_as_real(x).reshape(-1)
    if cfg.fmt == "cf32":
        return torch.view_as_complex(v.reshape(-1, 2).contiguous())
    if cfg.fmt == "cs16":
        return torch.clamp(torch.round(v * 32767), -32767, 32767).to(torch.int16)
    if cfg.fmt == "cs8":
        return torch.clamp(torch.round(v * 127), -127, 127).to(torch.int8)
    raise ValueError(cfg.fmt)


def frames_for_samples(cfg: SignalCfg, nsamples):
    bps = 1 if cfg.constellation == "bpsk" else 2
    if cfg.decoder == "turbo":  # turbo frames of ASM + codeword bits
        nbits = turbo_codeword_bits(cfg.turbo_rate, cfg.turbo_base) + TURBO_ASM_BITS[cfg.turbo_rate]
        return int(nsamples * bps / (cfg.samplerate / cfg.symbolrate) / nbits) + 2
    if cfg.decoder == "meteor":  # LRPT CADUs of 8192 bits, 16384 coded bits each
        return int(nsamples * bps / (cfg.samplerate / cfg.symbolrate) / 16384) + 2
    if cfg.decoder in ("noaa_hrpt", "meteor_hrpt"):  # bits on air: 110900 per NOAA minor frame, 8192 per METEOR CADU
        return int(nsamples / (cfg.samplerate / cfg.symbolrate) / (NOAA_WORDS * 10 if cfg.decoder == "noaa_hrpt" else 8192)) + 2
    if cfg.decoder in ("noaa_gac", "dmsp_rtd"):  # bits on air: 33270 per GAC frame, 150 per DMSP frame
        return int(nsamples / (cfg.samplerate / cfg.symbolrate) / (GAC_BITS if cfg.decoder == "noaa_gac" else DMSP_BITS)) + 2
    if cfg.decoder in ("meteor_mtvza", "meteor_kmss_bpsk"):  # bits on air per inner frame: its share of the records
        per = MTVZA_FRM * 8 * 384 / 368 if cfg.decoder == "meteor_mtvza" else KMSS_FRM * 8 * 1536 / 1504
        return int(nsamples / (cfg.samplerate / cfg.symbolrate) / per) + 2
    if cfg.decoder == "terra_db":  # 16384 code symbols per CADU, one per sample period of the half-symbol rate
        return int(nsamples / (cfg.samplerate / cfg.symbolrate) / 16384) + 2
    if cfg.decoder in ("ldpc", "dump", "aqua_db"):  # LDPC frames / MetOp dump and Aqua DB CADUs of 8192 bits
        return int(nsamples * bps / (cfg.samplerate / cfg.symbolrate) / 8192) + 2
    rate = {"1/2": 0.5, "3/4": 0.75, "none": 1.0, "p2/3": 2 / 3, "p3/4": 0.75, "p5/6": 5 / 6, "p7/8": 7 / 8}[cfg.conv]
    bits_per_sample = bps * rate / (cfg.samplerate / cfg.symbolrate)
    return int(nsamples * bits_per_sample / (cfg.cadu_bytes * 8)) + 4


def make_signal(cfg: SignalCfg, nsamples, seed=0xB2000000, device="cpu"):
    """Returns (raw torch tensor in cfg.fmt with exactly <= nsamples samples, clear CADUs (nframes, cadu_bytes) numpy)."""
    nframes = frames_for_samples(cfg, nsamples)
    coded, clear = make_bitstream(cfg, nframes, seed)
    raw = modulate(cfg, coded, seed, nsamples, device)
    return raw, clear


# ---------------------------------------------------------------------------------------------------------------- AOS frames with space packets
def build_aos_frames(nframes, seed, vcids=(9, 12, 3, 34), mpdu=884, insert_zone=0, cadu_size=1024, corrupt=0.0, drop=0.0, idle=0.05):
    """A CADU stream whose virtual channels carry CCSDS space packets in M-PDUs (the input of ccsds_aos::Demuxer, demuxer.cpp): per channel a
    byte stream of packets (lengths from 1 byte to several frames, so headers straddle frames and first-header-pointers of 2047 occur),
    cut into `mpdu`-byte zones with the first header pointer of each; channels interleaved at random, idle frames (VCID 63, pointer 2046)
    in between. corrupt: fraction of the frames with random damage to the pointer / packet headers / payload (exercises the demuxer's
    behaviour on inconsistent input); drop: fraction of the frames removed after packing (discontinuities). Returns uint8 [frames, cadu_size]."""
    rng = np.random.default_rng(seed)
    base = 10 + (insert_zone if insert_zone else 0)
    assert base + 2 + mpdu <= cadu_size
    streams = {}

    def more(v, need):
        st = streams.setdefault(v, dict(buf=bytearray(), starts=[], pos=0, seq=0))
        while len(st["buf"]) - st["pos"] < need:
            r = rng.random()
            n = int(rng.integers(1, 300)) if r < 0.7 else (int(rng.integers(300, 2000)) if r < 0.9 else int(rng.integers(2000, 14000)))
            apid = int(rng.choice([34, 39, 103, 104, 130, 384, 6]))
            sec = int(rng.integers(0, 2))
            st["seq"] = (st["seq"] + 1) & 0x3FFF
            hdr = bytes([(sec << 3) | (apid >> 8), apid & 0xFF, 0xC0 | (st["seq"] >> 8), st["seq"] & 0xFF, ((n - 1) >> 8) & 0xFF, (n - 1) & 0xFF])
            st["starts"].append(len(st["buf"]))
            st["buf"] += hdr + rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        return st

    out = np.zeros((nframes, cadu_size), np.uint8)
    out[:] = rng.integers(0, 256, (nframes, cadu_size), dtype=np.uint8)
    counters = {}
    for f in range(nframes):
        v = 63 if rng.random() < idle else int(rng.choice(vcids))
        fr = out[f]
        fr[0:4] = (0x1A, 0xCF, 0xFC, 0x1D)
        scid = 0x0B
        fr[4] = (1 << 6) | (scid >> 2)
        fr[5] = ((scid & 3) << 6) | v
        c = counters.get(v, 0)
        counters[v] = (c + 1) & 0xFFFFFF
        fr[6], fr[7], fr[8], fr[9] = (c >> 16) & 0xFF, (c >> 8) & 0xFF, c & 0xFF, 0
        if v == 63:
            fhp = 2046
        else:
            st = more(v, mpdu)
            p0 = st["pos"]
            fr[base + 2:base + 2 + mpdu] = np.frombuffer(bytes(st["buf"][p0:p0 + mpdu]), np.uint8)
            nxt = [s for s in st["starts"] if p0 <= s < p0 + mpdu]
            fhp = nxt[0] - p0 if nxt else 2047
            st["pos"] = p0 + mpdu
            st["starts"] = [s for s in st["starts"] if s >= p0 + mpdu]
            if st["pos"] > 1 << 20:  # keep the buffer short
                st["buf"] = st["buf"][st["pos"]:]
                st["starts"] = [s - st["pos"] for s in st["starts"]]
                st["pos"] = 0
        fr[base] = (int(rng.integers(0, 32)) << 3) | (fhp >> 8)
        fr[base + 1] = fhp & 0xFF
    if corrupt:
        for f in np.nonzero(rng.random(nframes) < corrupt)[0]:
            kind = int(rng.integers(0, 4))
            if kind == 0:  # a random first header pointer
                fhp = int(rng.integers(0, 2048))
                out[f, base] = (out[f, base] & 0xF8) | (fhp >> 8)
                out[f, base + 1] = fhp & 0xFF
            elif kind == 1:  # pointer "no header" although there is one / short pointers
                fhp = int(rng.choice([2047, 0, 1, 2, 3, 4, 5, mpdu - 1, mpdu - 3, mpdu - 6, mpdu - 7, mpdu, mpdu + 1]))
                out[f, base] = (out[f, base] & 0xF8) | (fhp >> 8)
                out[f, base + 1] = fhp & 0xFF
            elif kind == 2:  # a burst of wrong bytes somewhere in the data zone (packet lengths go wrong)
                a = int(rng.integers(0, mpdu - 16))
                out[f, base + 2 + a:base + 2 + a + 16] = rng.integers(0, 256, 16, dtype=np.uint8)
            else:  # the frame lands in another virtual channel
                out[f, 5] = (out[f, 5] & 0xC0) | int(rng.choice(vcids))
    if drop:
        out = out[rng.random(nframes) >= drop]
    return np.ascontiguousarray(out)


def craft_leftover_frames(mpdu, variant=0, vcid=9, cadu_size=1024):
    """Six frames that drive ccsds_aos::Demuxer into its rarest corner: a header straddles a frame boundary, the next frame claims to hold no
    header (pointer 2047) although the packet ends inside it, so the continuation takes more than what remained (demuxer.cpp:109) and the
    packet never completes; its bytes then stay in front of the next packet (readPacket does not clear them, :26-33). variant 0: that next
    packet completes inside its frame; variant 1: it runs on into the following frames."""
    rng = np.random.default_rng(100 + variant)
    fr = rng.integers(0, 256, (6, cadu_size), dtype=np.uint8)
    base = 10

    def head(f, fhp):
        fr[f, 5] = (fr[f, 5] & 0xC0) | vcid
        fr[f, base] = fhp >> 8
        fr[f, base + 1] = fhp & 0xFF

    def d(f):
        return fr[f, base + 2:]

    head(0, mpdu - 3)  # three header bytes at the end of the zone
    fr[0, base + 2 + mpdu - 3] &= 0xF7
    head(1, 2047)
    pl = (mpdu - 3 - 1) - 1  # remaining = mpdu - 4 with offset 3: (rem + 3) > mpdu - 3 but rem < mpdu - 3
    d(1)[1], d(1)[2] = pl >> 8, pl & 0xFF
    head(2, 10)
    n = 20 if variant == 0 else 3000
    d(2)[10 + 4], d(2)[10 + 5] = (n - 1) >> 8, (n - 1) & 0xFF
    if variant == 0:
        d(2)[10 + 6 + n + 4], d(2)[10 + 6 + n + 5] = 0, 49
    head(3, 2047 if variant else 100)
    head(4, 50)
    head(5, 7)
    for f in (3, 4, 5):
        p = ((int(fr[f, base]) & 7) << 8) | int(fr[f, base + 1])
        if p < 2047:
            d(f)[p + 4], d(f)[p + 5] = 0, 30
    return fr


# ---- CCSDS C2 LDPC (8176, 7154), the code behind ccsds_ldpc_decoder's ldpc_rate "7/8" -----------------------------------------------
LDPC_CIRC, LDPC_BX, LDPC_BY = 511, 16, 2
LDPC_N, LDPC_ROWS, LDPC_SHORT = 8176, 1022, 18  # code length, parity checks, leading positions that are always 0 (not sent)
LDPC_INFO = 7154 - LDPC_SHORT                   # info bits sent per codeword (7136)


@functools.lru_cache(maxsize=1)
def ldpc_c2_offsets():
    """The circulant offsets of satdump_b200/csrc/ldpc_c2_table.inc (tools/gen_ldpc_c2_table.py) as int [2, 16, 2]."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "ldpc_c2_table.inc")).read()
    nums = [int(v) for v in re.findall(r"\d+", src.split("= {", 1)[1])]
    return np.array(nums, np.int64).reshape(LDPC_BY, LDPC_BX, 2)


@functools.lru_cache(maxsize=1)
def ldpc_c2_cols():
    """H's rows (row block 0's 511 rows, then row block 1's) as the ascending column indices of their 32 ones: int [1022, 32]."""
    off = ldpc_c2_offsets()
    r = np.arange(LDPC_CIRC)
    cols = np.zeros((LDPC_ROWS, 2 * LDPC_BX), np.int64)
    for y in range(LDPC_BY):
        for x in range(LDPC_BX):
            a, b = (off[y, x, 0] + r) % LDPC_CIRC, (off[y, x, 1] + r) % LDPC_CIRC
            cols[y * LDPC_CIRC:(y + 1) * LDPC_CIRC, 2 * x] = LDPC_CIRC * x + np.minimum(a, b)
            cols[y * LDPC_CIRC:(y + 1) * LDPC_CIRC, 2 * x + 1] = LDPC_CIRC * x + np.maximum(a, b)
    return cols


def ldpc_c2_h():
    H = np.zeros((LDPC_ROWS, LDPC_N), np.uint8)
    H[np.repeat(np.arange(LDPC_ROWS), 2 * LDPC_BX), ldpc_c2_cols().reshape(-1)] = 1
    return H


@functools.lru_cache(maxsize=1)
def _ldpc_parity_solver():
    """Gaussian elimination of H's parity part (columns 7154..8175, rank 1020) over GF(2): the pivot columns and the row operations
    that turn a syndrome into their values (the two non-pivot parity positions are set to 0)."""
    H = ldpc_c2_h()
    A = np.concatenate([H[:, 7154:], np.eye(LDPC_ROWS, dtype=np.uint8)], axis=1)
    piv_cols, r = [], 0
    for c in range(LDPC_ROWS):
        rows = np.nonzero(A[r:, c])[0]
        if rows.size == 0:
            continue
        p = r + rows[0]
        A[[r, p]] = A[[p, r]]
        hit = np.nonzero(A[:, c])[0]
        hit = hit[hit != r]
        A[hit] ^= A[r]
        piv_cols.append(c)
        r += 1
    return np.array(piv_cols), A[:r, LDPC_ROWS:].astype(np.int64)


def ldpc_c2_encode(info):
    """info: uint8 [n, 7136] -> codewords uint8 [n, 8176] with H c = 0: 18 zeros, the info bits, 1022 parity bits."""
    info = np.atleast_2d(np.asarray(info, np.uint8))
    n = info.shape[0]
    H = ldpc_c2_h().astype(np.int64)
    cw = np.zeros((n, LDPC_N), np.uint8)
    cw[:, LDPC_SHORT:7154] = info
    syn = (cw[:, :7154].astype(np.int64) @ H[:, :7154].T) % 2
    piv, E = _ldpc_parity_solver()
    cw[:, 7154 + piv] = ((syn @ E.T) % 2).astype(np.uint8)
    assert not ((cw.astype(np.int64) @ H.T) % 2).any(), "H c != 0"
    return cw


def ldpc_pn_bits(n):
    """The CCSDS pseudo-random sequence one bit per entry (period 255), as derand_ccsds_soft applies it to the 8160 code soft bytes."""
    return np.resize(np.unpackbits(ccsds_pn(32))[:255], n)


def ldpc_frames(nframes, seed=0, info=None):
    """(tx bits uint8 [n, 8192] = ASM + PN-randomised (code bits 18..8175 + 2 zero fill bits), codewords [n, 8176], the CADUs the decoder
    writes for them [n, 1024]: the ASM 0x1ACFFC1D as a little-endian uint32, then the 8158 code bits and the 2 zero fill bits)."""
    if info is None:
        info = np.random.default_rng(seed).integers(0, 2, (nframes, LDPC_INFO), dtype=np.uint8)
    cw = ldpc_c2_encode(info)
    sent = np.concatenate([cw[:, LDPC_SHORT:], np.zeros((cw.shape[0], 2), np.uint8)], axis=1)
    asm = np.unpackbits(np.frombuffer(ASM, np.uint8))
    tx = np.concatenate([np.tile(asm, (cw.shape[0], 1)), sent ^ ldpc_pn_bits(8160)[None, :]], axis=1)
    cadu = np.concatenate([np.tile(np.array([0x1D, 0xFC, 0xCF, 0x1A], np.uint8), (cw.shape[0], 1)), np.packbits(sent, axis=1)], axis=1)
    return tx, cw, cadu


def ldpc_soft(tx_bits, constellation, amp=60.0, sigma=0.0, rot=0, q_late=False, seed=0):
    """int8 soft stream of the bit stream as psk_demod writes it: bit 1 -> +amp. BPSK: one byte per bit (rot 0 / 2 = 0 / 180 degrees).
    QPSK / OQPSK: (I, Q) pairs of consecutive bits, the symbols rotated by rot * 90 degrees; q_late: Q lags I by one symbol."""
    b = np.asarray(tx_bits, np.uint8).reshape(-1).astype(np.float64) * 2 - 1
    rng = np.random.default_rng(seed)
    if constellation == "bpsk":
        s = b * (-1 if rot == 2 else 1) * amp
    else:
        z = (b[0::2] + 1j * b[1::2]) * np.exp(1j * np.pi / 2 * rot)
        I, Q = np.round(z.real), np.round(z.imag)
        if q_late:
            Q = np.concatenate([[0.0], Q[:-1]])
        s = np.empty(2 * I.size)
        s[0::2], s[1::2] = I * amp, Q * amp
    if sigma:
        s = s + rng.normal(0, sigma, s.size)
    return np.clip(np.round(s), -127, 127).astype(np.int8)


def ldpc_inner_frames(nframes, cadu_size, asm, seed):
    """internal_stream: inner CADUs of cadu_size bits (asm + random bits) packed back to back into the 7136 info bits of nframes codewords.
    Returns (info uint8 [nframes, 7136], the whole inner frames the info bits carry, uint8 [k, cadu_size / 8])."""
    rng = np.random.default_rng(seed + 1)
    total = nframes * LDPC_INFO
    k = total // cadu_size
    asm_bits = np.unpackbits(np.frombuffer(int(asm).to_bytes(4, "big"), np.uint8))
    inner = np.concatenate([np.tile(asm_bits, (k, 1)), rng.integers(0, 2, (k, cadu_size - 32), dtype=np.uint8)], axis=1)
    bits = np.concatenate([inner.reshape(-1), rng.integers(0, 2, total - k * cadu_size, dtype=np.uint8)])
    return bits.reshape(nframes, LDPC_INFO), np.packbits(inner, axis=1)


# ---- MetOp X-band dump (metop_dump_decoder) ---------------------------------------------------------------------------------------------
def dump_frames(nframes, seed=0):
    """(tx bits uint8 [n, 8192] of randomised CADUs with RS(255,223) I=4 dual basis, the CADUs metop_dump_decoder writes for them
    [n, 1024]: the ASM and the derandomised codewords)."""
    payload = np.random.default_rng(seed).integers(0, 256, size=(nframes, 4 * 223), dtype=np.uint8)
    tx, clear = build_cadus(payload, 4)
    return np.unpackbits(tx, axis=1), clear


def dump_soft(tx_bits, phase=0, swap=False, amp=60.0, sigma=0.0, seed=0):
    """int8 soft stream of the bit stream (I, Q = consecutive bits) that metop_dump_decoder decodes with phase `phase` (0..3 = 0 .. 270
    degrees) and `swap`: the symbols the correlator's syncword 4 + phase (swap: phase) matches. The decoder inverts its hard decisions, so
    bit 1 is -amp after rotate_soft(phase, swap); here the inverse of that rotation is applied: rotation by -phase, then the IQ swap."""
    b = np.asarray(tx_bits, np.uint8).reshape(-1).astype(np.float64)
    s = (1 - 2 * b) * amp
    I, Q = s[0::2], s[1::2]
    for _ in range((4 - phase) % 4):  # rotate_soft's PHASE_90 step: (I, Q) -> (Q, -I)
        I, Q = Q, -I
    if swap:
        I, Q = Q, I
    out = np.empty(2 * I.size)
    out[0::2], out[1::2] = I, Q
    if sigma:
        out = out + np.random.default_rng(seed).normal(0, sigma, out.size)
    return np.clip(np.round(out), -127, 127).astype(np.int8)


# ---- METEOR-M LRPT (meteor_lrpt_decoder) ------------------------------------------------------------------------------------------------
def lrpt_frames(nframes, seed=0, nrzm=False, inverted=()):
    """The LRPT transmitter: random payloads, RS(255,223) I=4 in the conventional basis, the randomiser, NRZ-M when `nrzm`, then r=1/2 k=7
    over the whole stream (conv_encode). Returns (coded bits uint8 [nframes * 16384]: I = first, Q = second output of each step, the CADUs
    meteor_lrpt_decoder writes for them [n, 1024]: 1D CF FC 1D + the derandomised codewords). Frames listed in `inverted` are sent with
    bytes 4 .. 1023 inverted and a payload whose derandomised byte 9 is 0x00: the decoder finds 0xFF there and inverts the frame back."""
    payload = np.random.default_rng(seed).integers(0, 256, size=(nframes, 4 * 223), dtype=np.uint8)
    for k in inverted:
        payload[k, 5] = 0  # CADU byte 9 = byte 5 of the interleaved codewords = message byte 1 of codeword 1 = payload byte 1 * 4 + 1
    tx, clear = build_cadus(payload, 4, dual=False)
    for k in inverted:
        tx[k, 4:] ^= 0xFF
    bits = np.unpackbits(tx.reshape(-1))
    if nrzm:
        bits = nrzm_encode(bits)
    written = clear.copy()
    written[:, :4] = (0x1D, 0xCF, 0xFC, 0x1D)
    return conv_encode(bits), written


def lrpt_soft(coded, phase=0, swap=False, amp=60.0, sigma=0.0, seed=0):
    """int8 soft stream of coded bits (bit 1 = +amp, I and Q = consecutive bits) as a receiver with a phase ambiguity `phase` (0..3 = 0 ..
    270 degrees) and an IQ swap sees it: the inverse of rotate_soft(phase, swap), i.e. rotation by -phase, then the swap."""
    b = np.asarray(coded, np.uint8).reshape(-1).astype(np.float64)
    s = (2 * b - 1) * amp
    I, Q = s[0::2], s[1::2]
    for _ in range((4 - phase) % 4):  # rotate_soft's PHASE_90 step: (I, Q) -> (Q, -I)
        I, Q = Q, -I
    if swap:
        I, Q = Q, I
    out = np.empty(2 * I.size)
    out[0::2], out[1::2] = I, Q
    if sigma:
        out = out + np.random.default_rng(seed).normal(0, sigma, out.size)
    return np.clip(np.round(out), -127, 127).astype(np.int8)


# ---- NOAA and METEOR HRPT (noaa_hrpt_decoder, meteor_hrpt_decoder): bit streams without FEC -------------------------------------------
NOAA_SYNC_WORDS = (0x284, 0x16F, 0x35C, 0x19D, 0x20F, 0x095)  # the 60-bit minor-frame sync 0x0A116FD719D83C95 as six 10-bit words
NOAA_WORDS = 11090
METEOR_HRPT_ASM = bytes([0x1A, 0xCF, 0xFC, 0x1D])


def noaa_hrpt_frames(nframes, seed=0):
    """(bits uint8 [n, 110900] as sent, MSB first; words uint16 [n, 11090]): NOAA HRPT minor frames of 10-bit words, the six sync words
    then 11084 random words"""
    words = np.random.default_rng(seed).integers(0, 1024, size=(nframes, NOAA_WORDS)).astype(np.uint16)
    words[:, :6] = NOAA_SYNC_WORDS
    bits = ((words[..., None] >> np.arange(9, -1, -1, dtype=np.uint16)) & 1).astype(np.uint8).reshape(nframes, -1)
    return bits, words


def meteor_hrpt_frames(nframes, seed=0):
    """(bits uint8 [n, 8192] as sent; CADUs uint8 [n, 1024]): the ASM 1ACFFC1D and 1020 random bytes per frame"""
    cadu = np.random.default_rng(seed).integers(0, 256, size=(nframes, 1024)).astype(np.uint8)
    cadu[:, :4] = np.frombuffer(METEOR_HRPT_ASM, np.uint8)
    return np.unpackbits(cadu, axis=1), cadu


def hrpt_soft(bits, inverted=False, amp=60.0, sigma=0.0, seed=0, slips=(), gaps=()):
    """int8 soft stream of a bit stream as pm_demod writes it (bit 1 -> +amp; inverted: the other polarity). slips: bit indices dropped
    from the stream (a bit slip); gaps: (bit index, length) stretches of noise inserted there. Indices refer to `bits`."""
    b = np.asarray(bits, np.uint8).reshape(-1)
    s = (2.0 * b - 1.0) * amp * (-1.0 if inverted else 1.0)
    rng = np.random.default_rng(seed)
    if sigma:
        s = s + rng.normal(0, sigma, s.size)
    keep = np.ones(s.size, bool)
    keep[list(slips)] = False
    pieces, a = [], 0
    for at, n in sorted(gaps):
        pieces += [s[a:at][keep[a:at]], rng.normal(0, 1.5 * amp, n)]
        a = at
    pieces.append(s[a:][keep[a:]])
    return np.clip(np.round(np.concatenate(pieces)), -127, 127).astype(np.int8)


# ---- NOAA GAC and DMSP RTD (noaa_gac_decoder, dmsp_rtd_decoder): bit streams without FEC ------------------------------------------------
GAC_BITS, GAC_BYTES = 33270, 4159
GAC_SYNC, GAC_SYNC_BACKWARD = 0xA116FD71, 0x33C3E4A6
DMSP_BITS, DMSP_BYTES, DMSP_ASM = 150, 19, 0b1010110011111


def gac_pn_bits():
    """The GAC PN sequence (1023 bits): b[i] = b[i-1] ^ b[i-5] ^ b[i-6] ^ b[i-8] ^ b[i-11] from 0 0 0 0 0 1 1 1 0 1 0"""
    b = [0, 0, 0, 0, 0, 1, 1, 1, 0, 1, 0]
    for i in range(11, 1023):
        b.append(b[i - 1] ^ b[i - 5] ^ b[i - 6] ^ b[i - 8] ^ b[i - 11])
    return np.array(b, np.uint8)


def gac_pn_bytes():
    """The 4159 bytes noaa_gac_decoder XORs onto each frame: 60 zero bits, then the PN bits repeated, MSB first"""
    bits = np.concatenate([np.zeros(60, np.uint8), np.resize(gac_pn_bits(), GAC_BYTES * 8 - 60)])
    return np.packbits(bits)


def frame_image(bits, nbytes):
    """The byte image write_bit leaves of frames of len(bits) bits: MSB first, the partial last byte right-aligned. bits [n, nbits]"""
    bits = np.asarray(bits, np.uint8)
    full = bits.shape[1] // 8 * 8
    img = np.zeros((bits.shape[0], nbytes), np.uint8)
    img[:, :full // 8] = np.packbits(bits[:, :full], axis=1)
    if full < bits.shape[1]:
        img[:, full // 8] = (bits[:, full:] << np.arange(bits.shape[1] - full - 1, -1, -1, dtype=np.uint8)).sum(axis=1)
    return img


def gac_post(img, backward):
    """noaa_gac_decoder after the deframer (module_noaa_gac_decoder.cpp:84-98): with backward, output bit ii = bit 33269 - ii of the byte
    image read MSB first (written back with write_bit's right-aligned last byte); then the PN bytes. img uint8 [n, 4159]"""
    img = np.asarray(img, np.uint8)
    if backward:
        rd = np.unpackbits(img, axis=1)[:, GAC_BITS - 1::-1]
        img = frame_image(rd, GAC_BYTES)
    return img ^ gac_pn_bytes()


def gac_frames(nframes, seed=0, backward=False):
    """(bits uint8 [n, 33270] as sent; frames uint8 [n, 4159] as noaa_gac_decoder writes them): the sync word (0x33C3E4A6 when backward)
    and 33238 random bits per frame"""
    bits = np.random.default_rng(seed).integers(0, 2, size=(nframes, GAC_BITS)).astype(np.uint8)
    sync = GAC_SYNC_BACKWARD if backward else GAC_SYNC
    bits[:, :32] = (sync >> np.arange(31, -1, -1)) & 1
    return bits, gac_post(frame_image(bits, GAC_BYTES), backward)


def dmsp_frames(nframes, seed=0):
    """(bits uint8 [n, 150] as sent; frames uint8 [n, 19] as dmsp_rtd_decoder writes them): the 13-bit sync and 137 random bits"""
    bits = np.random.default_rng(seed).integers(0, 2, size=(nframes, DMSP_BITS)).astype(np.uint8)
    bits[:, :13] = (DMSP_ASM >> np.arange(12, -1, -1)) & 1
    return bits, frame_image(bits, DMSP_BYTES)


# ---- METEOR-M X-band dumps (meteor_xband_decoder) -------------------------------------------------------------------------------------
MTVZA_FRM, KMSS_FRM = 380, 60160
MTVZA_SYNC = bytes.fromhex("38FB456A")
KMSS_SYNCS = [bytes.fromhex("AF5FFF50AA5AA0"), bytes.fromhex("AE5EEC61BB7982"), bytes.fromhex("AB5BB394EED628")]


def kmss_frame_process(frame, d):
    """kmssFrameProcessor (module_meteor_xband_decoder.cpp:44-53) on one 60160-byte frame of deframer d (0, 1, 2), with the module's lane
    moves for deframers 2 and 3: the 60160 bytes the module writes"""
    b = np.unpackbits(np.asarray(frame, np.uint8) ^ 0xF0).reshape(KMSS_FRM // 4, 4, 2, 4)  # [c, byte i, nibble, bit in nibble]
    lanes = np.packbits(b.transpose(3, 0, 1, 2).reshape(4, -1), axis=1)  # lane o: bits o and 4 + o of bytes 4c .. 4c + 3
    if d:
        mv = [2, 3] if d == 1 else [0, 1]
        lanes[mv, 1:] = lanes[mv, :-1].copy()
    return lanes.reshape(-1)


def meteor_xband_records(kmss, packets, rng):
    """Records carrying the packet stream `packets` (a whole number of records' worth): MTVZA 384 bytes with its four patterns and eight
    46-byte packets XOR 0xAA at byte 2 + 48k; KMSS 1536 bytes with 0x0035 at its start, zeros at byte 382 and eight 188-byte packets at
    byte 2 + 192k. The bytes between the packets are random where no pattern lies."""
    P, stride, size = (188, 192, 1536) if kmss else (46, 48, 384)
    pk = np.asarray(packets, np.uint8).reshape(-1, 8, P)
    rec = rng.integers(0, 256, size=(pk.shape[0], size), dtype=np.uint8)
    for k in range(8):
        rec[:, 2 + stride * k:2 + stride * k + P] = pk[:, k] if kmss else pk[:, k] ^ 0xAA
    if kmss:
        rec[:, 0], rec[:, 1], rec[:, 382:386] = 0x00, 0x35, 0
    else:
        rec[:, 0], rec[:, 48], rec[:, 96], rec[:, 240] = 0xB3, 0xE3, 0x75, 0
        rec[:, 241] &= 0x7F
    return rec


def meteor_xband_frames(kmss, nframes, seed=0, cut=None):
    """(bits on air uint8: the records NRZ-M encoded; the frames meteor_xband_decoder writes, [n, 380] | [n, 60160]). Inner frames are the
    sync and random bytes (KMSS: the three deframers' syncs in turn). cut = (k, nbytes): frame k is sent only up to nbytes, so the next
    sync cuts it and the decoder writes it filled with zeros after that sync."""
    rng = np.random.default_rng(seed)
    F = KMSS_FRM if kmss else MTVZA_FRM
    frames = rng.integers(0, 256, size=(nframes, F), dtype=np.uint8)
    ds = [i % 3 if kmss else 0 for i in range(nframes)]
    if kmss and cut is not None and cut[0] + 1 < nframes:  # (the cut frame is followed by one of the same deframer)
        ds = ds[:cut[0] + 1] + [(d + 2) % 3 for d in ds[cut[0] + 1:]]
    syncs = [KMSS_SYNCS[d] if kmss else MTVZA_SYNC for d in ds]
    for i in range(nframes):
        frames[i, :len(syncs[i])] = np.frombuffer(syncs[i], np.uint8)
    sent, written = [], []
    for i in range(nframes):
        f = w = frames[i]
        if cut is not None and cut[0] == i and i + 1 < nframes:
            f = f[:cut[1]]
            w = np.zeros(F, np.uint8)
            w[:cut[1]] = f
            w[cut[1]:cut[1] + len(syncs[i + 1])] = np.frombuffer(syncs[i + 1], np.uint8)
        sent.append(f)
        written.append(kmss_frame_process(w, ds[i]) if kmss else w)
    stream = np.concatenate(sent)
    npb = 1504 if kmss else 368
    stream = np.concatenate([stream, rng.integers(0, 256, size=(-stream.size) % npb + npb, dtype=np.uint8)])
    rec = meteor_xband_records(kmss, stream, rng)
    return nrzm_encode(np.unpackbits(rec.reshape(-1))), np.stack(written)


# ---- EOS Aqua / Aura DB (aqua_db_decoder): randomised CADUs on two NRZ-M rails -----------------------------------------------------------
# ---- FengYun-3 AHRPT / DPT (fengyun_ahrpt_decoder) ---------------------------------------------------------------------------------------
def fengyun_diff_encode(bits):
    """The inverse of FengyunDiff::work2 (diff.cpp:45-74) from Xin = Yin = 0: the branch bits (x, y) (x = in1 = the Q branch's, y = in2 =
    the I branch's) of every pair, such that the decoder returns `bits` (even length). For output bits (h, l) and the previous pair
    (xp, yp): x != y gives h = yp ^ y, l = xp ^ x, and x == y gives h = xp ^ x, l = yp ^ y; exactly one of the two is consistent."""
    # Both branches give x ^ y = xp ^ yp ^ h ^ l, so d = x ^ y is the running XOR of h ^ l, and x steps by l where d = 1, else by h.
    b = np.asarray(bits, np.uint8).reshape(-1, 2)
    h, l = b[:, 0], b[:, 1]
    d = np.bitwise_xor.accumulate(h ^ l)
    x = np.bitwise_xor.accumulate(np.where(d == 1, l, h)).astype(np.uint8)
    return x, (x ^ d).astype(np.uint8)


def puncture_34_fengyun(coded):
    """From each 6 coded symbols e0..e5 transmit e0, e1, e3, e4 (the inverse of Viterbi3_4::depuncture in fymode, shift 0: "110")."""
    n = coded.size // 6 * 6
    return coded[:n].reshape(-1, 6)[:, [0, 1, 3, 4]].reshape(-1)


def fengyun_diff_branches(nframes, seed=0, errors=()):
    """What both FengYun-3 transmitters send before the convolutional code: (the I branch's bits y, the Q branch's bits x, the CADUs the
    decoders write [n, 1024]). Randomised CADUs with RS(255,223) I=4 dual basis (`errors`: (frame, codeword, nbytes) byte errors added on
    air), then the inverse of the differential decoder."""
    tx_bits, clear = dump_frames(nframes, seed)
    tx = np.packbits(tx_bits, axis=1)
    rng = np.random.default_rng(seed + 1)
    for fr, cw, nb in errors:  # codeword cw holds bytes 4 + cw, 4 + cw + 4, ... of the frame
        pos = 4 + cw + 4 * rng.choice(255, nb, replace=False)
        tx[fr, pos] ^= rng.integers(1, 256, nb, dtype=np.uint8)
    x, y = fengyun_diff_encode(np.unpackbits(tx, axis=1).reshape(-1))
    return y, x, clear


def fengyun_frames(nframes, seed=0, errors=()):
    """The FengYun-3 AHRPT transmitter: (tx soft-symbol branches (I bits, Q bits) as uint8, the CADUs fengyun_ahrpt_decoder writes
    [n, 1024]). fengyun_diff_branches, then per branch the r=1/2 k=7 (79, 109) code punctured to 3/4 as FengYun does."""
    y, x, clear = fengyun_diff_branches(nframes, seed, errors)
    return puncture_34_fengyun(conv_encode(y)), puncture_34_fengyun(conv_encode(x)), clear


def fengyun_soft(i_bits, q_bits, amp=60.0, sigma=0.0, seed=0, invert_second=False, swap_branches=False):
    """int8 soft pairs that fengyun_ahrpt_decoder reads: bit 1 -> +amp; the module swaps I and Q of every pair first, so the Q branch goes
    in byte 0 and the I branch in byte 1. invert_second: the Q branch sent negated (the module complements it back); swap_branches: the
    two branches exchanged on air."""
    I, Q = (q_bits, i_bits) if swap_branches else (i_bits, q_bits)
    n = min(I.size, Q.size)
    out = np.empty(2 * n, np.float32)
    out[1::2] = (2.0 * I[:n] - 1.0) * amp
    out[0::2] = (2.0 * Q[:n] - 1.0) * amp * (-1.0 if invert_second else 1.0)
    if sigma:
        out += np.random.default_rng(seed).normal(0, sigma, out.size).astype(np.float32)
    return np.clip(np.round(out), -127, 127).astype(np.int8)


# ---- FengYun-3 MPT (fengyun_mpt_decoder) ------------------------------------------------------------------------------------------------
def fengyun_mpt_frames(nframes, seed=0, errors=()):
    """The FengYun-3 MPT transmitter: (the I and Q branches' code symbols as uint8, the CADUs fengyun_mpt_decoder writes [n, 1024]).
    fengyun_diff_branches, then per branch the unpunctured r=1/2 k=7 (79, 109) code."""
    y, x, clear = fengyun_diff_branches(nframes, seed, errors)
    return conv_encode(y), conv_encode(x), clear


def fengyun_mpt_pairs(i_bits, q_bits, phase90=False):
    """The code symbols in the order fengyun_mpt_decoder reads them, as (byte 0 bits, byte 1 bits) of each soft pair. The module takes I
    from byte 1 and the complement of byte 0 as Q, then exchanges the two symbols of every branch pair, so branch symbol k of a read
    rides on pair k ^ 1. phase90: each branch pair (a, b) sent as (not b, a), which Viterbi1_2's PHASE_90 rotation undoes."""
    n = min(i_bits.size, q_bits.size) & ~1

    def rot(c):
        c = np.asarray(c[:n], np.uint8)
        if not phase90:
            return c
        r = np.empty_like(c)
        r[0::2], r[1::2] = 1 - c[1::2], c[0::2]
        return r
    idx = np.arange(n) ^ 1
    return 1 - rot(q_bits)[idx], rot(i_bits)[idx]


def fengyun_mpt_soft(i_bits, q_bits, amp=60.0, sigma=0.0, seed=0, swap_branches=False, phase90=False):
    """int8 soft pairs that fengyun_mpt_decoder reads (bit 1 -> +amp, see fengyun_mpt_pairs). swap_branches: the two branches exchanged
    on air; phase90: see fengyun_mpt_pairs."""
    b0, b1 = fengyun_mpt_pairs(*((q_bits, i_bits) if swap_branches else (i_bits, q_bits)), phase90=phase90)
    out = np.empty(2 * b0.size, np.float32)
    out[0::2] = (2.0 * b0 - 1.0) * amp
    out[1::2] = (2.0 * b1 - 1.0) * amp
    if sigma:
        out += np.random.default_rng(seed).normal(0, sigma, out.size).astype(np.float32)
    return np.clip(np.round(out), -127, 127).astype(np.int8)


def aqua_db_frames(nframes, seed=0):
    """(decoded bits uint8 [n, 8192]: randomised CADUs with RS(255,223) I=4 dual basis, the CADUs aqua_db_decoder writes for them
    [n, 1024]: the ASM and the derandomised codewords). The decoder's frame format is metop_dump_decoder's."""
    return dump_frames(nframes, seed)


def aqua_db_rails(bits):
    """The hard symbols on air for the decoded stream A0 B0 A1 B1 ... (even length): each rail NRZ-M encoded on its own (the decoder's two
    NRZMDiff::decode_bits, each starting from 0, undo it), rail A on Q and rail B on I, as constellation_t::soft_demod's 2*(Q>0) + (I>0)
    and the module's demod >> 1, demod & 1 read them. Returns (I, Q) uint8."""
    b = np.asarray(bits, np.uint8).reshape(-1)
    return np.bitwise_xor.accumulate(b[1::2]), np.bitwise_xor.accumulate(b[0::2])


def aqua_db_soft(bits, amp=60.0, sigma=0.0, seed=0, swap_iq=False):
    """int8 soft pairs (I, Q) that aqua_db_decoder decodes to `bits` (bit 1 -> +amp); swap_iq: the rails on the wrong axes."""
    I, Q = aqua_db_rails(bits)
    if swap_iq:
        I, Q = Q, I
    out = np.empty(2 * I.size, np.float32)
    out[0::2], out[1::2] = (2.0 * I - 1.0) * amp, (2.0 * Q - 1.0) * amp
    if sigma:
        out += np.random.default_rng(seed).normal(0, sigma, out.size).astype(np.float32)
    return np.clip(np.round(out), -127, 127).astype(np.int8)


def terra_db_frames(nframes, seed=0):
    """(BPSK symbols on air as bits uint8, the CADUs ccsds_conv_concat_decoder writes for them [n, 1024]) of EOS.json "terra_db"'s decoder
    (bpsk_90, nrzm, RS(255,223) I=4 dual basis, derand_after_rs from byte 10). The CADUs are sent as RS codewords without randomisation
    (the receiver derandomises after RS), NRZ-M encoded and convolutionally encoded. The module swaps each soft pair and rotates it by 90
    degrees, (s0, s1) -> (s0, -s1), so a code pair (a, b) goes on air as (a, not b)."""
    payload = np.random.default_rng(seed).integers(0, 256, size=(nframes, 4 * 223), dtype=np.uint8)
    tx, _ = build_cadus(payload, 4, randomize=False)
    written = tx.copy()
    written[:, 10:] ^= ccsds_pn(1014)[None, :]
    coded = conv_encode(nrzm_encode(np.unpackbits(tx.reshape(-1))))
    coded[1::2] ^= 1
    return coded, written


# ---- CCSDS turbo code (CCSDS 131.0-B section 6), as ccsds_turbo_decoder receives it ---------------------------------------------------
TURBO_ASM = {2: 0x034776C7272895B0, 3: 0x25D5C0CE8990F6C9461BF79C, 4: 0x034776C7272895B0FCB88938D8D76A4F,
             6: 0x25D5C0CE8990F6C9461BF79CDA2A3F31766F0936B9E40863}   # attached sync marker per rate 1/2, 1/3, 1/4, 1/6
TURBO_ASM_BITS = {2: 64, 3: 96, 4: 128, 6: 192}
TURBO_BASES = (223, 446, 892, 1115)
# feed-forward polynomials of the upper and lower component codes (taps 0..4; the first one is the systematic output), feedback 0011
TURBO_CODES = {2: (("10011", "11011"), ("11011",)), 3: (("10011", "11011"), ("11011",)), 4: (("10011", "10101", "11111"), ("11011",)),
               6: (("10011", "11011", "10101", "11111"), ("11011", "11111"))}


def turbo_interleaver(base):
    """The CCSDS turbo interleaver pi for k = 8 base bits (CCSDS 131.0-B 6.3): the lower encoder reads info[pi[j]] at step j."""
    p = (31, 37, 43, 47, 53, 59, 61, 67)
    k1, k2 = 8, base
    s = np.arange(8 * base)
    m = s % 2
    i = s // (2 * k2)
    j = s // 2 - i * k2
    t = (19 * i + 1) % (k1 // 2)
    q = t % 8
    c = (np.array(p)[q] * j + 21 * m) % k2
    return 2 * (t + c * (k1 // 2) + 1) - m - 1


def turbo_codeword_bits(rate, base):
    n = 8 * base + 4
    return 2 * n if rate == 2 else rate * n


def _rsc_encode(bits, taps):
    """Recursive systematic component encoder with feedback 1 + D^3 + D^4 ("0011" on registers 1..4) over bits [nframes, K], terminated
    by 4 tail steps that feed the feedback back in. Returns uint8 [nframes, K + 4, len(taps)]."""
    nf, K = bits.shape
    reg = np.zeros((nf, 4), np.uint8)   # registers 1..4
    fwd = np.array([[int(ch) for ch in t] for t in taps], np.uint8)
    out = np.zeros((nf, K + 4, len(taps)), np.uint8)
    for k in range(K + 4):
        fb = reg[:, 2] ^ reg[:, 3]
        u = bits[:, k] if k < K else fb
        first = u ^ fb
        for c in range(len(taps)):
            o = fwd[c, 0] & first
            for r in range(4):
                o = o ^ (fwd[c, r + 1] & reg[:, r])
            out[:, k, c] = o
        reg = np.concatenate([first[:, None], reg[:, :3]], axis=1)
    return out


def turbo_encode(info_bytes, rate):
    """uint8 [nframes, base] -> the turbo codewords as sent, bits uint8 [nframes, codeword bits]: per trellis step the upper code's outputs
    then the lower code's (on the interleaved bits); rate 1/2 keeps the systematic bit and alternately the upper and the lower parity."""
    info_bytes = np.atleast_2d(np.asarray(info_bytes, np.uint8))
    nf, base = info_bytes.shape
    bits = np.unpackbits(info_bytes, axis=1)
    up_taps, lo_taps = TURBO_CODES[rate]
    up = _rsc_encode(bits, up_taps)
    lo = _rsc_encode(bits[:, turbo_interleaver(base)], lo_taps)
    full = np.concatenate([up, lo], axis=2).reshape(nf, -1)
    if rate != 2:
        return full
    k = np.arange(full.shape[1])
    keep = (k % 3 == 0) | np.where((k // 3) % 2 == 1, k % 3 == 2, k % 3 == 1)
    return full[:, keep]


def crc16_ccitt(data):
    """CRC-16, polynomial 0x1021, initial value 0xFFFF, no reflection, no final xor, over each row of uint8 [n, len]."""
    data = np.atleast_2d(np.asarray(data, np.uint8))
    crc = np.full(data.shape[0], 0xFFFF, np.uint32)
    for col in range(data.shape[1]):
        crc ^= data[:, col].astype(np.uint32) << 8
        for _ in range(8):
            crc = np.where(crc & 0x8000, (crc << 1) ^ 0x1021, crc << 1) & 0xFFFF
    return crc


def turbo_frames(nframes, rate, base, seed=0):
    """(tx bits uint8 [n, ASM + codeword bits] = the rate's ASM + the PN-randomised codeword, the CADUs the decoder writes for them
    [n, 4 + base] = 1A CF FC 1D + the information bytes, whose last two are the CRC-16 of the others)."""
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, (nframes, base - 2), dtype=np.uint8)
    crc = crc16_ccitt(data)
    info = np.concatenate([data, (crc >> 8).astype(np.uint8)[:, None], (crc & 0xFF).astype(np.uint8)[:, None]], axis=1)
    cw = turbo_encode(info, rate)
    nasm = TURBO_ASM_BITS[rate]
    asm = np.unpackbits(np.frombuffer(TURBO_ASM[rate].to_bytes(nasm // 8, "big"), np.uint8))
    tx = np.concatenate([np.tile(asm, (nframes, 1)), cw ^ ldpc_pn_bits(cw.shape[1])[None, :]], axis=1)
    cadu = np.concatenate([np.tile(np.frombuffer(ASM, np.uint8), (nframes, 1)), info], axis=1)
    return tx, cadu


def fsk_signal(nsamples, samplerate, symbolrate, h=0.7, seed=0, bits=None, carrier=0.0, rate_offset=0.0, snr_db=None, zeros=(), fmt="cf32",
               amp=0.5):
    """Continuous-phase FSK: the bits (random from seed when None) mapped 0 -> -1, 1 -> +1, held for a symbol each, frequency deviation
    h * symbolrate / 2, plus a carrier offset (Hz), a sample-rate offset (relative), AWGN at snr_db (None: none) and stretches of zero
    samples zeros = ((start, length), ...). Returns (iq as cf32 complex64 / cs16 or cs8 interleaved int, the bits)."""
    rng = np.random.default_rng(seed)
    sps = samplerate / symbolrate * (1.0 + rate_offset)
    nsym = int(np.ceil(nsamples / sps)) + 2
    if bits is None:
        bits = rng.integers(0, 2, nsym, dtype=np.uint8)
    bits = np.resize(np.asarray(bits, np.uint8), nsym)
    k = np.minimum((np.arange(nsamples) / sps).astype(np.int64), nsym - 1)
    f = (2.0 * bits[k].astype(np.float64) - 1.0) * (h * symbolrate / 2.0) + carrier
    phase = 2.0 * np.pi * np.cumsum(f) / samplerate
    x = amp * np.exp(1j * phase)
    if snr_db is not None:
        sigma = amp / np.sqrt(2.0) * 10.0 ** (-snr_db / 20.0)
        x = x + sigma * (rng.standard_normal(nsamples) + 1j * rng.standard_normal(nsamples))
    for a, n in zeros:
        x[a:a + n] = 0
    if fmt == "cf32":
        return x.astype(np.complex64), bits
    scale = 32767.0 if fmt == "cs16" else 127.0
    dt = np.int16 if fmt == "cs16" else np.int8
    out = np.empty(2 * nsamples, dt)
    out[0::2] = np.clip(np.round(x.real * scale), -scale, scale)
    out[1::2] = np.clip(np.round(x.imag * scale), -scale, scale)
    return out, bits


def fsk_frames(nframes, cadu_size, seed=0):
    """(coded bits on air, the CADUs ccsds_conv_concat_decoder writes for them [n, cadu_size / 8]) of BlueWalker3.json's decoder: bpsk_90,
    cadu_size bits (ASM + payload, no Reed-Solomon), randomised from byte 4, rate 1/2 convolutional code. As for terra_db_frames, the
    module swaps each soft pair and rotates it by 90 degrees, so a code pair (a, b) goes on air as (a, not b)."""
    nb = cadu_size // 8
    payload = np.random.default_rng(seed).integers(0, 256, size=(nframes, nb - 4), dtype=np.uint8)
    clear = np.concatenate([np.tile(np.frombuffer(ASM, np.uint8), (nframes, 1)), payload], axis=1)
    tx = clear.copy()
    tx[:, 4:] ^= ccsds_pn(nb - 4)[None, :]
    coded = conv_encode(np.unpackbits(tx.reshape(-1)))
    coded[1::2] ^= 1
    return coded, clear
