"""CPU: the oracle itself. (1) our C restatement (oracle.c) == the reference's own code (oracle/_ref) bit for bit, stage by
stage — against the reference's committed results where oracle/_ref is not built (tests/refpin.py); (2) both reproduce the committed
golden fixtures (made from the reference by tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from tests.common import ROOT, oracle_demod, oracle_fec, signal, simple_soft_cases
from tests.refpin import Pin
from satdump_b200 import synth

GOLD = os.path.join(ROOT, "tests", "golden")
CONFIGS = ["metop_ahrpt", "bpsk_half", "jpss_hrd", "dvbs2_front", "hrpt_bpsk", "metop_oversampled", "bpsk_decim8", "qpsk_undersampled", "psk8", "bpsk_simple", "qpsk_simple",
           "qpsk_p34", "qpsk_p78",  # ccsds_conv_concat_decoder with conv_rate 3/4, 7/8 (Viterbi_Depunc)
           "pm_bpsk"]  # pm_demod in front of ccsds_conv_concat_decoder


def _ref():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    return ref


def bitwise(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("name", CONFIGS)
def test_port_matches_golden(built, name):
    from oracle import port
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    cfg = synth.CONFIGS[name]
    o = oracle_demod(port, cfg).run(g["raw"])
    assert o["mm"].size == int(g["nsym"])
    assert bitwise(o["agc"][:4096], g["agc_head"]) and bitwise(o["fir"][:4096], g["fir_head"]) and bitwise(o["mm"][:4096], g["mm_head"])
    if "costas_head" in g:
        assert bitwise(o["costas"][:4096], g["costas_head"])
    if "pll_head" in g:  # pm_demod: carrier PLL and PMToBPSK outputs
        assert bitwise(o["pll"][:4096], g["pll_head"]) and bitwise(o["pm"][:4096], g["pm_head"])
    if "resamp_head" in g:  # front-end resampler: output, length and polyphase bank
        dc = oracle_demod(port, cfg).cfg
        assert bitwise(port.resample(dc, g["raw"])[:4096], g["resamp_head"]) and o["front"] == int(g["front"])
        assert bitwise(port.resampler_taps(int(dc.final_samplerate), int(dc.samplerate)), g["resamp_bank"])
    assert np.array_equal(o["soft"], g["soft"])
    if cfg.decoder in ("metop", "ccsds", "simple"):
        f = oracle_fec(port, cfg).run(o["soft"])
        assert np.array_equal(f["cadu"], g["cadu"])
        assert np.array_equal(np.packbits(f["bits"]), g["bits"]) and f["bits"].size == int(g["nbits"])
        assert np.array_equal(f["vit_state"], g["vit_state"]) and np.array_equal(f["defr_state"], g["defr_state"])
        assert np.array_equal(f["rs_err"], g["rs_err"])


@pytest.mark.parametrize("name", CONFIGS)
def test_ref_matches_golden(built, name):
    ref = _ref()
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    cfg = synth.CONFIGS[name]
    o = oracle_demod(ref, cfg).run(g["raw"])
    assert np.array_equal(o["soft"], g["soft"]) and bitwise(o["mm"][:4096], g["mm_head"])
    if cfg.decoder in ("metop", "ccsds", "simple"):
        assert np.array_equal(oracle_fec(ref, cfg).run(o["soft"])["cadu"], g["cadu"])


@pytest.mark.parametrize("name", CONFIGS)
def test_port_equals_reference_fresh_signal(built, name):
    """A signal that is not in the fixtures, longer, different seed."""
    from oracle import port
    pin = Pin(f"fresh_signal[{name}]")
    cfg, raw, _ = signal(name, 18, seed=11)
    a, b = pin.run(lambda R: oracle_demod(R, cfg).run(raw)), oracle_demod(port, cfg).run(raw)
    for k in ("agc", "fir", "costas", "mm", "soft"):
        if b[k] is not None:
            pin.equal(k, a and a[k], b[k])
    if cfg.decoder in ("metop", "ccsds", "simple"):  # (the soft bytes are the reference's: checked above)
        fa, fb = pin.run(lambda R: oracle_fec(R, cfg).run(b["soft"])), oracle_fec(port, cfg).run(b["soft"])
        for k in ("cadu", "bits", "vit_state", "defr_state", "rs_err"):
            pin.equal("fec_" + k, fa and fa[k], fb[k])


def test_simple_psk_decoder_port_equals_reference_and_golden(built):
    """ccsds_simple_psk_decoder: the C restatement follows the reference's module loop in every mode; the committed fixture
    (tests/golden/simple_psk.npz, made from the reference) pins both."""
    from oracle import port
    cases, clear = simple_soft_cases()
    g = np.load(os.path.join(GOLD, "simple_psk.npz"))
    for name, kw, soft in cases:
        cfg = port.simple_cfg(cadu_size=8192, rs_i=4, **kw)
        f = port.Fec(cfg)
        n = soft.size // f.chunk * f.chunk
        b = f.run(soft[:n])
        assert np.array_equal(soft, g[f"{name}_soft"]), name  # the generator is deterministic
        assert np.array_equal(b["cadu"], g[f"{name}_cadu"]) and np.array_equal(np.packbits(b["bits"]), g[f"{name}_bits"]), name
        from oracle import ref
        if ref.available():
            a = ref.Fec(cfg).run(soft[:n])
            for k in ("cadu", "bits", "defr_state", "vit_state", "rs_err"):
                assert np.array_equal(a[k], b[k]), (name, k)
        fr = b["cadu"].reshape(-1, 1024)[:, :4 + 4 * 223]  # RS replaces the message bytes only: compare those with what was sent
        sent = clear[:, :4 + 4 * 223]
        assert fr.shape[0] >= 20 and sum(any(np.array_equal(x, c) for c in sent) for x in fr) >= fr.shape[0] - 2, name


def test_dc_block_port_equals_reference(built):
    """CorrectIQBlock in front (dc_block), alone and with iq_swap and the resampler behind it."""
    from oracle import port
    from tests.common import demod_kwargs
    pin = Pin("dc_block")
    for i, (name, kw) in enumerate([("metop_ahrpt", dict(dc_block=True)), ("metop_ahrpt", dict(dc_block=True, iq_swap=True)), ("hrpt_bpsk", dict(dc_block=True)),
                                    ("bpsk_half", dict(post_costas_dc=True)), ("metop_ahrpt", dict(dc_block=True, post_costas_dc=True))]):
        cfg, raw, _ = signal(name, 17, seed=4)
        raw = raw + np.complex64(0.02 + 0.01j) if cfg.fmt == "cf32" else raw + np.int16(300)
        a = pin.run(lambda R: R.Demod(R.demod_cfg(**kw, **demod_kwargs(cfg))).run(raw))
        b = port.Demod(port.demod_cfg(**kw, **demod_kwargs(cfg))).run(raw)
        for k in ("agc", "fir", "costas", "mm", "soft"):
            pin.equal(f"{i}_{name}_{k}", a and a[k], b[k])


def test_final_samplerate_rule():
    """BaseDemodModule::initb's choice of the working rate (module_demod_base.cpp:59-80), Python restatement vs the C ABI helper."""
    from oracle import port
    from satdump_b200 import capi
    cases = [(3e6, 665400, "bpsk", 2400000.0), (6e6, 2333333, "qpsk", 6e6), (30e6, 15e6, "oqpsk", 30e6), (2.6e6, 2.4e6, "qpsk", 2640000.0),
             (50e6, 15e6, "oqpsk", None), (1e6, 72000, "bpsk", None), (12.5e6, 3.5e6, "qpsk", 12.5e6)]
    for fs, rs, con, want in cases:
        a, b = port.final_samplerate_of(fs, rs, con), capi.final_samplerate_of(fs, rs, con)
        assert a == b, (fs, rs, con, a, b)
        if want is not None:
            assert a == want, (fs, rs, con, a)
    assert port.final_samplerate_of(6e6, 2e6, "qpsk", min_sps=2.0, max_sps=2.0) == capi.final_samplerate_of(6e6, 2e6, "qpsk", 2.0, 2.0) == 4e6
    assert capi.final_samplerate_of(6e6, 2e6, "qpsk", custom=5e6) == 5e6


def test_resampler_streaming_equals_one_shot(built):
    """The rational resampler's carried counters / history: any chunking gives the same stream (reference and restatement)."""
    from oracle import port, ref
    cfg, raw, _ = signal("hrpt_bpsk", 17, seed=3)
    pin = Pin("resampler_streaming")
    for O in ((ref, port) if pin.live else (port,)):
        one = oracle_demod(O, cfg).run(raw)
        d = oracle_demod(O, cfg)
        parts = [d.run(raw[a:b]) for a, b in [(0, 33333), (33333, 33334), (33334, 100001), (100001, raw.size)]]
        assert bitwise(np.concatenate([p["agc"] for p in parts]), one["agc"])
        assert np.array_equal(np.concatenate([p["soft"] for p in parts]), one["soft"])
        if O is port:
            a = pin.run(lambda R: oracle_demod(R, cfg).run(raw))
            pin.equal("agc", a and a["agc"], one["agc"])
            pin.equal("soft", a and a["soft"], one["soft"])


def test_port_low_snr_matches_reference(built):
    """Es/N0 5.5 dB: Viterbi makes errors, RS corrects most of them; the restatement must follow the reference through it."""
    from oracle import port
    pin = Pin("low_snr")
    cfg, raw, _ = signal("metop_ahrpt", 19, seed=5, esn0=5.5)
    a = pin.run(lambda R: oracle_demod(R, cfg).run(raw, stages=False))
    soft = oracle_demod(port, cfg).run(raw, stages=False)["soft"]
    pin.equal("soft", a and a["soft"], soft)
    fa, fb = pin.run(lambda R: oracle_fec(R, cfg).run(soft)), oracle_fec(port, cfg).run(soft)
    assert fb["rs_err"].sum() > 0, "the stress case should exercise RS"
    for k in ("cadu", "bits", "vit_state", "defr_state", "rs_err"):
        pin.equal(k, fa and fa[k], fb[k])


def test_rs_stress_golden(built):
    """RS(255,223) I=4 with 0..20 byte errors per codeword: corrections, the 'parity bytes stay as received' rule and the
    failure verdicts (libcorrect: locator degree != root count) all match the reference's output."""
    from oracle import port
    g = np.load(os.path.join(GOLD, "rs_stress.npz"))
    nfail = 0
    for f in range(g["noisy"].shape[0]):
        d, e = port.rs_decode_interleaved(g["noisy"][f], True, 4)
        assert np.array_equal(d, g["decoded"][f]) and np.array_equal(e, g["errors"][f])
        nfail += int((e < 0).sum())
    assert nfail > 10


def test_primitives_vs_reference(built):
    from oracle import port
    pin = Pin("primitives")
    rng = np.random.default_rng(3)
    bits = rng.integers(0, 2, 5000, dtype=np.uint8)
    pin.equal("cc_encode", pin.run(lambda R: R.cc_encode(bits)), port.cc_encode(bits))
    syms = rng.integers(0, 256, 3 * 2 * 1024 + 12, dtype=np.uint8)
    pin.equal("cc_decode", pin.run(lambda R: R.cc_decode(syms, 1024, 3)), port.cc_decode(syms, 1024, 3))
    soft = rng.integers(-128, 128, 4096, dtype=np.int8)
    for ph in range(4):
        for sw in (0, 1):
            pin.equal(f"rotate_soft_{ph}_{sw}", pin.run(lambda R: R.rotate_soft(soft, ph, sw)), port.rotate_soft(soft, ph, sw))
    pin.equal("derand", pin.run(lambda R: R.derand(np.zeros(1020, np.uint8))), port.derand(np.zeros(1020, np.uint8)))
    pin.equal("rrc_design", pin.run(lambda R: R.rrc_design(1, 6e6, 2333333, 0.5, 31)), port.rrc_design(1, 6e6, 2333333, 0.5, 31))
    pin.equal("mm_taps", pin.run(lambda R: R.mm_taps()), port.mm_taps())


def test_simple_psk_decoder_options_port_equals_reference(built):
    """rs_i = 0, RS(255,239), derandomiser off / after RS, rs_usecheck, another ASM, 10232-bit CADUs with I = 5, the derandomiser from byte 0
    (over the ASM) and from byte 10 after RS — restatement vs reference."""
    from oracle import port
    pin = Pin("simple_psk_options")
    rng = np.random.default_rng(9)
    for kw in [dict(rs_i=0, derandomize=False), dict(rs_i=4, rs_type=1), dict(rs_i=4, derand_after_rs=True), dict(rs_i=4, rs_usecheck=True),
               dict(rs_i=4, asm_sync=0xFAF3200D), dict(rs_i=5, cadu_size=10232), dict(rs_i=1, cadu_size=2072), dict(rs_i=4, derand_start=0),
               dict(rs_i=4, derand_start=10, derand_after_rs=True)]:
        kw = dict(kw)
        cadu_size = kw.pop("cadu_size", 8192)
        body = rng.integers(0, 256, size=(12, cadu_size // 8 - 4), dtype=np.uint8)
        asm = np.frombuffer(int(kw.get("asm_sync", 0x1ACFFC1D)).to_bytes(4, "big"), np.uint8)
        bits = np.unpackbits(np.concatenate([np.tile(asm, (12, 1)), body], axis=1).reshape(-1))
        soft = np.clip(np.round((bits * 2.0 - 1) * 60 + rng.normal(0, 15, bits.size)), -127, 127).astype(np.int8)
        for con in ("bpsk", "qpsk"):
            cfg = port.simple_cfg(con, cadu_size, **kw)
            fb = port.Fec(cfg)
            n = soft.size // fb.chunk * fb.chunk
            a, b = pin.run(lambda R: R.Fec(cfg).run(soft[:n])), fb.run(soft[:n])
            for k in ("cadu", "bits", "defr_state", "vit_state", "rs_err"):
                pin.equal(f"{sorted(kw.items())}_{cadu_size}_{con}_{k}", a and a[k], b[k])
        assert b["bits"].size == n


def test_resampler_port_equals_reference_over_rates_and_formats(built):
    """The front-end resampler restatement vs the reference over decimating and interpolating ratios, every sample format, with and
    without iq_swap / dc_block, and over ratios that put the power-of-two decimator in front."""
    from oracle import port
    pin = Pin("resampler_rates_formats")
    rng = np.random.default_rng(5)
    cases = [(3e6, 665400, "bpsk"), (12e6, 2333333, "qpsk"), (2.6e6, 2.4e6, "qpsk"), (1.05e6, 1e6, "bpsk"), (7e6, 1.5e6, "qpsk"), (40e6, 15e6, "oqpsk"),
             (10.5e6, 2.5e6, "qpsk")]
    for fs, rs, con in cases:
        for fmt in ("cs16", "cs8", "cf32"):
            n = 40000
            if fmt == "cf32":
                raw = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) * 0.3
            else:
                raw = (rng.standard_normal(2 * n) * (3000 if fmt == "cs16" else 30)).astype(np.int16 if fmt == "cs16" else np.int8)
            for extra in (dict(), dict(iq_swap=True, dc_block=True)):
                cfg = port.demod_cfg(fs, rs, con, 0.5, fmt=fmt, **extra)
                assert cfg.final_samplerate > 0 and cfg.samplerate / cfg.final_samplerate < 2, (fs, rs)
                pin.equal(f"{fs}_{rs}_{con}_{fmt}_{len(extra)}", pin.run(lambda R: R.resample(cfg, raw)), port.resample(cfg, raw))
    # the product's host-side design of the same banks (b200_demod_resampler_bank needs no device): bitwise
    from satdump_b200 import capi
    for fs, rs, con in cases:
        fin = port.final_samplerate_of(fs, rs, con)
        bank, i, d = capi.resampler_bank(fs, fin)
        pin.equal(f"bank_{fs}_{fin}", pin.run(lambda R: R.resampler_taps(int(fin), int(fs))), bank)
    # ratios >= 2: SmartResamplerBlock's power-of-two decimator in front (one to three DecimatingFIR stages), with and without a
    # rational part behind it
    for fs, rs, con in [(6e6, 233333, "qpsk"), (24e6, 2333333, "qpsk"), (32e6, 1e6, "bpsk"), (100e6, 1.2e6, "bpsk"), (90e6, 2e6, "qpsk")]:
        for fmt in ("cs16", "cf32"):
            n = 300000
            raw = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) * 0.3 if fmt == "cf32"
                   else (rng.standard_normal(2 * n) * 3000).astype(np.int16))
            cfg = port.demod_cfg(fs, rs, con, 0.5, fmt=fmt)
            assert cfg.samplerate / cfg.final_samplerate >= 2
            b = port.resample(cfg, raw)
            assert b.size > 1000
            pin.equal(f"decim_{fs}_{rs}_{con}_{fmt}", pin.run(lambda R: R.resample(cfg, raw)), b)


@pytest.mark.parametrize("name", ["qpsk_p23", "qpsk_p34", "qpsk_p56", "qpsk_p78"])
def test_viterbi_depunc_port_equals_reference(built, name):
    """Viterbi_Depunc (viterbi_punc.cpp, depunc.h) at its four rates: the C restatement follows the reference bit for bit - decoded bits,
    lock state and BER per module call, CADUs - also through noise -> signal -> noise (lock search on the persistent test buffer, unlock after
    viterbi_outsync_after bad calls, a second lock with the sliding buffer's leftover and the held-back symbol carried over)."""
    from oracle import port
    pin = Pin(f"viterbi_depunc[{name}]")
    cfg = synth.CONFIGS[name]
    raw, _ = synth.make_signal(cfg, 1 << 20, seed=0x600D + 1)
    soft = oracle_demod(port, cfg).run(raw.numpy(), stages=False)["soft"]
    pin.equal("soft", pin.run(lambda R: oracle_demod(R, cfg).run(raw.numpy(), stages=False)["soft"]), soft)
    rng = np.random.default_rng(5)
    noise = lambda n: rng.integers(-60, 61, n).astype(np.int8)
    stream = np.concatenate([noise(8192 * 5 + 16), soft[:400000], noise(8192 * 40 + 2), soft[400000:], noise(8192 * 3)])
    r, p = pin.run(lambda R: oracle_fec(R, cfg).run(stream)), oracle_fec(port, cfg).run(stream)
    assert (p["vit_state"] == 0).any() and (p["vit_state"] > 0).any() and p["bits"].size > 300000 and p["cadu"].size >= 10 * cfg.cadu_bytes
    for k in ("bits", "cadu", "vit_state", "defr_state", "rs_err", "vit_ber"):
        pin.equal(k, r and r[k], p[k])


def test_fast_trig_restatement_equals_reference(built):
    """fast_atan2f (table regenerated from atan() through seven significant digits), fast_cos, fast_sin of common/dsp/utils/fast_trig.cpp:
    every table cell, every quadrant, the small-ratio branch and random arguments, bit for bit."""
    from oracle import port
    pin = Pin("fast_trig")
    P = port.lib()
    rng = np.random.default_rng(7)
    zs = np.concatenate([np.linspace(0, 1, 256 * 4 + 1), rng.random(4000), [0.0, 0.0039, 0.00393, 1.0]]).astype(np.float32)
    yx = [(y, x) for z in zs for y, x in ((z, 1.0), (1.0, z), (-z, 1.0), (z, -1.0), (-1.0, -z), (-z, -1.0), (1.0, -z), (-1.0, z))] + [(0.0, 0.0)]
    at = lambda L: np.array([L.ref_fast_atan2f(float(y), float(x)) for y, x in yx], np.float32)
    pin.equal("atan2", pin.run(lambda R: at(R.lib())), at(P))
    assert P.ref_fast_atan2f(0.0, 0.0) == 0.0
    vs = np.concatenate([np.linspace(-3.3, 3.3, 6001), rng.standard_normal(2000) * 2]).astype(np.float32)
    cs = lambda L: np.array([(L.ref_fast_cos(float(v)), L.ref_fast_sin(float(v))) for v in vs], np.float32)
    pin.equal("cos_sin", pin.run(lambda R: cs(R.lib())), cs(P))


def test_psk_demod_carrier_mode_port_equals_reference(built):
    """psk_demod with "has_carrier" (module_psk_demod.cpp:93-116): RRC -> PLLCarrierTrackingBlock -> CorrectIQBlock -> Costas (limit 0.2)."""
    from oracle import port
    from tests.common import match_frames
    pin = Pin("carrier_mode")
    cfg, raw, clear = signal("bpsk_carrier", 20, seed=11)
    b = oracle_demod(port, cfg)
    ra, rb = pin.run(lambda R: (lambda a: (a.run(raw), a.pm_state()))(oracle_demod(R, cfg))), b.run(raw)
    for k in ("agc", "fir", "pll", "carrier_dc", "costas", "mm", "soft"):
        pin.equal(k, ra and ra[0][k], rb[k])
    pin.equal("pm_state", ra and np.array(list(ra[1].values()), np.float32), np.array(list(b.pm_state().values()), np.float32))
    fr = oracle_fec(port, cfg).run(rb["soft"])["cadu"].reshape(-1, cfg.cadu_bytes)
    assert fr.shape[0] >= 10 and match_frames(fr, clear)[1]


@pytest.mark.parametrize("name", ["pm_bpsk", "pm_bpsk_after", "pm_bpsk_front"])
def test_pm_demod_port_equals_reference(built, name):
    """pm_demod's chain (AGC -> carrier PLL -> PMToBPSK -> [resampler -> AGC2] -> RRC -> Costas -> M&M), restatement against the
    compiled reference modules stage by stage, and the decoded CADUs against the transmitted frames."""
    from oracle import port
    from tests.common import match_frames
    pin = Pin(f"pm_demod[{name}]")
    cfg, raw, clear = signal(name, 20, seed=11)
    b = oracle_demod(port, cfg)
    ra, rb = pin.run(lambda R: (lambda a: (a.run(raw), a.pm_state()))(oracle_demod(R, cfg))), b.run(raw)
    for k in ("agc", "pll", "pm", "fir", "costas", "mm", "soft"):
        pin.equal(k, ra and ra[0][k], rb[k])
    pin.equal("front", ra and np.array([ra[0]["front"]], np.int64), np.array([rb["front"]], np.int64))
    pin.equal("pm_state", ra and np.array(list(ra[1].values()), np.float32), np.array(list(b.pm_state().values()), np.float32))
    fr = oracle_fec(port, cfg).run(rb["soft"])["cadu"].reshape(-1, cfg.cadu_bytes)
    first, ok = match_frames(fr, clear)
    assert fr.shape[0] >= 1 and ok, (fr.shape, first)  # (24 samples per symbol: 2^20 samples hold two to three CADUs)


def test_freq_shift_port_equals_reference(built):
    """FreqShiftBlock in front of psk_demod (module_demod_base.cpp:122-123): a carrier 150 kHz off is brought back; restatement against
    the compiled block (both on the shim's VOLK rotator), and the chain decodes."""
    import dataclasses
    from oracle import port
    from tests.common import demod_kwargs, match_frames
    pin = Pin("freq_shift")
    cfg = dataclasses.replace(synth.CONFIGS["metop_ahrpt"], carrier_rad=2 * np.pi * 150e3 / 6e6 + 1e-3)
    raw, clear = synth.make_signal(cfg, 1 << 19, seed=5)
    raw = raw.numpy()
    kw = demod_kwargs(cfg)
    b = port.Demod(port.demod_cfg(freq_shift=-150000.0, **kw))
    ra, rb = pin.run(lambda R: R.Demod(R.demod_cfg(freq_shift=-150000.0, **kw)).run(raw)), b.run(raw)
    for k in ("agc", "fir", "costas", "mm", "soft"):
        pin.equal(k, ra and ra[k], rb[k])
    assert abs(b.state()["freq"] - 1e-3) < 3e-4  # the Costas loop sees only the residual offset
    fr = oracle_fec(port, cfg).run(rb["soft"])["cadu"].reshape(-1, cfg.cadu_bytes)
    assert fr.shape[0] >= 2 and match_frames(fr, clear)[1]


@pytest.mark.parametrize("mpdu,iz,corrupt,drop", [(884, 0, 0.0, 0.0), (882, 2, 0.2, 0.05), (60, 0, 0.5, 0.1)])
def test_packet_demux_port_equals_reference(built, mpdu, iz, corrupt, drop):
    """CADU -> CCSDS space packets (ccsds_aos::Demuxer per virtual channel): restatement against the compiled reference on clean and
    damaged streams, with the secondary-header option, and on the crafted leftover-bytes corner."""
    from oracle import port
    pin = Pin(f"packet_demux[{mpdu}-{iz}-{corrupt}-{drop}]")
    fr = synth.build_aos_frames(6000, seed=12, mpdu=mpdu, insert_zone=iz, corrupt=corrupt, drop=drop)
    for ext in (False, True):
        a, b = pin.run(lambda R: R.Demux(mpdu, iz, ext).run(fr)), port.Demux(mpdu, iz, ext).run(fr)
        assert b[1].shape[0] > 100
        pin.equal(f"bytes_{ext}", a and a[0], b[0])
        pin.equal(f"records_{ext}", a and a[1], b[1])
    for variant in (0, 1):
        q = synth.craft_leftover_frames(mpdu, variant)
        a, b = pin.run(lambda R: R.Demux(mpdu, 0).run(q)), port.Demux(mpdu, 0).run(q)
        assert b[1][0, 2] > mpdu
        pin.equal(f"leftover_bytes_{variant}", a and a[0], b[0])
        pin.equal(f"leftover_records_{variant}", a and a[1], b[1])
