"""Soft and IQ streams of the aqua_db_decoder tests, rebuilt from seeds on any machine. tests/golden/make_eos_pins.py pins the reference's
output for each of them in tests/golden/eos_pins.json, which the tests read where the reference is absent.

A case edits the DECODED bit stream (the CADUs as the deframer sees them) before its two rails are NRZ-M encoded, so an ASM gets an exact
number of bit errors, a frame its exact RS errors, and a bit slip stays one bit; a symbol slip drops one soft pair."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests.common import after_lock as _after_lock, digest, load_pins

HERE = os.path.dirname(os.path.abspath(__file__))
PINS = os.path.join(HERE, "golden", "eos_pins.json")
READ = 65536      # the module's read (BUFFER_SIZE)
FRAME = 8192      # decoded bits per CADU = soft bytes per CADU

# name -> frames, edits (see stream()); every case starts with `lead` noise bytes and ends with noise up to a whole read
CASES = {
    "clean": dict(frames=60, lead=3000),
    "inverted": dict(frames=60, lead=2000, invert_from=25),                     # the stream flips polarity in frame 25: SYNCED -> NOSYNC -> inverted ASM
    "inverted_start": dict(frames=30, lead=0, invert_from=0),
    "synced_asm_9_10": dict(frames=60, lead=1000, asm_errors={20: 9, 30: 10}),  # SYNCED accepts < 10 errors: 9 passes, 10 is a hard NOSYNC
    "syncing_5_6": dict(frames=60, lead=1000, asm_errors={3: 5, 5: 6}),          # SYNCING accepts < 6: 5 passes, 6 is invalid
    "syncing_invalid": dict(frames=60, lead=1000, asm_errors={4: 16, 5: 16, 6: 16, 7: 16}),  # invalid > 2 in SYNCING
    "bit_slip": dict(frames=50, lead=1000, drop_bit=20 * FRAME + 4001),
    "symbol_slip": dict(frames=50, lead=1000, drop_symbol=20 * FRAME + 3000),
    "iq_swapped": dict(frames=30, lead=1000, swap_iq=True),                      # the rails on the wrong axes: never syncs
    "noise_signal_noise": dict(frames=40, lead=200000, tail=300000),
    "rs": dict(frames=30, lead=1000, rs_errors={5: (0, 3), 8: (1, 16), 11: (2, 17), 12: (3, 17)}),  # frame: (codeword, byte errors); 17 = t + 1
}
SIGMA = 12.0
RAGGED = (1, 3, 65535, 65537)  # piece sizes of the ragged pushes
LARGE_FRAMES = 8320            # >= 2^26 soft bytes in one push


pins = functools.partial(load_pins, PINS)


def _noise(rng, n):
    return np.clip(np.round(rng.normal(0, 60, n)), -127, 127).astype(np.int8)


def stream(name):
    """(soft int8, the sent CADUs [frames, 1024], index of the first decoded bit of frame 0 in the soft stream's bit numbering)"""
    c = CASES[name]
    seed = 100 + sorted(CASES).index(name)
    rng = np.random.default_rng(seed)
    bits, clear = synth.aqua_db_frames(c["frames"], seed)
    bits = bits.copy()
    for f, k in c.get("asm_errors", {}).items():
        bits[f, rng.choice(32, k, replace=False)] ^= 1
    for f, (cw, k) in c.get("rs_errors", {}).items():
        byte = 4 + 4 * rng.choice(223, k, replace=False) + cw  # byte i of the 1020 belongs to codeword i % 4
        bits[f, 8 * byte + rng.integers(0, 8, k)] ^= 1
    bits = bits.reshape(-1)
    if "invert_from" in c:
        bits[c["invert_from"] * FRAME:] ^= 1
    if "drop_bit" in c:
        bits = np.concatenate([bits[:c["drop_bit"]], bits[c["drop_bit"] + 1:], bits[:1]])
    soft = synth.aqua_db_soft(bits, sigma=SIGMA, seed=seed + 1, swap_iq=c.get("swap_iq", False))
    if "drop_symbol" in c:
        soft = np.concatenate([soft[:c["drop_symbol"]], soft[c["drop_symbol"] + 2:]])
    lead, tail = c["lead"], c.get("tail", 0)
    body = np.concatenate([_noise(rng, lead), soft, _noise(rng, tail)])
    return np.concatenate([body, _noise(rng, (-body.size) % READ)]), clear


def read_cuts(n, every=2):
    """Pushes of `every` whole reads"""
    return list(range(every * READ, n, every * READ))


def ragged_cuts(n, lead):
    """Pieces cycling through RAGGED, plus cuts inside a symbol and inside the ASMs of frames 1 and 2"""
    cuts, a, k = {lead + FRAME + 13, lead + 2 * FRAME + 21, lead + 5 * FRAME + 7}, 0, 0
    while True:
        a += RAGGED[k % len(RAGGED)]
        k += 1
        if a >= n:
            return sorted(c for c in cuts if 0 < c < n)
        cuts.add(a)


def large_stream():
    """One push of at least 2^26 soft bytes: LARGE_FRAMES frames (64 distinct ones, repeated) between noise"""
    rng = np.random.default_rng(77)
    bits, clear = synth.aqua_db_frames(64, 77)
    reps = LARGE_FRAMES // 64
    soft = synth.aqua_db_soft(np.tile(bits.reshape(-1), reps), sigma=SIGMA, seed=78)
    body = np.concatenate([_noise(rng, 5000), soft, _noise(rng, 100000)])
    return np.concatenate([body, _noise(rng, (-body.size) % READ)]), clear


# IQ -> psk_demod OQPSK -> aqua_db_decoder: baseband format, log2 of the sample count at 15 MS/s, seed
CHAIN = {"cs16": ("cs16", 21, 41), "cf32": ("cf32", 20, 42)}


def aqua_demod_kwargs(fmt):
    """psk_demod's parameters of EOS.json "aqua_db" / "aura_db" (costas_max_offset 1 MHz at the 15 MS/s working rate)"""
    return dict(samplerate=15e6, symbolrate=7.5e6, constellation="oqpsk", rrc_alpha=0.5, pll_bw=0.006, fmt=fmt, clock_gain_omega=0.8,
                clock_mu=0.9, clock_gain_mu=0.037, clock_omega_limit=1e-4, costas_max_offset=float(2 * np.pi * 1e6 / 15e6))


def chain_signal(name):
    """(SignalCfg, raw IQ numpy in its format, the sent CADUs)"""
    import dataclasses
    fmt, log2n, seed = CHAIN[name]
    cfg = dataclasses.replace(synth.CONFIGS["aqua_db"], fmt=fmt)
    raw, clear = synth.make_signal(cfg, 1 << log2n, seed=seed, device="cpu")
    raw = raw.numpy()
    if fmt == "cf32":
        raw = raw.view(np.float32).reshape(-1)
    return cfg, raw, clear


def chain_reference(name):
    """The reference chain's CADUs: its psk_demod's soft symbols (tests.common.oracle()) into its Aqua DB module loop"""
    from oracle import eos as O
    from tests.common import oracle
    cfg, raw, clear = chain_signal(name)
    Od = oracle()
    soft = Od.Demod(Od.demod_cfg(**aqua_demod_kwargs(cfg.fmt))).run(raw, stages=False)["soft"]
    return O.Aqua().run(soft[:soft.size // READ * READ])["cadu"], clear


# a CADU's data: its first 896 bytes
after_lock = functools.partial(_after_lock, prefix=896)


def stats_rows(stats):
    return [[s["frames"], s["state"], s["corrected"], s["failed"]] for s in stats]


# ---- Terra DB: IQ -> terra_db_demod -> ccsds_conv_concat_decoder (EOS.json "terra_db") ------------------------------------------------
TERRA_RATE = (45e6, 13125000)   # samplerate, symbolrate
TERRA_LOG2N = 21
TERRA_SEED = 51
TERRA_FEC = dict(rs_i=4, nrzm=True, derand_after_rs=True, derand_start=10)  # with "bpsk_90", cadu_size 8192, BER 0.3, outsync 20


def terra_signal():
    """(raw cs16 IQ numpy, the CADUs the decoder writes for the sent frames)"""
    raw, clear = synth.make_signal(synth.CONFIGS["terra_db"], 1 << TERRA_LOG2N, seed=TERRA_SEED, device="cpu")
    return raw.numpy(), clear


def terra_demod_kwargs():
    from satdump_b200 import capi
    return capi.terra_db_demod_kwargs(*TERRA_RATE, fmt="cs16")


def terra_reference(stages=True):
    """The reference's terra_db_demod chain (tests.common.oracle()) on terra_signal(): its demodulator outputs"""
    from tests.common import oracle
    O = oracle()
    raw, _ = terra_signal()
    return O, O.demod_cfg(**terra_demod_kwargs()), O.Demod(O.demod_cfg(**terra_demod_kwargs())).run(raw, stages=stages)


def terra_chain_reference():
    """The reference chain's CADUs for terra_signal(): demodulator soft bytes into ccsds_conv_concat_decoder"""
    O, _, o = terra_reference(stages=False)
    soft = o["soft"][:o["soft"].size // 8192 * 8192]
    return O.Fec(O.ccsds_cfg("bpsk_90", 8192, 0.3, 20, **TERRA_FEC)).run(soft)["cadu"].reshape(-1, 1024)


def terra_floor():
    """tests/floors.py's M&M floor for the Terra configuration: the worst deviation of the reference's M&M output and soft bytes from
    themselves when its input is perturbed (8 seeds at 1e-6, 16 more at 1e-5 for the extremes), with the CRC of the signal it belongs to.
    The pinned value is used when the signal here is the one it was measured on, else it is measured again."""
    import zlib
    from tests import floors as F
    raw, _ = terra_signal()
    crc = zlib.crc32(np.ascontiguousarray(raw).view(np.uint8))
    pin = pins().get("terra_floor", {}) if os.path.exists(PINS) else {}
    if pin.get("sig") == crc:
        return pin
    O, oc, o = terra_reference()
    runs = []
    for sd in range(1, 9):
        got = O.run_stage(oc, "mm", F.perturb(o["costas"], 1e-6, sd))
        s = F.diff_stats(got, o["mm"])
        s |= {"soft_" + k: v for k, v in F.soft_stats(F.quantise(got, True), o["soft"]).items()}
        runs.append(s)
    w = F._worst(runs)
    for sd in range(1, 17):
        got = O.run_stage(oc, "mm", F.perturb(o["costas"], 1e-5, sd))
        w["max"] = max(w["max"], F.diff_stats(got, o["mm"])["max"])
        q = F.soft_stats(F.quantise(got, True), o["soft"])
        w["soft_gt1"], w["soft_max"] = max(w["soft_gt1"], q["gt1"]), max(w["soft_max"], q["max"])
    return {"mm_frac": w["frac"], "mm_max": w["max"], "soft_diff": w["soft_diff"], "soft_gt1": w["soft_gt1"], "soft_max": w["soft_max"],
            "sig": crc}
