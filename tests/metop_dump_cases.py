"""Soft streams of the metop_dump_decoder tests, rebuilt from seeds on any machine. tests/golden/make_metop_dump_pins.py runs the reference
on each of them and stores digests of its output in tests/golden/metop_dump_pins.json, which the tests read where the reference is absent."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests.common import after_lock, digest, load_pins  # noqa: F401

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metop_dump_pins.json")
F = 8192
SYNC = 0x1ACFFC1D


def noise(rng, n, sigma=40.0):
    return np.clip(np.round(rng.normal(0, sigma, n)), -127, 127).astype(np.int8)


def syncword(p):
    """Correlator32's QPSK syncword p (correlator32.cpp:54-63) as 32 hard bits"""
    def rot64(w, ph):
        i, q = w & 0xAAAAAAAA, w & 0x55555555
        if ph == 1:
            w = ((i ^ 0xAAAAAAAA) >> 1) | ((q << 1) & 0xFFFFFFFF)
        elif ph == 2:
            w ^= 0xFFFFFFFF
        elif ph == 3:
            w = (i >> 1) | (((q ^ 0x55555555) << 1) & 0xFFFFFFFF)
        return (((w & 0x55555555) << 1) & 0xFFFFFFFF) | ((w & 0xAAAAAAAA) >> 1)
    swapped = ((SYNC & 0xAAAAAAAA) >> 1) | ((SYNC & 0x55555555) << 1)
    w = rot64(SYNC, p) if p < 4 else rot64(swapped ^ 0xFFFFFFFF, p - 4)
    return np.array([(w >> (31 - k)) & 1 for k in range(32)], np.uint8)


def tail_window(rng, lane, p=5):
    """F soft bytes of noise whose last 30 - 2 lane bits are the first ones of syncword p (hard bit 1 = soft >= 0): the window's best
    correlation lies at offset 8162 + 2 lane, where the correlator reads those bits followed by zeros"""
    w = noise(rng, F, 30.0)
    n = 30 - 2 * lane
    w[F - n:] = np.where(syncword(p)[:n] == 1, 50, -50).astype(np.int8)
    return w


def flip_bytes(soft, frame_off, nbytes, seed):
    """Negates one soft byte in each of CADU bytes 4 .. 4 + nbytes of the frame at frame_off (one bit error per byte: nbytes / 4 per RS
    codeword of the I=4 interleave)"""
    rng = np.random.default_rng(seed)
    for j in range(4, 4 + nbytes):
        k = frame_off + 8 * j + int(rng.integers(0, 8))
        soft[k] = -soft[k] if soft[k] != 0 else 60


def stream(case):
    """(soft int8, transmitted CADUs, push cut points) of a case dict: nframes, sigma, seed, and optionally phase / swap (synth.dump_soft),
    lead (soft bytes of noise in front), edit, cuts (push boundaries)."""
    seed = case["seed"]
    rng = np.random.default_rng(seed + 1000)
    tx, cadu = synth.dump_frames(case["nframes"], seed)
    soft = synth.dump_soft(tx, case.get("phase", 0), case.get("swap", False), sigma=case["sigma"], seed=seed + 1)
    edit = case.get("edit")
    if edit == "shift_small":  # 314 bytes inserted, then 1000 deleted: shifts below F / 2
        a, b = F + 100, 3 * F + 50
        soft = np.concatenate([soft[:a], noise(rng, 314), soft[a:b], soft[b + 1000:]])
    elif edit == "shift_large":  # 6000 bytes inserted: a shift above F / 2
        a = 2 * F + 1234
        soft = np.concatenate([soft[:a], noise(rng, 6000), soft[a:]])
    elif edit == "odd_slip":  # one byte inserted: the QPSK pairs slip and the even positions never find the ASM again
        a = 2 * F + 77
        soft = np.concatenate([soft[:a], noise(rng, 1), soft[a:]])
    elif edit == "nsn":  # noise -> signal -> noise -> signal -> noise
        soft = np.concatenate([soft[:2 * F], noise(rng, F + F // 2 + 1234), soft[2 * F:], noise(rng, F + 78)])
    elif edit == "tail":  # a window whose winner lies in the window tail, in front of the signal
        soft = np.concatenate([tail_window(rng, case["lane"]), soft])
    elif edit == "rs":  # frame 1: 10 byte errors per codeword (corrected); frame 3: 20 per codeword (not decodable, still written)
        soft = soft.copy()
        flip_bytes(soft, F, 40, seed + 2)
        flip_bytes(soft, 3 * F, 80, seed + 3)
    elif edit == "noise":
        soft = noise(rng, soft.size)
    soft = np.concatenate([noise(rng, case.get("lead", 0)), soft, noise(rng, 7)])
    cuts = [c if c >= 0 else soft.size + c for c in case.get("cuts", [])]
    return soft, cadu, cuts


def piece_cuts(n, sizes=(1, 3, 777, 8191, 8193, 20001, 5, 2 * F + 3)):
    """Push boundaries of pieces cycling through odd sizes from 1 byte to more than two frames"""
    cuts, a, k = [], 0, 0
    while True:
        a += sizes[k % len(sizes)]
        k += 1
        if a >= n:
            return cuts
        cuts.append(a)


CASES = {}
for _p in range(4):
    for _s in (0, 1):
        CASES[f"phase{_p}_swap{_s}"] = dict(nframes=4, sigma=14.0, seed=100 + 2 * _p + _s, lead=36 + 2 * _p, phase=_p, swap=bool(_s))
CASES.update({
    "noise_signal_noise": dict(nframes=6, sigma=14.0, seed=11, lead=3000, edit="nsn"),
    "shift_small": dict(nframes=6, sigma=14.0, seed=12, phase=1, edit="shift_small"),
    "shift_large": dict(nframes=6, sigma=14.0, seed=13, phase=3, swap=True, edit="shift_large"),
    "odd_slip": dict(nframes=5, sigma=14.0, seed=14, edit="odd_slip"),
    "tail_8162": dict(nframes=4, sigma=14.0, seed=15, edit="tail", lane=0),
    "tail_8164": dict(nframes=4, sigma=14.0, seed=16, phase=2, edit="tail", lane=1),
    "rs_errors": dict(nframes=6, sigma=0.0, seed=17, phase=1, swap=True, edit="rs"),
    "noise": dict(nframes=6, sigma=14.0, seed=18, edit="noise"),
    "long": dict(nframes=40, sigma=18.0, seed=19, lead=1234, phase=2),
})
PIECES = ("noise_signal_noise", "shift_small", "shift_large", "tail_8162", "rs_errors", "long")

# IQ -> psk_demod -> metop_dump_decoder: satdump_b200.synth configuration, baseband format, log2 of the sample count, seed
CHAIN = {"metop_dump_cs16": ("metop_dump", "cs16", 20, 5), "metop_dump_cs8": ("metop_dump", "cs8", 20, 6)}


pins = functools.partial(load_pins, PINS)


def chain_signal(name):
    """(SignalCfg, raw IQ, transmitted CADUs) of a CHAIN entry"""
    import dataclasses
    cfg_name, fmt, log2n, seed = CHAIN[name]
    cfg = dataclasses.replace(synth.CONFIGS[cfg_name], fmt=fmt)
    raw, clear = synth.make_signal(cfg, 1 << log2n, seed=seed, device="cpu")
    return cfg, raw.numpy(), clear


def chain_reference(name):
    """The reference's CADUs for a CHAIN signal: its demodulator's soft symbols (tests.common.oracle()) into its dump decoder"""
    from oracle import dump as O
    from tests.common import demod_kwargs, oracle
    cfg, raw, clear = chain_signal(name)
    Od = oracle()
    soft = Od.Demod(Od.demod_cfg(**demod_kwargs(cfg))).run(raw, stages=False)["soft"]
    return O.Dump().run(soft)["cadu"], clear
