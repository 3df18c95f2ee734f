"""Soft and IQ streams of the meteor_lrpt_decoder tests, rebuilt from seeds on any machine. tests/golden/make_meteor_lrpt_pins.py runs the
reference on each of them and stores its records, stats and digests of its output in tests/golden/meteor_lrpt_pins.json, which the tests
read where the reference is absent."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests.common import after_lock, digest, load_pins  # noqa: F401

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "meteor_lrpt_pins.json")
F = 16384
MSG = 4 + 4 * 223


def noise(rng, n, sigma=40.0):
    return np.clip(np.round(rng.normal(0, sigma, n)), -127, 127).astype(np.int8)


def stream(case):
    """(soft int8, the CADUs the decoder writes for the transmitted frames, push cut points) of a case dict: nframes, sigma, seed, and
    optionally diff (NRZ-M), phase / swap (synth.lrpt_soft), inverted (frame indices), lead (noise bytes in front), edit, cuts."""
    seed = case["seed"]
    rng = np.random.default_rng(seed + 1000)
    coded, cadu = synth.lrpt_frames(case["nframes"], seed, nrzm=case.get("diff", False), inverted=case.get("inverted", ()))
    soft = synth.lrpt_soft(coded, case.get("phase", 0), case.get("swap", False), sigma=case["sigma"], seed=seed + 1)
    edit = case.get("edit")
    if edit == "shifts":  # 314 bytes inserted, 1000 deleted (shifts below F / 2), then 11000 inserted (a shift above F / 2)
        a, b, c = F + 100, 3 * F + 50, 5 * F + 4321
        soft = np.concatenate([soft[:a], noise(rng, 314), soft[a:b], soft[b + 1000:c], noise(rng, 11000), soft[c:]])
    elif edit == "nsn":  # noise -> signal -> noise -> signal -> noise
        soft = np.concatenate([noise(rng, 3 * F + 1234), soft[:4 * F], noise(rng, F + F // 2 + 78), soft[4 * F:], noise(rng, 2 * F + 10)])
    elif edit == "noise":
        soft = noise(rng, soft.size)
    soft = np.concatenate([noise(rng, case.get("lead", 0)), soft, noise(rng, 7)])
    cuts = [c if c >= 0 else soft.size + c for c in case.get("cuts", [])]
    return soft, cadu, cuts


def piece_cuts(n, sizes=(1, 3, 777, 16383, 16385, 40001, 5, 2 * F + 3, 9000)):
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
        CASES[f"phase{_p}_swap{_s}"] = dict(nframes=5, sigma=30.0, seed=200 + 2 * _p + _s, lead=36 + 2 * _p, phase=_p, swap=bool(_s))
CASES.update({
    "plain": dict(nframes=24, sigma=35.0, seed=21, lead=1000, inverted=(3, 17)),
    "diff": dict(nframes=24, sigma=35.0, seed=22, lead=2000, diff=True, inverted=(5,)),
    "diff_phase3": dict(nframes=10, sigma=35.0, seed=23, diff=True, phase=3, swap=True),
    "shifts": dict(nframes=10, sigma=30.0, seed=24, phase=1, edit="shifts"),
    "noise_signal_noise": dict(nframes=8, sigma=30.0, seed=25, edit="nsn"),
    "rs_corrected": dict(nframes=12, sigma=46.0, seed=28, lead=300),
    "low_esn0": dict(nframes=24, sigma=50.0, seed=26, lead=500),
    "noise": dict(nframes=6, sigma=30.0, seed=27, edit="noise"),
})
PIECES = ("plain", "diff", "shifts", "noise_signal_noise", "low_esn0")

# m2x_mode (Viterbi1_2 -> NRZ-M bits -> deframer -> RS): diff_decode, ber_thresold, outsync_after of the 80k pipeline; streams of 8192-bit
# CADUs behind the r=1/2 code, with noise stretches for unlock and relock
M2X = {
    "m2x_diff": dict(nframes=16, sigma=30.0, seed=31, diff=True, lead=5000, edit="nsn"),
    "m2x_plain_phase1": dict(nframes=12, sigma=30.0, seed=32, phase=1, swap=True),
}
M2X_PARAMS = dict(viterbi_ber_thresold=0.3, viterbi_outsync_after=20)

# IQ -> psk_demod -> meteor_lrpt_decoder: satdump_b200.synth configuration, baseband format, log2 of the sample count, seed
CHAIN = {"meteor_lrpt_cs16": ("meteor_lrpt", "cs16", 20, 5), "meteor_lrpt_1m_cs16": ("meteor_lrpt_1m", "cs16", 21, 6)}


pins = functools.partial(load_pins, PINS)


def chain_signal(name):
    """(SignalCfg, raw IQ, transmitted CADUs as the decoder writes them) of a CHAIN entry"""
    import dataclasses
    cfg_name, fmt, log2n, seed = CHAIN[name]
    cfg = dataclasses.replace(synth.CONFIGS[cfg_name], fmt=fmt)
    raw, clear = synth.make_signal(cfg, 1 << log2n, seed=seed, device="cpu")
    return cfg, raw.numpy(), clear


def chain_reference(name):
    """The reference's CADUs for a CHAIN signal: its demodulator's soft symbols (tests.common.oracle()) into its METEOR decoder"""
    from oracle import meteor as O
    from tests.common import demod_kwargs, oracle
    cfg, raw, clear = chain_signal(name)
    Od = oracle()
    soft = Od.Demod(Od.demod_cfg(**demod_kwargs(cfg))).run(raw, stages=False)["soft"]
    return O.Meteor(cfg.nrzm).run(soft)["cadu"], clear
