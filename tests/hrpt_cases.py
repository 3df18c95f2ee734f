"""Soft streams of the noaa_hrpt_decoder and meteor_hrpt_decoder tests, rebuilt from seeds on any machine. tests/golden/make_hrpt_pins.py
runs the reference on each stream and stores its records, per-push stats and a digest of its output in tests/golden/hrpt_pins.json, which
the tests read where the reference is absent."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests.common import after_lock, digest, load_pins  # noqa: F401

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hrpt_pins.json")
NOAA_BITS = synth.NOAA_WORDS * 10
MH_BITS = 8192
# where the mixed-window case's crafted ASM is matched, relative to the start of its noise (see meteor_stream)
MIX_AT = 40993 + 16


def _flip(bits, n, width, rng):
    bits[rng.choice(width, size=n, replace=False)] ^= 1


def noaa_stream(case):
    """(soft int8, push cut points) of a NOAA case: nframes, seed, thr, and optionally sync_errors {frame: n}, sigma, lead (noise bits in
    front), tail, inverted, flip_at (frame from which the polarity flips), slip (bit index dropped inside the frames), gap ((bit index,
    noise bits) inserted), drop_head (bits of the first sync not sent: the sync completes against the zero shifter), cuts."""
    rng = np.random.default_rng(case["seed"] + 500)
    bits, _ = synth.noaa_hrpt_frames(case["nframes"], case["seed"])
    for k, n in case.get("sync_errors", {}).items():
        _flip(bits[int(k)], n, 60, rng)
    flip = case.get("flip_at", case["nframes"])
    parts = [(bits[:flip].reshape(-1), case.get("inverted", False)), (bits[flip:].reshape(-1), not case.get("inverted", False))]
    soft = []
    for i, (b, inv) in enumerate(parts):
        if i == 0:
            b = b[case.get("drop_head", 0):]
        slips = [case["slip"]] if "slip" in case and i == 0 else []
        gaps = [tuple(case["gap"])] if "gap" in case and i == 0 else []
        soft.append(synth.hrpt_soft(b, inv, sigma=case.get("sigma", 0.0), seed=case["seed"] + i, slips=slips, gaps=gaps))
    soft = np.concatenate([noise(rng, case.get("lead", 0)), *soft, noise(rng, case.get("tail", 0))])
    return soft, [c if c >= 0 else soft.size + c for c in case.get("cuts", [])]


def meteor_stream(case):
    """(soft int8, push cut points) of a METEOR case: a list of items, each ("f", n frames, ASM errors of the first), ("n", noise bits),
    ("x", 1: one extra bit), or ("mix",): 60000 noise bits that time out state 2 (entered from 12 at the first failed test) and hold a
    crafted ASM across the inversion change, matched at noise start + MIX_AT. Case keys: items, seed, and optionally inverted, sigma,
    drop_head (bits of the first ASM not sent), cuts."""
    rng = np.random.default_rng(case["seed"] + 700)
    out, k = [], 0
    for it in case["items"]:
        if it[0] == "f":
            bits, _ = synth.meteor_hrpt_frames(it[1], case["seed"] + k)
            k += 1
            _flip(bits[0], it[2], 32, rng)
            out.append(bits.reshape(-1))
        elif it[0] == "n" or it[0] == "x":
            out.append(rng.integers(0, 2, it[1]).astype(np.uint8))
        else:
            b = rng.integers(0, 2, 60000).astype(np.uint8)
            asm = np.unpackbits(np.frombuffer(synth.METEOR_HRPT_ASM, np.uint8))
            t = MIX_AT - 16  # the timeout test; the stream is inverted, so bits up to t reach the shifter as sent, later ones flipped
            b[t - 15:t + 1] = asm[:16]
            b[t + 1:t + 17] = asm[16:] ^ 1
            out.append(b)
    bits = np.concatenate(out)[case.get("drop_head", 0):]
    soft = synth.hrpt_soft(bits, case.get("inverted", False), sigma=case.get("sigma", 0.0), seed=case["seed"])
    return soft, [c if c >= 0 else soft.size + c for c in case.get("cuts", [])]


def noise(rng, n, sigma=60.0):
    return np.clip(np.round(rng.normal(0, sigma, n)), -127, 127).astype(np.int8)


NOAA = {
    "noaa_plain": dict(nframes=5, seed=1, thr=10, lead=5000, tail=300, sigma=20.0),
    "noaa_inverted": dict(nframes=4, seed=2, thr=10, lead=777, inverted=True, sigma=20.0),
    "noaa_flip": dict(nframes=6, seed=3, thr=10, lead=100, flip_at=3, sigma=15.0),
    "noaa_thr_edges": dict(nframes=5, seed=4, thr=10, lead=50, sync_errors={1: 10, 2: 11, 4: 10}),
    "noaa_thr0": dict(nframes=4, seed=5, thr=0, lead=200, sync_errors={2: 1}),
    "noaa_thr26_splice": dict(nframes=4, seed=6, thr=26, lead=0),
    "noaa_zero_shifter": dict(nframes=3, seed=7, thr=10, drop_head=10),
    "noaa_nsn": dict(nframes=4, seed=8, thr=10, lead=150000, tail=130000, sigma=25.0),
    "noaa_slip": dict(nframes=5, seed=9, thr=10, lead=3000, slip=NOAA_BITS + 50000),
}
METEOR = {
    # 0->6, 6->12, 12 with 12 errors, 12->6 (13 errors), 6->2, 2 rejects 3 errors, 2->6 with 2, 6 takes 6 and rejects 7, then state 2
    # again, 6 good frames to 12
    "meteor_transitions": dict(seed=11, items=[("n", 3000), ("f", 7, 0), ("f", 2, 12), ("f", 1, 13), ("f", 1, 3), ("f", 1, 2),
                                                ("f", 1, 6), ("f", 1, 7), ("f", 1, 2), ("f", 7, 0)]),
    # a one-bit-late frame in state 6 (the test fails, the next bit matches), then lock
    "meteor_late": dict(seed=12, items=[("n", 500), ("f", 2, 0), ("x", 1), ("f", 8, 0)]),
    # lock, then noise: 12 -> 6 -> 2, a state-2 timeout to 0 while inverted, and an ASM matched in a window of mixed inversion
    "meteor_mixed": dict(seed=13, inverted=True, items=[("n", 100), ("f", 7, 0), ("mix",), ("n", 2000), ("f", 4, 0)]),
    "meteor_zero_shifter": dict(seed=14, drop_head=3, items=[("f", 3, 0)]),
    "meteor_nsn": dict(seed=15, sigma=20.0, items=[("n", 70000), ("f", 9, 0), ("n", 90000), ("f", 3, 0), ("n", 5000)]),
    "meteor_inverted": dict(seed=16, inverted=True, sigma=25.0, items=[("n", 1234), ("f", 10, 0)]),
}
PIECE_SIZES = (1, 3, 9, 777, 8191)


def stream(name):
    return noaa_stream(NOAA[name]) if name in NOAA else meteor_stream(METEOR[name])


def params(name):
    """(meteor, thr) of a case"""
    return (False, NOAA[name]["thr"]) if name in NOAA else (True, 0)


def piece_cuts(n, sizes=PIECE_SIZES, extra=()):
    """Push boundaries of pieces cycling through `sizes`, plus the cut points `extra`"""
    cuts, a, k = set(extra), 0, 0
    while True:
        a += sizes[k % len(sizes)]
        k += 1
        if a >= n:
            return sorted(c for c in cuts if 0 < c < n)
        cuts.add(a)


def boundary_cuts(name):
    """Cuts inside a word, inside a frame and inside a sync of the case's first frame"""
    soft, _ = stream(name)
    if name in NOAA:
        s0 = NOAA[name].get("lead", 0) - NOAA[name].get("drop_head", 0)
        return [s0 + 30, s0 + 60 + 10 * 37 + 4, s0 + NOAA_BITS // 2 + 3, s0 + NOAA_BITS + 59 + 7]
    return [600, 3000 + 17, 3000 + 32 + 8 * 400 + 5, 3000 + MH_BITS + 20]


pins = functools.partial(load_pins, PINS)


def stats_rows(stats):
    """[units, state] after every push (units: NOAA words / METEOR frames written so far)"""
    return [[s["units"], s["state"]] for s in stats]


# large pushes: 220 NOAA frames (thr 10) and 2000 METEOR frames, behind noise and followed by noise, in two pushes
LARGE = {"noaa_large": (False, 10, 220), "meteor_large": (True, 0, 2000)}


def large_stream(name):
    """(soft, cuts, meteor, thr) of a LARGE entry"""
    meteor, thr, n = LARGE[name]
    rng = np.random.default_rng(n)
    bits, _ = (synth.meteor_hrpt_frames if meteor else synth.noaa_hrpt_frames)(n, n + 1)
    soft = np.concatenate([noise(rng, 4321), synth.hrpt_soft(bits, sigma=10.0, seed=n + 2), noise(rng, 300000)])
    return soft, [soft.size // 3], meteor, thr


# IQ -> pm_demod -> decoder: satdump_b200.synth configuration, log2 of the sample count (cs16 at 3 MS/s), seed
CHAIN = {"noaa_hrpt": ("noaa_hrpt", 22, 31), "meteor_hrpt": ("meteor_hrpt", 20, 32)}


def demod_kwargs(cfg):
    """pm_demod's parameters of the two pipelines: tests.common.demod_kwargs plus "clock_omega_relative_limit" 0.001 (NOAA.json,
    Meteor-M.json)"""
    from tests.common import demod_kwargs as base
    return dict(base(cfg), clock_omega_limit=0.001)


def chain_signal(name):
    """(SignalCfg, raw cs16 IQ, the transmitted frames: NOAA words [n, 11090] / METEOR CADUs [n, 1024]) of a CHAIN entry"""
    cfg_name, log2n, seed = CHAIN[name]
    cfg = synth.CONFIGS[cfg_name]
    raw, clear = synth.make_signal(cfg, 1 << log2n, seed=seed, device="cpu")
    return cfg, raw.numpy(), clear


def frames_of(out, meteor):
    """The decoder's output as frames: METEOR CADU rows; NOAA the 11090-word runs that start with the six sync words"""
    if meteor:
        return out.reshape(-1, 1024)
    w = np.asarray(out, np.uint16)
    starts, i = [], 0
    while i + synth.NOAA_WORDS <= w.size:
        if tuple(w[i:i + 6]) == synth.NOAA_SYNC_WORDS:
            starts.append(i)
            i += synth.NOAA_WORDS
        else:
            i += 1
    return np.array([w[s:s + synth.NOAA_WORDS] for s in starts], np.uint16).reshape(-1, synth.NOAA_WORDS)


def chain_reference(name):
    """The reference's output for a CHAIN signal: its pm_demod's soft symbols (tests.common.oracle()) into its deframer"""
    from oracle import hrpt as O
    from tests.common import oracle
    cfg, raw, clear = chain_signal(name)
    Od = oracle()
    soft = Od.Demod(Od.demod_cfg(**demod_kwargs(cfg))).run(raw, stages=False)["soft"]
    meteor = cfg.decoder == "meteor_hrpt"
    return O.Hrpt(meteor, cfg.deframer_thresold).run(soft)["out"], clear, meteor
