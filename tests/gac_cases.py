"""Soft streams of the noaa_gac_decoder and dmsp_rtd_decoder tests, rebuilt from seeds on any machine. tests/golden/make_gac_pins.py runs
the reference on each stream and stores a digest of its frames and timestamps, its frame count and final state in
tests/golden/gac_pins.json, which the tests read where the reference is absent. Every stream is a whole number of the modules' 8192-byte
reads, so the reference decodes all of it."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests import common

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gac_pins.json")
START_TS = 1700000000.25  # dmsp_rtd_decoder's start_timestamp in the DMSP cases

# nframes, seed; sync_errors {frame: bits flipped in its sync}; sigma; lead / tail (noise bits); inverted; slip (bit dropped); gap
# ((bit, noise bits) inserted); flip_at (frame from which the polarity flips); backward (GAC)
GAC = {
    "gac_clean": dict(nframes=14, seed=1, lead=3000, tail_reads=0),
    "gac_noisy_inverted": dict(nframes=15, seed=2, lead=777, sigma=22.0, inverted=True, sync_errors={4: 5, 12: 11, 13: 12}),
    "gac_syncing_fail": dict(nframes=14, seed=3, lead=100, sync_errors={3: 6}),
    "gac_slip_gap": dict(nframes=16, seed=4, lead=50, slip=13 * 33270 + 900, gap=(6 * 33270 + 5, 4321)),
    "gac_flip": dict(nframes=15, seed=5, lead=20000, flip_at=12),
    "gac_backward": dict(nframes=14, seed=6, lead=2000, backward=True, sigma=30.0),
    "gac_backward_inverted": dict(nframes=5, seed=7, lead=64, backward=True, inverted=True),
}
DMSP = {
    "dmsp_clean": dict(nframes=400, seed=11, lead=5000),
    "dmsp_noisy_inverted": dict(nframes=500, seed=12, lead=3000, sigma=45.0, inverted=True, sync_errors={20: 4, 21: 5, 22: 6}),
    "dmsp_syncing_fail": dict(nframes=300, seed=13, lead=100, sync_errors={2: 2, 5: 1, 40: 3}),
    "dmsp_synced_drop": dict(nframes=600, seed=14, lead=20, sync_errors={100: 6, 300: 13}),
    "dmsp_slip_gap_flip": dict(nframes=900, seed=15, lead=1, slip=200 * 150 + 77, gap=(500 * 150 + 3, 7001), flip_at=700),
    "dmsp_noise": dict(nframes=0, seed=16, lead=60000),
}
CASES = [*GAC, *DMSP]


def is_dmsp(name):
    return name in DMSP


def params(name):
    """(dmsp, backward) of a case"""
    c = GAC.get(name) or DMSP[name]
    return is_dmsp(name), bool(c.get("backward", False))


def stream(name):
    """soft int8 of a case, a whole number of 8192-byte reads"""
    dmsp = is_dmsp(name)
    c = DMSP[name] if dmsp else GAC[name]
    rng = np.random.default_rng(c["seed"] + 500)
    bits, _ = (synth.dmsp_frames(c["nframes"], c["seed"]) if dmsp else synth.gac_frames(c["nframes"], c["seed"], c.get("backward", False)))
    width = 13 if dmsp else 32
    for k, n in c.get("sync_errors", {}).items():
        bits[int(k), rng.choice(width, size=n, replace=False)] ^= 1
    flip = c.get("flip_at", c["nframes"])
    inv = c.get("inverted", False)
    parts = [(bits[:flip].reshape(-1), inv), (bits[flip:].reshape(-1), not inv)]
    soft = [rng.normal(0, 90, c.get("lead", 0))]
    for i, (b, pol) in enumerate(parts):
        slips = [c["slip"]] if "slip" in c and i == 0 else []
        gaps = [tuple(c["gap"])] if "gap" in c and i == 0 else []
        soft.append(synth.hrpt_soft(b, pol, sigma=c.get("sigma", 0.0), seed=c["seed"] + i, slips=slips, gaps=gaps))
    n = sum(s.size for s in soft)
    soft.append(rng.normal(0, 90, (-n) % 8192 + 8192 * c.get("tail_reads", 1)))
    return np.clip(np.round(np.concatenate(soft)), -127, 127).astype(np.int8)


def cuts_for(name, n, sizes):
    """push cut points: pieces of the given sizes in turn, plus cuts inside the first syncs and frames (a sync split, a frame split)"""
    dmsp = is_dmsp(name)
    lead = (DMSP if dmsp else GAC)[name].get("lead", 0)
    period = 150 if dmsp else 33270
    extra = {lead + 5, lead + 20, lead + period + 7, lead + 2 * period + period // 2}
    cuts, at, k = set(), 0, 0
    while True:
        at += sizes[k % len(sizes)]
        k += 1
        if at >= n:
            break
        cuts.add(at)
    return sorted(c for c in cuts | extra if 0 < c < n)


digest = functools.partial(common.digest, hexlen=24)


def ts_digest(ts):
    """the timestamps as the module writes them (std::to_string: %f)"""
    return digest(np.frombuffer("".join("%f\n" % t for t in ts).encode(), np.uint8))


pins = functools.partial(common.load_pins, PINS)


def ref_result(name):
    """the reference's frames digest, frame count, final state and timestamps digest of a case: from oracle/_ref, else the pins"""
    from oracle import gac as O
    if O.available():
        dmsp, backward = params(name)
        r = O.Ref(dmsp, backward, START_TS if dmsp else -1.0).run(stream(name))
        return dict(out=digest(r["out"]), frames=int(r["out"].shape[0]), state=r["stats"]["state"], ts=ts_digest(r["ts"]))
    return pins()["cases"][name]
