"""The fengyun_mpt_decoder case streams (soft bytes, a multiple of the module's 16384-byte reads) shared by the oracle and GPU tests, and
the reference's result for each: oracle/_ref when built, else tests/golden/fengyun_mpt_pins.json."""
import functools
import hashlib
import os

import numpy as np

from satdump_b200 import synth
from tests import common

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fengyun_mpt_pins.json")
READ = 16384
OUTSYNC, BER = 20, 0.3  # FengYun-3.json "fengyun3_abc_mpt": viterbi_outsync_after, viterbi_ber_thresold


def _noise(n, rng):
    return rng.integers(-127, 128, size=n).astype(np.int8)


def _pad(soft, rng):
    return np.concatenate([soft, _noise((-soft.size) % READ, rng)])


def _signal(rng, nframes, errors=(), swap=False, phase90=False, sigma=14.0):
    i_bits, q_bits, clear = synth.fengyun_mpt_frames(nframes, int(rng.integers(1 << 30)), errors)
    return synth.fengyun_mpt_soft(i_bits, q_bits, sigma=sigma, seed=int(rng.integers(1 << 30)), swap_branches=swap, phase90=phase90)


def _build(name):
    rng = np.random.default_rng(int(hashlib.sha256(("mpt_" + name).encode()).hexdigest()[:8], 16))
    if name == "clean":
        return _pad(np.concatenate([_noise(3 * READ, rng), _signal(rng, 40)]), rng)
    if name == "swapped":  # the branches exchanged on air: invert_branches flips after ten deframer NOSYNC reads
        return _pad(np.concatenate([_noise(2 * READ, rng), _signal(rng, 60, swap=True)]), rng)
    if name == "slip":  # one symbol off the read grid: shift toggles once viterbiNoSyncRun reaches 10
        return _pad(np.concatenate([_noise(3 * READ + 2, rng), _signal(rng, 80)]), rng)
    if name == "slips":  # symbols lost mid-stream, twice: the second time viterbiNoSyncRun is past 10, so every NOSYNC read toggles
        s = _signal(rng, 140)
        a, b = s.size // 3 & ~1, 2 * s.size // 3 & ~1
        s = np.concatenate([s[:a], s[a + 2:b], s[b + 6:]])
        return _pad(np.concatenate([_noise(READ, rng), s]), rng)
    if name == "noise_signal_noise":
        s1, s2 = _signal(rng, 35), _signal(rng, 35)
        return _pad(np.concatenate([_noise(5 * READ + 1000, rng), s1, _noise(30 * READ, rng), s2, _noise(4 * READ, rng)]), rng)
    if name == "rs_errors":  # up to t = 16 byte errors per codeword corrected, t + 1 and more not (the frames are written anyway)
        s = _signal(rng, 30, errors=[(3, 0, 5), (5, 1, 16), (7, 2, 17), (9, 3, 25), (12, 0, 16), (12, 1, 17)], sigma=8.0)
        return _pad(np.concatenate([_noise(2 * READ, rng), s]), rng)
    if name in ("q_buried", "i_buried"):  # one branch buried in noise for 30 reads. The module's shift test reads viterbi1's state twice:
        # viterbi2 losing its lock (Q buried) never toggles shift, viterbi1 losing it (I buried) does
        s = _signal(rng, 110)
        a = 20 * READ + (0 if name == "q_buried" else 1)  # the Q branch rides on byte 0 of each pair, the I branch on byte 1
        s[a:a + 30 * READ:2] = _noise(15 * READ, rng)
        return _pad(np.concatenate([_noise(READ, rng), s]), rng)
    if name == "phase90":  # every branch pair rotated: both Viterbis lock on PHASE_90
        return _pad(np.concatenate([_noise(2 * READ, rng), _signal(rng, 40, phase90=True)]), rng)
    if name == "noise":
        return _noise(40 * READ, rng)
    if name == "large":  # 2^26 bytes: the clean stream over and over
        return np.resize(stream("clean"), 1 << 26)
    raise KeyError(name)


CASES = ["clean", "swapped", "slip", "slips", "noise_signal_noise", "rs_errors", "q_buried", "i_buried", "phase90", "noise"]
LARGE = ["large"]
_cache = {}


def stream(name):
    if name not in _cache:
        _cache[name] = _build(name)
    return _cache[name]


digest = functools.partial(common.digest, dtype=np.uint8)


def recs_digest(recs):
    """the per-read records (float64 [reads, 9], float32 values) as one digest"""
    return common.digest(np.asarray(recs, np.float32))


def reference(name):
    from oracle import fengyun_mpt
    r = fengyun_mpt.RefMpt(OUTSYNC, BER).run(stream(name))
    return dict(frames=int(r["out"].shape[0]), out=digest(r["out"]), recs=recs_digest(r["recs"]), reads=int(r["recs"].shape[0]),
                rs_avg=r["rs_avg"], deframer_lock=r["deframer_lock"])


def ref_result(name):
    from oracle import fengyun_mpt
    if fengyun_mpt.available():
        return reference(name)
    return common.load_pins(PINS)[name]
