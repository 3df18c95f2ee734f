"""The fengyun_ahrpt_decoder case streams (soft bytes, a multiple of the module's 16384-byte reads) shared by the oracle and GPU tests,
and the reference's result for each: oracle/_ref when built, else tests/golden/fengyun_pins.json."""
import functools
import hashlib
import os

import numpy as np

from satdump_b200 import synth
from tests import common

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fengyun_pins.json")
READ = 16384
OUTSYNC, BER = 20, 0.26  # the shipped FengYun-3 pipelines' viterbi_outsync_after and viterbi_ber_thresold


def _noise(n, rng):
    return rng.integers(-127, 128, size=n).astype(np.int8)


def _pad(soft, rng):
    return np.concatenate([soft, _noise((-soft.size) % READ, rng)])


def _signal(name, rng, nframes, inv, errors=(), swap=False, sigma=14.0):
    i_bits, q_bits, clear = synth.fengyun_frames(nframes, int(rng.integers(1 << 30)), errors)
    return synth.fengyun_soft(i_bits, q_bits, sigma=sigma, seed=int(rng.integers(1 << 30)), invert_second=inv, swap_branches=swap), clear


def invert_second(name):
    return name.endswith("_inv2")


def _build(name):
    rng = np.random.default_rng(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    inv = invert_second(name)
    base = name[:-5] if inv else name
    if base == "clean":
        s, _ = _signal(name, rng, 60, inv)
        return _pad(np.concatenate([_noise(3 * READ, rng), s]), rng)
    if base == "swapped":  # the branches exchanged on air: invert_branches flips after ten deframer NOSYNC reads
        s, _ = _signal(name, rng, 80, inv, swap=True)
        return _pad(np.concatenate([_noise(2 * READ, rng), s]), rng)
    if base == "slip":  # one symbol off the read grid: shift toggles once viterbiNoSyncRun reaches 10, then stays 1 for many reads
        s, _ = _signal(name, rng, 120, inv)
        return _pad(np.concatenate([_noise(3 * READ + 2, rng), s]), rng)
    if base == "slips":  # symbols lost mid-stream, twice: the second time viterbiNoSyncRun is already past 10, so every NOSYNC read toggles
        s, _ = _signal(name, rng, 200, inv)
        a, b = s.size // 3 & ~1, 2 * s.size // 3 & ~1
        s = np.concatenate([s[:a], s[a + 2:b], s[b + 6:]])
        return _pad(np.concatenate([_noise(READ, rng), s]), rng)
    if base == "noise_signal_noise":
        s1, _ = _signal(name, rng, 50, inv)
        s2, _ = _signal(name, rng, 50, inv)
        return _pad(np.concatenate([_noise(5 * READ + 1000, rng), s1, _noise(30 * READ, rng), s2, _noise(4 * READ, rng)]), rng)
    if base == "rs_errors":  # up to t = 16 byte errors per codeword corrected, t + 1 and more not (the frames are written anyway)
        s, _ = _signal(name, rng, 40, inv, errors=[(3, 0, 5), (5, 1, 16), (7, 2, 17), (9, 3, 25), (12, 0, 16), (12, 1, 17)], sigma=8.0)
        return _pad(np.concatenate([_noise(2 * READ, rng), s]), rng)
    if base == "v1_ne_v2":  # the Q branch buried in noise for 30 reads: viterbi2 loses the lock and finds it again, viterbi1 keeps it
        s, _ = _signal(name, rng, 150, inv)
        a = 20 * READ
        s[a:a + 30 * READ:2] = _noise(15 * READ, rng)
        return _pad(np.concatenate([_noise(READ, rng), s]), rng)
    if base == "noise":
        return _noise(40 * READ, rng)
    if base == "large":  # 2^26 bytes: the clean stream over and over
        return np.resize(stream("clean"), 1 << 26)
    raise KeyError(name)


BASES = ["clean", "swapped", "slip", "slips", "noise_signal_noise", "rs_errors", "v1_ne_v2", "noise"]
CASES = BASES + [b + "_inv2" for b in BASES]
LARGE = ["large"]
_cache = {}


def stream(name):
    if name not in _cache:
        _cache[name] = _build(name)
    return _cache[name]


digest = functools.partial(common.digest, dtype=np.uint8)


def reference(name):
    from oracle import fengyun
    r = fengyun.Ref(OUTSYNC, BER, invert_second(name)).run(stream(name))
    return dict(frames=int(r["out"].shape[0]), out=digest(r["out"]), recs=recs_digest(r["recs"]), reads=int(r["recs"].shape[0]),
                rs_avg=r["rs_avg"], deframer_lock=r["deframer_lock"])


def recs_digest(recs):
    """the per-read records (float64 [reads, 9], float32 values) as one digest"""
    return common.digest(np.asarray(recs, np.float32))


def ref_result(name):
    from oracle import fengyun
    if fengyun.available():
        return reference(name)
    return common.load_pins(PINS)[name]
