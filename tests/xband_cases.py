"""The meteor_xband_decoder case streams (soft bytes, a multiple of the module's 8192-byte reads) shared by the oracle, model and GPU
tests, and the reference's result for each: oracle/_ref when built, else tests/golden/meteor_xband_pins.json."""
import hashlib
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests import common

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "meteor_xband_pins.json")
READ = 8192
AMP = 60


def _soft(bits, rng, sigma=20.0):
    s = (bits.astype(np.float32) * 2 - 1) * AMP + rng.normal(0, sigma, bits.size).astype(np.float32)
    return np.clip(np.round(s), -127, 127).astype(np.int8)


def _noise(n, rng):
    return rng.integers(-127, 128, size=n).astype(np.int8)


def _slip(bits, at, insert):
    return np.concatenate([bits[:at], [1 - bits[at]], bits[at:]]) if insert else np.delete(bits, at)


def _pad(soft, rng):
    return np.concatenate([soft, _noise((-soft.size) % READ, rng)])


def _build(name):
    kmss = name.startswith("kmss")
    rng = np.random.default_rng(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    n = 5 if kmss else 60
    seed = int(rng.integers(1 << 30))
    if name.endswith("_clean"):
        bits, _ = synth.meteor_xband_frames(kmss, n, seed)
        return _pad(np.concatenate([_noise(3001, rng), _soft(bits, rng)]), rng)
    if name.endswith("_slips"):
        bits, _ = synth.meteor_xband_frames(kmss, n, seed)
        for at, ins in [(bits.size // 5, True), (bits.size // 2, False), (bits.size * 3 // 4 + 17, True)]:
            bits = _slip(bits, at, ins)
        return _pad(np.concatenate([_noise(777, rng), _soft(bits, rng)]), rng)
    if name.endswith("_noise_signal_noise"):
        bits, _ = synth.meteor_xband_frames(kmss, n, seed)
        soft = _soft(bits, rng)
        soft[soft.size // 3:soft.size // 3 + 20000] = _noise(20000, rng)
        return _pad(np.concatenate([_noise(50000, rng), soft, _noise(40000, rng)]), rng)
    if name.endswith("_resync"):
        bits, _ = synth.meteor_xband_frames(kmss, n, seed, cut=(2, 200 if not kmss else 30000))
        return _pad(np.concatenate([_noise(123, rng), _soft(bits, rng)]), rng)
    if name == "mtvza_three_patterns":  # records whose fourth pattern is broken: accepted only while not synced
        bits, _ = synth.meteor_xband_frames(False, n, seed)
        rec_bits = 3072
        for k in range(1, bits.size // rec_bits, 3):  # NRZ-M: flipping one line bit flips two decoded bits (1925, 1926)
            bits[k * rec_bits + 1925] ^= 1
        return _pad(np.concatenate([_noise(4096, rng), _soft(bits, rng)]), rng)
    if name == "kmss_all_deframers_one_read":  # short frames of deframers 2, 1, 2, 1, 3, 3: several deframers complete frames within
        # one read, deframer 2 before deframer 1 in the stream (the module writes deframer 1's first), then whole frames of all three
        parts = []
        for d, nb in [(1, 100), (0, 100), (1, 100), (0, 100), (2, 150), (2, 300), (1, None), (0, None), (2, None), (1, None)]:
            f = rng.integers(0, 256, size=synth.KMSS_FRM if nb is None else nb, dtype=np.uint8)
            f[:7] = np.frombuffer(synth.KMSS_SYNCS[d], np.uint8)
            parts.append(f)
        pk = np.concatenate([rng.integers(0, 256, size=3000, dtype=np.uint8)] + parts)
        pk = np.concatenate([pk, rng.integers(0, 256, size=(-pk.size) % 1504 + 1504, dtype=np.uint8)])
        bits = synth.nrzm_encode(np.unpackbits(synth.meteor_xband_records(True, pk, rng).reshape(-1)))
        return _pad(np.concatenate([_noise(9000, rng), _soft(bits, rng, 0.0)]), rng)
    if name.endswith("_large"):  # 2^26 bytes: the clean stream over and over
        return np.resize(stream(name[:-6] + "_clean"), 1 << 26)
    if name.endswith("_noise"):
        return _noise(48 * READ, rng)
    raise KeyError(name)


CASES = ["mtvza_clean", "mtvza_slips", "mtvza_noise_signal_noise", "mtvza_resync", "mtvza_three_patterns", "mtvza_noise",
         "kmss_clean", "kmss_slips", "kmss_noise_signal_noise", "kmss_resync", "kmss_all_deframers_one_read", "kmss_noise"]
LARGE = ["mtvza_large", "kmss_large"]
_cache = {}


def stream(name):
    if name not in _cache:
        _cache[name] = _build(name)
    return _cache[name]


def kind(name):
    return 1 if name.startswith("kmss") else 0


digest = functools.partial(common.digest, dtype=np.uint8)


def reference(name):
    from oracle import xband
    r = xband.Ref(kind(name)).run(stream(name))
    return dict(frames=int(r["out"].shape[0]), out=digest(r["out"]), frame_count=r["frame_count"])


def ref_result(name):
    from oracle import xband
    if xband.available():
        return reference(name)
    return common.load_pins(PINS)[name]
