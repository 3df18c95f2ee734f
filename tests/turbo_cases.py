"""Soft streams of the ccsds_turbo_decoder tests, rebuilt from seeds on any machine. tests/golden/make_turbo_pins.py runs the reference on
each of them and stores digests of its output in tests/golden/turbo_pins.json, which the tests read where the reference is absent."""
import functools
import os

import numpy as np

from satdump_b200 import synth
from tests.common import digest, load_pins  # noqa: F401

PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "turbo_pins.json")
LLR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "turbo_llr.npz")
LLR_CASES = ("llr_2_223", "llr_6_223")
RATE_NAME = {2: "1/2", 3: "1/3", 4: "1/4", 6: "1/6"}


def frame_size(rate, base):
    return synth.turbo_codeword_bits(rate, base) + synth.TURBO_ASM_BITS[rate]


def noise(rng, n, sigma=40.0):
    return np.clip(np.round(rng.normal(0, sigma, n)), -127, 127).astype(np.int8)


def stream(case):
    """(soft int8, transmitted CADUs, push cut points) of a case dict: rate, base, iters, nframes, sigma, seed, and optionally lead (soft
    bytes of noise in front), swap (negated soft bits), edits ("insdel": bytes inserted and deleted mid-stream; "nsn": noise -> signal ->
    noise -> signal, with a shift above F / 2), cuts (push boundaries)."""
    rate, base, seed = case["rate"], case["base"], case["seed"]
    F = frame_size(rate, base)
    rng = np.random.default_rng(seed + 1000)
    tx, cadu = synth.turbo_frames(case["nframes"], rate, base, seed)
    soft = synth.ldpc_soft(tx.reshape(-1), "bpsk", amp=60.0, sigma=case["sigma"], rot=2 if case.get("swap") else 0, seed=seed + 1)
    lead = noise(rng, case.get("lead", 0))
    edit = case.get("edit")
    if edit == "insdel":
        a, b = case.get("lead", 0) + F + 100, 3 * F + 50
        soft = np.concatenate([soft[:a], noise(rng, 314), soft[a:b], soft[b + 1000:]])
    elif edit == "nsn":
        soft = np.concatenate([soft[:2 * F], noise(rng, F + F // 2 + 1234), soft[2 * F:], noise(rng, F + 77)])
    soft = np.concatenate([lead, soft, noise(rng, 7)])
    cuts = [c if c >= 0 else soft.size + c for c in case.get("cuts", [])]
    return soft, cadu, cuts


def _combo(rate, base, iters):
    return dict(rate=rate, base=base, iters=iters, nframes=2, sigma=35.0, seed=rate * 10000 + base, lead=37)


CASES = {}
for _r in (2, 3, 4, 6):
    for _b in synth.TURBO_BASES:
        CASES[f"combo_{_r}_{_b}"] = _combo(_r, _b, 1 if _b > 446 else 2)
CASES.update({
    "r2_1115_it1": dict(rate=2, base=1115, iters=1, nframes=3, sigma=36.0, seed=11, lead=500),
    "r2_1115_it5": dict(rate=2, base=1115, iters=5, nframes=2, sigma=50.0, seed=12, lead=11),
    "r2_1115_it50": dict(rate=2, base=1115, iters=50, nframes=2, sigma=55.0, seed=13, lead=0),
    "r4_1115_it2": dict(rate=4, base=1115, iters=2, nframes=2, sigma=60.0, seed=14, lead=3),
    "r6_1115_it1": dict(rate=6, base=1115, iters=1, nframes=2, sigma=60.0, seed=15, lead=100),
    "r6_1115_it20": dict(rate=6, base=1115, iters=20, nframes=2, sigma=75.0, seed=16, lead=0),
    "r2_223_it10": dict(rate=2, base=223, iters=10, nframes=4, sigma=52.0, seed=17, lead=1),
    "crc_failures": dict(rate=2, base=223, iters=1, nframes=10, sigma=42.0, seed=18, lead=0),
    "swapped": dict(rate=3, base=223, iters=2, nframes=4, sigma=50.0, seed=19, lead=21, swap=True),
    "inserted_deleted": dict(rate=2, base=446, iters=2, nframes=6, sigma=45.0, seed=20, lead=0, edit="insdel"),
    "noise_signal_noise": dict(rate=2, base=223, iters=2, nframes=6, sigma=45.0, seed=21, lead=2000, edit="nsn"),
    "llr_2_223": dict(rate=2, base=223, iters=3, nframes=2, sigma=55.0, seed=31, lead=0),
    "llr_6_223": dict(rate=6, base=223, iters=2, nframes=2, sigma=80.0, seed=32, lead=0),
    "ragged": dict(rate=4, base=223, iters=2, nframes=6, sigma=45.0, seed=22, lead=500,
                   cuts=[1, 500 + 40, 500 + 7212 + 3000, 500 + 7212 + 3001, 500 + 3 * 7212 + 17, -9]),
})


pins = functools.partial(load_pins, PINS)


def encoder_info(rate, base):
    """the information bytes the encoder pins encode"""
    return np.random.default_rng(rate * 7 + base).integers(0, 256, base, dtype=np.uint8)


# IQ -> demodulator -> ccsds_turbo_decoder: satdump_b200.synth configurations, log2 of the sample count, seed
CHAIN = {"turbo_pm": (21, 3), "turbo_bpsk": (21, 3)}


def chain_demod_kwargs(cfg):
    from tests.common import demod_kwargs
    kw = demod_kwargs(cfg)
    if cfg.post_costas_dc:
        kw["post_costas_dc"] = True
    return kw


def chain_reference(name):
    """The reference's CADUs for a CHAIN signal: its demodulator's soft symbols (tests.common.oracle()) into its turbo decoder."""
    from oracle import turbo as O
    from tests.common import oracle, signal
    log2n, seed = CHAIN[name]
    cfg, raw, clear = signal(name, log2n, seed=seed)
    Od = oracle()
    soft = Od.Demod(Od.demod_cfg(**chain_demod_kwargs(cfg))).run(raw, stages=False)["soft"]
    return O.Turbo(RATE_NAME[cfg.turbo_rate], cfg.turbo_base, cfg.turbo_iters).run(soft)["cadu"]


def frame_streams(soft, off, swapped, rate, base):
    """The decoder's input of a frame read at its place (pos 0): derandomised code bytes / 127 in float32, negated when swapped, widened,
    depunctured (rate 1/2: zeros at the punctured places) and split into the upper and lower code streams (float64)."""
    nasm, cw = synth.TURBO_ASM_BITS[rate], synth.turbo_codeword_bits(rate, base)
    b = np.asarray(soft[off + nasm:off + nasm + cw], np.int8)
    b = np.where(synth.ldpc_pn_bits(cw).astype(bool), ~b, b)
    x = b.astype(np.float32) / np.float32(127)
    x = (-x if swapped else x).astype(np.float64)
    n = 8 * base + 4
    cu, cl = len(synth.TURBO_CODES[rate][0]), len(synth.TURBO_CODES[rate][1])
    if rate == 2:
        k = np.arange(3 * n)
        keep = (k % 3 == 0) | np.where((k // 3) % 2 == 1, k % 3 == 2, k % 3 == 1)
        full = np.zeros(3 * n)
        full[keep] = x
        x = full
    blocks = x.reshape(n, cu + cl)
    return blocks[:, :cu].reshape(-1).copy(), blocks[:, cu:].reshape(-1).copy()


def reference_llr(rate, base, iters, up, lo):
    """turbo_decode's loop (libturbocodes.c:160-184) around the reference's own convcode_extrinsic: the a-priori arrays after the last
    iteration"""
    from oracle import turbo as O
    K = 8 * base
    pi = synth.turbo_interleaver(base)
    m0, m1 = np.full(K, np.log(0.5)), np.full(K, np.log(0.5))
    for _ in range(iters):
        m0, m1, _ = O.half(RATE_NAME[rate], base, 0, up, m0, m1)
        i0, i1, _ = O.half(RATE_NAME[rate], base, 1, lo, m0[pi], m1[pi])
        m0, m1 = np.empty(K), np.empty(K)
        m0[pi], m1[pi] = i0, i1
    return m0, m1


def llr_frames(name):
    """(frame index in the case's stream, upper stream, lower stream) of every frame of an LLR case read at its place"""
    case = CASES[name]
    soft, _, _ = stream(case)
    recs = np.array(pins()["cases"][name]["recs"], np.int64).reshape(-1, 6)
    return [(k, *frame_streams(soft, int(r[0]), bool(r[3]), case["rate"], case["base"])) for k, r in enumerate(recs) if r[1] == 0]
