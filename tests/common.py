"""Shared helpers of the test-suite: config plumbing between the synthetic transmitter, the oracle and the C ABI."""
import copy
import functools
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle._checker import pieces  # noqa: E402,F401  (the (start, end) of each push, shared with the checkers)
from satdump_b200 import synth  # noqa: E402


def oracle():
    """The checker: the compiled reference (oracle/_ref) when present, else our C restatement."""
    from oracle import ref
    if ref.available():
        return ref
    from oracle import port
    return port


def reference(O):
    """The checker module O (oracle.hrpt, ...) when its library was built from the reference, else skip: without the reference the
    tests compare with the pins."""
    if not O.available():
        import pytest
        pytest.skip(f"{O.__name__}: oracle/_ref not built (the reference is absent): the tests compare with the pins")
    return O


def digest(a, dtype=None, hexlen=None):
    """sha256 of the array's bytes (cast to dtype first when given) in hex, its first hexlen digits when given"""
    return hashlib.sha256(np.ascontiguousarray(a, dtype).tobytes()).hexdigest()[:hexlen]


@functools.cache
def _read_json(path):
    with open(path) as f:
        return json.load(f)


def load_pins(path):
    """A golden JSON file, read from disk once; each caller gets its own copy."""
    return copy.deepcopy(_read_json(path))


def assert_pin(pin, golden, **live):
    """The reference's results now (live: field -> value) equal the pinned ones (pin[field]). The pins stand in for the reference where it
    is absent: otherwise the golden file `golden` is stale."""
    stale = sorted(k for k, v in live.items() if pin[k] != v)
    assert not stale, f"{golden} is stale: {stale}"


def after_lock(frames, clear, prefix=None):
    """The frames from the third one whose data (its first `prefix` bytes when given) is a transmitted frame's on: the first ones are
    read while the demodulator's loops acquire, where its soft bytes sit on the float floor (DESIGN §5)"""
    for i, row in enumerate(frames):
        if any(np.array_equal(row[:prefix], c[:prefix]) for c in clear):
            return frames[i + 2:]
    return frames[:0]


def run_chain(dcfg, fcfg, raw, fmt, pipelined):
    """raw IQ through a capi.Chain of the two configs in three pushes (the second ends off a third of the stream), synchronous or
    pipelined: the frames concatenated, and the decoder's stats"""
    from satdump_b200 import capi
    per = 1 if fmt == "cf32" else 2
    n = raw.size // per
    ch = capi.Chain(dcfg, fcfg)
    if pipelined:
        ch.set_pipelined(True)
    out = []
    for a, b in [(0, n // 3), (n // 3, 2 * n // 3 + 1001), (2 * n // 3 + 1001, n)]:
        ch.push(raw[per * a:per * b])
        out.append(ch.frames())
    if pipelined:
        ch.sync()
        out.append(ch.frames())
    _, fs = ch.stats()
    ch.close()
    return np.concatenate(out), fs


def run_cli(pipe, inp, hint, *args, fused=False, timeout=300):
    """b200_pipeline <pipe> baseband <inp> <hint> <args>, two-stage or --fused; the completed process, which must have exited 0"""
    tool = os.path.join(ROOT, "satdump_b200", "host", "b200_pipeline")
    r = subprocess.run([tool, pipe, "baseband", str(inp), hint, *args] + (["--fused"] if fused else []), capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0, r.stderr
    return r


def rx_const(cfg):
    return cfg.constellation if cfg.decoder != "none" else "none"  # decoder "demod": psk_demod alone, with its Costas loop


def demod_kwargs(cfg):
    kw = dict(samplerate=cfg.samplerate, symbolrate=cfg.symbolrate, constellation=rx_const(cfg), rrc_alpha=cfg.rrc_alpha, pll_bw=cfg.pll_bw,
              fmt=cfg.fmt)
    if cfg.clock_alpha:
        kw["clock_alpha"] = cfg.clock_alpha
    if cfg.has_carrier:
        kw.update(has_carrier=True, carrier_pll_bw=cfg.carrier_pll_bw)
    elif cfg.pm_index:
        kw.update(pm=True, pm_pll_bw=cfg.pm_pll_bw, pm_pll_max_offset=cfg.pm_pll_max_offset, resample_after_pll=cfg.resample_after_pll,
                  subcarrier_offset=cfg.subcarrier)
    return kw


def oracle_demod(O, cfg):
    return O.Demod(O.demod_cfg(**demod_kwargs(cfg)))


def conv_rate_of(cfg):
    return cfg.conv[1:] if cfg.conv.startswith("p") else "1/2"


def oracle_fec(O, cfg):
    if cfg.decoder == "simple":
        return O.Fec(O.simple_cfg(cfg.constellation, cfg.cadu_bytes * 8, cfg.interleave, nrzm=cfg.nrzm, qpsk_swap_iq=cfg.constellation == "qpsk"))
    if cfg.decoder == "metop":
        return O.Fec(O.metop_cfg(cfg.ber_thresold, cfg.outsync_after))
    return O.Fec(O.ccsds_cfg(cfg.constellation, cfg.cadu_bytes * 8, cfg.ber_thresold, cfg.outsync_after, cfg.interleave, nrzm=cfg.nrzm,
                             rs_usecheck=cfg.rs_usecheck, conv_rate=conv_rate_of(cfg)))


def gpu_demod(cfg, n, keep_stages=False):
    from satdump_b200 import capi
    return capi.Demod(capi.demod_cfg(max_batch=max(n, 4096), keep_stages=keep_stages, **demod_kwargs(cfg)))


def gpu_fec_cfg(cfg, max_soft):
    from satdump_b200 import capi
    if cfg.decoder == "simple":
        return capi.simple_cfg(cfg.constellation, cfg.cadu_bytes * 8, cfg.interleave, nrzm=cfg.nrzm, qpsk_swap_iq=cfg.constellation == "qpsk",
                               max_soft=max(max_soft, 65536))
    if cfg.decoder == "metop":
        return capi.metop_cfg(cfg.ber_thresold, cfg.outsync_after, max_soft=max(max_soft, 65536))
    return capi.ccsds_cfg(cfg.constellation, cfg.cadu_bytes * 8, cfg.ber_thresold, cfg.outsync_after, cfg.interleave, nrzm=cfg.nrzm,
                          rs_usecheck=cfg.rs_usecheck, max_soft=max(max_soft, 65536))


def gpu_chain(cfg, n):
    from satdump_b200 import capi
    return capi.Chain(capi.demod_cfg(max_batch=max(n, 4096), **demod_kwargs(cfg)), gpu_fec_cfg(cfg, 2 * n))


def simple_soft_cases(seed=1, nframes=24, sigma=20.0):
    """Soft-symbol streams for ccsds_simple_psk_decoder (no convolutional code): (name, simple_cfg kwargs, int8 soft) for every mode
    built: BPSK, BPSK + NRZ-M, QPSK at the four carrier phases (two deframers), QPSK with qpsk_swap_iq + oqpsk_delay, QPSK + NRZ-M
    (QPSKDiff) with and without qpsk_swap_diff. RS(255,223) I=4 frames; noise so that RS has work to do."""
    rng = np.random.default_rng(seed)
    pay = rng.integers(0, 256, size=(nframes, 4 * 223), dtype=np.uint8)
    tx, clear = synth.build_cadus(pay, 4)
    bits = np.unpackbits(tx.reshape(-1))
    lead = rng.integers(0, 2, size=3001, dtype=np.uint8)  # the stream does not start on a frame (nor byte) boundary
    bits = np.concatenate([lead, bits, lead[:777]])

    def noisy(v):
        return np.clip(np.round(v + rng.normal(0, sigma, v.size)), -127, 127).astype(np.int8)

    def iq(I, Q, rot=0):
        z = ((I * 2.0 - 1) + 1j * (Q * 2.0 - 1)) * np.exp(1j * np.pi / 2 * rot)
        s = np.empty(2 * I.size)
        s[0::2], s[1::2] = z.real * 60, z.imag * 60
        return noisy(s)

    cases = [("bpsk", dict(constellation="bpsk"), noisy((bits * 2.0 - 1) * 60)),
             ("bpsk_nrzm", dict(constellation="bpsk", nrzm=True), noisy((synth.nrzm_encode(bits) * 2.0 - 1) * 60))]
    b = bits[:bits.size // 2 * 2]
    for rot in range(4):  # bit order of the simple decoder: Q rail first (constellation_t::soft_demod, :190-199)
        cases.append((f"qpsk_rot{rot}", dict(constellation="qpsk"), iq(b[1::2], b[0::2], rot)))
    cases.append(("qpsk_swapiq_delay", dict(constellation="qpsk", qpsk_swap_iq=True, oqpsk_delay=True), iq(b[1::2], b[0::2], 0)))
    for swap in (True, False):
        sy = synth.qpsk_diff_encode(b[0::2].astype(np.int64) * 2 + b[1::2], swap)
        cases.append((f"qpsk_diff_swap{int(swap)}", dict(constellation="qpsk", nrzm=True, qpsk_swap_diff=swap), iq(sy & 1, sy >> 1, 1)))
    return cases, clear


def nsamples(raw, cfg):
    return raw.size if cfg.fmt == "cf32" else raw.size // 2


@functools.lru_cache(maxsize=16)
def signal(name, log2n, seed=1, esn0=None):
    """(raw numpy array in the config's format, clear CADUs). Generated on the CPU: the realisation of the noise depends on the generator
    (torch's CUDA generator gives another one on every GPU model), and the committed parity floors (tests/floors.py) belong to this one."""
    import dataclasses
    cfg = synth.CONFIGS[name]
    if esn0 is not None:
        cfg = dataclasses.replace(cfg, esn0_db=esn0)
    raw, clear = synth.make_signal(cfg, 1 << log2n, seed=seed, device="cpu")
    return cfg, raw.numpy(), clear


def match_frames(got, clear):
    """Index in `clear` of got[0] and whether got is the consecutive run of transmitted frames from there."""
    if got.shape[0] == 0:
        return None, False
    for i in range(min(256, clear.shape[0])):
        if np.array_equal(clear[i], got[0]):
            ok = i + got.shape[0] <= clear.shape[0] and np.array_equal(got, clear[i:i + got.shape[0]])
            return i, ok
    return None, False
