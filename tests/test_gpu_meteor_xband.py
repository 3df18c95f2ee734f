"""GPU: meteor_xband_decoder (B200_FEC_METEOR_XBAND, mtvza and kmss_bpsk) against the reference (oracle/_ref, else the pins of
tests/golden/meteor_xband_pins.json) on every case stream: frames, their order and frame_count, pushed whole, in ragged pieces (1, 3, 8191,
8193 bytes, so that the record windows, the NRZ-M bit, an open inner frame and a partial read cross pushes) and as one push of 2^26 bytes;
IQ (cs16, cf32) -> psk_demod BPSK -> the decoder through b200_chain, synchronous and pipelined, against the reference chain and the sent
frames; b200_pipeline meteor_mtvza | meteor_kmss_bpsk, two-stage and fused."""
import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests import xband_cases as X
from tests.common import pieces, run_chain, run_cli

pytestmark = pytest.mark.gpu

TYPES = {0: "mtvza", 1: "kmss_bpsk"}


def _decode(name, soft, cuts=(), max_soft=1 << 22):
    f = capi.Fec(capi.meteor_xband_cfg(TYPES[X.kind(name)], max_soft=max_soft))
    out = []
    for a, b in pieces(soft.size, cuts):
        f.push(soft[a:b])
        out.append(f.frames())
    st = f.stats()
    f.close()
    return np.concatenate(out), st


def _check(name, out, st):
    pin = X.ref_result(name)
    assert out.shape[0] == pin["frames"] and X.digest(out) == pin["out"]
    assert st["frames_out"] == pin["frame_count"]


@pytest.mark.parametrize("name", X.CASES)
def test_whole_stream(name):
    _check(name, *_decode(name, X.stream(name)))


def _cuts(n, sizes, limit=3000):
    """cuts cycling through `sizes` for the first `limit` pieces, then whole reads"""
    cuts, at, i = [], 0, 0
    while at < n and len(cuts) < limit:
        at += sizes[i % len(sizes)]
        i += 1
        if at < n:
            cuts.append(at)
    nxt = (at // X.READ + 1) * X.READ
    return cuts + list(range(nxt, n, X.READ))


@pytest.mark.parametrize("sizes", [(1, 3, 8191, 8193), (8191,), (8193, 1), (100003,)])
@pytest.mark.parametrize("name", X.CASES)
def test_pieces(name, sizes):
    soft = X.stream(name)
    _check(name, *_decode(name, soft, _cuts(soft.size, sizes)))


def test_one_byte_pushes_across_a_read():
    """every push of one byte around a read boundary: nothing comes out before the read is whole"""
    name = "kmss_all_deframers_one_read"
    soft = X.stream(name)
    f = capi.Fec(capi.meteor_xband_cfg("kmss_bpsk", max_soft=1 << 22))
    f.push(soft[:5 * X.READ - 40])
    out = [f.frames()]
    n0 = sum(o.shape[0] for o in out)
    for k in range(5 * X.READ - 40, 5 * X.READ + 40):
        f.push(soft[k:k + 1])
        got = f.frames()
        assert got.shape[0] == 0 or k == 5 * X.READ - 1
        out.append(got)
    f.push(soft[5 * X.READ + 40:])
    out.append(f.frames())
    st = f.stats()
    f.close()
    assert n0 >= 0
    _check(name, np.concatenate(out), st)


@pytest.mark.parametrize("name", X.LARGE)
def test_large_push(name):
    soft = X.stream(name)
    assert soft.size == 1 << 26
    _check(name, *_decode(name, soft, max_soft=soft.size))


def _signal(name, fmt):
    cfg = synth.CONFIGS[name]
    cfg = synth.SignalCfg(**{**cfg.__dict__, "fmt": fmt})
    n = 1 << 21 if name == "meteor_mtvza" else 1 << 23
    raw, clear = synth.make_signal(cfg, n, seed=5)
    return cfg, raw.numpy(), clear


def _chain(cfg, raw, pipelined):
    n = raw.size // 2 if cfg.fmt != "cf32" else raw.size
    return run_chain(capi.demod_cfg_for(cfg, max_batch=n), capi.fec_cfg_for(cfg, max_soft=n), raw, cfg.fmt, pipelined)


@pytest.mark.parametrize("fmt", ["cs16", "cf32"])
@pytest.mark.parametrize("name", ["meteor_mtvza", "meteor_kmss_bpsk"])
def test_chain(name, fmt):
    """IQ -> psk_demod BPSK with the pipeline's parameters -> the decoder through b200_chain, in three pushes: synchronous and pipelined
    write the same frames, the reference chain writes them too, and they are the sent frames"""
    cfg, raw, clear = _signal(name, fmt)
    sync, fs = _chain(cfg, raw, False)
    pipe, fp = _chain(cfg, raw, True)
    assert np.array_equal(sync, pipe) and fs["frames_out"] == fp["frames_out"] == sync.shape[0]
    sent = {bytes(r) for r in np.asarray(clear)}
    good = sum(bytes(r) in sent for r in sync)
    assert sync.shape[0] >= (100 if name == "meteor_mtvza" else 4) and good >= sync.shape[0] - 1
    try:
        from oracle import ref as orc
        if not orc.available():
            raise ImportError
    except ImportError:
        from oracle import port as orc
    from oracle import xband
    soft = orc.Demod(orc.demod_cfg(cfg.samplerate, cfg.symbolrate, cfg.constellation, cfg.rrc_alpha, cfg.pll_bw, cfg.fmt)).run(raw, stages=False)["soft"]
    if xband.available():
        want = xband.Ref(1 if name == "meteor_kmss_bpsk" else 0).run(soft)["out"]
        assert np.array_equal(sync, want)


@pytest.mark.parametrize("name", ["meteor_mtvza", "meteor_kmss_bpsk"])
def test_cli(built, tmp_path, name):
    """b200_pipeline meteor_mtvza | meteor_kmss_bpsk (the pipelines' psk_demod and decoder parameters), two-stage and fused, write the
    same .frm, the sent frames"""
    cfg, raw, clear = _signal(name, "cs16")
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    nb = clear.shape[1]
    got = {}
    for mode in ("two_stage", "fused"):
        hint = str(tmp_path / mode)
        r = run_cli(name, inp, hint, "--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16", fused=mode == "fused",
                    timeout=600)
        got[mode] = np.fromfile(hint + ".frm", np.uint8).reshape(-1, nb)
        assert f"frame_count {got[mode].shape[0]}\n" in r.stdout
    assert np.array_equal(got["two_stage"], got["fused"])
    sent = {bytes(x) for x in np.asarray(clear)}
    assert got["fused"].shape[0] >= 4 and sum(bytes(x) in sent for x in got["fused"]) >= got["fused"].shape[0] - 1
