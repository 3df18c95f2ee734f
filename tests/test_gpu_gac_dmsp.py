"""GPU: noaa_gac_decoder (B200_FEC_NOAA_GAC) and dmsp_rtd_decoder (B200_FEC_DMSP_RTD) against the reference (oracle/_ref, else the pins
of tests/golden/gac_pins.json) on every case stream: frames, final deframer state and DMSP timestamps, pushed whole and in pieces (1 byte,
sizes that split a sync word and a frame, so that the machine's state and an open frame cross pushes); the completion bits against the
bit-serial model; b200_chain synchronous and pipelined."""
import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests import gac_cases as G
from tests import gac_model as M
from tests.common import pieces, run_chain, run_cli

pytestmark = pytest.mark.gpu


def _cfg(name, max_soft=1 << 20):
    dmsp, backward = G.params(name)
    return capi.dmsp_rtd_cfg(max_soft=max_soft) if dmsp else capi.noaa_gac_cfg(backward, max_soft=max_soft)


def _decode(name, soft, cuts=()):
    f = capi.Fec(_cfg(name))
    out, bits = [], []
    for a, b in pieces(soft.size, cuts):
        f.push(soft[a:b])
        out.append(f.frames())
        bits.append(f.frame_bits())
    st = f.stats()
    f.close()
    return np.concatenate(out), np.concatenate(bits), st


def _check(name, out, bits, st):
    pin = G.ref_result(name)
    assert out.shape[0] == pin["frames"] and G.digest(out) == pin["out"]
    assert st["deframer_state"] == pin["state"] and st["frames_out"] == pin["frames"]
    assert bits.size == out.shape[0]
    if G.is_dmsp(name):
        assert G.ts_digest(capi.dmsp_timestamps(bits, G.START_TS)) == pin["ts"]


@pytest.mark.parametrize("name", G.CASES)
def test_whole_stream(name):
    soft = G.stream(name)
    out, bits, st = _decode(name, soft)
    _check(name, out, bits, st)
    assert np.array_equal(bits, M.run(soft, *G.params(name))["done"])


@pytest.mark.parametrize("sizes", [(8192,), (13, 4099, 151), (33269, 40000), (1, 2, 3, 5, 8, 12, 31, 149, 150, 1500)])
@pytest.mark.parametrize("name", G.CASES)
def test_pieces(name, sizes):
    soft = G.stream(name)
    cuts = G.cuts_for(name, soft.size, sizes)
    if len(cuts) > 4000:  # (small pieces over the stream's start, where the first syncs and frames lie, then whole reads)
        lim = cuts[3999]
        cuts = [c for c in cuts if c <= lim] + list(range((lim // 8192 + 1) * 8192, soft.size, 8192))
    _check(name, *_decode(name, soft, cuts))


def test_one_byte_pushes_across_a_dmsp_frame_and_gac_sync():
    for name in ("dmsp_clean", "gac_clean"):
        soft = G.stream(name)
        lead = (G.DMSP if G.is_dmsp(name) else G.GAC)[name]["lead"]
        cuts = list(range(lead - 40, lead + 400)) + list(range(((lead + 400) // 8192 + 1) * 8192, soft.size, 8192))
        _check(name, *_decode(name, soft, cuts))


@pytest.mark.parametrize("name", ["gac_clean", "gac_backward", "dmsp_synced_drop"])
def test_large_push(name):
    reps = 40
    soft = np.concatenate([G.stream(name)] * reps)
    f = capi.Fec(_cfg(name, max_soft=soft.size))
    f.push(soft)
    out = f.frames()
    bits = f.frame_bits()
    m = M.run(G.stream(name), *G.params(name))
    assert out.shape[0] >= reps * (m["out"].shape[0] - 1) and bits.size == out.shape[0] and np.all(np.diff(bits) > 0)
    # every copy of the stream starts in noise, so each decodes as the stream alone
    per = G.stream(name).size
    k0 = bits < per
    assert np.array_equal(out[k0], m["out"])


def test_other_kinds_refuse_frame_bits():
    f = capi.Fec(capi.meteor_hrpt_cfg(max_soft=1 << 17))
    with pytest.raises(capi.B200Error, match="noaa_gac_decoder and dmsp_rtd_decoder"):
        f.frame_bits()


def _chain(cfg, raw, pipelined):
    n = raw.size // 2
    return run_chain(capi.demod_cfg_for(cfg, max_batch=n), capi.fec_cfg_for(cfg, max_soft=n), raw, cfg.fmt, pipelined)


@pytest.mark.parametrize("name", ["noaa_gac", "dmsp_rtd"])
def test_chain(name):
    """IQ (cs16) -> psk_demod BPSK with the pipeline's parameters -> the decoder through b200_chain, in three pushes: synchronous and
    pipelined write the same bytes, and after the lock they are the sent frames"""
    cfg = synth.CONFIGS[name]
    raw, clear = synth.make_signal(cfg, 1 << 21, seed=5)
    raw = raw.numpy()
    sync, fs = _chain(cfg, raw, False)
    pipe, fp = _chain(cfg, raw, True)
    assert np.array_equal(sync, pipe) and fs["frames_out"] == fp["frames_out"] == sync.shape[0]
    sent = {bytes(r) for r in np.asarray(clear).reshape(-1, sync.shape[1])}
    good = sum(bytes(r) in sent for r in sync)
    assert sync.shape[0] >= (5 if name == "noaa_gac" else 1000) and good >= sync.shape[0] - 2


@pytest.mark.parametrize("name", ["noaa_gac", "dmsp_rtd"])
@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli(built, tmp_path, name, mode):
    """b200_pipeline noaa_gac | dmsp_rtd (the pipelines' psk_demod and decoder parameters) writes the sent frames to .frm after the lock;
    DMSP's two-stage run writes one timestamp per frame by the reference's rule; a backward GAC run leaves no .frm.tmp behind"""
    import os
    cfg = synth.CONFIGS[name]
    raw, clear = synth.make_signal(cfg, 1 << 21, seed=5)
    inp = tmp_path / "in.cs16"
    raw.numpy().tofile(inp)
    hint = str(tmp_path / "out")
    args = ["--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16"]
    if mode == "two_stage" and name == "dmsp_rtd":
        args += ["--start_timestamp", "1700000000.5"]
    r = run_cli(name, inp, hint, *args, fused=mode == "fused")
    nb = 4159 if name == "noaa_gac" else 19
    got = np.fromfile(hint + ".frm", np.uint8).reshape(-1, nb)
    sent = {bytes(x) for x in np.asarray(clear).reshape(-1, nb)}
    assert got.shape[0] >= 5 and sum(bytes(x) in sent for x in got) >= got.shape[0] - 2
    if name == "noaa_gac":
        assert f"frame_count {got.shape[0] // 11090}\n" in r.stdout
        run_cli(name, inp, hint, *args, "--backward", "true", fused=mode == "fused")
        assert os.path.exists(hint + ".frm") and not os.path.exists(hint + ".frm.tmp")
    else:
        assert "deframer_state " in r.stdout
        if mode == "two_stage":
            lines = open(hint + "_timestamps.txt").read().splitlines()
            assert len(lines) == got.shape[0] and all(float(v) >= 1700000000.5 for v in lines)
