"""GPU: meteor_lrpt_decoder parity. The decoder is all-integer (hard correlator, Viterbi27, byte stage, RS), so the CUDA path must
reproduce the reference bit for bit: every frame's (offset, pos, corr, phase, swap, RS errors, BER) record, every CADU byte and the stats
after every push, against oracle/_ref where it was built, else against tests/golden/meteor_lrpt_pins.json."""
import numpy as np
import pytest

from tests.common import assert_pin, pieces, run_chain, run_cli
from tests.meteor_lrpt_cases import (CASES, CHAIN, M2X, M2X_PARAMS, MSG, PIECES, after_lock, chain_signal, digest, piece_cuts, pins,
                                     stream)

pytestmark = pytest.mark.gpu


def expected(name, pieces=False):
    """The reference's pin of a case: CADU digest and count, records, stats after the last push"""
    from oracle import meteor as O
    pin = pins()["pieces" if pieces else "cases"][name]
    if O.available():
        case = CASES[name]
        soft, _, cuts = stream(case)
        r = O.run_pieces(soft, piece_cuts(soft.size) if pieces else cuts, case.get("diff", False))
        assert_pin(pin, "meteor_lrpt_pins.json", cadu=digest(r["cadu"]), recs=r["recs"].tolist())
    return pin


def run_gpu(soft, cuts, diff, max_soft=None):
    from satdump_b200 import capi
    g = capi.Fec(capi.meteor_lrpt_cfg(diff, max_soft=max_soft or max(1 << 16, soft.size)))
    frames, recs = [], []
    for a, b in pieces(soft.size, cuts):
        g.push(soft[a:b])
        frames.append(g.frames())
        recs.append(g.meteor_frames())
    return np.concatenate(frames), np.concatenate(recs), g.stats()


def check(name, pieces=False):
    pin = expected(name, pieces)
    case = CASES[name]
    soft, _, cuts = stream(case)
    got, grec, s = run_gpu(soft, piece_cuts(soft.size) if pieces else cuts, case.get("diff", False))
    want = np.array(pin["recs"], np.int64).reshape(-1, 10)
    assert np.array_equal(grec, want), (grec, want)
    assert got.shape[0] == pin["ncadu"] and digest(got) == pin["cadu"]
    st = pin["stats"][-1]
    assert s["correlator_lock"] == st["correlator_lock"] and s["rs_avg"] == st["rs_avg"]
    assert np.float32(s["viterbi_ber"]).view(np.uint32) == st["viterbi_ber"]
    rs = want[:, 5:9]
    assert s["frames_out"] == pin["ncadu"] and s["ldpc_resyncs"] == int((want[:, 1] != 0).sum())
    assert s["rs_failed"] == int((rs == -1).sum()) and s["rs_corrected"] == int(rs[rs > 0].sum())
    if want.shape[0]:
        assert s["correlator_corr"] == want[-1, 2]
    return got, grec


@pytest.mark.parametrize("name", sorted(CASES))
def test_records_cadus_and_stats_equal_the_reference(built, name):
    check(name)


@pytest.mark.parametrize("name", PIECES)
def test_ragged_pushes(built, name):
    """The same streams pushed in pieces of 1, 3, 777, 16383, 16385, 40001, 5, 32771 and 9000 bytes (most shorter than a frame)"""
    check(name, pieces=True)


def test_the_cases_reach_their_branches(built):
    """What each case is for: all 8 ambiguities, shifts below and above F / 2, the inversion test, RS corrections and drops"""
    recs = {n: np.array(pins()["cases"][n]["recs"], np.int64).reshape(-1, 10) for n in CASES}
    seen = {(int(p), int(s)) for n in CASES if n.startswith("phase") for p, s in recs[n][:, 3:5]}
    assert len(seen) == 8
    pos = recs["shifts"][:, 1]
    assert ((pos > 0) & (pos < 8192)).any() and (pos > 8192).any()
    assert (recs["rs_corrected"][:, 5:9] > 0).any() and (recs["low_esn0"][:, 5:9] == -1).any()
    assert pins()["cases"]["low_esn0"]["ncadu"] < recs["low_esn0"].shape[0]
    got, _ = check("plain")
    from satdump_b200 import synth
    _, written = synth.lrpt_frames(24, 21, inverted=(3, 17))
    assert np.array_equal(got, written)  # frames 3 and 17 went through the inversion branch


def test_large_push(built):
    """Thousands of frames in one push (the frame walk's rounds of 128 frames, thousands of Viterbi chunks) after a shift, then noise
    (one frame per walk round)"""
    from oracle import meteor as O
    from satdump_b200 import synth
    from tests.meteor_lrpt_cases import noise
    coded, written = synth.lrpt_frames(1500, seed=77)
    rng = np.random.default_rng(5)
    soft = np.concatenate([noise(rng, 4242), synth.lrpt_soft(coded, 1, False, sigma=30.0, seed=3), noise(rng, 20 * 16384)])
    got, grec, s = run_gpu(soft, [soft.size // 3], False)
    assert got.shape[0] == 1500 and (grec[1:1500, 1] == 0).all()
    # a frame whose derandomised byte 9 happens to be 0xFF (about 1 in 256) takes the inversion branch and comes out inverted
    inv = written[:, 9] == 0xFF
    assert 0 < inv.sum() < 20
    assert np.array_equal(got[~inv, :MSG], written[~inv, :MSG]) and np.array_equal(got[inv, 4:MSG], written[inv, 4:MSG] ^ 0xFF)
    if O.available():
        r = O.run_pieces(soft, [soft.size // 3])
        assert np.array_equal(grec, r["recs"]) and np.array_equal(got, r["cadu"])


@pytest.mark.parametrize("name", sorted(M2X))
def test_m2x_mode(built, name):
    """m2x_mode (the conv_concat OQPSK configuration) through lock, unlock and relock: the reference's CADUs and stats"""
    from satdump_b200 import capi
    case = M2X[name]
    soft, _, _ = stream(case)
    pin = pins()["m2x"][name]
    g = capi.Fec(capi.meteor_lrpt_cfg(case.get("diff", False), m2x_mode=True, max_soft=soft.size + 65536, **M2X_PARAMS))
    out = []
    for a, b in [(0, soft.size // 3), (soft.size // 3, soft.size)]:
        g.push(soft[a:b])
        out.append(g.frames())
    got = np.concatenate(out)
    s = g.stats()
    assert got.shape[0] == pin["ncadu"] and digest(got) == pin["cadu"]
    st = pin["stats"]
    assert s["deframer_state"] == st["deframer_state"] and s["viterbi_state"] == st["viterbi_lock"] and s["rs_avg"] == st["rs_avg"]
    assert np.float32(s["viterbi_ber"]).view(np.uint32) == st["viterbi_ber"]


def chain_expected(name):
    from oracle import meteor as O
    pin = pins()["chain"][name]
    if O.available():
        from tests.meteor_lrpt_cases import chain_reference
        cadu, clear = chain_reference(name)
        assert_pin(pin, "meteor_lrpt_pins.json", ncadu=cadu.shape[0], tail=digest(after_lock(cadu, clear)))
    return pin["ncadu"], pin["ntail"], pin["tail"]


def same_as_reference(got, name, clear):
    """The reference's CADUs from the third transmitted one on (the first are read while the demodulator's loops acquire, on its float
    floor), and they are the transmitted ones"""
    n, ntail, tail_digest = chain_expected(name)
    tail = after_lock(got, clear)
    assert got.shape[0] == n and tail.shape[0] == ntail and digest(tail) == tail_digest
    assert ntail > 10 and all(any(np.array_equal(row, c) for c in clear) for row in tail)


@pytest.mark.parametrize("name", sorted(CHAIN))
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain(built, name, pipelined):
    """IQ -> psk_demod (QPSK, 72 ksym/s, pll_bw 0.002; at 200 kS/s and through the front-end resampler at 1 MS/s) -> meteor_lrpt_decoder
    through the fused chain, in three pushes"""
    from satdump_b200 import capi
    from tests.common import demod_kwargs
    cfg, raw, clear = chain_signal(name)
    n = raw.size // 2
    got, fs = run_chain(capi.demod_cfg(max_batch=n, **demod_kwargs(cfg)), capi.fec_cfg_for(cfg, max_soft=4 * n), raw, cfg.fmt, pipelined)
    same_as_reference(got, name, clear)
    assert fs["correlator_lock"] == 1


@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli_meteor_lrpt(built, tmp_path, mode):
    """b200_pipeline meteor_lrpt (the 72k pipeline's psk_demod parameters, module id meteor_lrpt_decoder, diff_decode false) at the
    pipeline's default 1 MS/s: the .cadu file holds the reference's frames and the module reports lock_state"""
    name = "meteor_lrpt_1m_cs16"
    cfg, raw, clear = chain_signal(name)
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    r = run_cli("meteor_lrpt", inp, hint, "--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16", fused=mode == "fused")
    assert "lock_state SYNCED" in r.stdout
    same_as_reference(np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024), name, clear)


def test_host_refusals(built):
    """The library refuses interleaved as not built, and m2x_mode has no mode-A frame records"""
    from satdump_b200 import capi
    with pytest.raises(capi.B200Error) as e:
        capi.Fec(capi.meteor_lrpt_cfg(True, m2x_mode=True, interleaved=True, **M2X_PARAMS))
    assert "interleaved" in str(e.value) and "not built" in str(e.value)
    g = capi.Fec(capi.meteor_lrpt_cfg(False, m2x_mode=True, **M2X_PARAMS))  # (run as ccsds_conv_concat_decoder: no frame records)
    g.push(np.zeros(10, np.int8))
    with pytest.raises(capi.B200Error, match="not a METEOR LRPT decoder"):
        g.meteor_frames()
