"""GPU: noaa_hrpt_decoder and meteor_hrpt_decoder parity. Both deframers are bit machines without FEC, so the CUDA path must reproduce the
reference bit for bit: every accepted sync's (bit, inverted, state) record, every output word / CADU byte and the stats after every push,
against oracle/_ref where it was built, else against tests/golden/hrpt_pins.json."""
import numpy as np
import pytest

from tests.common import assert_pin, pieces, run_chain, run_cli
from tests.hrpt_cases import (LARGE, METEOR, MIX_AT, NOAA, boundary_cuts, digest, large_stream, params, piece_cuts, pins, stats_rows,
                              stream)

pytestmark = pytest.mark.gpu
CASES = [*NOAA, *METEOR]


def run_gpu(soft, cuts, meteor, thr):
    """The decoder over soft pushed in the pieces cut at `cuts`: output, records, [units, state] after every push, final stats"""
    from satdump_b200 import capi
    cfg = capi.meteor_hrpt_cfg(max_soft=max(1 << 16, soft.size)) if meteor else capi.noaa_hrpt_cfg(thr, max_soft=max(1 << 16, soft.size))
    g = capi.Fec(cfg)
    out, recs, rows = [], [], []
    for a, b in pieces(soft.size, cuts):
        g.push(soft[a:b])
        f = g.frames()
        out.append(f.reshape(-1).view(np.uint16) if not meteor else f)
        recs.append(g.hrpt_frames())
        s = g.stats()
        rows.append([s["frames_out"], s["deframer_state"]])
    return np.concatenate(out), np.concatenate(recs), rows, g.stats()


def check(pin, soft, cuts, meteor, thr):
    from oracle import hrpt as O
    if O.available():
        r = O.run_pieces(soft, cuts, meteor, thr)
        assert_pin(pin, "hrpt_pins.json", out=digest(r["out"]), recs=r["recs"].tolist())
    got, recs, rows, s = run_gpu(soft, cuts, meteor, thr)
    assert recs.tolist() == pin["recs"]
    assert got.shape[0] == pin["units"] and digest(got) == pin["out"]
    assert (rows if isinstance(pin["stats"], list) else digest(rows)) == pin["stats"]
    return got, recs, s


@pytest.mark.parametrize("name", CASES)
def test_output_records_and_stats_equal_the_reference(built, name):
    soft, cuts = stream(name)
    check(pins()["cases"][name], soft, cuts, *params(name))


@pytest.mark.parametrize("name", CASES)
def test_ragged_pushes(built, name):
    """The same streams in pieces of 1, 3, 9, 777 and 8191 bytes, with cuts inside a word, a frame and a sync"""
    soft, _ = stream(name)
    check(pins()["pieces"][name], soft, piece_cuts(soft.size, extra=boundary_cuts(name)), *params(name))


@pytest.mark.parametrize("name", sorted(LARGE))
def test_large_push(built, name):
    """Hundreds of frames in one push (a frame-length jump per frame), then noise; the frames come out as sent"""
    from satdump_b200 import synth
    soft, cuts, meteor, thr = large_stream(name)
    got, recs, s = check(pins()["large"][name], soft, cuts, meteor, thr)
    n = LARGE[name][2]
    _, sent = (synth.meteor_hrpt_frames if meteor else synth.noaa_hrpt_frames)(n, n + 1)
    if meteor:
        assert np.array_equal(got[:n], sent)
    else:
        assert np.array_equal(got[:n * synth.NOAA_WORDS].reshape(n, -1), sent) and s["frames_out"] // synth.NOAA_WORDS >= n


def test_the_cases_reach_their_branches(built):
    """What each case is for, read from the reference's records: polarity and its flip, thr and thr + 1 errors, a splice window accepted
    at thr 26, syncs completed against the zero shifter, a bit slip, every METEOR state transition, a one-bit-late frame, a match in a
    window of mixed inversion after a state-2 timeout"""
    rec = {n: np.array(pins()["cases"][n]["recs"], np.int64).reshape(-1, 3) for n in CASES}
    F = 110900
    assert (rec["noaa_inverted"][:, 1] == 1).all() and rec["noaa_flip"][:, 1].tolist() == [0, 0, 0, 1, 1, 1]
    assert rec["noaa_thr_edges"].shape[0] == 4 and np.diff(rec["noaa_thr_edges"][:, 0]).tolist() == [F, 2 * F, F]  # 10 in, 11 out
    assert rec["noaa_thr0"].shape[0] == 3
    d = np.diff(rec["noaa_thr26_splice"][:, 0])
    assert ((d > 110840) & (d < F)).all()  # accepted in a splice: 1 .. 59 bits after the frame's last data bit (sync + 110840)
    assert rec["noaa_zero_shifter"][0, 0] == 49 and rec["meteor_zero_shifter"][0, 0] == 28
    assert (np.diff(rec["noaa_slip"][:, 0]) == [F, F - 1, F, F]).all()
    m = rec["meteor_transitions"]
    trans = {(int(a), int(b)) for a, b in zip(m[:-1, 2], m[1:, 2])}
    assert {(0, 6), (6, 12), (12, 2), (2, 6), (6, 2)} <= trans and (m[:, 2] == 12).any()
    late = rec["meteor_late"]
    assert 8193 in np.diff(late[:, 0]).tolist() and late[np.diff(late[:, 0]).tolist().index(8193) + 1, 2] == 6
    mix = rec["meteor_mixed"]
    assert mix[-1].tolist() == [100 + 7 * 8192 + MIX_AT, 0, 0] and mix[-2, 1] == 1  # 2 -> 0 by the timeout, then the mixed window
    assert rec["meteor_nsn"][:, 2].tolist().count(0) == 2


def test_refusals(built):
    from satdump_b200 import capi
    with pytest.raises(capi.B200Error, match="deframer_thresold"):
        capi.Fec(capi.noaa_hrpt_cfg(61))
    g = capi.Fec(capi.meteor_hrpt_cfg())
    g.push(np.zeros(10, np.int8))
    with pytest.raises(capi.B200Error, match="not a METEOR LRPT decoder"):
        g.meteor_frames()


def same_as_reference(got, name, meteor, clear):
    """The reference's frames from the third transmitted one on (the first are read while the demodulator's loops acquire, on its float
    floor), and they are the transmitted ones"""
    from tests.hrpt_cases import after_lock, chain_reference, frames_of
    pin = pins()["chain"][name]
    from oracle import hrpt as O
    if O.available():
        o, _, _ = chain_reference(name)
        assert_pin(pin, "hrpt_pins.json", units=o.shape[0], tail=digest(after_lock(frames_of(o, meteor), clear)))
    tail = after_lock(frames_of(got, meteor), clear)
    assert got.shape[0] == pin["units"] and tail.shape[0] == pin["ntail"] and digest(tail) == pin["tail"]
    assert pin["ntail"] >= 5 and all(any(np.array_equal(row, c) for c in clear) for row in tail)


@pytest.mark.parametrize("name", ["noaa_hrpt", "meteor_hrpt"])
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain(built, name, pipelined):
    """IQ (cs16, 3 MS/s) -> pm_demod (665 400 sym/s, pll_bw 0.01, clock_omega_relative_limit 0.001) -> the decoder through the fused chain,
    in three pushes; NOAA's 2-byte output unit goes through the chain's frame buffers as words"""
    from satdump_b200 import capi
    from tests.hrpt_cases import chain_signal, demod_kwargs
    cfg, raw, clear = chain_signal(name)
    n = raw.size // 2
    got, fs = run_chain(capi.demod_cfg(max_batch=n, **demod_kwargs(cfg)), capi.fec_cfg_for(cfg, max_soft=n), raw, cfg.fmt, pipelined)
    meteor = name == "meteor_hrpt"
    got = got.reshape(-1)
    same_as_reference(got.reshape(-1, 1024) if meteor else got.view(np.uint16), name, meteor, clear)
    assert fs["deframer_state"] == (12 if meteor else 0)


@pytest.mark.parametrize("name", ["noaa_hrpt", "meteor_hrpt"])
@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli(built, tmp_path, name, mode):
    """b200_pipeline noaa_hrpt | meteor_hrpt (the pipelines' pm_demod and decoder parameters) writes the reference's .raw16 / .cadu after
    the lock and reports the module's stats"""
    from tests.hrpt_cases import chain_signal
    cfg, raw, clear = chain_signal(name)
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    r = run_cli(name, inp, hint, "--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16", fused=mode == "fused")
    meteor = name == "meteor_hrpt"
    got = np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024) if meteor else np.fromfile(hint + ".raw16", np.uint16)
    same_as_reference(got, name, meteor, clear)
    n = pins()["chain"][name]["units"]
    if meteor:
        assert f"frame_count {n}\n" in r.stdout and "deframer_lock 1" in r.stdout and "deframer_state SYNCED" in r.stdout
    else:
        assert f"frame_count {n // 11090}\n" in r.stdout
