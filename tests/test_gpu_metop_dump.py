"""GPU: metop_dump_decoder parity. The decoder is all-integer, so the CUDA path must reproduce the reference bit for bit: every frame's
(offset, pos, corr, phase, swap, RS errors) record and every CADU byte, against oracle/_ref where it was built, else against
tests/golden/metop_dump_pins.json."""
import numpy as np
import pytest

from tests.common import assert_pin, pieces, run_chain, run_cli
from tests.metop_dump_cases import CASES, CHAIN, PIECES, after_lock, chain_signal, digest, piece_cuts, pins, stream

pytestmark = pytest.mark.gpu
MSG = 4 + 4 * 223


def expected(name):
    """The reference's (CADU digest, number of CADUs, records) for a case"""
    from oracle import dump as O
    pin = pins()["cases"][name]
    if O.available():
        soft, _, _ = stream(CASES[name])
        r = O.Dump().run(soft)
        assert_pin(pin, "metop_dump_pins.json", cadu=digest(r["cadu"]), recs=r["recs"].tolist())
    return pin["cadu"], pin["ncadu"], np.array(pin["recs"], np.int64).reshape(-1, 9)


def run_gpu(soft, cuts, max_soft=None):
    from satdump_b200 import capi
    g = capi.Fec(capi.dump_cfg(max_soft=max_soft or max(1 << 16, soft.size)))
    frames, recs = [], []
    for a, b in pieces(soft.size, cuts):
        g.push(soft[a:b])
        frames.append(g.frames())
        recs.append(g.dump_frames())
    return np.concatenate(frames), np.concatenate(recs), g.stats()


def check(name, cuts):
    want_digest, ncadu, want_recs = expected(name)
    soft, _, _ = stream(CASES[name])
    got, grec, s = run_gpu(soft, cuts)
    assert np.array_equal(grec, want_recs), (grec, want_recs)
    assert got.shape[0] == ncadu and digest(got) == want_digest
    rs = want_recs[:, 5:]
    assert s["frames_out"] == ncadu and s["ldpc_resyncs"] == int((want_recs[:, 1] != 0).sum())
    assert s["rs_failed"] == int((rs == -1).sum()) and s["rs_corrected"] == int(rs[rs > 0].sum())
    if want_recs.shape[0]:
        assert s["correlator_lock"] == int(want_recs[-1, 1] == 0) and s["correlator_corr"] == want_recs[-1, 2]
    return got, grec


@pytest.mark.parametrize("name", sorted(CASES))
def test_records_and_cadus_equal_the_reference(built, name):
    check(name, stream(CASES[name])[2])


@pytest.mark.parametrize("name", PIECES)
def test_odd_sized_pieces(built, name):
    """The same streams pushed in pieces of 1, 3, 777, 8191, 8193, 20001, 5 and 16387 bytes"""
    soft, _, _ = stream(CASES[name])
    check(name, piece_cuts(soft.size))


def test_rs_results_and_lock_state(built):
    _, grec = check("rs_errors", [])
    assert (grec[1, 5:] == 10).all() and (grec[3, 5:] == -1).all()
    from satdump_b200 import capi, synth
    tx, clear = synth.dump_frames(3, seed=9)
    soft = synth.dump_soft(tx, 3, True)
    g = capi.Fec(capi.dump_cfg(max_soft=1 << 16))
    g.push(soft)
    assert np.array_equal(g.frames(), clear)
    s = g.stats()
    assert s["correlator_lock"] == 1 and s["correlator_corr"] == 32 and s["ldpc_resyncs"] == 0 and s["rs_failed"] == 0
    g.push(np.full(3 * 8192, 5, np.int8))  # a constant stream: no ASM at position 0
    assert g.stats()["correlator_lock"] == 0 and g.stats()["ldpc_resyncs"] > 0


def test_large_push(built):
    """Thousands of frames in one push (the frame walk's rounds of 128 frames) after a shift, then noise (one frame per round)"""
    from satdump_b200 import synth
    from tests.metop_dump_cases import noise
    tx, clear = synth.dump_frames(3000, seed=77)
    rng = np.random.default_rng(5)
    soft = np.concatenate([noise(rng, 4242), synth.dump_soft(tx, 1, False, sigma=10.0, seed=3), noise(rng, 40 * 8192)])
    got, grec, s = run_gpu(soft, [soft.size // 3])
    assert got.shape[0] > 3000 and np.array_equal(got[1:3000, :MSG], clear[1:, :MSG])  # (frame 0 is read across the shift)
    from oracle import dump as O
    impl = "ref" if O.available() else "port"
    r = O.Dump(impl).run(soft)
    assert np.array_equal(grec, r["recs"]) and np.array_equal(got, r["cadu"])


def chain_expected(name):
    """(number of CADUs, number after the lock, digest of those) of the reference's demodulator + decoder where it was built, else the pins"""
    from oracle import dump as O
    pin = pins()["chain"][name]
    if O.available():
        from tests.metop_dump_cases import chain_reference
        cadu, clear = chain_reference(name)
        tail = after_lock(cadu, clear)
        assert_pin(pin, "metop_dump_pins.json", ncadu=cadu.shape[0], tail=digest(tail))
    return pin["ncadu"], pin["ntail"], pin["tail"]


def same_as_reference(got, name, clear):
    """The reference's CADUs from the third transmitted one on (the first are read while the demodulator's loops acquire, on its float
    floor), and their message bytes are the transmitted ones"""
    from tests.common import match_frames
    n, ntail, tail_digest = chain_expected(name)
    tail = after_lock(got, clear)
    assert got.shape[0] == n and tail.shape[0] == ntail and digest(tail) == tail_digest
    i, _ = match_frames(tail[:1], clear)
    assert i is not None and np.array_equal(tail[:, :MSG], clear[i:i + tail.shape[0], :MSG])


@pytest.mark.parametrize("name", sorted(CHAIN))
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain(built, name, pipelined):
    """IQ -> psk_demod (QPSK, 35 Msym/s at 45 MS/s, pll_bw 0.03) -> metop_dump_decoder through the fused chain, in three pushes"""
    from satdump_b200 import capi
    from tests.common import demod_kwargs
    cfg, raw, clear = chain_signal(name)
    n = raw.size // 2
    got, fs = run_chain(capi.demod_cfg(max_batch=n, **demod_kwargs(cfg)), capi.fec_cfg_for(cfg, max_soft=4 * n), raw, cfg.fmt, pipelined)
    same_as_reference(got, name, clear)
    assert fs["correlator_lock"] == 1


@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli_metop_dump(built, tmp_path, mode):
    """b200_pipeline metop_dump (MetOp.json's psk_demod parameters, module id metop_dump_decoder): the .cadu file holds the reference's
    frames and the module reports lock_state"""
    name = "metop_dump_cs16"
    cfg, raw, clear = chain_signal(name)
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    r = run_cli("metop_dump", inp, hint, "--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16", fused=mode == "fused")
    assert "lock_state SYNCED" in r.stdout
    same_as_reference(np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024), name, clear)
