"""CPU: the checkers of metop_dump_decoder. The C restatement (oracle/dump_port.c) equals the reference's own parts wired as the module
runs them (oracle/dump_harness.cpp) on records and CADU bytes, both equal the pins (tests/golden/metop_dump_pins.json), and synthesised
streams decode through the reference to the transmitted frames."""
import numpy as np
import pytest

from oracle import dump as O
from satdump_b200 import synth
from tests.common import reference
from tests.metop_dump_cases import CASES, F, digest, pins, stream


@pytest.mark.parametrize("name", sorted(CASES))
def test_pins_are_the_reference(name):
    reference(O)
    soft, _, _ = stream(CASES[name])
    r = O.Dump().run(soft)
    pin = pins()["cases"][name]
    assert r["recs"].tolist() == pin["recs"]
    assert r["cadu"].shape[0] == pin["ncadu"] and digest(r["cadu"]) == pin["cadu"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_the_reference(name):
    soft, _, _ = stream(CASES[name])
    p = O.Dump("port").run(soft)
    pin = pins()["cases"][name]
    assert p["recs"].tolist() == pin["recs"]
    assert p["cadu"].shape[0] == pin["ncadu"] and digest(p["cadu"]) == pin["cadu"]
    if O.available():
        r = O.Dump().run(soft)
        assert np.array_equal(p["recs"], r["recs"]) and np.array_equal(p["cadu"], r["cadu"])


def test_restatement_in_pieces():
    """The module loop continues across pushes: a frame whose shifted window is incomplete waits for the bytes behind it"""
    soft, _, _ = stream(CASES["shift_large"])
    whole = O.Dump("port").run(soft)
    cuts = [1, 8193, 2 * F + 1300, 3 * F + 6001, soft.size - 3]
    parts = O.run_pieces(soft, cuts, impl="port")
    assert np.array_equal(parts["recs"], whole["recs"]) and np.array_equal(parts["cadu"], whole["cadu"])


def test_cases_cover_the_quirks():
    """All 8 phase / swap results, shifts below and above F / 2, a window-tail winner, corrected and undecodable RS codewords"""
    recs = {name: np.array(p["recs"], np.int64).reshape(-1, 9) for name, p in pins()["cases"].items()}
    every = np.concatenate(list(recs.values()))
    assert {(int(a), int(b)) for a, b in every[:, 3:5]} == {(p, s) for p in range(4) for s in (0, 1)}
    pos = every[:, 1]
    assert ((pos > 0) & (pos < F // 2)).any() and ((pos > F // 2) & (pos < F - 32)).any()
    assert recs["tail_8162"][0, 1] == 8162 and recs["tail_8164"][0, 1] == 8164
    rs = recs["rs_errors"][:, 5:]
    assert (rs == 10).all(axis=1).any() and (rs == -1).all(axis=1).any()
    assert pins()["cases"]["rs_errors"]["ncadu"] == recs["rs_errors"].shape[0]  # undecodable frames are written too


@pytest.mark.parametrize("phase", range(4))
@pytest.mark.parametrize("swap", [False, True])
def test_synthesised_stream_decodes_to_the_transmitted_frames(phase, swap):
    """dump_frames + dump_soft: the reference writes the transmitted CADUs. Swapped streams at 0 and 180 degrees are the exception: the
    correlator's swapped syncwords at those phases stand for the other one of the two (DESIGN §9), so the reference writes every bit
    inverted (the complemented CCSDS RS codeword decodes too)."""
    impl = "ref" if O.available() else "port"
    tx, clear = synth.dump_frames(5, seed=40 + phase)
    soft = synth.dump_soft(tx, phase, swap, sigma=12.0, seed=phase)
    r = O.Dump(impl).run(soft)
    assert (r["recs"][:, 1] == 0).all() and (r["recs"][:, 5:] == 0).all()
    want = clear.copy()
    if swap and phase in (0, 2):
        want[:, 4:] ^= 0xFF
    assert np.array_equal(r["cadu"], want)


def test_signal_config():
    cfg = synth.CONFIGS["metop_dump"]
    assert (cfg.samplerate, cfg.symbolrate, cfg.constellation, cfg.pll_bw, cfg.rrc_alpha) == (45e6, 35e6, "qpsk", 0.03, 0.5)
    assert cfg.cadu_bytes == 1024 and abs(cfg.sps - 45 / 35) < 1e-6
