"""CPU: the checker of noaa_hrpt_decoder and meteor_hrpt_decoder. The compiled reference harness (oracle/_ref/libsatref_hrpt.so) equals
its committed pins on every test stream, its record-keeping single-byte calls change nothing against the module's 8192-byte reads, the
synthesised frames come out as sent, the numpy model of the GPU decomposition (tests/hrpt_model.py) equals the reference (or its pins) on
every case, and a missing deframer_thresold is refused by name."""
import numpy as np
import pytest

from oracle import hrpt as O
from tests.common import reference
from tests.hrpt_cases import METEOR, NOAA, boundary_cuts, digest, params, piece_cuts, pins, stats_rows, stream

CASES = [*NOAA, *METEOR]


def _same(r, pin):
    rows = stats_rows(r["stats"])
    assert r["recs"].tolist() == pin["recs"] and digest(r["out"]) == pin["out"] and r["out"].shape[0] == pin["units"]
    assert (rows if isinstance(pin["stats"], list) else digest(rows)) == pin["stats"]


@pytest.mark.parametrize("name", CASES)
def test_reference_equals_pins(name):
    reference(O)
    soft, cuts = stream(name)
    _same(O.run_pieces(soft, cuts, *params(name)), pins()["cases"][name])
    _same(O.run_pieces(soft, piece_cuts(soft.size, extra=boundary_cuts(name)), *params(name)), pins()["pieces"][name])


@pytest.mark.parametrize("name", CASES)
def test_record_keeping_changes_nothing(name):
    """One work() call per byte (to see each accepted sync) writes what the module's 8192-byte reads write"""
    reference(O)
    soft, _ = stream(name)
    a, b = O.Hrpt(*params(name)).run(soft), O.Hrpt(*params(name)).run(soft, records=False)
    assert np.array_equal(a["out"], b["out"]) and a["stats"] == b["stats"]


@pytest.mark.parametrize("meteor", [False, True])
def test_synthesised_frames_come_out_as_sent(meteor):
    reference(O)
    from satdump_b200 import synth
    bits, sent = (synth.meteor_hrpt_frames if meteor else synth.noaa_hrpt_frames)(12, seed=3)
    lead = np.random.default_rng(5).integers(0, 2, 1000).astype(np.uint8)
    r = O.Hrpt(meteor, 10).run(synth.hrpt_soft(np.concatenate([lead, bits.reshape(-1)]), inverted=True, sigma=10.0, seed=4))
    assert (r["recs"][:, 1] == 1).all()
    assert np.array_equal(r["out"].reshape(sent.shape), sent)


@pytest.mark.parametrize("name", CASES)
def test_model_equals_the_reference(name):
    """The numpy model of the GPU decomposition (candidate bitmap, frame-level walk, splice and mixed windows): pushed whole, the
    reference's records, output and stats; in pieces cut inside words, frames and syncs, the same records and output"""
    from tests import hrpt_model as M
    soft, cuts = stream(name)
    pin = pins()["cases"][name]
    _same(M.run_pieces(soft, cuts, *params(name)), pin)
    r = M.run_pieces(soft, piece_cuts(soft.size, sizes=(9, 777, 8191, 50000), extra=boundary_cuts(name)), *params(name))
    assert r["recs"].tolist() == pin["recs"] and digest(r["out"]) == pin["out"]


def test_missing_threshold_is_refused_by_name():
    from satdump_b200 import capi
    with pytest.raises(ValueError, match="deframer_thresold"):
        capi.noaa_hrpt_cfg()
