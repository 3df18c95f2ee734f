"""CPU: meteor_xband_decoder's decomposition (tests/xband_model.py) against the compiled reference module loop (oracle/_ref, else the pins
of tests/golden/meteor_xband_pins.json) on every case stream of both modes; synthesised streams decode to the sent frames in the
reference; the refusals (instrument_type, hard_symbols) name the option before any device is looked at."""
import numpy as np
import pytest

from oracle import xband
from satdump_b200 import capi, synth
from tests import xband_cases as X
from tests import xband_model as M
from tests.common import load_pins, reference

@pytest.mark.parametrize("name", X.CASES)
def test_model_equals_reference(name):
    out = M.run(X.stream(name), X.kind(name))
    pin = X.ref_result(name)
    assert out.shape[0] == pin["frames"] == pin["frame_count"] and X.digest(out) == pin["out"]


@pytest.mark.parametrize("name", X.CASES)
def test_pins_are_current(name):
    """the pins hold what the reference computes (they stand in for it where it is absent)"""
    pin = load_pins(X.PINS)[name]
    if xband.available():
        assert pin == X.reference(name)
    assert pin["frames"] == pin["frame_count"]


@pytest.mark.parametrize("kmss,cut", [(False, None), (False, (7, 200)), (True, None), (True, (1, 30000))])
def test_synthesised_streams_decode_to_the_sent_frames(kmss, cut):
    reference(xband)
    rng = np.random.default_rng(3)
    bits, sent = synth.meteor_xband_frames(kmss, 5 if kmss else 40, seed=11, cut=cut)
    bits = np.concatenate([[0], bits])  # (a clean first bit: the frame in the first record is then found too)
    soft = X._pad(np.concatenate([np.full(999, -60, np.int8), X._soft(bits, rng, 0.0)]), rng)
    got = xband.Ref(int(kmss)).run(soft)["out"]
    assert np.array_equal(got, sent)


def test_reference_in_pieces_equals_whole():
    """the harness decodes whole reads only, whatever the pieces"""
    reference(xband)
    soft = X.stream("kmss_all_deframers_one_read")
    r = xband.Ref(1)
    out = np.concatenate([r.run(soft[a:a + 100003])["out"] for a in range(0, soft.size, 100003)])
    assert X.digest(out) == X.ref_result("kmss_all_deframers_one_read")["out"]


def test_refusals_name_the_option():
    with pytest.raises(ValueError, match="Invalid METEOR instrument type!"):
        capi.meteor_xband_cfg("kmss_qpsk")
    with pytest.raises(ValueError, match="Invalid METEOR instrument type!"):
        capi.meteor_xband_cfg()
    cfg = capi.meteor_xband_cfg("mtvza")
    cfg.instrument_type = 2
    with pytest.raises(capi.B200Error, match="Invalid METEOR instrument type!"):  # before the device is looked at
        capi.Fec(cfg)
