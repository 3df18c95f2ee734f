"""CPU: the checker of noaa_gac_decoder and dmsp_rtd_decoder. The PN sequence generated from its recurrence equals the reference's table
(entry 1022 included); the compiled reference harness (oracle/_ref/libsatref_gac.so) equals its committed pins on every case stream; the
synthesised frames come out of the reference as sent, forward and backward; the bit-serial model (tests/gac_model.py) equals the
reference (or its pins) on every case; the timestamp rule follows the reference's 8192-byte reads; a missing backward is refused."""
import numpy as np
import pytest

from oracle import gac as O
from satdump_b200 import capi, synth
from tests.common import reference
from tests import gac_cases as G
from tests import gac_model as M


def test_pn_table_equals_the_reference():
    pn = synth.gac_pn_bits()
    assert pn.size == 1023 and pn[1022] == 0
    assert G.digest(pn) == G.pins()["pn_table"]
    from oracle import gac as O
    if O.available():
        assert np.array_equal(O.pn_table(), pn)


def test_pn_recurrence_has_period_1023():
    b = list(synth.gac_pn_bits())
    for i in range(1023, 3 * 1023):
        b.append(b[i - 1] ^ b[i - 5] ^ b[i - 6] ^ b[i - 8] ^ b[i - 11])
    assert b[1023:2046] == b[:1023] and b[2046:] == b[:1023]


@pytest.mark.parametrize("name", G.CASES)
def test_reference_equals_pins(name):
    reference(O)
    dmsp, backward = G.params(name)
    r = O.Ref(dmsp, backward, G.START_TS if dmsp else -1.0).run(G.stream(name))
    pin = G.pins()["cases"][name]
    assert G.digest(r["out"]) == pin["out"] and r["out"].shape[0] == pin["frames"] and r["stats"]["state"] == pin["state"]
    assert G.ts_digest(r["ts"]) == pin["ts"]


@pytest.mark.parametrize("name", G.CASES)
def test_model_equals_the_reference(name):
    pin = G.ref_result(name)
    r = M.run(G.stream(name), *G.params(name))
    assert G.digest(r["out"]) == pin["out"] and r["out"].shape[0] == pin["frames"] and r["state"] == pin["state"]
    if G.is_dmsp(name):  # the completion bits give the reference's timestamps
        assert G.ts_digest(capi.dmsp_timestamps(r["done"], G.START_TS)) == pin["ts"]


@pytest.mark.parametrize("backward", [False, True])
def test_synthesised_gac_frames_come_out_as_sent(backward):
    reference(O)
    bits, sent = synth.gac_frames(13, seed=3, backward=backward)
    soft = synth.hrpt_soft(np.concatenate([np.zeros(999, np.uint8), bits.reshape(-1)]), inverted=True, sigma=10.0, seed=4)
    soft = np.concatenate([soft, np.zeros((-soft.size) % 8192, np.int8)])
    r = O.Ref(False, backward).run(soft)
    assert np.array_equal(r["out"], sent)


def test_synthesised_dmsp_frames_come_out_as_sent():
    reference(O)
    bits, sent = synth.dmsp_frames(500, seed=3)
    soft = synth.hrpt_soft(bits.reshape(-1), sigma=10.0, seed=4)
    soft = np.concatenate([soft, np.zeros((-soft.size) % 8192, np.int8)])
    assert np.array_equal(O.Ref(True).run(soft)["out"], sent)


def test_missing_backward_is_refused_by_name():
    with pytest.raises(ValueError, match="backward"):
        capi.noaa_gac_cfg()
