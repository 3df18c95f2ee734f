"""CPU: the checker of meteor_lrpt_decoder. The compiled reference harness (oracle/_ref/libsatref_meteor.so) equals its committed pins on
every test stream, the synthesised LRPT frames decode to the transmitted ones, m2x_mode is exactly ccsds_conv_concat_decoder's OQPSK
configuration, and the decoder's refusals name their option before a device is touched."""
import numpy as np
import pytest

from oracle import meteor as O
from tests.common import reference
from tests.meteor_lrpt_cases import CASES, M2X, M2X_PARAMS, PIECES, digest, piece_cuts, pins, stream


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_equals_pins(name):
    reference(O)
    case = CASES[name]
    soft, _, cuts = stream(case)
    r = O.run_pieces(soft, cuts, case.get("diff", False))
    pin = pins()["cases"][name]
    assert r["recs"].tolist() == pin["recs"] and digest(r["cadu"]) == pin["cadu"] and r["stats"] == pin["stats"]


@pytest.mark.parametrize("name", PIECES)
def test_reference_in_pieces_equals_pins(name):
    reference(O)
    case = CASES[name]
    soft, _, _ = stream(case)
    r = O.run_pieces(soft, piece_cuts(soft.size), case.get("diff", False))
    pin = pins()["pieces"][name]
    assert r["recs"].tolist() == pin["recs"] and digest(r["cadu"]) == pin["cadu"] and r["stats"] == pin["stats"]
    whole = pins()["cases"][name]
    assert pin["recs"] == whole["recs"] and pin["cadu"] == whole["cadu"]  # pushing in pieces changes nothing but the stats' timing


@pytest.mark.parametrize("diff", [False, True])
def test_synthesised_frames_decode_to_the_transmitted_ones(diff):
    """The LRPT transmitter (synth.lrpt_frames / lrpt_soft) against the reference: without NRZ-M every frame, the inverted one included.
    With NRZ-M the transmitted ASM is the syncword or its complement, depending on the parity before it; the correlator then also finds
    the table's IQ-swapped entries, whose frames the Viterbi decoder cannot decode and RS drops, so the frames written are transmitted ones,
    in order."""
    reference(O)
    from satdump_b200 import synth
    coded, written = synth.lrpt_frames(10, seed=5, nrzm=diff, inverted=(4,))
    r = O.Meteor(diff).run(synth.lrpt_soft(coded, sigma=25.0, seed=6))
    assert (r["recs"][:, 1] == 0).all() and r["recs"].shape[0] == 10
    if not diff:
        assert np.array_equal(r["cadu"], written)
    else:
        ok = [k for k in range(10) if (r["recs"][k, 5:9] >= 0).all()]
        assert len(ok) >= 5 and np.array_equal(r["cadu"], written[ok])


@pytest.mark.parametrize("name", sorted(M2X))
def test_m2x_mode_is_the_conv_concat_oqpsk_configuration(name):
    """module_meteor_lrpt_decoder.cpp:103-197 against ccsds_conv_concat_decoder (constellation oqpsk, cadu_size 8192, nrzm = diff_decode,
    rs_i 4, rs_dualbasis false, rs_usecheck): the same frames are written and the stats agree, so the decoder runs m2x_mode as that
    configuration. The stats keys are the same in both modules (deframer_lock, viterbi_ber, viterbi_lock, rs_avg, viterbi_state,
    deframer_state)."""
    reference(O)
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    case = M2X[name]
    soft, _, _ = stream(case)
    m = O.MeteorM2x(case.get("diff", False), M2X_PARAMS["viterbi_ber_thresold"], M2X_PARAMS["viterbi_outsync_after"]).run(soft)
    c = ref.Fec(ref.ccsds_cfg("oqpsk", 8192, M2X_PARAMS["viterbi_ber_thresold"], M2X_PARAMS["viterbi_outsync_after"], 4,
                              nrzm=case.get("diff", False), rs_usecheck=True, rs_dualbasis=False)).run(soft)
    assert m["cadu"].shape[0] > 5 and np.array_equal(m["cadu"].reshape(-1), c["cadu"])
    assert m["stats"]["deframer_state"] == int(c["defr_state"][-1]) and m["stats"]["viterbi_lock"] == int(c["vit_state"][-1])
    assert np.array([m["stats"]["viterbi_ber"]], np.uint32).view(np.float32)[0] == c["vit_ber"][-1]
    pin = pins()["m2x"][name]
    assert digest(m["cadu"]) == pin["cadu"] and m["stats"] == pin["stats"]


def test_refusals_name_their_option(built):
    """diff_decode is required, the Viterbi parameters are required with m2x_mode, and interleaved is refused as not built; all before a
    device is touched (this machine may have none)"""
    from satdump_b200 import capi
    with pytest.raises(ValueError, match="diff_decode"):
        capi.meteor_lrpt_cfg()
    with pytest.raises(ValueError, match="viterbi_outsync_after"):
        capi.meteor_lrpt_cfg(False, m2x_mode=True, viterbi_ber_thresold=0.3)
    with pytest.raises(ValueError, match="viterbi_ber_thresold"):
        capi.meteor_lrpt_cfg(False, m2x_mode=True, viterbi_outsync_after=20)
    with pytest.raises(capi.B200Error) as e:
        capi.Fec(capi.meteor_lrpt_cfg(True, m2x_mode=True, interleaved=True, **M2X_PARAMS))
    assert "interleaved" in str(e.value) and "not built" in str(e.value) and "never delivers a sample" in str(e.value)
