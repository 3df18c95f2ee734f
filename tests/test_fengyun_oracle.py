"""CPU: the fengyun_ahrpt_decoder checker (oracle/_ref, the reference's own blocks wired as the module) against its pins, the synthetic
FengYun-3 transmitter decoded by it to the frames that were sent (both invert_second_viterbi values), and the configuration's refusals."""
import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests import common
from tests import fengyun_cases as X

needs_ref = pytest.mark.skipif("not __import__('oracle.fengyun').fengyun.available()", reason="oracle/_ref not built (the pins stand in)")


@needs_ref
@pytest.mark.parametrize("name", X.CASES + X.LARGE)
def test_pins(name):
    assert X.reference(name) == common.load_pins(X.PINS)[name]


@needs_ref
@pytest.mark.parametrize("inv", [False, True])
def test_transmitter(inv):
    from oracle import fengyun
    i_bits, q_bits, clear = synth.fengyun_frames(40, seed=11)
    soft = synth.fengyun_soft(i_bits, q_bits, sigma=12.0, seed=5, invert_second=inv)
    soft = np.concatenate([np.zeros(2 * X.READ, np.int8), soft])
    soft = np.concatenate([soft, np.zeros((-soft.size) % X.READ, np.int8)])
    r = fengyun.Ref(X.OUTSYNC, X.BER, inv).run(soft)
    # every sent frame in order, but the first (the differential decoder's first pair follows the zeros in front) and the last (its
    # tail runs into the zero padding) may be lost
    got = [int(np.nonzero((clear == o).all(1))[0][0]) for o in r["out"] if (clear == o).all(1).any()]
    assert got[-38:] == list(range(1, 39)) and len(got) >= 38
    assert (r["recs"][-15:-1, 8] == 16).all()


def test_fengyun_diff_encode_inverts_work2():
    """the transmitter's differential encoder against a restatement of FengyunDiff::work2"""
    bits = np.random.default_rng(3).integers(0, 2, 4000).astype(np.uint8)
    x, y = synth.fengyun_diff_encode(bits)
    xp = yp = 0
    out = []
    for a, b in zip(x.tolist(), y.tolist()):
        if a != b:
            out += [yp ^ b, xp ^ a]
        else:
            out += [xp ^ a, yp ^ b]
        xp, yp = a, b
    assert np.array_equal(np.array(out, np.uint8), bits)


@pytest.mark.parametrize("missing", ["viterbi_outsync_after", "viterbi_ber_thresold", "invert_second_viterbi"])
def test_missing_parameter(missing):
    """each of the three is required, refused by name before a device is looked at"""
    kw = dict(viterbi_outsync_after=20, viterbi_ber_thresold=0.26, invert_second_viterbi=True)
    del kw[missing]
    with pytest.raises(ValueError, match=missing):
        capi.fengyun_ahrpt_cfg(**kw)
