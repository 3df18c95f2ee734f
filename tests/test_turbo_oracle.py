"""CPU: the checker of ccsds_turbo_decoder and the parts of it that need no GPU. The synthetic encoder (satdump_b200.synth, written from the
CCSDS standard) equals the reference's CCSDSTurbo::encode for every rate and base, the interleaver is the reference's, the pinned reference
results (tests/golden/turbo_pins.json) are what the reference computes and the transmitted frames of clean streams, glibc's pow(x, 2) is
x * x on every value the decoder squares, and the decoder's refusals name their option."""
import ctypes
import ctypes.util

import numpy as np
import pytest

from satdump_b200 import synth
from tests.common import reference
from tests.turbo_cases import CASES, RATE_NAME, digest, encoder_info, frame_size, pins, stream


def _ref():
    from oracle import turbo as O
    return O if O.available() else None


@pytest.mark.parametrize("base", synth.TURBO_BASES)
def test_interleaver(base):
    pi = synth.turbo_interleaver(base).astype(np.int32)
    assert np.array_equal(np.sort(pi), np.arange(8 * base))
    assert digest(pi) == pins()["perm"][str(base)]
    O = _ref()
    if O:
        assert np.array_equal(O.perm(base), pi)


@pytest.mark.parametrize("rate", [2, 3, 4, 6])
@pytest.mark.parametrize("base", synth.TURBO_BASES)
def test_encoder_equals_reference(rate, base):
    bits = synth.turbo_encode(encoder_info(rate, base)[None], rate)[0]
    assert bits.size == synth.turbo_codeword_bits(rate, base)
    assert digest(bits.astype(np.uint8)) == pins()["encode"][f"{rate}_{base}"]
    O = _ref()
    if O:
        assert np.array_equal(O.encode(RATE_NAME[rate], base, encoder_info(rate, base)), bits)


def test_crc_matches_frame_layout():
    _, cadu = synth.turbo_frames(3, 2, 223, seed=4)
    assert (cadu[:, :4] == [0x1A, 0xCF, 0xFC, 0x1D]).all()
    crc = synth.crc16_ccitt(cadu[:, 4:-2])
    assert np.array_equal(crc, cadu[:, -2].astype(np.uint32) << 8 | cadu[:, -1])
    assert synth.crc16_ccitt(np.frombuffer(b"123456789", np.uint8))[0] == 0x29B1  # CRC-16/CCITT-FALSE check value


@pytest.mark.parametrize("name", ["combo_2_223", "combo_6_223", "swapped", "noise_signal_noise", "crc_failures"])
def test_pins_are_the_reference(name):
    """Where the reference was built, it reproduces the pinned records and CADUs."""
    from oracle import turbo
    O = reference(turbo)
    case = CASES[name]
    soft, _, _ = stream(case)
    r = O.Turbo(RATE_NAME[case["rate"]], case["base"], case["iters"]).run(soft)
    pin = pins()["cases"][name]
    assert r["recs"].tolist() == pin["recs"] and digest(r["cadu"]) == pin["cadu"]


@pytest.mark.parametrize("name", ["swapped", "noise_signal_noise", "ragged", "inserted_deleted"])
def test_pinned_frames_are_the_transmitted_ones(name):
    """On the low-noise streams every frame read at its place (pos 0) passes its CRC and the written CADUs are the transmitted ones, in
    order. A frame read after a shift by 0 < pos <= F / 2 keeps F - 2 pos stale bytes in its middle and fails; after a shift by pos > F / 2
    the new bytes overwrite everything the memmove wrote past the buffer, so the frame is whole and passes."""
    case = CASES[name]
    _, clear, _ = stream(case)
    pin = pins()["cases"][name]
    recs = np.array(pin["recs"], np.int64).reshape(-1, 6)
    F = frame_size(case["rate"], case["base"])
    whole = (recs[:, 1] == 0) | (recs[:, 1] > F // 2)
    assert (recs[~whole, 4] == 0).all() and (recs[recs[:, 1] > F // 2, 4] == 1).all()
    if case.get("edit") != "insdel":  # (there the frame with the inserted bytes fails at pos 0)
        assert (recs[whole, 4] == 1).all()
    ok = int(recs[:, 4].sum())
    assert ok == pin["ncadu"] and ok >= 3
    starts = [i for i in range(clear.shape[0] - ok + 1) if digest(clear[i:i + ok]) == pin["cadu"]]
    if case.get("edit") is None:
        assert starts, "the written CADUs should be consecutive transmitted frames"


def test_pow_square_is_the_product():
    """The decoder computes pow(rho - (2 out - 1), 2) as a product. rho is (double)(+-(float)v / 127) for an int8 v, or 0 where rate 1/2
    is punctured: glibc's pow(x, 2) equals x * x on every such x."""
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.pow.restype, libm.pow.argtypes = ctypes.c_double, [ctypes.c_double, ctypes.c_double]
    v = np.arange(-128, 128, dtype=np.float32)
    rho = np.concatenate([v / np.float32(127), -(v / np.float32(127)), [0.0]]).astype(np.float64)
    xs = np.concatenate([rho - 1.0, rho + 1.0])
    bad = [x for x in xs if libm.pow(float(x), 2.0) != float(x) * float(x)]
    assert not bad, bad[:5]


@pytest.mark.parametrize("kw,text", [(dict(turbo_rate=5, turbo_base=223, turbo_iters=1), "Invalid Turbo Rate"),
                                     (dict(turbo_rate="1/5", turbo_base=223, turbo_iters=1), "Invalid Turbo Rate"),
                                     (dict(turbo_rate="1/2", turbo_base=224, turbo_iters=1), "Turbo Base must be 223, 446, 892 or 1115"),
                                     (dict(turbo_rate="1/2", turbo_base=223, turbo_iters=0), "turbo_iters 0"),
                                     (dict(turbo_rate="1/2", turbo_base=223, turbo_iters=-3), "turbo_iters -3")])
def test_refusals_name_the_option(built, kw, text):
    """Refused before the device is checked, so the text is the same with and without a GPU."""
    from satdump_b200 import capi
    with pytest.raises(capi.B200Error) as e:
        capi.Fec(capi.turbo_cfg(**kw))
    assert text in str(e.value) and e.value.code == -1


@pytest.mark.parametrize("missing,text", [("turbo_rate", "Turbo Rate is required!"), ("turbo_base", "Turbo Base is required!"),
                                          ("turbo_iters", "Turbo Iters is required!")])
def test_missing_parameters(missing, text):
    from satdump_b200 import capi
    kw = dict(turbo_rate="1/2", turbo_base=223, turbo_iters=1)
    del kw[missing]
    with pytest.raises(ValueError, match=text):
        capi.turbo_cfg(**kw)


@pytest.mark.parametrize("name", ["llr_2_223", "llr_6_223"])
def test_llr_golden_is_the_reference(name):
    """tests/golden/turbo_llr.npz holds what the reference's convcode_extrinsic computes, bit for bit, for the frames of the LLR cases."""
    from tests.turbo_cases import LLR, llr_frames, reference_llr
    from oracle import turbo
    reference(turbo)
    case = CASES[name]
    gold = np.load(LLR)
    frames = llr_frames(name)
    assert len(frames) == 2
    for k, up, lo in frames:
        a0, a1 = reference_llr(case["rate"], case["base"], case["iters"], up, lo)
        assert np.array_equal(a0.view(np.uint64), gold[f"{name}_{k}_0"].view(np.uint64))
        assert np.array_equal(a1.view(np.uint64), gold[f"{name}_{k}_1"].view(np.uint64))


def _port():
    from oracle import turbo as O
    if not O.available("port"):
        import __graft_entry__ as g
        g.build()
    return O


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_reproduces_the_reference(name):
    """oracle/turbo_port.c (the module loop, correlator, shift quirk, derandomiser, BCJR and CRC restated in C) writes the reference's
    records and CADUs bit for bit on every stream: noisy, shifted (pos > F / 2 included), swapped, 1 to 50 iterations."""
    O = _port()
    case = CASES[name]
    soft, _, _ = stream(case)
    r = O.Turbo(RATE_NAME[case["rate"]], case["base"], case["iters"], impl="port").run(soft)
    pin = pins()["cases"][name]
    assert r["recs"].tolist() == pin["recs"] and digest(r["cadu"]) == pin["cadu"]


@pytest.mark.parametrize("name", ["llr_2_223", "llr_6_223"])
def test_restatement_extrinsic_arrays_bitwise(name):
    """The restatement's a-priori arrays after every half-iteration equal the reference's convcode_extrinsic bit for bit (same host libm),
    and after the last iteration they equal tests/golden/turbo_llr.npz."""
    from tests.turbo_cases import LLR, llr_frames
    O = _port()
    case = CASES[name]
    rate, base = RATE_NAME[case["rate"]], case["base"]
    pi = synth.turbo_interleaver(base)
    gold = np.load(LLR)
    bits = lambda a: np.asarray(a).view(np.uint64)  # noqa: E731
    for k, up, lo in llr_frames(name):
        m0, m1 = np.full(8 * base, np.log(0.5)), np.full(8 * base, np.log(0.5))
        for it in range(case["iters"]):
            last = it == case["iters"] - 1
            p0, p1, _ = O.half(rate, base, 0, up, m0, m1, impl="port")
            if _ref():
                r0, r1, _ = O.half(rate, base, 0, up, m0, m1)
                assert np.array_equal(bits(p0), bits(r0)) and np.array_equal(bits(p1), bits(r1))
            q0, q1, pd = O.half(rate, base, 1, lo, p0[pi], p1[pi], decision=last, impl="port")
            if _ref():
                r0, r1, rd = O.half(rate, base, 1, lo, p0[pi], p1[pi], decision=last)
                assert np.array_equal(bits(q0), bits(r0)) and np.array_equal(bits(q1), bits(r1))
                assert not last or np.array_equal(pd, rd)
            m0, m1 = np.empty(8 * base), np.empty(8 * base)
            m0[pi], m1[pi] = q0, q1
        assert np.array_equal(bits(m0), bits(gold[f"{name}_{k}_0"])) and np.array_equal(bits(m1), bits(gold[f"{name}_{k}_1"]))


@pytest.mark.parametrize("base", synth.TURBO_BASES)
def test_restatement_interleaver(base):
    assert np.array_equal(_port().perm(base, impl="port"), synth.turbo_interleaver(base))
