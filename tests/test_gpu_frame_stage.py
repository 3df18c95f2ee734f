"""GPU: the frame stage (k_deframe, k_frames with the derandomiser and the warp Reed-Solomon decoder, the rs_usecheck filter) driven with
exact bytes. Noise-free +-100 BPSK soft bytes through ccsds_simple_psk_decoder hand the deframer exactly the designed bit stream; frames,
RS counters and the deframer state after every push must equal the oracle's, and the frames and counters must equal the plain models of
tests/rs_model.py (computed without the oracle)."""
import numpy as np
import pytest

from tests import frame_cases as FC
from tests import rs_model as M
from tests.common import oracle

pytestmark = pytest.mark.gpu
LEAD, TAIL = 3001, 17000  # the tail outlasts the largest CADU (16352 bits): cutting the stream to whole chunks keeps every frame


def run_gpu(cfg_kw, soft, cuts=None):
    """Pushes soft (in pieces ending at cuts) through a simple PSK decoder. Returns (frames, stats, deframer state after each push)."""
    from satdump_b200 import capi
    g = capi.Fec(capi.simple_cfg("bpsk", max_soft=max(soft.size + 65536, 1 << 20), **cfg_kw))
    frames, states, prev = [], [], 0
    for c in (cuts or [soft.size]):
        frames.append(g.push(soft[prev:c]).frames())
        states.append(g.stats()["deframer_state"])
        prev = c
    return np.concatenate(frames), g.stats(), states, g.chunk


def check(cfg_kw, bits, model_frames, model_counts, cuts=None):
    """GPU vs oracle (frames, counters, deframer state per push) and vs the model (frames, counters)."""
    O = oracle()
    C = cfg_kw["cadu_size"]
    bits = bits[:bits.size // C * C]
    soft = FC.soft_of(bits)
    want = O.Fec(O.simple_cfg("bpsk", **cfg_kw)).run(soft)
    got, s, states, chunk = run_gpu(cfg_kw, soft, cuts)
    assert chunk == C
    assert np.array_equal(got.reshape(-1), want["cadu"])
    assert np.array_equal(got, model_frames)
    e = want["rs_err"]
    assert s["rs_corrected"] == int(e[e >= 0].sum()) == int(model_counts[model_counts >= 0].sum())
    assert s["rs_failed"] == int((e < 0).sum()) == int((model_counts < 0).sum())
    ends = [c // C for c in (cuts or [soft.size])]
    assert states == [int(want["defr_state"][k - 1]) if k else 2 for k in ends]
    return want


def model_stage(bits, rx, I, dual=True, rs_type=0, rs_usecheck=False):
    """The model's prediction: the deframer model on the bits (cut to whole chunks), then the frame stage model. The designed CADUs
    must be the first frames it finds (random tail bits may pass one more SYNCED test)."""
    C = rx.shape[1] * 8
    dfr = M.deframe(bits[:bits.size // C * C], C)["frames"]
    assert dfr.shape[0] >= rx.shape[0] and np.array_equal(dfr[:rx.shape[0]], rx)
    return M.frame_stage(dfr, I, dual, rs_type, rs_usecheck=rs_usecheck)


def rs_stream(rs_type, dual, I, seed, positions=True, derand=True):
    """CADUs of the designed codewords (ASM + interleaved words, randomised from byte 4), their bits with a lead-in and a tail, and the
    CADUs as the deframer hands them over (pre-derandomiser)."""
    c = FC.codeword_cases(rs_type, dual, I, seed, positions)
    nf = c["rx"].shape[0]
    asm = np.tile(np.frombuffer(M.SYNC.to_bytes(4, "big"), np.uint8), (nf, 1))
    rx = np.concatenate([asm, c["rx"]], axis=1)
    if derand:
        rx[:, 4:] ^= FC.synth.ccsds_pn(255 * I)[None, :]
    return c, rx, FC.cadu_stream(rx, LEAD, TAIL, seed)


SWEEP = [(rs_type, dual, I) for rs_type in (0, 1) for dual in (True, False) for I in range(1, 9)]


@pytest.mark.parametrize("rs_type,dual,I", SWEEP)
def test_rs_sweep(built, rs_type, dual, I):
    """Every code, basis and interleave depth: one error at each codeword position, 0 .. t+2 errors, parity-only errors, the designed
    miscorrection. With rs_usecheck the surviving frames carry the per-frame verdicts."""
    c, rx, bits = rs_stream(rs_type, dual, I, seed=1000 + 100 * rs_type + 10 * I + int(dual))
    C = rx.shape[1] * 8
    kw = dict(cadu_size=C, rs_i=I, rs_type=rs_type, rs_dualbasis=dual)
    mf, counts, kept = model_stage(bits, rx, I, dual, rs_type)
    # the model's verdicts are the designed ones, and the paths are reached: failures at t+1, moved bytes for the miscorrections
    m, cd = c["want_count"] > -2, counts[:c["kind"].shape[0]]
    assert np.array_equal(cd[m], c["want_count"][m])
    t = FC.t_of(rs_type)
    assert (cd[c["kind"] == f"n{t + 1}"] == -1).any() and (cd[c["kind"] == "mis"] > 0).all()
    check(kw, bits, mf, counts)
    uf, ucounts, ukept = model_stage(bits, rx, I, dual, rs_type, rs_usecheck=True)
    assert 0 < ukept.sum() < ukept.size
    check(dict(kw, rs_usecheck=True), bits, uf, ucounts)


SHIPPED = [(0, 1, False), (0, 4, False), (0, 5, False), (1, 4, False), (1, 5, False), (1, 8, False), (0, 1, True), (0, 5, True)]


@pytest.mark.parametrize("rs_type,I,usecheck", SHIPPED)
def test_shipped_configurations_ragged(built, rs_type, I, usecheck):
    """The shipped RS configurations with byte errors, in one push and in pushes of one chunk each (every push ends 13 bits into an
    ASM: the lead-in is chosen so) and of ragged sizes."""
    c, rx, _ = rs_stream(rs_type, True, I, seed=2000 + 10 * I + rs_type, positions=False)
    C = rx.shape[1] * 8
    bits = FC.cadu_stream(rx, 3 * C - 13, TAIL, 7)
    kw = dict(cadu_size=C, rs_i=I, rs_type=rs_type, rs_usecheck=usecheck)
    mf, counts, kept = model_stage(bits, rx, I, True, rs_type, rs_usecheck=usecheck)
    assert (counts > 0).any() and (counts < 0).any()
    if usecheck:  # the filter drops the frames with a failed word
        assert 0 < kept.sum() < kept.size
    n = bits.size // C * C
    check(kw, bits, mf, counts)
    check(kw, bits, mf, counts, cuts=list(range(C, n + 1, C)))
    check(kw, bits, mf, counts, cuts=[5001, 5001 + 3 * C + 1, n // 2 + 7, n])


@pytest.mark.parametrize("rs_type,I,extra", FC.SPARE)
def test_spare_bytes_after_the_codewords(built, rs_type, I, extra):
    """CADUs longer than 4 + 255*I: the first I spare bytes carry the row past the codewords that the reference decodes with
    rs_fill_bytes -1 (the corrected first message byte of each word that decodes, the byte as received otherwise), the others come out
    as received. With rs_fill_bytes 0 there is no such row and every spare byte comes out as received."""
    c, cadus = FC.spare_cadus(rs_type, I, extra, seed=60 + I)
    C = cadus.shape[1] * 8
    bits = FC.cadu_stream(cadus, LEAD, TAIL, 9)
    kw = dict(cadu_size=C, rs_i=I, rs_type=rs_type)
    mf, counts, _ = model_stage(bits, cadus, I, True, rs_type)
    J = min(I, extra)  # spare bytes that hold the row past the codewords
    ok = counts[:cadus.shape[0], :J] >= 0
    assert ok.any() and (~ok).any()
    clear_tail = cadus[:, 4 + 255 * I:] ^ FC.synth.ccsds_pn(C // 8 - 4)[255 * I:]
    assert np.array_equal(mf[:cadus.shape[0], 4 + 255 * I + J:], clear_tail[:, J:])
    assert not np.array_equal(mf[:cadus.shape[0], 4 + 255 * I:4 + 255 * I + J][ok], clear_tail[:, :J][ok])
    check(kw, bits, mf, counts)
    dfr = M.deframe(bits[:bits.size // C * C], C)["frames"]
    f0, counts0, _ = M.frame_stage(dfr, I, True, rs_type, row256=False)
    assert np.array_equal(f0[:cadus.shape[0], 4 + 255 * I:], clear_tail)
    check(dict(kw, rs_fill_bytes=0), bits, f0, counts0)


def test_eos_db_configuration(built):
    """The Terra / Aqua / Aura DB decoder of the shipped pipelines: ccsds_conv_concat_decoder (plain BPSK here), NRZ-M, RS(255,223) I=4,
    the derandomiser after RS from byte 10. Noise-free +-60 soft bytes of the r=1/2 code hand the frame stage the designed bytes: frames
    equal the oracle's and the model's, and the designed byte errors are corrected before the derandomiser runs."""
    from satdump_b200 import capi
    I, C, nf = 4, 8192, 40
    rng = np.random.default_rng(31)
    pay = rng.integers(0, 256, (nf, 223 * I), dtype=np.uint8)
    tx, _ = FC.synth.build_cadus(pay, I, randomize=False)  # sent as encoded: the receiver derandomises after RS
    for f in range(6, nf, 3):
        tx[f, 4 + rng.choice(255 * I, 6 * I, replace=False)] ^= rng.integers(1, 256, 6 * I, dtype=np.uint8)
    tx[nf - 5, 4 + rng.choice(255, 17, replace=False) * I + 1] ^= 0x3C  # t+1 errors in one word
    bits = FC.synth.nrzm_encode(np.unpackbits(tx.reshape(-1)))
    soft = np.where(FC.synth.conv_encode(bits) > 0, 60, -60).astype(np.int8)
    soft = soft[:soft.size // 8192 * 8192]
    kw = dict(rs_i=I, nrzm=True, derand_after_rs=True, derand_start=10)
    O = oracle()
    want = O.Fec(O.ccsds_cfg("bpsk", C, 0.3, 20, **kw)).run(soft)
    g = capi.Fec(capi.ccsds_cfg("bpsk", C, 0.3, 20, max_soft=soft.size, **kw))
    got = g.push(soft).frames()
    s = g.stats()
    assert np.array_equal(got.reshape(-1), want["cadu"])
    mf, counts, _ = M.frame_stage(tx, I, derand_after_rs=True, derand_start=10)
    i0 = next(i for i in range(nf) if np.array_equal(mf[i], got[0]))
    k = got.shape[0]
    assert k >= nf - 8 and np.array_equal(got, mf[i0:i0 + k])
    e = want["rs_err"]
    assert s["rs_corrected"] == int(e[e >= 0].sum()) == int(counts[i0:i0 + k][counts[i0:i0 + k] >= 0].sum()) > 0
    assert s["rs_failed"] == int((e < 0).sum()) == int((counts[i0:i0 + k] < 0).sum()) == 1
    assert s["deframer_state"] == int(want["defr_state"][-1])


def test_large_push_grid_stride_and_filter_rounds(built):
    """One push of 2200 CADUs (RS(255,223) I=4, rs_usecheck): k_frames runs its grid-stride loop (grid 1056) and k_frames_filter carries
    its scan over three 1024-frame rounds. Failing frames sit at the loop and round edges."""
    nf, I, C = 2200, 4, 8192
    fail = [0, 1023, 1024, 1055, 1056, 2047, 2048, nf - 1]
    rng = np.random.default_rng(77)
    pay = rng.integers(0, 256, (nf, 223 * I), dtype=np.uint8)
    tx, _ = FC.synth.build_cadus(pay, I)
    for f in fail:
        pos = 4 + rng.choice(255, 17, replace=False) * I + rng.integers(0, I)  # t+1 errors in one word
        tx[f, pos] ^= rng.integers(1, 256, 17, dtype=np.uint8)
    for f in range(5, nf, 97):  # and corrections elsewhere
        tx[f, 4 + rng.choice(1020, 20, replace=False)] ^= 0x5A
    bits = FC.cadu_stream(tx, LEAD, TAIL, 3)
    kw = dict(cadu_size=C, rs_i=I, rs_usecheck=True)
    mf, counts, kept = model_stage(bits, tx, I, rs_usecheck=True)
    assert sorted(np.nonzero(~kept[:nf])[0].tolist()) == fail and (counts > 0).sum() > 20
    want = check(kw, bits, mf, counts)
    assert want["nframes"] >= nf > 1056


@pytest.mark.parametrize("name,kw,synced", [c for c in FC.deframer_cases() if c[2] == 12], ids=lambda v: v if isinstance(v, str) else "")
@pytest.mark.parametrize("lead", FC.DEFRAMER_LEADS)
def test_deframer_edges(built, name, kw, synced, lead):
    """SYNCING at 5 / 6 ASM bit errors, SYNCED at 11 / 12, slips of 1 / 2 / 3 bits, a polarity flip, the first failing ASM at lookahead
    127 / 128 / 129 / 256 of the SYNCED walk: frames and the state after every chunk equal the oracle's and the model's. Pushed whole, one
    chunk per push (each ending 13 bits into an ASM, or 513 bits into a frame) and in ragged pieces."""
    C = FC.DEFRAMER_CADU
    bits, ends, bodies = FC.deframer_stream(cadu_size=C, lead=lead, seed=sum(map(ord, name)), **kw)
    bits = bits[:bits.size // C * C]
    n = bits.size
    m = M.deframe(bits, C, synced, checkpoints=range(C, n + 1, C))
    FC.check_deframer_path(name, m, ends, bodies, synced)
    cfg = dict(cadu_size=C, rs_i=0, derandomize=False)
    want = check(cfg, bits, m["frames"], np.zeros(0, np.int64))
    assert np.array_equal(want["defr_state"], m["states"])
    check(cfg, bits, m["frames"], np.zeros(0, np.int64), cuts=list(range(C, n + 1, C)))
    check(cfg, bits, m["frames"], np.zeros(0, np.int64), cuts=[777, 777 + 5 * C, n // 3, n // 3 + 1, n])
