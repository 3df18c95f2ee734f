"""CPU: the frame stage models (tests/rs_model.py) against the C restatement (oracle/port) and the reference (oracle/_ref, or its committed
results through tests/refpin.py): the Reed-Solomon decode of every shipped code, basis and interleave depth on designed error patterns,
the locator invariants the warp decoder relies on, and the deframer on designed bit streams."""
import numpy as np
import pytest

from tests import frame_cases as FC
from tests import rs_model as M
from tests.refpin import Pin

RS_CASES = [(rs_type, dual, I) for rs_type in (0, 1) for dual in (True, False) for I in (1, 2, 3, 4, 5, 8)]


@pytest.mark.parametrize("rs_type,dual,I", RS_CASES)
def test_rs_model_equals_restatement_and_reference(built, rs_type, dual, I):
    """One error at each of the 255 codeword positions, 0 / 1 / t-1 / t / t+1 / t+2 random errors, t errors in the parity bytes only, and
    the designed miscorrection: bytes and return codes of the model, the restatement and the reference agree, and the designed outcomes
    hold."""
    from oracle import port
    pin = Pin(f"rs_model[{rs_type}-{int(dual)}-{I}]")
    c = FC.codeword_cases(rs_type, dual, I, seed=100 * rs_type + 10 * I + int(dual))
    got, cnt, info = M.rs_decode_interleaved(c["rx"], dual, I, rs_type)
    pb = [port.rs_decode_interleaved(r, dual, I, rs_type) for r in c["rx"]]
    pd, pe = np.array([d for d, _ in pb]), np.array([e for _, e in pb])
    assert np.array_equal(got, pd) and np.array_equal(cnt, pe)
    ra = pin.run(lambda R: [R.rs_decode_interleaved(r, dual, I, rs_type) for r in c["rx"]])
    pin.equal("bytes", ra and np.array([d for d, _ in ra]), pd)
    pin.equal("counts", ra and np.array([e for _, e in ra]).astype(np.int32), pe.astype(np.int32))
    # designed outcomes: every position located, parity left as received, the miscorrection lands on c + w
    t = FC.t_of(rs_type)
    m = c["want_count"] > -2
    assert np.array_equal(cnt[m], c["want_count"][m])
    whole = m.all(axis=1)
    assert np.array_equal(got[whole], c["want"][whole])
    kind = c["kind"]
    assert (cnt[kind == "mis"] > 0).all() and (cnt[kind == "parity"] == 0).all()
    assert (cnt[kind == f"n{t + 1}"] == -1).any() and (cnt[kind == f"n{t + 2}"] == -1).any()
    # the path each word took: L = order = number of roots = errors for the corrected words
    L, order, roots = (info[k].reshape(kind.shape) for k in ("L", "order", "roots"))
    for k in [f"n{n}" for n in (1, t - 1, t)] + ["parity", "mis"]:
        want = {"parity": t, "mis": t}.get(k, int(k[1:]) if k.startswith("n") else 0)
        sel = kind == k
        assert (L[sel] == want).all() and (order[sel] == want).all() and (roots[sel] == want).all(), k
    assert (L[np.char.startswith(kind, "pos")] == 1).all()


@pytest.mark.parametrize("rs_type", [0, 1])
def test_locator_order_equals_bm_length(rs_type):
    """Over random syndrome vectors (every syndrome vector is reached by some received word): libcorrect's locator order equals the
    Berlekamp-Massey length L <= nroots, and a word the decoder accepts has L <= t. The warp decoder gives one lane to each root and to
    each derivative coefficient (lane < order, 32 lanes), which needs exactly this."""
    nroots, _ = M.params(rs_type)
    t = nroots // 2
    rng = np.random.default_rng(20 + rs_type)
    S = rng.integers(0, 256, (60000, nroots), dtype=np.int64)
    S[:200] = 0
    S[200:400, ::2] = 0
    lam, L, order = M.berlekamp_massey(S)
    assert (order == L).all() and (L <= nroots).all()
    assert (L == 0).sum() == 200 and (L == t).sum() > 30000 and (L > t).sum() > 100
    # acceptance (roots == order) only where L <= t
    big = np.nonzero(L > t)[0]
    for a in range(0, big.size, 8192):
        rows = big[a:a + 8192]
        roots = (M.poly_eval_all(lam[rows]) == 0).sum(axis=1)
        assert (roots != order[rows]).all()


@pytest.mark.parametrize("rs_type,I,extra", FC.SPARE)
def test_row_past_the_codewords(built, rs_type, I, extra):
    """With rs_fill_bytes -1 the reference decodes one row past the interleaved codewords: in a CADU longer than 4 + 255*I, spare byte b
    comes out as the corrected first message byte of word b when it decodes and as received when it does not, the later spare bytes as
    received. The model, the restatement and the reference agree through the simple PSK decoder."""
    from oracle import port
    pin = Pin(f"rs_row256[{rs_type}-{I}-{extra}]")
    c, cadus = FC.spare_cadus(rs_type, I, extra, seed=40 + I)
    C = cadus.shape[1] * 8
    bits = FC.cadu_stream(cadus, 3001, C + 100, 5)
    soft = FC.soft_of(bits[:bits.size // C * C])
    cfg = port.simple_cfg("bpsk", C, I, rs_type=rs_type)
    b = port.Fec(cfg).run(soft)
    fr = b["cadu"].reshape(-1, C // 8)[:cadus.shape[0]]
    mf, counts, _ = M.frame_stage(cadus, I, True, rs_type)
    assert np.array_equal(fr, mf) and (counts == -1).any() and (counts >= 0).any()
    pn = FC.synth.ccsds_pn(C // 8 - 4)
    clear_tail, J = cadus[:, 4 + 255 * I:] ^ pn[255 * I:], min(I, extra)
    assert np.array_equal(fr[:, 4 + 255 * I + J:], clear_tail[:, J:])                            # later spare bytes: as received
    bad = counts[:, :J] < 0
    assert bad.any() and np.array_equal(fr[:, 4 + 255 * I:4 + 255 * I + J][bad], clear_tail[:, :J][bad])
    for k in ("cadu", "rs_err"):
        pin.equal(k, pin.run(lambda R: R.Fec(cfg).run(soft)[k]), b[k])


def test_row_past_the_codewords_reaches_the_next_frame(built):
    """When the CADU ends with the codewords, the extra row is the first bytes of the next frame in the decoder's frame buffer: with
    2072-bit frames behind the r=1/2 decoder (4096 bits per call) two frames often complete in one call, and the second one's first ASM
    byte comes out as the first message byte of the first one's word. The restatement follows the reference."""
    from oracle import port
    pin = Pin("rs_row256_next_frame")
    rng = np.random.default_rng(6)
    pay = rng.integers(0, 256, (40, 223), dtype=np.uint8)
    tx, _ = FC.synth.build_cadus(pay, 1)
    tx[5:, 4 + np.arange(3)] ^= 7
    soft = np.where(FC.synth.conv_encode(np.unpackbits(tx.reshape(-1))) > 0, 60, -60).astype(np.int8)
    soft = soft[:soft.size // 8192 * 8192]
    cfg = port.ccsds_cfg("bpsk", 2072, 0.3, 20, 1)
    b = port.Fec(cfg).run(soft)
    fr = b["cadu"].reshape(-1, 259)
    assert fr.shape[0] > 30 and (fr[:, 0] != 0x1A).sum() > 10 and (b["rs_err"] > 0).sum() > 20
    for k in ("cadu", "rs_err"):
        pin.equal(k, pin.run(lambda R: R.Fec(cfg).run(soft)[k]), b[k])


def _deframer_streams():
    for name, kw, synced in FC.deframer_cases():
        for lead in FC.DEFRAMER_LEADS:
            bits, ends, bodies = FC.deframer_stream(cadu_size=FC.DEFRAMER_CADU, lead=lead, seed=sum(map(ord, name)), **kw)
            yield name, lead, synced, bits[:bits.size // FC.DEFRAMER_CADU * FC.DEFRAMER_CADU], ends, bodies


def test_deframer_model_equals_restatement_and_reference(built):
    """The bit-serial deframer model on the designed streams: frames equal the restatement's and the reference's deframer; the state
    after every cadu_size bits equals the state the simple PSK decoder reports per chunk (SYNCED threshold 12)."""
    from oracle import port
    pin = Pin("deframer_model")
    C = FC.DEFRAMER_CADU
    for name, lead, synced, bits, ends, bodies in _deframer_streams():
        m = M.deframe(bits, C, synced, checkpoints=range(C, bits.size + 1, C))
        FC.check_deframer_path(name, m, ends, bodies, synced)
        b = port.deframe(bits, C, synced)
        assert np.array_equal(m["frames"], b), (name, lead)
        pin.equal(f"{name}_{lead}_frames", pin.run(lambda R: R.deframe(bits, C, synced)), b)
        if synced == 12:
            cfg = port.simple_cfg("bpsk", C, 0, derandomize=False)
            r = port.Fec(cfg).run(FC.soft_of(bits))
            assert np.array_equal(r["defr_state"], m["states"]) and np.array_equal(r["cadu"].reshape(-1, C // 8), m["frames"]), (name, lead)
            pin.equal(f"{name}_{lead}_states", pin.run(lambda R: R.Fec(cfg).run(FC.soft_of(bits))["defr_state"]), r["defr_state"])
