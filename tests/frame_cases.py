"""Designed inputs of the frame stage tests (tests/test_rs_model.py on the CPU, tests/test_gpu_frame_stage.py on the GPU): Reed-Solomon
codewords with chosen errors, and bit streams that drive the deframer through chosen transitions. Everything is rebuilt from seeds."""
import numpy as np

from satdump_b200 import synth
from tests import rs_model

ASM_BITS = np.unpackbits(np.frombuffer(rs_model.SYNC.to_bytes(4, "big"), np.uint8))


def t_of(rs_type):
    return rs_model.params(rs_type)[0] // 2


def min_weight_word(rs_type, shift):
    """x^shift g(x): a codeword of the minimum weight nroots + 1, as conventional bytes (255,) in codeword byte order."""
    nroots, fcr = rs_model.params(rs_type)
    g = synth.rs_generator(nroots, fcr)
    assert np.count_nonzero(g) == nroots + 1, "the generator polynomial should have full weight"
    w = np.zeros(255, np.int64)
    w[254 - (shift + np.arange(nroots + 1))] = g
    return w


def codeword_cases(rs_type, dual, I, seed, positions=True):
    """RS codewords with designed errors, interleaved I deep. Returns dict(sent, rx: (nframes, 255*I) bytes as the CADU holds them from byte
    4 (dual basis if dual), kind: (nframes, I) labels, want_count: (nframes, I) the count a correct decoder returns or -2 where the
    outcome is not designed (t+1, t+2 errors), want: (nframes, 255*I) the decoded bytes where designed).

    Word kinds: 'pos<p>' one error at codeword byte p for every p in 0..254 (positions=True); 'n<k>' k random errors for
    k = 0, 1, t-1, t, t+1, t+2 (three words each); 'parity' t errors inside the parity bytes; 'mis' t+1 of the nroots+1 nonzero symbols
    of a shifted generator polynomial w added to a codeword c, which lies at distance t from c + w: every decoder must return c + w."""
    nroots, _ = rs_model.params(rs_type)
    t, k = nroots // 2, 255 - nroots
    rng = np.random.default_rng(seed)
    kinds, errs, fix = [], [], []
    if positions:
        for p in range(255):
            e = np.zeros(255, np.int64)
            e[p] = rng.integers(1, 256)
            kinds.append(f"pos{p}")
            errs.append(e)
            fix.append(None)
    for n in (0, 1, t - 1, t, t + 1, t + 2):
        for _ in range(3):
            e = np.zeros(255, np.int64)
            e[rng.choice(255, n, replace=False)] = rng.integers(1, 256, n)
            kinds.append(f"n{n}")
            errs.append(e)
            fix.append(None)
    for _ in range(2):
        e = np.zeros(255, np.int64)
        e[k + rng.choice(nroots, t, replace=False)] = rng.integers(1, 256, t)
        kinds.append("parity")
        errs.append(e)
        fix.append(None)
    for shift in (10, 200):
        w = min_weight_word(rs_type, shift)
        nz = np.nonzero(w)[0]
        add = rng.choice(nz, t + 1, replace=False)
        e = np.zeros(255, np.int64)
        e[add] = w[add]
        kinds.append("mis")
        errs.append(e)
        fix.append(w)
    while len(kinds) % I:
        kinds.append("n0")
        errs.append(np.zeros(255, np.int64))
        fix.append(None)
    nw = len(kinds)
    msg = rng.integers(0, 256, (nw, k), dtype=np.uint8)
    c = synth.rs_encode(msg, dual=False, nroots=nroots).astype(np.int64)
    e = np.array(errs)
    r = c ^ e
    want = r.copy()
    want_count = np.full(nw, -2, np.int64)
    for i, kd in enumerate(kinds):
        if kd == "mis":
            target = c[i] ^ fix[i]
            want[i, :k] = target[:k]
            want_count[i] = int((target[:k] != r[i, :k]).sum())
            assert 0 < want_count[i] <= t
        elif kd.startswith("pos") or kd == "parity" or (kd.startswith("n") and int(kd[1:]) <= t):
            want[i, :k] = c[i, :k]
            want_count[i] = int((e[i, :k] != 0).sum())
    if dual:
        c, r, want = synth.TO_DUAL[c], synth.TO_DUAL[r], synth.TO_DUAL[want]
    nf = nw // I
    lay = lambda a: np.asarray(a, np.uint8).reshape(nf, I, 255).transpose(0, 2, 1).reshape(nf, 255 * I)
    return dict(sent=lay(c), rx=lay(r), want=lay(want), kind=np.array(kinds).reshape(nf, I), want_count=want_count.reshape(nf, I))


def spare_cadus(rs_type, I, extra, seed, derand_start=4):
    """CADUs 4 + 255*I + extra bytes long: ASM, the designed words of codeword_cases (no position sweep), `extra` random spare bytes, all
    randomised from derand_start as the deframer hands them over. Returns (codeword_cases dict, CADUs)."""
    c = codeword_cases(rs_type, True, I, seed, positions=False)
    nf = c["rx"].shape[0]
    rng = np.random.default_rng(seed + 1)
    asm = np.tile(np.frombuffer(rs_model.SYNC.to_bytes(4, "big"), np.uint8), (nf, 1))
    cadus = np.concatenate([asm, c["rx"], rng.integers(0, 256, (nf, extra), dtype=np.uint8)], axis=1)
    cadus[:, derand_start:] ^= synth.ccsds_pn(cadus.shape[1] - derand_start)[None, :]
    return c, cadus


SPARE = [(0, 4, 8), (1, 8, 3), (0, 1, 5)]  # (rs_type, I, spare bytes)


def random_bits(rng, n):
    """n random bits that hold no exact or inverted ASM (the deframer's NOSYNC search must not stop in them)."""
    while True:
        b = rng.integers(0, 2, n, dtype=np.uint8)
        w = rs_model.windows(b)[31:]
        if not ((w == rs_model.SYNC) | (w == (~rs_model.SYNC & 0xFFFFFFFF))).any():
            return b


def cadu_stream(cadus, lead, tail, seed):
    """Bits of lead random bits, the CADUs (their ASM included), tail random bits."""
    rng = np.random.default_rng(seed)
    return np.concatenate([random_bits(rng, lead), np.unpackbits(np.asarray(cadus, np.uint8).reshape(-1)), random_bits(rng, tail)])


def soft_of(bits, amp=100):
    """Noise-free BPSK soft bytes: bit 1 -> +amp."""
    return np.where(np.asarray(bits) > 0, amp, -amp).astype(np.int8)


def deframer_stream(nframes, cadu_size, lead, seed, asm_errors=None, inverted_from=None, slips=None, tail=700):
    """A bit stream for the deframer: lead random bits, then nframes frames of ASM + random body, then tail bits. asm_errors {frame: bit
    errors in its ASM}; inverted_from: frames from this index on are sent inverted; slips {frame: extra random bits inserted before it}.
    Returns (bits, asm_end: the bit index of each ASM's last bit, bodies (nframes, cadu_size/8 - 4) as meant)."""
    rng = np.random.default_rng(seed)
    asm_errors, slips = asm_errors or {}, slips or {}
    parts, ends, n = [random_bits(rng, lead)], [], lead
    bodies = rng.integers(0, 2, (nframes, cadu_size - 32), dtype=np.uint8)
    for f in range(nframes):
        if f in slips:
            parts.append(rng.integers(0, 2, slips[f], dtype=np.uint8))
            n += slips[f]
        a = ASM_BITS.copy()
        if asm_errors.get(f):
            a[rng.choice(32, asm_errors[f], replace=False)] ^= 1
        fr = np.concatenate([a, bodies[f]])
        if inverted_from is not None and f >= inverted_from:
            fr = fr ^ 1
        parts.append(fr)
        ends.append(n + 31)
        n += cadu_size
    parts.append(random_bits(rng, tail))
    return np.concatenate(parts), np.array(ends), np.packbits(bodies, axis=1)


DEFRAMER_CADU = 1024


def deframer_cases():
    """(name, deframe kwargs, SYNCED threshold). SYNCED is entered on frame 11 (the exact ASM of frame 0 and 11 good ones), so frame
    12 + l is the l-th ASM the SYNCED walk tests after entering."""
    cases = [("syncing_5", dict(nframes=30, asm_errors={3: 5}), 12), ("syncing_6", dict(nframes=30, asm_errors={3: 6}), 12),
             ("synced_11", dict(nframes=40, asm_errors={20: 11}), 12), ("synced_12", dict(nframes=40, asm_errors={20: 12}), 12),
             ("synced18_17", dict(nframes=40, asm_errors={20: 17}), 18), ("synced18_18", dict(nframes=40, asm_errors={20: 18}), 18),
             ("slip_1", dict(nframes=30, slips={4: 1}), 12), ("slip_2", dict(nframes=30, slips={4: 2}), 12),
             ("slip_3", dict(nframes=30, slips={4: 3}), 12), ("flip", dict(nframes=40, inverted_from=20), 12)]
    for l in (127, 128, 129, 256):
        cases.append((f"lookahead_{l}", dict(nframes=12 + l + 8, asm_errors={12 + l: 16}), 12))
    return cases


# lead-in lengths: the chunk boundaries (every cadu_size bits) fall 13 bits into every ASM, or 513 bits into every frame body
DEFRAMER_LEADS = (3 * DEFRAMER_CADU - 13, 3 * DEFRAMER_CADU - 513)


def check_deframer_path(name, m, ends, bodies, synced):
    """The transitions each designed stream is for, read from the model's trace."""
    tr = {p: (s, d, ok) for p, s, d, ok in m["trace"]}
    ev = m["events"]
    # SYNCED after 11 good tests in a row: a failed test resets the count (slips: the first ASM re-found on a later bit passes after 1
    # or 2 failed tests), NOSYNC starts over from the next exact ASM
    enter = {"syncing_6": 15, "slip_1": 14, "slip_2": 14, "slip_3": 15}.get(name, 11)
    assert ev[0] == (ends[0], 6) and (ends[enter], synced) in ev, name
    if name.startswith("syncing_"):
        k = int(name[-1])
        assert tr[ends[3]] == (6, k, k < 6), name
        if k == 6:  # three failed tests one bit apart, then the exact search finds the next ASM
            assert (ends[3] + 2, 2) in ev and (ends[4], 6) in ev
    if name.startswith("synced"):
        k = int(name.split("_")[1])
        assert tr[ends[20]] == (synced, k, k < synced), name
        assert ((ends[20], 2) in ev) == (k >= synced) and ((ends[21], 6) in ev) == (k >= synced)
    if name.startswith("slip_"):
        k = int(name[-1])
        # the ASM shifted by 1..3 bits differs from itself in >= 11 bits: k failed tests, the k-th one is NOSYNC for k = 3
        for j in range(k):
            assert tr[ends[4] - k + j][1] >= 11
        if k < 3:
            assert tr[ends[4]] == (6, 0, True) and not any(s == 2 for p, s in ev if ends[0] < p <= ends[4])
        else:
            assert (ends[4] - 1, 2) in ev and (ends[4], 6) in ev
    if name == "flip":
        assert tr[ends[20]] == (synced, 32, False) and (ends[20], 2) in ev and (ends[21], 6) in ev
        i = list(m["asm_end"]).index(ends[21])
        assert m["inversion"][i] == 1 and np.array_equal(m["frames"][i, 4:], bodies[21])
    if name.startswith("lookahead_"):
        f = 12 + int(name.split("_")[1])
        assert tr[ends[f]] == (synced, 16, False) and (ends[f], 2) in ev and (ends[f + 1], 6) in ev
    # every frame the model keeps carries its designed body (inversion undone)
    for i, e in enumerate(m["asm_end"]):
        j = list(ends).index(e)
        assert np.array_equal(m["frames"][i, 4:], bodies[j]), (name, i)
