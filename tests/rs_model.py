"""Plain models of the frame stage (deframer, derandomiser, Reed-Solomon), written from the textbook algorithms and the decoder modules'
documented rules, for the CPU and GPU tests of that stage.

Reed-Solomon (CCSDS 131.0-B): GF(256) with polynomial 0x187, code roots beta^(fcr+i), beta = alpha^11, fcr = 112 (32 roots, RS(255,223))
or 120 (16 roots, RS(255,239)). A codeword byte k is the coefficient of x^(254-k). Syndromes in numpy over all codewords at once;
Berlekamp-Massey vectorised over codewords; Chien search over the 255 nonzero elements; error positions straight from the roots
(X = root^-1, position = log(X) / 11 mod 255); Forney for the values. On top of that the module-level rules of the reference decoder:

- acceptance: a word is accepted iff its number of Chien roots equals the locator's "order", the degree bound libcorrect keeps next
  to the Berlekamp-Massey length L (both are returned);
- write-back: only message bytes are written back, parity stays as received;
- return value: the number of message bytes changed, -1 when the word is not accepted;
- layout: codeword b of an interleave depth I holds bytes data[i*I + b]; dual-basis bytes are converted before decoding and after;
- the row past the codewords: with rs_fill_bytes -1 (the modules' default) the reference's (de)interleave loops run 256 rows, and byte
  255*I + b goes through the first byte of its message buffer. It comes back as the corrected first message byte (conventional basis)
  when word b decodes, and unchanged when it does not. A CADU longer than 4 + 255*I holds that byte; later spare bytes stay as received.

Deframer (the bit-serial ASM machine of the CCSDS deframer): a 32-bit shifter tested against the ASM at chosen bits.
- NOSYNC (2): every bit, an exact ASM or inverted ASM opens a frame and goes to SYNCING;
- SYNCING (6): a test passes with < 6 bit errors; good > 10 goes to SYNCED, bad > 2 back to NOSYNC; after a failed test the next bit is tested;
- SYNCED (12, 18 in MetOp's decoder): a test passes with < that many errors; the first failure goes back to NOSYNC;
- a passed test opens a frame: its ASM bytes are the clean sync word, its body the next cadu_size - 32 bits with the inversion applied,
  and the next test falls on the last bit of the following 32 (the next ASM)."""
import numpy as np

from satdump_b200 import synth

EXP = synth.GF_EXP.astype(np.int64)   # EXP[i] = alpha^i, i < 510
LOG = synth.GF_LOG.astype(np.int64)   # LOG[alpha^i] = i (LOG[0] is meaningless)
GAP = 11
GAP_INV = pow(GAP, -1, 255)
SYNC = 0x1ACFFC1D


def params(rs_type):
    """(nroots, fcr) of rs_type 0 = RS(255,223), 1 = RS(255,239)."""
    return (16, 120) if rs_type == 1 else (32, 112)


def gmul(a, b):
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    return np.where((a == 0) | (b == 0), 0, EXP[(LOG[a] + LOG[b]) % 255])


def ginv(a):
    return EXP[(255 - LOG[np.asarray(a, np.int64)]) % 255]


def poly_eval_all(P):
    """P: (n, K) coefficients, lowest order first -> (n, 255) values at x = alpha^e, e = 0..254 (Horner)."""
    n, K = P.shape
    e = np.arange(255, dtype=np.int64)[None, :]
    v = np.zeros((n, 255), np.int64)
    for i in range(K - 1, -1, -1):
        v = np.where(v == 0, 0, EXP[(LOG[v] + e) % 255]) ^ P[:, i:i + 1]
    return v


def syndromes(cw, nroots, fcr):
    """cw: (n, 255) conventional-basis codewords -> (n, nroots) syndromes S_j = r(beta^(fcr+j))."""
    cw = np.asarray(cw, np.int64)
    p = 254 - np.arange(255, dtype=np.int64)                       # power of x of codeword byte k
    out = np.zeros((cw.shape[0], nroots), np.int64)
    for a in range(0, cw.shape[0], 256):
        c = cw[a:a + 256]
        lg = LOG[c][:, None, :] + (GAP * (fcr + np.arange(nroots))[:, None] * p[None, :])[None] % 255
        t = np.where(c[:, None, :] == 0, 0, EXP[lg % 255])
        out[a:a + 256] = np.bitwise_xor.reduce(t, axis=2)
    return out


def berlekamp_massey(S):
    """S: (n, N) syndromes -> (locator (n, N + 2) lowest order first, BM length L (n,), libcorrect's order (n,)).

    Massey's algorithm: C(x) the connection polynomial, B(x) the copy from the last length change, m the shift since then, b its
    discrepancy. libcorrect keeps the degree bound of C next to L: on a length change order = the bound of B + m (and B's bound becomes
    the old order); on any other correction order = max(order, bound of B + m)."""
    S = np.asarray(S, np.int64)
    n, N = S.shape
    K = N + 2
    C = np.zeros((n, K), np.int64)
    B = np.zeros((n, K), np.int64)
    C[:, 0] = B[:, 0] = 1
    L = np.zeros(n, np.int64)
    order = np.zeros(n, np.int64)
    border = np.zeros(n, np.int64)
    m = np.ones(n, np.int64)
    b = np.ones(n, np.int64)
    cols = np.arange(K)[None, :]
    for i in range(N):
        d = S[:, i].copy()
        for j in range(1, i + 1):
            d ^= np.where(j <= L, gmul(C[:, j], S[:, i - j]), 0)
        nz = d != 0
        grow = nz & (2 * L <= i)
        idx = cols - m[:, None]
        Bs = np.where(idx >= 0, np.take_along_axis(B, np.clip(idx, 0, K - 1), axis=1), 0)
        coef = gmul(d, ginv(b))
        Cn = C ^ gmul(coef[:, None], Bs)
        B = np.where(grow[:, None], C, B)
        C = np.where(nz[:, None], Cn, C)
        new_order = np.where(grow, border + m, np.where(nz, np.maximum(order, border + m), order))
        border = np.where(grow, order, border)
        order = new_order
        L = np.where(grow, i + 1 - L, L)
        b = np.where(grow, d, b)
        m = np.where(grow, 1, m + 1)
    return C, L, order


def rs_decode(cw, rs_type=0):
    """Conventional-basis codewords (n, 255) -> dict(out = the words with the message bytes corrected where accepted, count = message
    bytes changed or -1, L, order, roots = number of Chien roots, positions = list of the corrected codeword byte indices per word)."""
    nroots, fcr = params(rs_type)
    k = 255 - nroots
    cw = np.asarray(cw, np.int64)
    n = cw.shape[0]
    S = syndromes(cw, nroots, fcr)
    lam, L, order = berlekamp_massey(S)
    V = poly_eval_all(lam)                                   # Lambda(alpha^e)
    isroot = (V == 0) & (order[:, None] > 0)
    nr = isroot.sum(axis=1)
    ok = nr == order
    out = cw.copy()
    count = np.where(ok, 0, -1)
    positions = [[] for _ in range(n)]
    fix = np.nonzero(ok & (order > 0))[0]
    if fix.size:
        # Omega = S(x) Lambda(x) mod x^nroots; Lambda' = the odd-degree terms shifted down
        Sf, lf = S[fix], lam[fix]
        om = np.zeros((fix.size, nroots), np.int64)
        for i in range(nroots):
            for j in range(nroots - i):
                om[:, i + j] ^= gmul(lf[:, i], Sf[:, j])
        der = np.zeros_like(lf)
        der[:, 0:-1:2] = lf[:, 1::2]
        num, den = poly_eval_all(om), poly_eval_all(der)
        e = np.arange(255, dtype=np.int64)
        for r, w in enumerate(fix):
            for ee in e[isroot[w]]:
                logx = (255 - ee) % 255                              # X = root^-1 = alpha^(-e)
                p = logx * GAP_INV % 255                             # X = beta^p
                val = gmul(EXP[(logx * (1 - fcr)) % 255], gmul(num[r, ee], ginv(den[r, ee]) if den[r, ee] else 0))
                byte = 254 - p
                positions[w].append(int(byte))
                if byte < k and val:
                    out[w, byte] ^= val
                    count[w] += 1
    return dict(out=out.astype(np.uint8), count=count, L=L, order=order, roots=nr, positions=positions)


def rs_decode_interleaved(data, dual=True, interleave=4, rs_type=0, row256=True):
    """The decoder module's decode of I interleaved codewords: data (nframes, >= 255*I) bytes (a CADU from byte 4) -> (decoded bytes,
    counts (nframes, I), the rs_decode dict of the nframes*I words, frame-major). row256: the row past the codewords, where data has it."""
    data = np.atleast_2d(np.asarray(data, np.uint8))
    nf, I = data.shape[0], interleave
    cw = data[:, :255 * I].reshape(nf, 255, I).transpose(0, 2, 1).reshape(nf * I, 255)
    if dual:
        cw = synth.FROM_DUAL[cw]
    r = rs_decode(cw, rs_type)
    o = r["out"]
    if dual:
        o = synth.TO_DUAL[o]
    out = data.copy()
    out[:, :255 * I] = o.reshape(nf, I, 255).transpose(0, 2, 1).reshape(nf, 255 * I)
    counts = r["count"].reshape(nf, I)
    if row256:
        msg0 = r["out"][:, 0].reshape(nf, I)                    # conventional basis
        for b in range(min(I, data.shape[1] - 255 * I)):
            out[:, 255 * I + b] = np.where(counts[:, b] >= 0, msg0[:, b], out[:, 255 * I + b])
    return out, counts, r


def frame_stage(cadus, rs_i, dual=True, rs_type=0, derandomize=True, derand_after_rs=False, derand_start=4, rs_usecheck=False, row256=True):
    """Deframed CADUs (n, cadu_bytes) -> (the frames the decoder writes, counts (n, rs_i), kept mask): the derandomiser (from byte
    derand_start to the end of the CADU, before or after RS), RS on the bytes from 4, and rs_usecheck's drop of frames with a failed word.
    row256: rs_fill_bytes -1 (the row past the codewords is decoded), False for rs_fill_bytes 0."""
    f = np.array(cadus, np.uint8, copy=True)
    nb = f.shape[1]
    pn = None
    if derandomize and derand_start < nb:
        pn = synth.ccsds_pn(nb - derand_start)
    if pn is not None and not derand_after_rs:
        f[:, derand_start:] ^= pn[None, :]
    counts = np.zeros((f.shape[0], max(rs_i, 0)), np.int64)
    if rs_i:
        f[:, 4:], counts, _ = rs_decode_interleaved(f[:, 4:], dual, rs_i, rs_type, row256)
    if pn is not None and derand_after_rs:
        f[:, derand_start:] ^= pn[None, :]
    kept = (counts >= 0).all(axis=1) if rs_usecheck else np.ones(f.shape[0], bool)
    return f[kept], counts, kept


# ---------------------------------------------------------------------------------------------------------------- deframer
def windows(bits):
    """The shifter after each bit: w[p] = bits[p-31 .. p] (zeros before the stream) as uint32."""
    b = np.asarray(bits, np.uint32)
    w = np.zeros(b.size, np.uint32)
    for k in range(32):
        w[k:] |= b[:b.size - k] << np.uint32(k)
    return w


def deframe(bits, cadu_size, synced=12, sync=SYNC, checkpoints=()):
    """Bit-serial deframer over the whole bit stream. Returns dict(frames (n, cadu_size / 8), asm_end (n,) bit index of each frame's
    ASM end, inversion (n,), trace = [(bit, state before, bit errors, passed)] of every test in SYNCING / SYNCED and every NOSYNC hit,
    events = [(bit, new state)], states = the state after the first c bits for each c in checkpoints)."""
    bits = np.asarray(bits, np.uint8)
    N = bits.size
    w = windows(bits)
    inv_sync = ~sync & 0xFFFFFFFF
    hits = np.nonzero((w == sync) | (w == inv_sync))[0]
    state, inv, good, bad, pos = 2, 0, 0, 0, 0
    trace, events, opened = [], [], []
    while pos < N:
        if state == 2:
            h = hits[np.searchsorted(hits, pos):]
            if h.size == 0:
                break
            q = int(h[0])
            inv = int(w[q] == inv_sync)
            trace.append((q, 2, 0, True))
            state, good, bad = 6, 0, 0
            events.append((q, 6))
            opened.append((q, inv))
            pos = q + cadu_size
            continue
        diff = bin(int(w[pos]) ^ (inv_sync if inv else sync)).count("1")
        passed = diff < state
        trace.append((pos, state, diff, passed))
        if state == 6:
            if passed:
                good, bad = good + 1, 0
                if good > 10:
                    state = synced
                    events.append((pos, synced))
            else:
                bad, good = bad + 1, 0
                if bad > 2:
                    state = 2
                    events.append((pos, 2))
        elif not passed:
            state, good, bad = 2, 0, 0
            events.append((pos, 2))
        if passed:
            opened.append((pos, inv))
            pos += cadu_size
        else:
            pos += 1
    done = [(q, v) for q, v in opened if q + cadu_size - 32 < N]
    C8 = cadu_size // 8
    frames = np.zeros((len(done), C8), np.uint8)
    for i, (q, v) in enumerate(done):
        frames[i, :4] = np.frombuffer(int(sync).to_bytes(4, "big"), np.uint8)
        frames[i, 4:] = np.packbits(bits[q + 1:q + cadu_size - 31] ^ v)
    states = []
    for c in checkpoints:
        st = 2
        for p, s in events:
            if p < c:
                st = s
        states.append(st)
    return dict(frames=frames, asm_end=np.array([q for q, _ in done], np.int64), inversion=np.array([v for _, v in done], np.int64),
                trace=trace, events=events, states=np.array(states, np.int64))
