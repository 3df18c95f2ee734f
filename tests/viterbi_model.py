"""A numpy model of how the device Viterbi decoder (satdump_b200/csrc/fec.cuh, api_fec.cu: decode_range / viterbi_segment) splits the
decoding of a locked stream, with the reference's integer arithmetic (volk_k7_r2_generic_fixed.h, cc_decoder.cpp):

  * the ACS over chunks x 64 states: (1 + a + b) >> 3 branch metric, uint8 wrap, ties pick m1, per-step renormalisation, first-minimum
    end state, biased (63 / 0 at the start state) and unbiased (all 31) initialisation;
  * the true chunk-by-chunk decode from the carried start state, and the lock machine of Viterbi3_4 / Viterbi1_2 around it (lock search,
    chained BER encoder, invalid counter);
  * what the device does instead: start-state speculation (k_vit_spec), chainback in blocks of TB_WORDS words that warm up over
    tb_overlap rows (k_vit_tb) with the edge check (k_vit_tb_check), the redo rounds with the successor BER recompute, and the adaptive
    windows (adapt_window).

It is the reference the CPU test pins against the oracle, and the tool that designs the GPU test streams of test_gpu_viterbi_paths.py:
it predicts which chunks the device mis-speculates and which block edges disagree."""
import numpy as np

TESTLEN = 2048
SPEC_STEPS_34, SPEC_STEPS_12 = 768, 512
TB_WORDS, TB_OVERLAP, TB_OVERLAP_MAX = 16, 256, 2048


def _parity(x):
    return bin(x).count("1") & 1


BT0 = np.array([255 if _parity((2 * i) & 79) else 0 for i in range(32)], np.int32)
BT1 = np.array([255 if _parity((2 * i) & 109) else 0 for i in range(32)], np.int32)


# ----------------------------------------------------------------------------- symbols
def rotate_soft(s, phase, swap):
    """rotation.cpp:4-63 on an int8 array (pairs I, Q)."""
    v = s.astype(np.int32)
    v[v == -128] = -127
    i, q = v[0::2].copy(), v[1::2].copy()
    if swap:
        i, q = q, i
    if phase == 1:
        i, q = q, -i
    elif phase == 2:
        i, q = -i, -q
    elif phase == 3:
        i, q = -q, i
    out = np.empty_like(v)
    out[0::2], out[1::2] = i, q
    return out


def soft_u8(v):
    """signed_soft_to_unsigned (utils.cpp:3-11) of rotated values."""
    u = (v + 127) & 255
    u[u == 128] = 127
    return u.astype(np.uint8)


def depunc34(u, shift):
    """Viterbi3_4::depuncture, MetOp branch (viterbi_3_4.cpp:84-104): 4 soft bytes -> 6 symbols."""
    g = u[:u.size // 4 * 4].reshape(-1, 4)
    e = np.full((g.shape[0], 6), 128, np.uint8)
    if not shift:
        e[:, 0], e[:, 1], e[:, 3], e[:, 4] = g[:, 0], g[:, 1], g[:, 3], g[:, 2]
    else:
        e[:, 1], e[:, 2], e[:, 4], e[:, 5] = g[:, 1], g[:, 0], g[:, 2], g[:, 3]
    return e.reshape(-1)


class Geom:
    """One decoder configuration: MetOp r=3/4 (16384 soft bytes per chunk) or CCSDS r=1/2 (chunk = max(cadu_size, 8192))."""

    def __init__(self, kind, cadu_size=8192, constellation="qpsk", nrzm=False):
        self.kind, self.nrzm = kind, nrzm
        if kind == "metop":
            self.rate34, self.chunk, self.F = True, 16384, 12288
            self.hyps = [(0, ph, sh) for ph in (0, 1) for sh in (0, 1)]
            self.kber, self.spec_base = np.float32(5.0), SPEC_STEPS_34
            self.tb = TESTLEN * 3 // 4
        else:
            self.rate34, self.chunk = False, max(cadu_size, 8192)
            self.F = self.chunk // 2
            phases = {"bpsk": [0], "bpsk_90": [1]}.get(constellation, [0, 1])
            swaps = [0, 1] if constellation == "oqpsk" else [0]
            self.hyps = [(s, ph, sh) for s in swaps for ph in phases for sh in (0, 1)]
            self.kber, self.spec_base = np.float32(2.5), SPEC_STEPS_12
            self.tb = TESTLEN // 2
        self.spec_cap = (self.F // 32) * 32
        self.nblocks = ((self.F + 31) // 32 + TB_WORDS - 1) // TB_WORDS

    def symbols(self, soft, hyp):
        """The 2 (F + 6) decoder symbols of one chunk of soft bytes under hypothesis (swap, phase, shift); the six flush steps read
        erasures (the symbol buffers are set to 128 at lock time)."""
        swap, phase, shift = hyp
        u = soft_u8(rotate_soft(soft, phase, swap and not self.rate34))
        out = np.full(2 * (self.F + 6), 128, np.uint8)
        if self.rate34:
            d = depunc34(u, shift)
            out[:d.size] = d
        else:
            d = u[shift:]
            out[:d.size] = d
        return out


# ----------------------------------------------------------------------------- ACS / chainback
def init_metrics(start):
    """start: (C,) start states, -1 = unbiased."""
    start = np.asarray(start)
    X = np.full((start.size, 64), 63, np.int32)
    X[np.arange(start.size), np.maximum(start, 0)] = 0
    X[start < 0] = 31
    return X


def acs(sym, X):
    """sym: (C, steps, 2) uint8; X: (C, 64) metrics. Returns (metrics after the last step, decisions (C, steps, 64) bool)."""
    C, steps = sym.shape[0], sym.shape[1]
    X = X.astype(np.int32).copy()
    dec = np.empty((C, steps, 64), bool)
    s = sym.astype(np.int32)
    Y = np.empty_like(X)
    for t in range(steps):
        m = (1 + (BT0[None, :] ^ s[:, t, 0:1]) + (BT1[None, :] ^ s[:, t, 1:2])) >> 3
        xl, xh = X[:, :32], X[:, 32:]
        m0, m1 = (xl + m) & 255, (xh + 63 - m) & 255
        m2, m3 = (xl + 63 - m) & 255, (xh + m) & 255
        d0, d1 = m0 >= m1, m2 >= m3
        Y[:, 0::2] = np.where(d0, m1, m0)
        Y[:, 1::2] = np.where(d1, m3, m2)
        dec[:, t, 0::2], dec[:, t, 1::2] = d0, d1
        Y -= Y.min(axis=1, keepdims=True)
        X, Y = Y, X
    return X, dec


def walk(dec, rows_top, nrows, st, collect=False, idx=None):
    """Chainback of every entry e: from state st[e], rows rows_top[e], rows_top[e] - 1, ... (nrows[e] rows) of dec[idx[e]] (idx defaults to
    e). Returns the final states (and the decision bits by row when `collect`)."""
    E = st.size
    st = st.copy()
    idx = np.arange(E) if idx is None else idx
    bits = np.zeros((E, int(nrows.max()) if E else 0), np.uint8) if collect else None
    for j in range(int(nrows.max()) if E else 0):
        act = j < nrows
        r = np.where(act, rows_top - j, 0)
        b = dec[idx, r, st].astype(np.int32)
        nst = (st >> 1) | (b << 5)
        st = np.where(act, nst, st)
        if collect:
            bits[:, j] = b
    return st, bits


def serial_chainback(dec, X, F):
    """cc_decoder.cpp:192-276: first-minimum end state, output bit i from row i + 6, next start = the state after the first six rows walked."""
    C = dec.shape[0]
    end = np.argmin(X, axis=1)
    st6, _ = walk(dec, np.full(C, F + 5), np.full(C, 6), end)
    _, b = walk(dec, np.full(C, F + 5), np.full(C, F), end, collect=True)
    return b[:, ::-1].copy(), st6, end


def tb_edges_bad(dec, end, F, overlap):
    """k_vit_tb + k_vit_tb_check: per chunk, whether any block edge disagrees (the device then chains the chunk back serially)."""
    C = dec.shape[0]
    nwords = (F + 31) // 32
    nb = (nwords + TB_WORDS - 1) // TB_WORDS
    q = np.repeat(np.arange(C), nb)
    k = np.tile(np.arange(nb), C)
    w_hi = nwords - k * TB_WORDS
    w_lo = np.maximum(0, w_hi - TB_WORDS)
    top = np.minimum(F, 32 * w_hi + overlap)
    warm = np.where(k == 0, 0, top - 32 * w_hi)
    st0 = np.where(k == 0, end[q], 0)
    assumed, _ = walk(dec, 6 + top - 1, warm, st0, idx=q)
    # the block itself: output rows 6 + 32 w_hi - 1 .. 6 + 32 w_lo (block 0 from row F + 5)
    btop = np.where(k == 0, F + 5, 6 + 32 * w_hi - 1)
    bend = 6 + 32 * w_lo
    left, _ = walk(dec, btop, btop - bend + 1, assumed, idx=q)
    assumed, left = assumed.reshape(C, nb), left.reshape(C, nb)
    return (assumed[:, 1:] != left[:, :-1]).any(axis=1)


def ber_counts(geom, sym, bits, enc_init):
    """k_vit_ber / get_ber: re-encode the first tb bits from the chained encoder register and compare with the hard decisions of the
    non-erased symbols. Returns (errors, total)."""
    tb = geom.tb
    b = np.concatenate([[(enc_init >> (5 - i)) & 1 for i in range(6)], bits[:tb]]).astype(np.uint8)
    s = lambda k: b[6 - k:6 - k + tb]
    e = np.stack([s(0) ^ s(1) ^ s(2) ^ s(3) ^ s(6), s(0) ^ s(2) ^ s(3) ^ s(5) ^ s(6)], axis=1).reshape(-1)
    raw = sym[:2 * tb]
    keep = raw != 128
    return int(((raw > 127) != e)[keep].sum()), int(keep.sum())


def enc_tail(bits, tb):
    t = 0
    for k in range(tb - 6, tb):
        t = (t << 1) | int(bits[k])
    return t


def ber_value(geom, errors, total):
    return np.float32(np.float32(errors) / np.float32(total)) * geom.kber


# ----------------------------------------------------------------------------- the device's split of one locked range
class Range:
    """Outcome of the device's decode of n consecutive chunks (decode_range): bits and records as the device leaves them, and the
    counters of the correction paths."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def spec_starts(geom, syms, spec):
    """k_vit_spec: chunk w's last `spec` steps + 6 flush steps from all-zero metrics, first-minimum end state, six rows back."""
    C = syms.shape[0]
    sy = syms[:, 2 * (geom.F - spec):2 * (geom.F + 6)].reshape(C, spec + 6, 2)
    X, dec = acs(sy, np.zeros((C, 64), np.int32))
    st, _ = walk(dec, np.full(C, spec + 5), np.full(C, 6), np.argmin(X, axis=1))
    return st


def decode_chunks(geom, syms, starts, overlap):
    """k_vit_acs3 + k_vit_tb (+ check) on the chunks given: bits (C, F), next_start, and which chunks' block edges disagree."""
    C = syms.shape[0]
    X, dec = acs(syms.reshape(C, geom.F + 6, 2), init_metrics(starts))
    bits, nxt, end = serial_chainback(dec, X, geom.F)
    bad = tb_edges_bad(dec, end, geom.F, overlap)
    return bits, nxt, bad


def decode_range(geom, syms, first_start, enc_state, spec, overlap, rounds=6):
    """decode_range (api_fec.cu): speculation, one pass, up to `rounds` redo rounds. syms: (n, 2 (F + 6)) symbols of a locked range."""
    n = syms.shape[0]
    start = np.empty(n, np.int64)
    start[0] = first_start
    spec_miss = np.zeros(n, bool)
    if n > 1:
        start[1:] = spec_starts(geom, syms[:-1], spec)
    bits, nxt, bad = decode_chunks(geom, syms, start, overlap)
    first_tail = [enc_tail(bits[i], geom.tb) for i in range(n)]  # what a successor's BER check reads before any redo
    tb_serial = int(bad.sum())
    tb_first = tb_serial
    enc_init = np.empty(n, np.int64)

    def bers(idx):
        out = {}
        for i in idx:
            init = enc_state if i == 0 else enc_tail(bits[i - 1], geom.tb)
            out[i] = ber_counts(geom, syms[i], bits[i], init)
        return out

    ber = bers(range(n))
    redone, nrounds, misses0 = 0, 0, 0
    redo_chunks, succ_stale = [], []
    for rnd in range(rounds):
        redo = [i for i in range(1, n) if start[i] != nxt[i - 1]]
        if rnd == 0:
            misses0 = len(redo)
        if not redo:
            break
        nrounds += 1
        redone += len(redo)
        redo_chunks.append(redo)
        start[redo] = nxt[np.array(redo) - 1]
        old_tail = {i: enc_tail(bits[i], geom.tb) for i in redo}
        b2, n2, bad2 = decode_chunks(geom, syms[redo], start[redo], overlap)
        bits[redo], nxt[redo] = b2, n2
        tb_serial += int(bad2.sum())
        # successors that are not redone themselves, whose BER check reads a predecessor tail the redo changed
        succ_stale += [i + 1 for i in redo if i + 1 < n and i + 1 not in redo and enc_tail(bits[i], geom.tb) != old_tail[i]]
        ber.update(bers(sorted(set(redo) | {i + 1 for i in redo if i + 1 < n})))
    consistent = all(start[i] == nxt[i - 1] for i in range(1, n))
    return Range(bits=bits, start=start, next_start=nxt, ber=[ber[i] for i in range(n)], misses=misses0, redone=redone, rounds=nrounds,
                 redo_chunks=redo_chunks, succ_stale=succ_stale, first_tail=first_tail, tb_serial=tb_serial, tb_first=tb_first, consistent=consistent)


def adapt_window(win, clean, miss_frac, base, cap):
    """api_fec.cu adapt_window: > 2 % misses doubles up to cap, 32 launches in a row with < 0.2 % halve towards base."""
    if miss_frac > 0.02:
        return min(cap, win * 2), 0
    if miss_frac < 0.002:
        clean += 1
        if clean >= 32:
            return max(base, win // 2), 0
    return win, clean


# ----------------------------------------------------------------------------- the reference's decoder, chunk by chunk
class Decoder:
    """Viterbi3_4 / Viterbi1_2 (viterbi_3_4.cpp:110-173, viterbi_1_2.cpp:52-116) over whole chunks: lock search while IDLE, the main
    decode from the carried start state while SYNCED. The SYNCED chunks of one call are decoded as the device does it (decode_range, with
    redo rounds until consistent) - which IS the serial decode once every start state agrees with its predecessor's next start.
    run() returns the decoded bits (after NRZ-M), vit_state / vit_ber per chunk like the oracle's, and the device's counters."""

    def __init__(self, geom, thr, outsync):
        self.g, self.thr, self.outsync = geom, np.float32(thr), outsync
        self.state, self.invalid = 0, 0
        self.hyp = None
        self.dec_ber_start, self.main_start, self.enc = -1, -1, 0
        self.bers = {h: np.float32(10) for h in geom.hyps}
        self.bdecoded = np.zeros(16, np.uint8)  # r=1/2: the lock test over-reads 12 bytes past its 2048 test bytes; they read as zeros
        self.nrzm_last = 0
        self.spec, self.overlap, self.spec_clean, self.tb_clean = geom.spec_base, TB_OVERLAP, 0, 0
        self.counters = dict(start_redone=0, tb_serial=0, misses=[], tb_first=[], rounds=[], redo=[], succ_stale=[])

    def _lock_test(self, soft):
        g = self.g
        best = np.float32(10)
        for hyp in g.hyps:
            swap, phase, shift = hyp
            u = soft_u8(rotate_soft(soft[:TESTLEN], phase, swap and not g.rate34))
            if g.rate34:
                d = depunc34(u, shift)
                sym = np.zeros(2 * (TESTLEN * 3 // 4 + 6), np.uint8)  # (the bytes behind the 3072 written are never written: zeros)
                sym[:d.size] = d
                nb, cmp = TESTLEN * 3 // 4, d
            else:
                sym = np.concatenate([u, self.bdecoded])[shift:shift + 2 * (TESTLEN // 2 + 6)]
                nb = TESTLEN // 2
            X, dec = acs(sym.reshape(1, nb + 6, 2), init_metrics([self.dec_ber_start]))
            bits, nxt, _ = serial_chainback(dec, X, nb)
            self.dec_ber_start = int(nxt[0])
            if not g.rate34:
                cmp = np.concatenate([u, self.bdecoded])[shift:shift + TESTLEN]
            b = np.concatenate([[(self.enc >> (5 - i)) & 1 for i in range(6)], bits[0]]).astype(np.uint8)
            s = lambda k: b[6 - k:6 - k + nb]
            e = np.stack([s(0) ^ s(1) ^ s(2) ^ s(3) ^ s(6), s(0) ^ s(2) ^ s(3) ^ s(5) ^ s(6)], axis=1).reshape(-1)
            self.enc = enc_tail(bits[0], nb)
            keep = cmp != 128
            ber = np.float32(np.float32(((cmp > 127) != e)[keep].sum()) / np.float32(keep.sum())) * g.kber
            self.bers[hyp] = ber
            if (best == 10 and ber < self.thr) or (best < 10 and ber < best):
                best, self.hyp, self.state, self.invalid = ber, hyp, 1, 0
        return best

    def run(self, soft):
        g = self.g
        nch = soft.size // g.chunk
        vs, vb, out = np.zeros(nch, np.int32), np.zeros(nch, np.float32), []
        c = 0
        while c < nch:
            if not self.state:
                chunk = soft[c * g.chunk:(c + 1) * g.chunk]
                self._lock_test(chunk)
                if not self.state:
                    vs[c], vb[c] = 0, min(self.bers.values())
                    c += 1
                    continue
            # SYNCED from chunk c on: the device decodes the rest of the call at once and replays the lock machine
            n = nch - c
            syms = np.stack([g.symbols(soft[(c + i) * g.chunk:(c + i + 1) * g.chunk], self.hyp) for i in range(n)])
            self.c0 = c
            r = decode_range(g, syms, self.main_start, self.enc, self.spec, self.overlap, rounds=1 << 20)
            self.last, self.last_syms = r, syms
            self._count(r, n)
            acc = 0
            for i in range(n):
                acc = i + 1
                ber = ber_value(g, *r.ber[i])
                if ber > self.thr:
                    self.invalid += 1
                    if self.invalid > self.outsync:
                        self.state = 0
                else:
                    self.invalid = 0
                vs[c + i] = self.state
                vb[c + i] = ber if self.state else min(self.bers.values())
                out.append(r.bits[i])
                if not self.state:
                    break
            self.main_start = int(r.next_start[acc - 1])
            self.enc = enc_tail(r.bits[acc - 1], g.tb)
            c += acc
        bits = np.concatenate(out).astype(np.uint8) if out else np.zeros(0, np.uint8)
        if g.nrzm and bits.size:
            prev = np.concatenate([[self.nrzm_last], bits[:-1]])
            self.nrzm_last = int(bits[-1])
            bits = bits ^ prev
        return dict(bits=bits, vit_state=vs, vit_ber=vb)

    def _count(self, r, n):
        k = self.counters
        k["start_redone"] += r.redone
        k["tb_serial"] += r.tb_serial
        k["misses"].append(r.misses)
        k["tb_first"].append(r.tb_first)
        k["rounds"].append(r.rounds)
        k["redo"].extend(r.redo_chunks)
        k["succ_stale"] += [self.c0 + i for i in r.succ_stale]
        if n > 64:
            self.overlap, self.tb_clean = adapt_window(self.overlap, self.tb_clean, r.tb_first / n, TB_OVERLAP, TB_OVERLAP_MAX)
            self.spec, self.spec_clean = adapt_window(self.spec, self.spec_clean, r.misses / n, self.g.spec_base, self.g.spec_cap)


# ----------------------------------------------------------------------------- stream builders (soft level)
def coded_stream(geom, nchunks, seed, cadu_size=8192, interleave=4, noframes=()):
    """Soft-level transmitter: CADUs (synth.build_cadus) -> NRZ-M when the geometry has it -> k=7 encoder -> MetOp puncturing for r=3/4.
    Returns the coded symbols (0/1), at least nchunks chunks of them. The decoded bits of chunks in `noframes` are random bits with no
    ASM (the Viterbi stays locked while the deframer loses its frames)."""
    from satdump_b200 import synth
    rng = np.random.default_rng(seed)
    nbits = geom.F * (nchunks + 1)
    nfr = nbits // cadu_size + 2
    tx, _ = synth.build_cadus(rng.integers(0, 256, size=(nfr, interleave * 223), dtype=np.uint8), interleave)
    pad = cadu_size // 8 - tx.shape[1]
    if pad:
        tx = np.concatenate([tx, rng.integers(0, 256, size=(nfr, pad), dtype=np.uint8)], axis=1)
    bits = np.unpackbits(tx.reshape(-1))[:nbits]
    for c in noframes:
        bits[c * geom.F:(c + 1) * geom.F] = rng.integers(0, 2, geom.F, dtype=np.uint8)
    if geom.nrzm:
        bits = (np.cumsum(bits.astype(np.int64)) & 1).astype(np.uint8)
    coded = synth.conv_encode(bits)
    return synth.puncture_34_metop(coded) if geom.rate34 else coded


def soft_stream(geom, coded, profile, seed):
    """Maps coded symbols to int8 soft bytes chunk by chunk: profile[c] = (amplitude, noise sigma) of chunk c."""
    rng = np.random.default_rng(seed + 1)
    out = np.empty(len(profile) * geom.chunk, np.int8)
    for c, p in enumerate(profile):
        x = coded[c * geom.chunk:(c + 1) * geom.chunk] * 2.0 - 1
        if p == HALF:  # WEAK first half, GOOD second half
            amp = np.where(np.arange(x.size) < x.size // 2, WEAK[0], GOOD[0])
            sigma = np.where(np.arange(x.size) < x.size // 2, WEAK[1], GOOD[1])
        else:
            amp, sigma = p
        out[c * geom.chunk:(c + 1) * geom.chunk] = np.clip(np.round(x * amp + rng.normal(0, 1, x.size) * sigma), -127, 127)
    return out


# Chunks where the survivors do not merge: soft bytes of +-1 plus noise of the same size. After the reference's `>> 3` the branch metrics
# carry almost no information, so neither the speculation window nor the chainback warm-up pins the state.
WEAK = (1, 1)
GOOD = (40, 20)
# a chunk whose end state speculates right (good second half) while its first half, the part the BER check reads, depends on its start
HALF = "half"


def weak_stretch(geom, nchunks, weak, seed, **kw):
    """Good chunks with the chunks in `weak` replaced by WEAK ones: (soft bytes, coded symbols)."""
    coded = coded_stream(geom, nchunks, seed, **kw)
    return soft_stream(geom, coded, [WEAK if c in weak else GOOD for c in range(nchunks)], seed), coded
