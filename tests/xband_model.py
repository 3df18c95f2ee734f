"""Bit-serial numpy model of meteor_xband_decoder's decomposition (satdump_b200/csrc/xband.cuh), pinned to the reference by
tests/test_meteor_xband_oracle.py: NRZ-M in closed form, the record candidates of every window start, the record machine walked over the
candidates only, the packet stream with the read of each record, each inner SimpleDeframer as its exact syncs (every sync opens a frame
and cuts the one before it), and the frames ordered by (read, deframer, position)."""
import numpy as np

from satdump_b200 import synth

READ = 8192
PAD = {0: 3071, 1: 12288}
REC = {0: 3072, 1: 12288}
PKT = {0: (46, 48), 1: (188, 192)}
SYNCS = {0: [(0x38FB456A, 32)], 1: [(0xAF5FFF50AA5AA0, 56), (0xAE5EEC61BB7982, 56), (0xAB5BB394EED628, 56)]}
FRM_BITS = {0: 3040, 1: 481280}


def _field(bits, starts, off, n):
    """the n-bit values at bits starts + off .. + n - 1, MSB first"""
    v = np.zeros(starts.size, np.int64)
    for k in range(n):
        v = (v << 1) | bits[starts + off + k]
    return v


def _popcount(v):
    return np.bitwise_count(v.astype(np.uint64)).astype(np.int64)


def records(soft, kind):
    """the accepted records' window starts (padded stream) over the whole reads of `soft`"""
    R = soft.size // READ * READ
    hard = (soft[:R] > 0).astype(np.uint8)
    dec = hard ^ np.concatenate([[0], hard[:-1]]).astype(np.uint8)  # NRZMDiff::decode_bits from lastBit 0
    bits = np.concatenate([np.zeros(PAD[kind], np.uint8), dec]).astype(np.int64)
    w = np.arange(R)
    if kind == 0:
        m = ((_field(bits, w, 0, 8) == 0xB3).astype(int) + (_field(bits, w, 384, 8) == 0xE3) + (_field(bits, w, 768, 8) == 0x75)
             + ((_field(bits, w, 1920, 9) & 0x1FD) == 0))
        cand = np.nonzero(m >= 3)[0]
        out, synced, runs, p = [], False, 0, 0
        for c in cand.tolist():
            if c > p:
                synced, runs = False, min(3, runs + 2 * (c - p))
            runs = min(3, runs + 1)
            if (m[c] == 4) if synced else True:
                out.append(c)
                if not synced and runs > 2:
                    synced, runs = True, 0
            else:
                runs, synced = min(3, runs + 1), False
            p = c + 1
        return bits, np.array(out, np.int64)
    v1 = _field(bits, w, 0, 16) ^ 0x35
    v2 = _field(bits, w, 3056, 32)
    e1, e2 = _popcount(v1), _popcount(v2)
    loose = (e1 < 6) & (e2 < 8)
    strict = (e1 < 1) & (e2 < 3)
    out, synced, p = [], False, 0
    cand = np.nonzero(loose)[0]
    while p < R:
        if synced:
            if loose[p]:
                out.append(p)
                p += REC[1]
            else:
                synced, p = False, p + 1
            continue
        i = np.searchsorted(cand, p)
        nxt = cand[i:][strict[cand[i:]]]
        if nxt.size == 0:
            break
        out.append(int(nxt[0]))
        synced, p = True, int(nxt[0]) + REC[1]
    return bits, np.array(out, np.int64)


def run(soft, kind):
    """the frames (uint8 [n, 380 | 60160]) meteor_xband_decoder writes for the whole reads of `soft`"""
    bits, recs = records(np.asarray(soft, np.int8), kind)
    P, stride = PKT[kind]
    if recs.size == 0:
        return np.zeros((0, FRM_BITS[kind] // 8), np.uint8)
    idx = (recs[:, None] + 8 * (2 + (np.arange(8 * P) // P) * stride + np.arange(8 * P) % P)[None, :])
    byte = np.zeros(idx.shape, np.int64)
    for k in range(8):
        byte = (byte << 1) | bits[idx + k]
    pk = byte.astype(np.uint8).reshape(-1)
    if kind == 0:
        pk ^= 0xAA
    rec_read = recs // READ
    pbits = np.unpackbits(pk).astype(np.int64)
    frames = []
    for d, (sync, n) in enumerate(SYNCS[kind]):
        w = np.arange(n - 1, pbits.size)
        ends = w[_exact(pbits, w, sync, n)]
        span = FRM_BITS[kind] - n
        for i, t in enumerate(ends.tolist()):
            e = t + span
            if i + 1 < ends.size and ends[i + 1] <= e:
                e = int(ends[i + 1])
            elif e >= pbits.size:
                continue
            body = np.zeros(span, np.uint8)
            body[:e - t] = pbits[t + 1:e + 1]
            fb = np.packbits(np.concatenate([(np.array([sync >> (n - 1 - k) & 1 for k in range(n)], np.uint8)), body]))
            if kind == 1:
                fb = synth.kmss_frame_process(fb, d)
            frames.append((int(rec_read[(e // 8) // (8 * P)]), d, e, fb))
    frames.sort(key=lambda f: (f[0], f[1], f[2]))
    return np.stack([f[3] for f in frames]) if frames else np.zeros((0, FRM_BITS[kind] // 8), np.uint8)


def _exact(pbits, w, sync, n):
    """windows of n bits ending at w equal to sync (bits before the stream read 0)"""
    ok = np.ones(w.size, bool)
    for k in range(n):
        ok &= pbits[w - (n - 1) + k] == (sync >> (n - 1 - k) & 1)
    return ok
