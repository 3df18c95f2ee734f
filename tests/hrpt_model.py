"""A numpy model of the GPU decomposition of the HRPT deframers (satdump_b200/csrc/hrpt.cuh, api_hrpt.cu), checked against the reference on
the CPU: per push, the hard bits of the soft FIFO, the candidate bitmap (windows within thr of the sync or its complement: NOAA thr, METEOR
2), the frame-level walk over it with the windows the bitmap cannot judge computed directly (NOAA's splices of the stale shifter after a
frame, METEOR's windows of mixed inversion after a state-2 timeout), the gathered output, and the FIFO keeping an open frame or 63 bits."""
import numpy as np

from oracle._checker import pieces

NOAA_WORDS, NOAA_DATA_BITS, NOAA_SYNC, NOAA_MASK = 11090, 11084 * 10, 0x0A116FD719D83C95, (1 << 60) - 1
NOAA_FIXED = np.array([0x284, 0x16F, 0x35C, 0x19D, 0x20F, 0x095], np.uint16)
MH_ASM, MH_DATA_BITS, MH_PERIOD, MH_S2_LIMIT = 0x1ACFFC1D, 8160, 8192, 5 * 1024 * 8
NONE = -(1 << 50)


def _pop(x):
    return bin(x).count("1")


class Model:
    def __init__(self, meteor, thr=0):
        self.meteor, self.thr = meteor, thr
        self.fifo = np.zeros(0, np.uint8)
        self.base = 0
        self.next, self.open, self.open_inv, self.open_done = 0, NONE, 0, 0
        self.stale, self.stale_end = 0, NONE
        self.state, self.inv, self.good, self.sep, self.s2, self.inv_old, self.inv_at = 0, 0, 0, 0, 0, 0, NONE
        self.units = 0

    def win(self, p, n):
        """the n-bit window ending at FIFO bit p (bits before the FIFO read 0)"""
        a = max(0, p - n + 1)
        v = 0
        for b in self.fifo[a:p + 1]:
            v = (v << 1) | int(b)
        return v

    def cands(self, h):
        L, word = (32, MH_ASM) if self.meteor else (60, NOAA_SYNC)
        thr = 2 if self.meteor else self.thr
        pad = np.concatenate([np.zeros(L - 1, np.uint8), h])
        sb = np.array([(word >> (L - 1 - k)) & 1 for k in range(L)], np.uint8)
        d = np.zeros(h.size, np.int32)
        for k in range(L):
            d += pad[k:k + h.size] != sb[k]
        return np.flatnonzero((d <= thr) | (L - d <= thr))

    def push(self, soft):
        self.fifo = np.concatenate([self.fifo, (np.asarray(soft, np.int8) > 0).astype(np.uint8)])
        have = self.fifo.size
        cand = self.cands(self.fifo)
        recs, segs = [], []
        (self._noaa if not self.meteor else self._meteor)(have, cand, recs, segs)
        out = []
        for s, inv, first, count in segs:
            if self.meteor:
                body = np.packbits(self.fifo[s + 1:s + 1 + MH_DATA_BITS] ^ inv)
                out.append(np.concatenate([np.array([0x1A, 0xCF, 0xFC, 0x1D], np.uint8), body])[None])
            else:
                nd = max(0, first + count - 6)  # data words up to the last one written
                w = np.concatenate([NOAA_FIXED, (self.fifo[s + 1:s + 1 + 10 * nd].reshape(-1, 10).astype(np.uint16)
                                                 @ (1 << np.arange(9, -1, -1)).astype(np.uint16)) ^ (0x3FF if inv else 0)])
                out.append(w[first:first + count].astype(np.uint16))
        keep_from = have - 63
        if self.open != NONE:
            keep_from = min(keep_from, self.open + 1 - self.base)
        used = max(0, keep_from)
        self.fifo = self.fifo[used:]
        self.base += used
        empty = np.zeros((0, 1024), np.uint8) if self.meteor else np.zeros(0, np.uint16)
        return dict(out=np.concatenate(out) if out else empty, recs=np.array(recs, np.int64).reshape(-1, 3),
                    stats=dict(units=self.units, state=self.state))

    def _scan(self, cand, p, lim):
        i = np.searchsorted(cand, p)
        return int(cand[i]) if i < cand.size and cand[i] <= lim else -1

    def _noaa(self, have, cand, recs, segs):
        base, thr = self.base, self.thr

        def emit(s, inv, first):
            last = min(NOAA_WORDS, 6 + (have - 1 - s) // 10)
            if last > first:
                segs.append((s, inv, first, last - first))
                self.units += last - first
            return last

        p = self.next - base
        if self.open != NONE:
            last = emit(self.open - base, self.open_inv, self.open_done)
            if last < NOAA_WORDS:
                self.open_done = last
                return
            self.stale_end, self.open = self.open + NOAA_DATA_BITS, NONE
            p = self.stale_end + 1 - base
        while p < have:
            hit, se = -1, self.stale_end - base
            while p <= min(se + 59, have - 1):  # splice windows
                j = p - se
                w = ((self.stale << j) | (self.win(p, j))) & NOAA_MASK
                if _pop(w ^ NOAA_SYNC) <= thr or _pop(w ^ NOAA_SYNC ^ NOAA_MASK) <= thr:
                    hit = p
                    break
                p += 1
            if hit < 0:
                hit = self._scan(cand, p, have - 1)
                if hit < 0:
                    p = have
                    break
                w = self.win(hit, 60)
            inv = 0 if _pop(w ^ NOAA_SYNC) <= thr else 1
            recs.append((hit + base, inv, 0))
            self.stale = w
            last = emit(hit, inv, 0)
            if last < NOAA_WORDS:
                self.open, self.open_inv, self.open_done = hit + base, inv, last
                p = have
                break
            self.stale_end = hit + base + NOAA_DATA_BITS
            p = hit + NOAA_DATA_BITS + 1
        self.next = max(p, have) + base

    def _mwin(self, q):
        w = self.win(q, 32) ^ (0xFFFFFFFF if self.inv else 0)
        d = q - (self.inv_at - self.base)
        if self.inv_old != self.inv and d < 32:
            w ^= 0xFFFFFFFF if d <= 0 else (0xFFFFFFFF << d) & 0xFFFFFFFF
        return w

    def _meteor(self, have, cand, recs, segs):
        base = self.base
        p = self.next - base
        if self.open != NONE:
            s = self.open - base
            if s + MH_DATA_BITS >= have:
                return
            segs.append((s, self.open_inv, 0, 1024))
            self.units += 1
            self.open = NONE
        while p < have:
            hit = -1
            if self.state in (6, 12):
                if _pop(self._mwin(p) ^ MH_ASM) <= self.state:
                    hit = p
                else:
                    if self.state == 12:
                        self.state, self.good, self.sep = 6, 0, 0
                    else:
                        self.sep += 1
                        if self.sep == 2:
                            self.state, self.s2, self.good, self.sep = 2, 0, 0, 0
                    p += 1
                    continue
            else:
                p0 = p
                timeout = p0 + (MH_S2_LIMIT - self.s2) - 1
                lim = min(have - 1, timeout) if self.state == 2 else have - 1

                def ok(w):
                    return (w == MH_ASM or w == MH_ASM ^ 0xFFFFFFFF) if self.state == 0 else _pop(w ^ MH_ASM) <= 2

                mlim = min(lim, self.inv_at - base + 31) if self.inv_old != self.inv else -1
                while p <= mlim:  # windows of mixed inversion
                    if ok(self._mwin(p)):
                        hit = p
                        break
                    p += 1
                while hit < 0 and p <= lim:
                    c = self._scan(cand, p, lim)
                    if c < 0:
                        p = lim + 1
                        break
                    if ok(self._mwin(c)):
                        hit = c
                    else:
                        p = c + 1
                if hit < 0:
                    if self.state == 2 and timeout <= have - 1:
                        self.state, self.inv_old, self.inv, self.inv_at, self.good, self.sep = 0, self.inv, 0, timeout + base, 0, 0
                        p = timeout + 1
                        continue
                    if self.state == 2:
                        self.s2 += have - p0
                    p = have
                    break
            frm = self.state
            if self.state == 0:
                w = self._mwin(hit)
                self.inv_old, self.inv, self.inv_at = self.inv, 0 if w == MH_ASM else 1, hit + base
                self.state, self.good, self.sep = 6, 0, 0
            elif self.state == 2:
                self.state, self.good, self.sep = 6, 0, 0
            elif self.state == 6:
                self.good += 1
                if self.good == 5:
                    self.state, self.good = 12, 0
            recs.append((hit + base, self.inv, frm))
            if hit + MH_DATA_BITS < have:
                segs.append((hit, self.inv, 0, 1024))
                self.units += 1
            else:
                self.open, self.open_inv = hit + base, self.inv
            p = hit + MH_PERIOD
        self.next = max(p, have) + base


def run_pieces(soft, cuts=(), meteor=False, thr=0):
    """As oracle.hrpt.run_pieces"""
    m = Model(meteor, thr)
    out, recs, stats = [], [], []
    for a, b in pieces(soft.size, cuts):
        r = m.push(soft[a:b])
        out.append(r["out"])
        recs.append(r["recs"])
        stats.append(r["stats"])
    return dict(out=np.concatenate(out), recs=np.concatenate(recs), stats=stats)
