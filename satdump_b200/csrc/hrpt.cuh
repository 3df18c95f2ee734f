// The NOAA and METEOR HRPT deframers (noaa_hrpt_decoder: noaa_deframer.cpp:42-117; meteor_hrpt_decoder: meteor/deframer.cpp:57-230):
// serial bit machines without FEC, replayed at frame level. k_sync_cand marks every bit position whose window is close to the sync word
// or its complement; one warp then walks the machine over that bitmap (k_noaa_walk, k_meteor_hrpt_walk), jumping a whole frame at a
// time in lock, and the gathers write the frames it accepted. Positions are FIFO bit indices (one soft byte = one bit); the carried
// state is in stream bits. Device code and types only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200
{

constexpr int NOAA_WORDS = 11090, NOAA_SYNC_WORDS = 6, NOAA_DATA_BITS = (NOAA_WORDS - NOAA_SYNC_WORDS) * 10, NOAA_SPLICE = 59;
constexpr unsigned long long NOAA_SYNC = 0x0A116FD719D83C95ull, NOAA_MASK = 0x0FFFFFFFFFFFFFFFull;
constexpr int MH_CADU = 1024, MH_DATA_BITS = (MH_CADU - 4) * 8, MH_PERIOD = MH_CADU * 8, MH_S2_LIMIT = 5 * 1024 * 8;
constexpr unsigned MH_ASM = 0x1ACFFC1Du;
constexpr long long HRPT_NONE = -(1LL << 50);

struct HrptRec { long long bit; int inverted, state; }; // the layout of b200_hrpt_frame
// What a gather writes: NOAA words [first, first + count) of the frame whose sync ends at FIFO bit `sync` (METEOR: the whole CADU), at
// output unit `out` of the push
struct HrptSeg { long long sync, out; int inv, first, count, pad; };
struct HrptOut { int nrec, nseg; long long units; };
// The machine between pushes (stream bits)
struct HrptState
{
    long long next;      // the next position tested
    long long open;      // the sync of the frame still being written, or HRPT_NONE
    int open_inv, open_done; // its inversion; NOAA: its words already written
    unsigned long long stale; // NOAA: the window that matched last (the shifter stays on it while SYNCED) ...
    long long stale_end;      // ... and the last bit of its frame: the windows ending at stale_end + 1 .. + 59 are splices
    int state, inv, good, sep, s2; // METEOR: state 0 / 2 / 6 / 12, bit_inversion, good, sep_errors, state_2_bits_count
    int inv_old;         // METEOR: bit_inversion before its last change ...
    long long inv_at;    // ... at the test at this position: the 31 windows after it mix the two
};

// the 64 hard bits ending at FIFO bit p, MSB first; bits before the FIFO's start read 0
__device__ __forceinline__ unsigned long long hrpt_win64(const uint32_t *__restrict__ hw, long long p)
{
    const long long k = p >> 5;
    const int s = 31 - (int)(p & 31);
    const unsigned long long w0 = hw[k], w1 = k >= 1 ? hw[k - 1] : 0u, w2 = k >= 2 ? hw[k - 2] : 0u;
    const unsigned long long lo = (w1 << 32) | w0;
    return s ? (lo >> s) | (w2 << (64 - s)) : lo;
}

// bit p of cand (LSB first within a word) = the `mask`-wide window ending at p is within thr bits of `word` or of its complement
__global__ void __launch_bounds__(256) k_sync_cand(const uint32_t *__restrict__ hw, long long nbits, unsigned long long word,
                                                   unsigned long long mask, int thr, uint32_t *__restrict__ cand)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (p < nbits) {
        const unsigned long long w = hrpt_win64(hw, p) & mask;
        hit = __popcll(w ^ word) <= thr || __popcll(w ^ word ^ mask) <= thr;
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && p < nbits)
        cand[p >> 5] = b;
}

// The first candidate in [p, lim] (lim < have), or -1: one warp, 1024 positions per step
__device__ __forceinline__ long long hrpt_scan(const uint32_t *__restrict__ cand, long long p, long long lim)
{
    const int lane = threadIdx.x & 31;
    while (p <= lim) {
        const long long w0 = p >> 5, wi = w0 + lane;
        unsigned c = 0;
        if (wi <= (lim >> 5)) {
            c = cand[wi];
            if (wi == w0)
                c &= ~0u << (p & 31);
            if (wi == (lim >> 5) && (lim & 31) != 31)
                c &= (2u << (lim & 31)) - 1;
        }
        const unsigned b = __ballot_sync(0xffffffffu, c != 0);
        if (b) {
            const int l = __ffs(b) - 1;
            const unsigned cl = __shfl_sync(0xffffffffu, c, l);
            return (w0 + l) * 32 + __ffs(cl) - 1;
        }
        p = (w0 + 32) * 32;
    }
    return -1;
}

// NOAA: the words of the frame with sync at FIFO bit s, from `first`, that are complete in the FIFO; true when the frame is complete
__device__ __forceinline__ bool noaa_emit(long long s, int inv, int first, long long have, HrptSeg *segs, int &nseg, long long &units,
                                          int &last)
{
    last = (int)min((long long)NOAA_WORDS, NOAA_SYNC_WORDS + (have - 1 - s) / 10);
    if (last > first) {
        if ((threadIdx.x & 31) == 0)
            segs[nseg] = HrptSeg{s, units, inv, first, last - first, 0};
        nseg++;
        units += last - first;
    }
    return last == NOAA_WORDS;
}

// NOAA's machine over FIFO bits [0, have) (stream bit base + i): IDLE tests every window; a window within thr of the sync (else of its
// complement: inverted) emits the six fixed words and 11084 data words (10 bits each, XOR the inversion), then IDLE again. While SYNCED the
// shifter stands still, so the 59 windows after a frame splice the matched window with the new bits: those are tested directly, all
// others through the bitmap. One warp; every lane runs the same control flow.
__global__ void __launch_bounds__(32) k_noaa_walk(const uint32_t *__restrict__ hw, const uint32_t *__restrict__ cand, long long have, long long base,
                                                  int thr, HrptState *__restrict__ st, HrptRec *__restrict__ recs, HrptSeg *__restrict__ segs,
                                                  HrptOut *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    HrptState S = *st;
    int nrec = 0, nseg = 0, last;
    long long units = 0, p = S.next - base;
    if (S.open != HRPT_NONE) {
        const long long s = S.open - base;
        if (!noaa_emit(s, S.open_inv, S.open_done, have, segs, nseg, units, last)) {
            S.open_done = last;
            p = have;
            goto done;
        }
        S.stale_end = S.open + NOAA_DATA_BITS;
        S.open = HRPT_NONE;
        p = S.stale_end + 1 - base;
    }
    while (p < have) {
        long long hit = -1;
        unsigned long long win = 0;
        const long long se = S.stale_end - base, slim = min(se + NOAA_SPLICE, have - 1), p_in = p;
        for (; p <= slim; p += 32) {
            const long long q = p + lane;
            unsigned long long w = 0;
            bool ok = false;
            if (q <= slim) {
                const int j = (int)(q - se);
                w = ((S.stale << j) | (hrpt_win64(hw, q) & ((1ull << j) - 1))) & NOAA_MASK;
                ok = __popcll(w ^ NOAA_SYNC) <= thr || __popcll(w ^ NOAA_SYNC ^ NOAA_MASK) <= thr;
            }
            const unsigned b = __ballot_sync(0xffffffffu, ok);
            if (b) {
                const int l = __ffs(b) - 1;
                hit = p + l;
                win = __shfl_sync(0xffffffffu, w, l);
                break;
            }
        }
        if (hit < 0) {
            if (p_in <= slim)
                p = slim + 1;
            hit = hrpt_scan(cand, p, have - 1);
            if (hit < 0) {
                p = have;
                break;
            }
            win = hrpt_win64(hw, hit) & NOAA_MASK;
        }
        const int inv = __popcll(win ^ NOAA_SYNC) <= thr ? 0 : 1;
        if (lane == 0)
            recs[nrec] = HrptRec{hit + base, inv, 0};
        nrec++;
        S.stale = win;
        if (!noaa_emit(hit, inv, 0, have, segs, nseg, units, last)) {
            S.open = hit + base;
            S.open_inv = inv;
            S.open_done = last;
            p = have;
            break;
        }
        S.stale_end = hit + base + NOAA_DATA_BITS;
        p = hit + NOAA_DATA_BITS + 1;
    }
done:
    if (lane == 0) {
        S.next = max(p, have) + base;
        *st = S;
        *out = HrptOut{nrec, nseg, units};
    }
}

// METEOR: the 32-bit shifter at FIFO bit q: each bit XOR the inversion current when it arrived (inv, or inv_old up to FIFO bit ia)
__device__ __forceinline__ unsigned mh_window(const uint32_t *__restrict__ hw, long long q, int inv, int inv_old, long long ia)
{
    unsigned w = (unsigned)hrpt_win64(hw, q) ^ (inv ? 0xffffffffu : 0u);
    const long long d = q - ia; // the top 32 - d bits arrived at or before ia
    if (inv_old != inv && d < 32)
        w ^= d <= 0 ? 0xffffffffu : ~0u << d;
    return w;
}

// METEOR's machine over FIFO bits [0, have). Frames: an accepted ASM at s is followed by 8160 written bits; the next test is at s + 8192.
// States 6 and 12 test one position; a failure tests the next bit. States 0 and 2 search: through the bitmap (distance <= 2 to the ASM or
// its complement, then checked exactly), except the windows after a state-2 timeout that still hold inverted bits, tested directly.
__global__ void __launch_bounds__(32) k_meteor_hrpt_walk(const uint32_t *__restrict__ hw, const uint32_t *__restrict__ cand, long long have,
                                                         long long base, HrptState *__restrict__ st, HrptRec *__restrict__ recs,
                                                         HrptSeg *__restrict__ segs, HrptOut *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    HrptState S = *st;
    int nrec = 0, nseg = 0;
    long long units = 0, p = S.next - base;
    if (S.open != HRPT_NONE) {
        const long long s = S.open - base;
        if (s + MH_DATA_BITS >= have) // (p stays on the test after it)
            goto done;
        if (lane == 0)
            segs[nseg] = HrptSeg{s, units, S.open_inv, 0, MH_CADU, 0};
        nseg++;
        units++;
        S.open = HRPT_NONE;
    }
    while (p < have) {
        long long hit = -1;
        if (S.state == 6 || S.state == 12) {
            const unsigned w = mh_window(hw, p, S.inv, S.inv_old, S.inv_at - base);
            if (__popc(w ^ MH_ASM) <= S.state) {
                hit = p;
            } else {
                if (S.state == 12) {
                    S.state = 6;
                    S.good = S.sep = 0;
                } else if (++S.sep == 2) {
                    S.state = 2;
                    S.s2 = 0;
                    S.good = S.sep = 0;
                }
                p++;
                continue;
            }
        } else {
            const long long p0 = p, lim = S.state == 2 ? min(have - 1, p + (MH_S2_LIMIT - S.s2) - 1) : have - 1;
            const long long iaf = S.inv_at - base;
            if (S.inv_old != S.inv) { // (state 0 right after a timeout) the windows holding bits of both inversions
                const long long mlim = min(lim, iaf + 31), p_in = p;
                for (; p <= mlim; p += 32) {
                    const long long q = p + lane;
                    bool ok = false;
                    if (q <= mlim) {
                        const unsigned w = mh_window(hw, q, S.inv, S.inv_old, iaf);
                        ok = S.state == 0 ? (w == MH_ASM || w == ~MH_ASM) : __popc(w ^ MH_ASM) <= 2;
                    }
                    const unsigned b = __ballot_sync(0xffffffffu, ok);
                    if (b) {
                        hit = p + __ffs(b) - 1;
                        break;
                    }
                }
                if (hit < 0 && p_in <= mlim)
                    p = mlim + 1;
            }
            while (hit < 0 && p <= lim) {
                const long long c = hrpt_scan(cand, p, lim);
                if (c < 0) {
                    p = lim + 1;
                    break;
                }
                const unsigned w = mh_window(hw, c, S.inv, S.inv_old, iaf);
                if (S.state == 0 ? (w == MH_ASM || w == ~MH_ASM) : __popc(w ^ MH_ASM) <= 2)
                    hit = c;
                else
                    p = c + 1;
            }
            if (hit < 0) {
                const long long timeout = p0 + (MH_S2_LIMIT - S.s2) - 1; // state 2: the test that makes state_2_bits_count reach the limit
                if (S.state == 2 && timeout <= have - 1) {
                    S.state = 0;
                    S.inv_old = S.inv;
                    S.inv = 0;
                    S.inv_at = timeout + base;
                    S.good = S.sep = 0;
                    p = timeout + 1;
                    continue;
                }
                if (S.state == 2)
                    S.s2 += (int)(have - p0);
                p = have;
                break;
            }
        }
        // accept at hit
        const int from = S.state;
        if (S.state == 0) {
            const unsigned w = mh_window(hw, hit, S.inv, S.inv_old, S.inv_at - base);
            S.inv_old = S.inv;
            S.inv = w == MH_ASM ? 0 : 1;
            S.inv_at = hit + base;
            S.state = 6;
            S.good = S.sep = 0;
        } else if (S.state == 2) {
            S.state = 6;
            S.good = S.sep = 0;
        } else if (S.state == 6 && ++S.good == 5) {
            S.state = 12;
            S.good = 0;
        }
        if (lane == 0)
            recs[nrec] = HrptRec{hit + base, S.inv, from};
        nrec++;
        if (hit + MH_DATA_BITS < have) {
            if (lane == 0)
                segs[nseg] = HrptSeg{hit, units, S.inv, 0, MH_CADU, 0};
            nseg++;
            units++;
        } else {
            S.open = hit + base;
            S.open_inv = S.inv;
        }
        p = hit + MH_PERIOD;
    }
done:
    if (lane == 0) {
        S.next = max(p, have) + base;
        *st = S;
        *out = HrptOut{nrec, nseg, units};
    }
}

// NOAA: one thread per output word: the six fixed words, then 10 bits MSB first XOR the inversion, as uint16
__global__ void __launch_bounds__(256) k_noaa_gather(const uint32_t *__restrict__ hw, const HrptSeg *__restrict__ segs, uint16_t *__restrict__ out)
{
    const HrptSeg g = segs[blockIdx.y];
    const int i = g.first + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.first + g.count)
        return;
    uint16_t v;
    if (i < NOAA_SYNC_WORDS) {
        const uint16_t fixed[NOAA_SYNC_WORDS] = {0x284, 0x16F, 0x35C, 0x19D, 0x20F, 0x095};
        v = fixed[i];
    } else {
        v = (uint16_t)((hrpt_win64(hw, g.sync + (long long)(i - NOAA_SYNC_WORDS + 1) * 10) & 0x3FF) ^ (g.inv ? 0x3FF : 0));
    }
    out[g.out + i - g.first] = v;
}

// METEOR: one thread per CADU byte: the clean ASM, then 8 bits MSB first XOR the inversion
__global__ void __launch_bounds__(256) k_meteor_hrpt_gather(const uint32_t *__restrict__ hw, const HrptSeg *__restrict__ segs, uint8_t *__restrict__ out)
{
    const HrptSeg g = segs[blockIdx.y];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    uint8_t v;
    if (j < 4)
        v = (uint8_t)(MH_ASM >> (24 - 8 * j));
    else
        v = (uint8_t)((hrpt_win64(hw, g.sync + (long long)(j - 3) * 8) & 0xFF) ^ (g.inv ? 0xFF : 0));
    out[g.out * MH_CADU + j] = v;
}

} // namespace b200
