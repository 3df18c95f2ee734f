// The METEOR-M X-band dump decoder (meteor_xband_decoder: module_meteor_xband_decoder.cpp:62-230), two modes, each a record deframer
// followed by exact-sync SimpleDeframers over the packets the records carry:
//   mtvza      MTVZA_ExtDeframer (meteor_rec_deframer.h:12-105) -> eight 46-byte packets XOR 0xAA per 384-byte record ->
//              SimpleDeframer(0x38FB456A, 32, 3040)
//   kmss_bpsk  RepackBitsByte + KMSS_BPSK_ExtDeframer (:107-261) -> eight 188-byte packets per 1536-byte record -> three
//              SimpleDeframers (56-bit syncs, 481280-bit frames) -> kmssFrameProcessor (XOR 0xF0, four-lane bit de-interleave, one
//              lane pair moved by a byte for deframers 2 and 3)
// Hard bits soft > 0 are packed by k_hard_pack<1> (walk.cuh) and NRZ-M decoded word by word (k_nrzm_words). k_xband_cand marks the record
// windows that could be accepted; one warp walks the record machine over that bitmap (k_xband_rec_walk); k_xband_packets writes the
// accepted records' packets into the packet FIFO; k_sync_cand (hrpt.cuh) marks each inner deframer's sync words there; one warp per inner
// deframer walks its frames (k_xband_inner_walk); k_mtvza_frames / k_kmss_frames write them.
// Positions: the record deframers see a stream of PAD zero bits (their zeroed shift buffers) and then the decoded bits; a record test is
// named by its window's first bit in that padded stream, w, and it belongs to the soft byte w of the stream (mtvza: the test runs when
// bit w + PAD arrives; kmss_bpsk: when the byte holding it does), hence to read w / 8192. Device code and types only; included after
// hrpt.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200
{

constexpr int XB_READ = 8192;                       // BUFFER_SIZE: the module's read
constexpr int MTVZA_PAD = 3071, MTVZA_REC = 3072;  // the window ends at the newest bit
constexpr int KMSS_PAD = 12288, KMSS_REC = 12288;  // the window starts 1536 bytes behind the newest byte
constexpr int MTVZA_PKT = 46, KMSS_PKT = 188;      // packet bytes, eight per record at byte 2 + k * 48 (mtvza) | 192 (kmss_bpsk)
constexpr int MTVZA_FRM = 380, KMSS_FRM = 60160;   // inner frame bytes (3040 / 481280 bits, sync included)
constexpr int KMSS_LANE = 15040;
constexpr unsigned MTVZA_SYNC = 0x38FB456Au;
__host__ __device__ __forceinline__ unsigned long long kmss_sync(int d)
{
    return d == 0 ? 0xAF5FFF50AA5AA0ull : (d == 1 ? 0xAE5EEC61BB7982ull : 0xAB5BB394EED628ull);
}

struct XbRec { long long w; };                     // an accepted record: its window's first bit (padded stream)
struct XbState { long long next; int synced, runs; }; // the record machine between pushes (mtvza's runs_since_sync saturates at 3)
// An inner frame: its sync's last bit t and the last stream bit e it holds (t + frame bits - sync bits, or the bit of the sync that cut
// it: the rest is zero), in packet-stream bits; `read` is the module read of the record that brought bit e.
struct XbFrame { long long t, e; unsigned read; int d; };
struct XbInner { long long next, open; };          // an inner deframer between pushes: the next position tested, the open frame's sync
struct XbOut { int nrec, nfrm[3]; };

// decoded bit q = hard bit q XOR hard bit q - 1 (NRZMDiff::decode_bits); bit 0 of the FIFO is the carried lastBit and decodes to nothing
__global__ void __launch_bounds__(256) k_nrzm_words(const uint32_t *__restrict__ hw, long nwords, uint32_t *__restrict__ db)
{
    const long w = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w < nwords)
        db[w] = hw[w] ^ ((hw[w] >> 1) | (w ? hw[w - 1] << 31 : 0u));
}

// MTVZA_ExtDeframer's four patterns in the window starting at FIFO bit q: bits 0, 384, 768 (8 bits each) and 1920 .. 1926 + 1928
__device__ __forceinline__ int mtvza_matches(const uint32_t *__restrict__ db, long long q)
{
    return ((hrpt_win64(db, q + 7) & 0xFF) == 0xB3) + ((hrpt_win64(db, q + 384 + 7) & 0xFF) == 0xE3) +
           ((hrpt_win64(db, q + 768 + 7) & 0xFF) == 0x75) + ((hrpt_win64(db, q + 1928) & 0x1FD) == 0);
}

// KMSS_BPSK_ExtDeframer's bit errors: 16 bits at the window start against 0x0035, 32 bits at byte 382 against 0
__device__ __forceinline__ void kmss_errors(const uint32_t *__restrict__ db, long long q, int &e1, int &e2)
{
    e1 = __popcll((hrpt_win64(db, q + 15) & 0xFFFF) ^ 0x35);
    e2 = __popcll(hrpt_win64(db, q + 3087) & 0xFFFFFFFFull);
}

// bit q of cand (q in [1, qend)) = the window starting at FIFO bit q passes the loose test: mtvza >= 3 patterns, kmss_bpsk the synced
// thresholds (sync1 < 6, sync2 < 8); the strict tests are a subset, checked by the walk
__global__ void __launch_bounds__(256) k_xband_cand(const uint32_t *__restrict__ db, long long qend, int kmss, uint32_t *__restrict__ cand)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (q >= 1 && q < qend) {
        if (kmss) {
            int e1, e2;
            kmss_errors(db, q, e1, e2);
            hit = e1 < 6 && e2 < 8;
        } else {
            hit = mtvza_matches(db, q) >= 3;
        }
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && q < qend)
        cand[q >> 5] = b;
}

// The record machine over the window starts [S.next, lim) (padded stream; FIFO bit q = w - base). One warp.
//   mtvza: every bit is a test. A window matching all four patterns, or at least three while not synced, is a record; it makes the
//     machine synced when runs_since_sync (+1 per test, +1 more per failed test) exceeds 2, and a failed test clears synced. Between two
//     candidates every test fails: synced clears and runs grows by 2 per test.
//   kmss_bpsk: synced, the test right after a record's 12287 skipped tests accepts the loose thresholds; otherwise only the strict ones
//     (sync1 < 1, sync2 < 3) accept. A failed test clears synced; a record skips the next 12287 tests.
__global__ void __launch_bounds__(32) k_xband_rec_walk(const uint32_t *__restrict__ db, const uint32_t *__restrict__ cand, long long base,
                                                       long long lim, int kmss, XbState *__restrict__ st, XbRec *__restrict__ recs,
                                                       int cap, XbOut *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    XbState S = *st;
    int nrec = 0;
    long long p = S.next;
    while (p < lim) {
        if (kmss && S.synced) {
            if (cand[(p - base) >> 5] >> ((p - base) & 31) & 1) {
                if (lane == 0 && nrec < cap)
                    recs[nrec] = XbRec{p};
                nrec++;
                p += KMSS_REC;
            } else {
                S.synced = 0;
                p++;
            }
            continue;
        }
        const long long c = hrpt_scan(cand, p - base, lim - 1 - base);
        const long long hit = c < 0 ? lim : c + base;
        if (!kmss && hit > p) {
            S.synced = 0;
            S.runs = (int)min(3LL, S.runs + 2 * (hit - p));
        }
        if (c < 0) {
            p = lim;
            break;
        }
        if (kmss) {
            int e1, e2;
            kmss_errors(db, c, e1, e2);
            if (e1 < 1 && e2 < 3) {
                if (lane == 0 && nrec < cap)
                    recs[nrec] = XbRec{hit};
                nrec++;
                S.synced = 1;
                p = hit + KMSS_REC;
            } else {
                p = hit + 1;
            }
            continue;
        }
        const int m = mtvza_matches(db, c);
        S.runs = min(3, S.runs + 1);
        if (S.synced ? m == 4 : m >= 3) {
            if (lane == 0 && nrec < cap)
                recs[nrec] = XbRec{hit};
            nrec++;
            if (!S.synced && S.runs > 2) {
                S.synced = 1;
                S.runs = 0;
            }
        } else {
            S.runs = min(3, S.runs + 1);
            S.synced = 0;
        }
        p = hit + 1;
    }
    if (lane == 0) {
        S.next = p;
        *st = S;
        out->nrec = nrec;
    }
}

// One thread per packet byte of the accepted records, appended to the packet FIFO from byte pk0. The FIFO is a bit stream in 32-bit
// words MSB first (as hrpt_win64 reads it), so byte j is stored at j ^ 3. The first thread of a record notes its read.
__global__ void __launch_bounds__(256) k_xband_packets(const uint32_t *__restrict__ db, long long base, const XbRec *__restrict__ recs,
                                                       int nrec, int kmss, uint8_t *__restrict__ pk, long pk0, uint32_t *__restrict__ pk_read,
                                                       long rec0)
{
    const int P = kmss ? KMSS_PKT : MTVZA_PKT, stride = kmss ? 192 : 48, NPB = 8 * P;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)nrec * NPB)
        return;
    const int k = (int)(t / NPB), b = (int)(t - (long)k * NPB);
    const long long w = recs[k].w;
    const int fb = 2 + (b / P) * stride + b % P;
    uint8_t v = (uint8_t)(hrpt_win64(db, w - base + 8 * fb + 7) & 0xFF);
    if (!kmss)
        v ^= 0xAA;
    pk[(pk0 + t) ^ 3] = v;
    if (b == 0)
        pk_read[rec0 + k] = (unsigned)(w / XB_READ);
}

// SimpleDeframer (threshold 0, bit by bit) over packet-stream bits [S.next, have) (FIFO bit u = stream bit u + pbase): every exact sync
// starts a frame; the frame open before it is cut there (its bits up to the sync's last bit, then zeros) unless it completed first.
// One warp per deframer (blockIdx.x); cand holds that deframer's bitmap at cand + blockIdx.x * cwords.
__global__ void __launch_bounds__(32) k_xband_inner_walk(const uint32_t *__restrict__ pk, const uint32_t *__restrict__ cand, long cwords,
                                                         long long have, long long pbase, int kmss, const uint32_t *__restrict__ pk_read,
                                                         XbInner *__restrict__ st, XbFrame *__restrict__ frames, int cap,
                                                         XbOut *__restrict__ out)
{
    const int lane = threadIdx.x & 31, d = blockIdx.x;
    const int NPB = 8 * (kmss ? KMSS_PKT : MTVZA_PKT);
    const unsigned long long sync = kmss ? kmss_sync(d) : MTVZA_SYNC, mask = kmss ? (1ull << 56) - 1 : 0xFFFFFFFFull;
    const long long span = kmss ? 481280 - 56 : 3040 - 32; // a frame's bits after the sync
    const uint32_t *cd = cand + d * cwords;
    XbFrame *fr = frames + (long)d * cap;
    XbInner S = st[d];
    int n = 0;
    long long u = S.next - pbase;
    auto emit = [&](long long e) {
        if (lane == 0 && n < cap) {
            const long long byte = (e - pbase) >> 3;
            fr[n] = XbFrame{S.open, e, pk_read[byte / NPB], d};
        }
        n++;
    };
    for (;;) {
        long long c = -1;
        while (u < have) {
            c = hrpt_scan(cd, u, have - 1);
            if (c < 0 || (hrpt_win64(pk, c) & mask) == sync)
                break;
            u = c + 1;
            c = -1;
        }
        if (S.open != HRPT_NONE) {
            const long long end = S.open + span - pbase;
            if (c >= 0 && c <= end) {
                emit(c + pbase);
            } else if (end < have) {
                emit(end + pbase);
                S.open = HRPT_NONE;
            } else {
                u = have;
                break;
            }
        }
        if (c < 0) {
            u = have;
            break;
        }
        S.open = c + pbase;
        u = c + 1;
    }
    if (lane == 0) {
        S.next = u + pbase;
        st[d] = S;
        out->nfrm[d] = n;
    }
}

// byte j of an inner frame before kmssFrameProcessor: the clean sync, then the stream bits after it up to e, zero after e
__device__ __forceinline__ unsigned xb_frame_byte(const uint32_t *__restrict__ pk, long long pbase, const XbFrame &f, int j, int sbytes,
                                                  unsigned long long sync)
{
    if (j < sbytes)
        return (unsigned)(sync >> (8 * (sbytes - 1 - j))) & 0xFF;
    const long long first = f.t + 1 + 8LL * (j - sbytes);
    const long long nv = min(8LL, f.e - first + 1);
    if (nv <= 0)
        return 0;
    const unsigned v = (unsigned)(hrpt_win64(pk, first + 7 - pbase) & 0xFF);
    return v & (0xFFu << (8 - nv)) & 0xFF;
}

// mtvza: one thread per byte of the frames frames[0 .. n) (in output order), written from out
__global__ void __launch_bounds__(256) k_mtvza_frames(const uint32_t *__restrict__ pk, long long pbase, const XbFrame *__restrict__ frames,
                                                      long n, uint8_t *__restrict__ out)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * MTVZA_FRM)
        return;
    const long k = t / MTVZA_FRM;
    out[t] = (uint8_t)xb_frame_byte(pk, pbase, frames[k], (int)(t - k * MTVZA_FRM), 4, MTVZA_SYNC);
}

// kmss_bpsk: one thread per output byte of the frames listed by `order` (indices into `frames`), kmssFrameProcessor fused: lane o byte c
// takes bits 7 - o and 3 - o of frame bytes 4c .. 4c + 3 (XOR 0xF0); deframer 2 moves lanes 2 and 3, deframer 3 lanes 0 and 1, one byte
// right (byte 0 stays)
__global__ void __launch_bounds__(256) k_kmss_frames(const uint32_t *__restrict__ pk, long long pbase, const XbFrame *__restrict__ frames,
                                                     const int *__restrict__ order, long n, uint8_t *__restrict__ out)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * KMSS_FRM)
        return;
    const long k = t / KMSS_FRM;
    const int r = (int)(t - k * KMSS_FRM), o = r / KMSS_LANE;
    int c = r - o * KMSS_LANE;
    const XbFrame f = frames[order[k]];
    if (c > 0 && ((f.d == 1 && o >= 2) || (f.d == 2 && o < 2)))
        c--;
    unsigned v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const unsigned b = xb_frame_byte(pk, pbase, f, 4 * c + i, 7, kmss_sync(f.d)) ^ 0xF0;
        v = (v << 2) | ((b >> (7 - o)) & 1) << 1 | ((b >> (3 - o)) & 1);
    }
    out[t] = (uint8_t)v;
}

} // namespace b200
