// The NOAA GAC and DMSP RTD decoders (noaa_gac_decoder: module_noaa_gac_decoder.cpp:65-102; dmsp_rtd_decoder: dmsp_deframer.cpp:24-111):
// serial bit machines without FEC, behind hard bits soft > 0.
//   GAC runs the BPSK_CCSDS_Deframer walk of the convolutional decoders (k_deframe, k_frames with 6 bits of padding) over a bit FIFO that
//   k_gac_bits fills; k_gac_post then reverses each frame's bits (backward playback) and XORs the PN bytes.
//   DMSP is replayed at frame level like the HRPT machines: k_sync_cand (hrpt.cuh) marks the exact 13-bit sync words, one warp walks the
//   machine (k_dmsp_walk) and k_dmsp_gather writes the 19-byte frames. Positions are FIFO bit indices; the carried state is in stream bits.
// Device code and types only; included after hrpt.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200
{

constexpr int GAC_BITS = 33270, GAC_BYTES = 4159, GAC_PN_ZERO = 60, GAC_PN_LEN = 1023;
constexpr unsigned GAC_SYNC = 0xA116FD71u, GAC_SYNC_BACKWARD = 0x33C3E4A6u;
constexpr int DMSP_BITS = 150, DMSP_BYTES = 19, DMSP_ASM_BITS = 13, DMSP_PAY = DMSP_BITS - DMSP_ASM_BITS;
constexpr unsigned DMSP_ASM = 0x159Fu, DMSP_MASK = 0x1FFFu; // 0b1010110011111

// ---------------------------------------------------------------- GAC
// Soft bytes -> hard bits soft > 0, MSB first into the bit FIFO from bit fifo_bits0 (the bits in front of it in the first word are kept).
// One warp writes one word.
__global__ void __launch_bounds__(256) k_gac_bits(const int8_t *__restrict__ soft, long nbits, uint32_t *__restrict__ fifo, long fifo_bits0)
{
    const int lane = threadIdx.x & 31;
    const long w0 = fifo_bits0 >> 5, w1 = (fifo_bits0 + nbits + 31) >> 5;
    const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
    for (long w = w0 + ((long)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < w1; w += nwarps) {
        const long j = (w << 5) - fifo_bits0 + lane;
        const bool in = j >= 0 && j < nbits;
        const bool bit = in && soft[j] > 0;
        const uint32_t v = __brev(__ballot_sync(0xffffffffu, bit)), mask = __brev(__ballot_sync(0xffffffffu, in));
        if (lane == 0)
            fifo[w] = mask == 0xffffffffu ? v : ((fifo[w] & ~mask) | v);
    }
}

// One CTA per 4159-byte frame, in place. backward (module :84-95): output bit ii (written MSB first into byte ii / 8, the last byte
// right-aligned like write_bit) is bit inv = 33269 - ii of the frame's byte image read MSB first, so the right-aligned last byte gives
// its two zero bits first. Then every byte is XORed with the PN byte (module :55-63, :97-98), the partial last byte included.
__global__ void __launch_bounds__(256) k_gac_post(uint8_t *__restrict__ frames, int backward, const uint8_t *__restrict__ pn)
{
    __shared__ uint8_t img[GAC_BYTES + 1];
    uint8_t *frm = frames + (long)blockIdx.x * GAC_BYTES;
    for (int i = threadIdx.x; i < GAC_BYTES; i += blockDim.x)
        img[i] = frm[i];
    __syncthreads();
    for (int i = threadIdx.x; i < GAC_BYTES; i += blockDim.x) {
        uint8_t b = img[i];
        if (backward) {
            const int n = min(8, GAC_BITS - 8 * i); // bits written into this byte
            unsigned v = 0;
            for (int k = 0; k < n; k++) {
                const int inv = GAC_BITS - 1 - (8 * i + k);
                v = (v << 1) | ((img[inv >> 3] >> (7 - (inv & 7))) & 1u);
            }
            b = (uint8_t)v;
        }
        frm[i] = b ^ pn[i];
    }
}

// ---------------------------------------------------------------- DMSP
struct DmspRec { long long bit; int inverted, state; }; // the sync's last bit (FIFO bits in a walk, stream bits on the host)
struct DmspOut { int nrec, nseg; };
// The machine between pushes (stream bits)
struct DmspState
{
    long long next;  // the next position tested
    long long open;  // the sync of the frame still being written, or HRPT_NONE
    int open_inv;
    int state, inv, good, bad; // 0 NOSYNC / 2 SYNCING / 6 SYNCED, bit_inversion, d_good_asm, d_invalid_asm
};

__device__ __forceinline__ unsigned dmsp_win(const uint32_t *__restrict__ hw, long long p) { return (unsigned)hrpt_win64(hw, p) & DMSP_MASK; }

// DMSP's machine over FIFO bits [0, have) (stream bit base + i). An accepted sync at s is followed by the frame's 137 bits, complete at
// s + 137, and the next test is at s + 150. NOSYNC searches the bitmap of exact syncs (either polarity); SYNCING tests one position,
// within 1 bit (< 2), a failure tests the next bit; SYNCED tests 128 frames ahead at once, within 5 bits (< 6), and one failure drops to
// NOSYNC at the next bit. Every accepted sync is a record and, once complete, a frame. One warp; every lane runs the same control flow.
__global__ void __launch_bounds__(32) k_dmsp_walk(const uint32_t *__restrict__ hw, const uint32_t *__restrict__ cand, long long have, long long base,
                                                  DmspState *__restrict__ st, DmspRec *__restrict__ recs, DmspRec *__restrict__ segs,
                                                  DmspOut *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    DmspState S = *st;
    int nrec = 0, nseg = 0;
    long long p = S.next - base;
    if (S.open != HRPT_NONE) {
        const long long s = S.open - base;
        if (s + DMSP_PAY >= have) // (p stays on the test after it)
            goto done;
        if (lane == 0)
            segs[nseg] = DmspRec{s, S.open_inv, 0};
        nseg++;
        S.open = HRPT_NONE;
    }
    while (p < have) {
        if (S.state == 6) {
            constexpr int G = 4;
            const unsigned want = S.inv ? DMSP_ASM ^ DMSP_MASK : DMSP_ASM;
            unsigned pm[G], cm[G];
#pragma unroll
            for (int g = 0; g < G; g++) {
                const long long e = p + (long long)(lane + 32 * g) * DMSP_BITS;
                const bool pass = e < have && __popc(dmsp_win(hw, e) ^ want) < 6;
                pm[g] = __ballot_sync(0xffffffffu, pass);
                cm[g] = __ballot_sync(0xffffffffu, pass && e + DMSP_PAY < have);
            }
            int n = 0, m = 0;
            bool nrun = true, mrun = true;
#pragma unroll
            for (int g = 0; g < G; g++) {
                if (nrun) {
                    const int k = pm[g] == 0xffffffffu ? 32 : __ffs(~pm[g]) - 1;
                    n += k;
                    nrun = k == 32;
                }
                if (mrun) {
                    const int k = cm[g] == 0xffffffffu ? 32 : __ffs(~cm[g]) - 1;
                    m += k;
                    mrun = k == 32;
                }
            }
            m = min(m, n);
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int f = lane + 32 * g;
                const long long e = p + (long long)f * DMSP_BITS;
                if (f < n)
                    recs[nrec + f] = DmspRec{e, S.inv, 6};
                if (f < m)
                    segs[nseg + f] = DmspRec{e, S.inv, 6};
            }
            nrec += n;
            nseg += m;
            const long long e_n = p + (long long)n * DMSP_BITS;
            if (m < n) { // accepted, its bits still arriving (n == m + 1: the next test lies beyond the FIFO)
                S.open = p + (long long)m * DMSP_BITS + base;
                S.open_inv = S.inv;
                p = e_n;
                break;
            }
            if (n == 32 * G || e_n >= have) {
                p = e_n;
                continue;
            }
            S.state = 0; // hard NOSYNC (dmsp_deframer.cpp:94-98)
            S.good = S.bad = 0;
            p = e_n + 1;
            continue;
        }
        long long hit = -1;
        const int from = S.state;
        if (S.state == 2) {
            const unsigned want = S.inv ? DMSP_ASM ^ DMSP_MASK : DMSP_ASM;
            if (__popc(dmsp_win(hw, p) ^ want) < 2) {
                hit = p;
                S.bad = 0;
                if (++S.good > 10)
                    S.state = 6;
            } else {
                S.good = 0;
                if (++S.bad > 2)
                    S.state = 0;
                p++;
                continue;
            }
        } else {
            while (p < have) {
                const long long c = hrpt_scan(cand, p, have - 1);
                if (c < 0) {
                    p = have;
                    break;
                }
                const unsigned w = dmsp_win(hw, c);
                if (w == DMSP_ASM || w == (DMSP_ASM ^ DMSP_MASK)) {
                    hit = c;
                    S.inv = w != DMSP_ASM;
                    S.state = 2;
                    S.good = S.bad = 0;
                    break;
                }
                p = c + 1;
            }
            if (hit < 0)
                break;
        }
        if (lane == 0)
            recs[nrec] = DmspRec{hit, S.inv, from};
        nrec++;
        if (hit + DMSP_PAY < have) {
            if (lane == 0)
                segs[nseg] = DmspRec{hit, S.inv, 0};
            nseg++;
        } else {
            S.open = hit + base;
            S.open_inv = S.inv;
        }
        p = hit + DMSP_BITS;
    }
done:
    if (lane == 0) {
        S.next = max(p, have) + base;
        *st = S;
        *out = DmspOut{nrec, nseg};
    }
}

// One thread per frame byte: frame bit k < 13 is the clean sync's, bit k >= 13 the stream bit sync + k - 12 XOR the inversion; bytes
// MSB first, the last one holding bits 144 .. 149 right-aligned.
__global__ void __launch_bounds__(256) k_dmsp_gather(const uint32_t *__restrict__ hw, const DmspRec *__restrict__ segs, long nseg, uint8_t *__restrict__ out)
{
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nseg * DMSP_BYTES)
        return;
    const long f = t / DMSP_BYTES;
    const int j = (int)(t - f * DMSP_BYTES);
    const DmspRec g = segs[f];
    const int n = min(8, DMSP_BITS - 8 * j);
    unsigned v = 0;
    for (int k = 8 * j; k < 8 * j + n; k++) {
        const unsigned b = k < DMSP_ASM_BITS ? (DMSP_ASM >> (DMSP_ASM_BITS - 1 - k)) & 1u
                                             : ((unsigned)hrpt_win64(hw, g.bit + k - (DMSP_ASM_BITS - 1)) & 1u) ^ (unsigned)g.inverted;
        v = (v << 1) | b;
    }
    out[t] = (uint8_t)v;
}

} // namespace b200
