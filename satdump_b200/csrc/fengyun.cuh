// FengYun-3 decoder kernels (sm_90a): the branch split in front of the two Viterbis and the FengYun differential decoder behind them.
//   fengyun_ahrpt_decoder: two Viterbi3_4 (fymode) (plugins/fengyun3_support/fengyun3/module_fengyun_ahrpt_decoder.cpp:42-136)
//   fengyun_mpt_decoder:   two Viterbi1_2, phases 0 / 90 (plugins/fengyun3_support/fengyun3/module_fengyun_mpt_decoder.cpp:42-135)
//   FengyunDiff::work2     plugins/fengyun3_support/fengyun3/diff.cpp:45-74
#pragma once
#include "fec.cuh"

namespace b200
{

constexpr int FY_READ = 16384;               // soft bytes of one module read
constexpr int FY_BRANCH = FY_READ / 2;       // soft bytes of one branch per read (one Viterbi work call)
constexpr int FY_BITS = FY_BRANCH * 3 / 4;   // bits one Viterbi3_4 call returns (6144)
constexpr int FY_MPT_BITS = FY_BRANCH / 2;   // bits one Viterbi1_2 call returns (4096)

// Reads r of the n at `soft` into the two branch streams, FY_BRANCH bytes per read each. The bytes past the read's end (shift = 1) are 0.
// MPT = false (AHRPT): rotate_soft(buf, 16384, PHASE_0, true) (-128 -> -127, I and Q of every pair swapped), then
//   i_soft[i] = buf[(i + shift) * 2], q_soft[i] = buf[(i + shift) * 2 + 1] (~ when invert_q). The branch bytes are stored with the two
//   bytes of every odd pair of the call exchanged: through the MetOp depuncture with I/Q swap = puncturing shift (k_vit_idle<true>,
//   VitHyp{shift, 0, shift}) that is FengYun's "110" depuncture (viterbi_3_4.cpp:55-76) exactly.
// MPT = true: the same split with q_soft always complemented, then rotate_soft(branch, 8192, PHASE_0, true) on each branch (module
//   :61-70): branch byte k of I is clamp(b[2 ((k ^ 1) + shift) + 1]), of Q clamp(~clamp(b[2 ((k ^ 1) + shift)])), stored as they are
//   for the rate-1/2 decoder (VitHyp{0, phase, shift}); invert_q is not read.
template <bool MPT>
__global__ void k_fy_split(const int8_t *__restrict__ soft, long n, int shift, int invert_q, int8_t *__restrict__ ib, int8_t *__restrict__ qb)
{
    const long total = n * FY_BRANCH;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long r = t / FY_BRANCH;
        const int k = (int)(t - r * FY_BRANCH);
        const int i = (MPT || ((k >> 1) & 1)) ? (k ^ 1) : k; // the branch byte stored at k
        const int8_t *b = soft + r * FY_READ;
        const int j = (i + shift) * 2;
        int vi = 0, vq = 0;
        if (j < FY_READ) {
            vi = b[j + 1]; // (swapped)
            vq = b[j];
            if (vi == -128) vi = -127;
            if (vq == -128) vq = -127;
        }
        ib[t] = (int8_t)vi;
        if (MPT) {
            const int v = (int8_t)~vq;
            qb[t] = (int8_t)(v == -128 ? -127 : v);
        } else
            qb[t] = (int8_t)(invert_q ? ~vq : vq);
    }
}

// bit k (MSB first) of chunk q of a Viterbi's chunk_bits
__device__ __forceinline__ int fy_bit(const uint32_t *__restrict__ bits, int bit_words, int q, int k)
{
    return (bits[(long)q * bit_words + (k >> 5)] >> (31 - (k & 31))) & 1;
}

// FengyunDiff::work2(in1, in2, BITS) over the reads `reads[0 .. nr)` (chunk indices of both Viterbis' chunk_bits; BITS = FY_BITS for
// AHRPT, FY_MPT_BITS for MPT), in1 = branch 2 (Q) and in2 = branch 1 (I), exchanged when `invert`; (x0, y0) = the carried Xin >> 1, Yin.
// Pair p gives the two bits (x != y) ? (yp ^ y, xp ^ x) : (xp ^ x, yp ^ y), written MSB first into the bit FIFO from bit fifo_bits0
// (2 BITS bits per read).
template <int BITS>
__global__ void k_fy_diff(const uint32_t *__restrict__ b1, const uint32_t *__restrict__ b2, int bit_words, const int *__restrict__ reads, int nr,
                          int invert, int x0, int y0, uint32_t *__restrict__ fifo, long fifo_bits0)
{
    const uint32_t *in1 = invert ? b1 : b2, *in2 = invert ? b2 : b1;
    const long total = (long)nr * 2 * BITS;
    const long w0 = fifo_bits0 >> 5, w1 = (fifo_bits0 + total + 31) >> 5;
    for (long w = w0 + (long)blockIdx.x * blockDim.x + threadIdx.x; w < w1; w += (long)gridDim.x * blockDim.x) {
        const long o0 = (w << 5) - fifo_bits0; // output bit of this word's MSB (may be negative in the first word)
        uint32_t v = 0, mask = 0;
        for (int b = 0; b < 32; b++) {
            const long o = o0 + b;
            if (o < 0 || o >= total)
                continue;
            const long p = o >> 1;
            const int a = (int)(p / BITS), k = (int)(p - (long)a * BITS), q = reads[a];
            const int x = fy_bit(in1, bit_words, q, k), y = fy_bit(in2, bit_words, q, k);
            int xp = x0, yp = y0;
            if (k > 0) {
                xp = fy_bit(in1, bit_words, q, k - 1);
                yp = fy_bit(in2, bit_words, q, k - 1);
            } else if (a > 0) {
                xp = fy_bit(in1, bit_words, reads[a - 1], BITS - 1);
                yp = fy_bit(in2, bit_words, reads[a - 1], BITS - 1);
            }
            const int hi = (x != y) ? (yp ^ y) : (xp ^ x), lo = (x != y) ? (xp ^ x) : (yp ^ y);
            v |= (uint32_t)((o & 1) ? lo : hi) << (31 - b);
            mask |= 1u << (31 - b);
        }
        fifo[w] = (mask == 0xffffffffu) ? v : ((fifo[w] & ~mask) | (v & mask));
    }
}
} // namespace b200
