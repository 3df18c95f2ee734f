// Kernels of meteor_lrpt_decoder with m2x_mode false (plugins/meteor_support/meteor/module_meteor_lrpt_decoder.cpp:198-262, the METEOR-M
// LRPT 72k pipeline): Correlator(QPSK, 64-bit ASM) (src-core/common/codings/correlator.cpp) on 16384-soft-byte windows, rotate_soft,
// Viterbi27 (one chained CCDecoder call per frame: the Viterbi kernels of fec.cuh), NRZ-M, derandomiser, inversion, RS(255,223) I=4 in
// the conventional basis. Included by api_meteor.cu only.
//   k_hard_pack<1> (walk.cuh) the hard bits soft > 0 of the FIFO, MSB first in 32-bit words (the correlator's hard_buf)
//   k_meteor_corr    the correlation (64 - Hamming distance) of the 8 syncwords at every even position + the maxima of 32-position blocks
//   Corr64Window     the module's window for k_frame_walk (walk.cuh): the position-0 early accept, else the first maximum
//   k_meteor_gather  the walked frames, rotate_soft applied, one after the other: the chunks the Viterbi kernels decode
//   k_meteor_frames  one CTA per frame: repack, NRZ-M, derandomiser, inversion, RS, CADU 1D CF FC 1D + bytes 4 .. 1023
#pragma once
#include "fec.cuh"
#include "walk.cuh"

namespace b200
{

constexpr int METEOR_F = 16384;               // soft bytes per frame (ENCODED_FRAME_SIZE)
constexpr int METEOR_BITS = METEOR_F / 2;     // Viterbi27(8192): decoded bits per frame
constexpr int METEOR_CADU = 1024;             // FRAME_SIZE
constexpr int METEOR_NPOS = (METEOR_F / 8 - 8) * 4; // even offsets 0 .. 16318 the correlator scans (i < length / 8 - 8, ii = 0, 2, 4, 6)
constexpr int METEOR_RS_I = 4;
constexpr int METEOR_EARLY = 45;              // position 0 is taken by the first syncword whose correlation exceeds this
constexpr uint32_t METEOR_SYNC_OUT = 0x1DCFFC1Du; // what the module writes in front of bytes 4 .. 1023 (its sync[] = 1d cf fc 1d)

// Correlator's QPSK syncwords (correlator.cpp:54-63), built on the host: rotate_64(asm, p) for p = 0..3, then rotate_64(~swapIQ(asm), p).
// Word p means phase p % 4 and swap = (p / 4) == 0 (:146-147, :164-165).
struct MeteorSync { unsigned long long w[8]; };

// 64 hard bits starting at bit `b` of the packed FIFO (MSB first)
__device__ __forceinline__ unsigned long long meteor_word(const uint32_t *__restrict__ hw, long b)
{
    const long w = b >> 5;
    const int o = (int)(b & 31);
    const unsigned long long x = (unsigned long long)hw[w] << 32 | hw[w + 1];
    return o ? x << o | hw[w + 2] >> (32 - o) : x;
}

// Score of every even position 2q, q < nq: the best corr_64 (correlator.cpp:28-35) of the 8 syncwords with the 64 hard bits there and the
// first syncword that reaches it. Block b's maximum over q = 32b .. 32b+31 (first index on ties) for every complete block (k_dump_corr's
// layout, dump.cuh). Indices are half positions.
__global__ void __launch_bounds__(256) k_meteor_corr(const uint32_t *__restrict__ hw, long nq, const MeteorSync sw, float *__restrict__ score,
                                                      unsigned char *__restrict__ best_sync, float *__restrict__ bval, int *__restrict__ bidx)
{
    const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
    int best = -1, p = 0;
    if (q < nq) {
        const unsigned long long word = meteor_word(hw, 2 * q);
#pragma unroll
        for (int s = 0; s < 8; s++) {
            const int c = 64 - __popcll(word ^ sw.w[s]);
            if (c > best) { best = c; p = s; }
        }
        score[q] = (float)best;
        best_sync[q] = (unsigned char)p;
    }
    float v = q < nq ? (float)best : -INFINITY;
    int vi = (int)q;
    first_max_warp(v, vi);
    const long b = q >> 5;
    if ((threadIdx.x & 31) == 0 && (b + 1) * 32 <= nq) {
        bval[b] = v;
        bidx[b] = vi;
    }
}

// The module's correlator on the window at w0 for k_frame_walk (walk.cuh), by one warp:
//   - position 0 first: the first syncword whose correlation there exceeds 45 gives pos 0 at once (not necessarily the best one);
//   - otherwise the first maximum over the even offsets 0 .. 16318, all of whose 64 bits lie inside the window (no tail, unlike
//     Correlator32).
// The module then moves the window by pos (memmove of F - pos bytes, pos new ones read behind): the frame is the F stream bytes from the
// window start + pos. Offsets are even. Syncword p means phase p % 4 and swap = p < 4.
struct Corr64Window
{
    const uint32_t *hw;
    const float *score;
    const unsigned char *best_sync;
    const float *bval;
    const int *bidx;
    MeteorSync sw;

    __device__ __forceinline__ WalkCand operator()(long w0) const
    {
        const unsigned long long first = meteor_word(hw, w0);
        int early = -1, c = 0;
#pragma unroll
        for (int s = 0; s < 8; s++) {
            const int cs = 64 - __popcll(first ^ sw.w[s]);
            if (early < 0 && cs > METEOR_EARLY) { early = s; c = cs; }
        }
        if (early >= 0)
            return WalkCand{0, (float)c, (early & 3) | (early < 4) << 2};
        float v;
        int vi;
        window_first_max(score, bval, bidx, w0 >> 1, METEOR_NPOS, v, vi);
        const int p = best_sync[vi];
        return WalkCand{2 * vi - (int)w0, v, (p & 3) | (p < 4) << 2};
    }
    __device__ static int shift(int pos, int F) { return pos != 0 && pos < F ? pos : 0; }
};

// Frame f of the walk, rotate_soft(phase, swap) applied (rot_soft), at out + f * F: the chunks of the Viterbi kernels. Grid (F / 1024, nf),
// four soft bytes (two symbols) per thread.
__global__ void __launch_bounds__(256) k_meteor_gather(const int8_t *__restrict__ soft, const WalkFrame *__restrict__ frames, int8_t *__restrict__ out)
{
    const WalkFrame r = frames[blockIdx.y];
    const int k = 4 * (blockIdx.x * blockDim.x + threadIdx.x);
    const int8_t *f = soft + r.off;
    char4 v;
    v.x = (int8_t)rot_soft(f, k, r.phase, r.swap);
    v.y = (int8_t)rot_soft(f, k + 1, r.phase, r.swap);
    v.z = (int8_t)rot_soft(f, k + 2, r.phase, r.swap);
    v.w = (int8_t)rot_soft(f, k + 3, r.phase, r.swap);
    reinterpret_cast<char4 *>(out + (size_t)blockIdx.y * METEOR_F)[k >> 2] = v;
}

// One CTA per frame (256 threads) over the Viterbi output of frame f (8192 bits, MSB first, at bits + f * bit_words): the 1024 bytes
// (Viterbi27's repack), NRZMDiff::decode when nrzm (bit k ^= bit k-1; bit -1 of frame 0 is `nrzm_in`, the last bit of the previous push),
// derand_ccsds on bytes 4 .. 1023, every byte inverted when byte 9 is then 0xFF, decode_interlaved(I = 4, conventional basis) on bytes
// 4 .. 1023, and the CADU 1D CF FC 1D + bytes 4 .. 1023 at out + f * 1024. rs_err[4 f + i]: -1 or corrections.
__global__ void __launch_bounds__(256) k_meteor_frames(const uint32_t *__restrict__ bits, int bit_words, int nrzm, int nrzm_in,
                                                        const RsTables *__restrict__ gtab, uint8_t *__restrict__ out, int *__restrict__ rs_err)
{
    __shared__ __align__(16) RsTables T;
    __shared__ __align__(16) uint8_t frame[METEOR_CADU];
    __shared__ __align__(16) uint8_t work[METEOR_RS_I * 704];
    __shared__ int inverted;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < (int)sizeof(RsTables) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(&T)[i] = reinterpret_cast<const uint32_t *>(gtab)[i];
    const uint32_t *b = bits + (size_t)blockIdx.x * bit_words;
    // word t = bytes 4t .. 4t+3
    uint32_t w = b[t];
    if (nrzm) {
        uint32_t prev; // (its last bit is the one before the word's first)
        if (t > 0) prev = b[t - 1];
        else if (blockIdx.x > 0) prev = (b - bit_words)[METEOR_BITS / 32 - 1];
        else prev = (uint32_t)nrzm_in;
        w ^= (w >> 1) | (prev << 31);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int i = 4 * t + j;
        uint8_t v = (uint8_t)(w >> (24 - 8 * j));
        if (i >= 4)
            v ^= T.pn[(i - 4) % 255];
        frame[i] = v;
    }
    __syncthreads();
    if (t == 0)
        inverted = frame[9] == 0xFF;
    __syncthreads();
    if (inverted)
        reinterpret_cast<uint32_t *>(frame)[t] ^= 0xFFFFFFFFu;
    __syncthreads();
    if (warp < METEOR_RS_I) {
        const FrameCfg fc{METEOR_CADU, METEOR_CADU * 8, 1, 0, 4, METEOR_RS_I, 0, 32, 112, METEOR_SYNC_OUT, 0};
        const int err = rs_decode_interleave(T, frame, fc, work + warp * 704, warp, lane);
        if (lane == 0) rs_err[(long)blockIdx.x * METEOR_RS_I + warp] = err;
    }
    __syncthreads();
    uint32_t *o = reinterpret_cast<uint32_t *>(out + (size_t)blockIdx.x * METEOR_CADU);
    o[t] = t == 0 ? __byte_perm(METEOR_SYNC_OUT, 0u, 0x0123u) : reinterpret_cast<const uint32_t *>(frame)[t];
}

} // namespace b200
