// Kernels of metop_dump_decoder (plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83, the MetOp X-band dump): no
// convolutional code, Correlator32(QPSK, 0x1ACFFC1D) (src-core/common/codings/correlator32.cpp) on 8192-soft-byte windows, RS(255,223) I=4
// dual basis. Included by api_dump.cu only.
//   k_hard_pack<0> (walk.cuh) the hard bits soft >= 0 of the FIFO, MSB first in 32-bit words (the correlator's hard_buf)
//   k_dump_corr    the correlation (32 - Hamming distance) of the 8 syncwords at every even position + the maxima of 32-position blocks
//   DumpWindow     the module's window for k_frame_walk (walk.cuh): the position-0 early accept, the first maximum, the tail past 8192 bits
//   k_dump_frames  one CTA per frame: the module's buffer after the shift, rotate_soft, hard decisions, inversion, derandomiser, RS, CADU
#pragma once
#include "fec.cuh"
#include "walk.cuh"

namespace b200
{

constexpr int DUMP_F = 8192;                // soft bytes per frame (ENCODED_FRAME_SIZE)
constexpr int DUMP_CADU = 1024;             // FRAME_SIZE
constexpr int DUMP_NPOS = DUMP_F / 2 - 15;  // even offsets 0 .. 8160 of a window whose 32 bits lie inside it
constexpr int DUMP_TAIL = 16;               // even offsets 8162 .. 8190 (bits past the window read as zeros) and 8192 (the all-zero word)
constexpr int DUMP_RS_I = 4;
constexpr int DUMP_EARLY = 27;              // position 0 is taken by the first syncword whose correlation exceeds this

// Correlator32's QPSK syncwords (correlator32.cpp:54-63), built on the host: rotate_64(asm, p) for p = 0..3, then
// rotate_64(swapIQ(asm) ^ ~0, p). Word p means phase p % 4 and swap = p < 4 (:145-146, :163-164).
struct DumpSync { uint32_t w[8]; };

// corr_64 (correlator32.cpp:28-35) of the 8 syncwords against `word`: the best value and the first syncword reaching it
__device__ __forceinline__ void dump_best(const DumpSync &sw, uint32_t word, int &best, int &p)
{
    best = -1;
    p = 0;
#pragma unroll
    for (int s = 0; s < 8; s++) {
        const int c = 32 - __popc(word ^ sw.w[s]);
        if (c > best) { best = c; p = s; }
    }
}

// 32 hard bits starting at bit `b` of the packed FIFO (MSB first)
__device__ __forceinline__ uint32_t dump_word(const uint32_t *__restrict__ hw, long b)
{
    const long w = b >> 5;
    const int o = (int)(b & 31);
    return o ? (hw[w] << o) | (hw[w + 1] >> (32 - o)) : hw[w];
}

// Score of every even position 2q, q < nq: the best correlation of the 8 syncwords with the 32 hard bits there and the first syncword that
// reaches it. Block b's maximum over q = 32b .. 32b+31 (first index on ties) for every complete block. Indices are half positions.
__global__ void __launch_bounds__(256) k_dump_corr(const uint32_t *__restrict__ hw, long nq, const DumpSync sw, float *__restrict__ score,
                                                    unsigned char *__restrict__ best_sync, float *__restrict__ bval, int *__restrict__ bidx)
{
    const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
    int best = -1, p = 0;
    if (q < nq) {
        dump_best(sw, dump_word(hw, 2 * q), best, p);
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

// The dump correlator's window at w0 for k_frame_walk (walk.cuh), by one warp:
//   - position 0 first: the first syncword whose correlation there exceeds 27 gives pos 0 at once (not necessarily the best one);
//   - otherwise the first maximum over the even offsets 0 .. 8160, then the window tail: the scan runs over 8184 BYTES of a hard_buf
//     of which only the window's 1024 were written, the rest being the zeros of a fresh allocation, so offsets 8162 .. 8190 see the
//     window's last bits followed by zeros and every offset from 8192 on sees the all-zero word (only 8192 can win under the strict '>').
// A winner at 8192 or later is not shifted (the module's "Safety" test) but its phase and swap apply. Offsets are even. Syncword p
// means phase p % 4 and swap = p < 4.
struct DumpWindow
{
    const uint32_t *hw;
    const float *score;
    const unsigned char *best_sync;
    const float *bval;
    const int *bidx;
    DumpSync sw;

    __device__ __forceinline__ WalkCand operator()(long w0) const
    {
        const int lane = threadIdx.x & 31;
        const uint32_t first = dump_word(hw, w0);
        int early = -1, c = 0;
#pragma unroll
        for (int s = 0; s < 8; s++) {
            const int cs = 32 - __popc(first ^ sw.w[s]);
            if (early < 0 && cs > DUMP_EARLY) { early = s; c = cs; }
        }
        if (early >= 0)
            return WalkCand{0, (float)c, (early & 3) | (early < 4) << 2};
        float v;
        int vi;
        window_first_max(score, bval, bidx, w0 >> 1, DUMP_NPOS, v, vi);
        // the tail: lane l < 15 at offset 8162 + 2l, lane 15 the all-zero word at 8192
        float tv = -INFINITY;
        int ti = 0x7fffffff, tp = 0;
        if (lane < DUMP_TAIL) {
            const int off = 2 * DUMP_NPOS + 2 * lane;
            const int valid = DUMP_F - off; // window bits in the word: 30 .. 2, 0 for the zero word
            const uint32_t word = valid > 0 ? dump_word(hw, w0 + off) & (~0u << (32 - valid)) : 0u;
            int tc;
            dump_best(sw, word, tc, tp);
            tv = (float)tc;
            ti = (int)(w0 >> 1) + DUMP_NPOS + lane;
        }
        const int my_tp = tp;
        first_max_warp(tv, ti);
        tp = __shfl_sync(0xffffffffu, my_tp, (ti - (int)(w0 >> 1) - DUMP_NPOS) & 31);
        const bool tail = tv > v; // (later offsets: only a strictly better value wins)
        const int p = tail ? tp : best_sync[vi];
        return WalkCand{2 * (tail ? ti : vi) - (int)w0, tail ? tv : v, (p & 3) | (p < 4) << 2};
    }
    __device__ static int shift(int pos, int F) { return pos != 0 && pos < F ? pos : 0; }
};

// One CTA per frame (256 threads). The module's buffer after a shift by sh = pos (0 < pos < F; module :50-55: memmove(buf, buf + pos, pos),
// then pos new bytes at the end) holds stream byte off + k at k < sh and k >= F - sh and the stale window byte off - sh + k in between;
// for sh > F/2 the memmove reads past the buffer, but the new bytes overwrite all it wrote (k_turbo_gather's layout). Then rotate_soft
// (phase, swap), hard decisions > 0 packed MSB first, every byte inverted, derand_ccsds on bytes 4 .. 1023, decode_interlaved(I = 4,
// dual basis) on them, and the CADU 1A CF FC 1D + bytes 4 .. 1023, written whatever RS returned. rs_err[4 f + i]: -1 or corrections.
__global__ void __launch_bounds__(256) k_dump_frames(const int8_t *__restrict__ soft, const WalkFrame *__restrict__ frames,
                                                      const RsTables *__restrict__ gtab, uint8_t *__restrict__ out, int *__restrict__ rs_err)
{
    __shared__ __align__(16) RsTables T;
    __shared__ __align__(16) uint8_t frame[DUMP_CADU];
    __shared__ __align__(16) uint8_t work[DUMP_RS_I * 704];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < (int)sizeof(RsTables) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(&T)[i] = reinterpret_cast<const uint32_t *>(gtab)[i];
    const WalkFrame r = frames[blockIdx.x];
    const int sh = r.pos > 0 && r.pos < DUMP_F ? r.pos : 0;
    const int8_t *cur = soft + r.off, *stale = soft + (r.off - sh);
    __syncthreads();
    for (int i = t; i < DUMP_CADU; i += blockDim.x) {
        uint8_t b = 0;
#pragma unroll
        for (int y = 0; y < 8; y += 2) { // (a symbol's two bytes lie in the same piece: sh and F - sh are even)
            const int k = 8 * i + y;
            const int8_t *f = (k < sh || k >= DUMP_F - sh) ? cur : stale;
            b = (uint8_t)(b << 2 | (rot_soft(f, k, r.phase, r.swap) > 0) << 1 | (rot_soft(f, k + 1, r.phase, r.swap) > 0));
        }
        b ^= 0xFF;
        if (i >= 4)
            b ^= T.pn[(i - 4) % 255];
        else
            b = (uint8_t)(0x1ACFFC1Du >> (24 - 8 * i));
        frame[i] = b;
    }
    __syncthreads();
    if (warp < DUMP_RS_I) {
        const FrameCfg fc{DUMP_CADU, DUMP_CADU * 8, 1, 0, 4, DUMP_RS_I, 1, 32, 112, 0x1ACFFC1Du};
        const int err = rs_decode_interleave(T, frame, fc, work + warp * 704, warp, lane);
        if (lane == 0) rs_err[(long)blockIdx.x * DUMP_RS_I + warp] = err;
    }
    __syncthreads();
    uint32_t *o = reinterpret_cast<uint32_t *>(out + (size_t)blockIdx.x * DUMP_CADU);
    o[t] = reinterpret_cast<const uint32_t *>(frame)[t];
}

} // namespace b200
