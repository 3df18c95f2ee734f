// Kernels of metop_dump_decoder (plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83, the MetOp X-band dump): no
// convolutional code, Correlator32(QPSK, 0x1ACFFC1D) (src-core/common/codings/correlator32.cpp) on 8192-soft-byte windows, RS(255,223) I=4
// dual basis. Included by api_dump.cu only.
//   k_dump_pack    the hard bits soft >= 0 of the FIFO, MSB first in 32-bit words (the correlator's hard_buf)
//   k_dump_corr    the correlation (32 - Hamming distance) of the 8 syncwords at every even position + the maxima of 32-position blocks
//   k_dump_walk    the module's frame walk: the position-0 early accept, the window's first maximum, and the window tail past the 8192 bits
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
constexpr int DUMP_WALK_WARPS = 32, DUMP_WALK_SPEC = 4 * DUMP_WALK_WARPS; // frames of the current lattice checked per round
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

// word w of the hard-bit FIFO = the signs (soft >= 0, correlator32.cpp:75-89) of soft bytes 32w .. 32w+31; bytes at or past `have` are 0
__global__ void __launch_bounds__(256) k_dump_pack(const int8_t *__restrict__ soft, long have, long nwords, uint32_t *__restrict__ hw)
{
    const long j = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned bits = __ballot_sync(0xffffffffu, j < have && soft[j] >= 0);
    if ((threadIdx.x & 31) == 0 && (j >> 5) < nwords)
        hw[j >> 5] = __brev(bits);
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
    ldpc_best_warp(v, vi);
    const long b = q >> 5;
    if ((threadIdx.x & 31) == 0 && (b + 1) * 32 <= nq) {
        bval[b] = v;
        bidx[b] = vi;
    }
}

// The frame walk over the `have` soft bytes of the FIFO from offset 0, k_ldpc_walk's round structure (ldpc.cuh) with what the dump
// correlator adds per window o (one warp per window):
//   - position 0 first: the first syncword whose correlation there exceeds 27 gives pos 0 at once (not necessarily the best one);
//   - otherwise the first maximum over the even offsets 0 .. 8160, then the window tail: the scan runs over 8184 BYTES of a hard_buf
//     of which only the window's 1024 were written, the rest being the zeros of a fresh allocation, so offsets 8162 .. 8190 see the
//     window's last bits followed by zeros and every offset from 8192 on sees the all-zero word (only 8192 can win under the strict '>').
// A winner at 8192 or later is not shifted (the module's "Safety" test) but its phase and swap apply. A frame whose shifted window is
// not complete in the FIFO waits for the next push. Offsets are even and < 2^31. Record: off = window start + shift, pos as the
// correlator returned it, cor, phase, swap.
__global__ void __launch_bounds__(1024) k_dump_walk(const uint32_t *__restrict__ hw, const float *__restrict__ score,
                                                     const unsigned char *__restrict__ best_sync, const float *__restrict__ bval,
                                                     const int *__restrict__ bidx, const DumpSync sw, long have, LdpcFrameRec *__restrict__ frames,
                                                     int max_frames, LdpcWalkOut *__restrict__ out)
{
    __shared__ int s_pos[DUMP_WALK_SPEC], s_cor[DUMP_WALK_SPEC], s_p[DUMP_WALK_SPEC];
    __shared__ long s_o;
    __shared__ int s_nf, s_shifted, s_done;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { s_o = 0; s_nf = 0; s_shifted = 0; s_done = 0; }
    __syncthreads();
    while (!s_done) {
        const long o = s_o;
        const long avail = have >= o + DUMP_F ? (have - o - DUMP_F) / DUMP_F + 1 : 0;
        const int n = (int)min(min(avail, (long)DUMP_WALK_SPEC), (long)(max_frames - s_nf));
        for (int j = warp; j < n; j += DUMP_WALK_WARPS) {
            const long w0 = o + (long)j * DUMP_F;
            const uint32_t first = dump_word(hw, w0);
            int early = -1, c = 0;
#pragma unroll
            for (int s = 0; s < 8; s++) {
                const int cs = 32 - __popc(first ^ sw.w[s]);
                if (early < 0 && cs > DUMP_EARLY) { early = s; c = cs; }
            }
            if (early >= 0) {
                if (lane == 0) { s_pos[j] = 0; s_cor[j] = c; s_p[j] = early; }
                continue;
            }
            float v;
            int vi;
            ldpc_window_max(score, bval, bidx, w0 >> 1, DUMP_NPOS, v, vi);
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
            ldpc_best_warp(tv, ti);
            tp = __shfl_sync(0xffffffffu, my_tp, (ti - (int)(w0 >> 1) - DUMP_NPOS) & 31);
            const bool tail = tv > v; // (later offsets: only a strictly better value wins)
            if (lane == 0) {
                const int wi = tail ? ti : vi;
                s_pos[j] = 2 * wi - (int)w0;
                s_cor[j] = (int)(tail ? tv : v);
                s_p[j] = tail ? tp : best_sync[vi];
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long oo = o;
            int nf = s_nf, j = 0;
            bool stop = n == 0;
            for (; j < n; j++) {
                const int pos = s_pos[j];
                const bool shift = pos != 0 && pos < DUMP_F;
                if (shift && oo + pos + DUMP_F > have) { stop = true; break; }
                LdpcFrameRec r;
                r.off = oo + (shift ? pos : 0);
                r.pos = pos;
                r.cor = (float)s_cor[j];
                r.phase = s_p[j] & 3;
                r.swap = s_p[j] < 4;
                r.corr = 0;
                r.pad = 0;
                frames[nf++] = r;
                oo = r.off + DUMP_F;
                if (shift) { s_shifted++; j++; break; }
            }
            if (n == 0 || nf >= max_frames) stop = true;
            s_o = oo;
            s_nf = nf;
            s_done = stop;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out->next = s_o;
        out->nf = s_nf;
        out->shifted = s_shifted;
    }
}

// One CTA per frame (256 threads). The module's buffer after a shift by sh = pos (0 < pos < F; module :50-55: memmove(buf, buf + pos, pos),
// then pos new bytes at the end) holds stream byte off + k at k < sh and k >= F - sh and the stale window byte off - sh + k in between;
// for sh > F/2 the memmove reads past the buffer, but the new bytes overwrite all it wrote (k_turbo_gather's layout). Then rotate_soft
// (phase, swap), hard decisions > 0 packed MSB first, every byte inverted, derand_ccsds on bytes 4 .. 1023, decode_interlaved(I = 4,
// dual basis) on them, and the CADU 1A CF FC 1D + bytes 4 .. 1023, written whatever RS returned. rs_err[4 f + i]: -1 or corrections.
__global__ void __launch_bounds__(256) k_dump_frames(const int8_t *__restrict__ soft, const LdpcFrameRec *__restrict__ frames,
                                                      const RsTables *__restrict__ gtab, uint8_t *__restrict__ out, int *__restrict__ rs_err)
{
    __shared__ __align__(16) RsTables T;
    __shared__ __align__(16) uint8_t frame[DUMP_CADU];
    __shared__ __align__(16) uint8_t work[DUMP_RS_I * 704];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < (int)sizeof(RsTables) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(&T)[i] = reinterpret_cast<const uint32_t *>(gtab)[i];
    const LdpcFrameRec r = frames[blockIdx.x];
    const int sh = r.pos > 0 && r.pos < DUMP_F ? r.pos : 0;
    const int8_t *cur = soft + r.off, *stale = soft + (r.off - sh);
    __syncthreads();
    for (int i = t; i < DUMP_CADU; i += blockDim.x) {
        uint8_t b = 0;
#pragma unroll
        for (int y = 0; y < 8; y += 2) { // (a symbol's two bytes lie in the same piece: sh and F - sh are even)
            const int k = 8 * i + y;
            const int8_t *f = (k < sh || k >= DUMP_F - sh) ? cur : stale;
            b = (uint8_t)(b << 2 | (ldpc_rot(f, k, r.phase, r.swap) > 0) << 1 | (ldpc_rot(f, k + 1, r.phase, r.swap) > 0));
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
