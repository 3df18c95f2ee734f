// What the correlator-driven decoders (ccsds_ldpc_decoder, ccsds_turbo_decoder, metop_dump_decoder) share: the frame walk k_frame_walk
// with its records, the first-maximum reductions over correlator scores, CorrWindow (the LDPC and turbo window; the dump window is
// DumpWindow in dump.cuh) and rot_soft. Device code and types only, so that more than one translation unit may include it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct WalkFrame { long long off; int pos; float cor; int phase, swap, corr, pad; };
struct WalkOut { long long next; int nf, shifted; };

// (value, index) of a maximum, first index on ties: the order in which the correlator's strict '>' keeps its best
__device__ __forceinline__ void first_max(float &v, int &i, float v2, int i2)
{
    if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}
__device__ __forceinline__ void first_max_warp(float &v, int &i)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        first_max(v, i, v2, i2);
    }
}

// first maximum of the scores over window [a, a + npos), by one warp: the partial blocks at both ends position by position, the
// complete blocks through their maxima
__device__ __forceinline__ void window_first_max(const float *__restrict__ score, const float *__restrict__ bval, const int *__restrict__ bidx,
                                                 long a, int npos, float &v, int &vi)
{
    const int lane = threadIdx.x & 31;
    const long e = a + npos;
    const long b0 = (a + 31) >> 5, b1 = e >> 5;
    v = -INFINITY;
    vi = 0x7fffffff;
    const long h = a + lane;
    if (h < (b0 << 5) && h < e) first_max(v, vi, score[h], (int)h);
    for (long b = b0 + lane; b < b1; b += 32) first_max(v, vi, bval[b], bidx[b]);
    const long t = (b1 << 5) + lane;
    if (b1 >= b0 && t < e) first_max(v, vi, score[t], (int)t);
    first_max_warp(v, vi);
}

// soft byte k (0 .. F-1) of a frame after rotate_soft(phase, swap) (rotation.cpp:4-63)
__device__ __forceinline__ int rot_soft(const int8_t *__restrict__ f, int k, int phase, int swap)
{
    int vi = f[k & ~1], vq = f[k | 1];
    if (vi == -128) vi = -127;
    if (vq == -128) vq = -127;
    if (swap) { const int t = vi; vi = vq; vq = t; }
    int oi, oq;
    switch (phase) {
    case 1: oi = vq; oq = -vi; break;
    case 2: oi = -vi; oq = -vq; break;
    case 3: oi = -vq; oq = vi; break;
    default: oi = vi; oq = vq; break;
    }
    return (k & 1) ? oq : oi;
}

namespace b200
{

constexpr int WALK_WARPS = 32, WALK_SPEC = 4 * WALK_WARPS; // frames of the current lattice checked per round
constexpr int WALK_SWAP_ONLY = -1; // CorrWindow's `constellation` for the turbo correlator: its table index is the sign (swap), no phase

// What a window tells the walk about its frame: the position the correlator returned (relative to the window's start), its correlation,
// and phase | swap << 2
struct WalkCand { int pos; float cor; int ps; };

// The window of the LDPC and turbo modules (k_ldpc_corr / k_turbo_corr scores, npos positions): pos = the first maximum's offset if it
// is > 0, else 0, and the frame starts there (shift = pos). The phase and swap of the table index (generic_correlator.cpp:233-262 by
// constellation; WALK_SWAP_ONLY: the index is the swap).
struct CorrWindow
{
    const float *score;
    const unsigned char *best_sync;
    const float *bval;
    const int *bidx;
    int npos, constellation;

    __device__ __forceinline__ WalkCand operator()(long w0) const
    {
        float v;
        int vi;
        window_first_max(score, bval, bidx, w0, npos, v, vi);
        const int bs = v > 0.0f ? best_sync[vi] : 0;
        int phase, swap = 0;
        if (constellation == WALK_SWAP_ONLY) { phase = 0; swap = bs; }
        else if (constellation == 0) phase = bs ? 2 : 0;
        else if (constellation == 1) phase = bs;
        else { phase = bs == 0 ? 1 : (bs == 1 ? 3 : (bs == 2 ? 0 : 2)); swap = bs >> 1; }
        return WalkCand{v > 0.0f ? (int)(vi - w0) : 0, v > 0.0f ? v : 0.0f, phase | swap << 2};
    }
    __device__ static int shift(int pos, int F) { return pos; }
};

// The frame walk over the `have` soft bytes of the FIFO, from offset 0, for frames of F soft bytes. Each round checks up to WALK_SPEC
// frames of the current lattice o + jF at once, one warp per window through `win`; thread 0 then takes the frames up to and including
// the first one that Window::shift moves: those are exact, since their windows start where the module would read them (so `win` may
// take w0 = o + jF as the window's start). The walk then continues on the shifted lattice. Without signal every frame shifts, and each
// round takes one frame. A frame whose shifted window leaves fewer than F bytes waits for the next push. Offsets are < 2^31 (the FIFO
// is sized by max_soft). Records: off = window start + shift, pos as the correlator returned it, cor, phase, swap.
template <class Window>
__global__ void __launch_bounds__(WALK_WARPS * 32) k_frame_walk(Window win, long have, int F, WalkFrame *__restrict__ frames, int max_frames,
                                                                WalkOut *__restrict__ out)
{
    __shared__ int s_pos[WALK_SPEC];
    __shared__ float s_cor[WALK_SPEC];
    __shared__ unsigned char s_ps[WALK_SPEC];
    __shared__ long s_o;
    __shared__ int s_nf, s_shifted, s_done;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { s_o = 0; s_nf = 0; s_shifted = 0; s_done = 0; }
    __syncthreads();
    while (!s_done) {
        const long o = s_o;
        const long rest = have - o - F; // (< 2^31: a 32-bit division; F is known only at run time, so a 64-bit one would cost every round)
        const int avail = rest >= 0 ? (int)rest / F + 1 : 0;
        const int n = min(min(avail, WALK_SPEC), max_frames - s_nf);
        for (int j = warp; j < n; j += WALK_WARPS) {
            const WalkCand c = win(o + (long)j * F);
            if (lane == 0) { s_pos[j] = c.pos; s_cor[j] = c.cor; s_ps[j] = (unsigned char)c.ps; }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long oo = o;
            int nf = s_nf;
            bool stop = n == 0;
            for (int j = 0; j < n; j++) {
                const int pos = s_pos[j], shift = Window::shift(pos, F);
                if (shift && oo + shift + F > have) { stop = true; break; }
                WalkFrame r;
                r.off = oo + shift;
                r.pos = pos;
                r.cor = s_cor[j];
                r.phase = s_ps[j] & 3;
                r.swap = s_ps[j] >> 2;
                r.corr = 0;
                r.pad = 0;
                frames[nf++] = r;
                oo = r.off + F;
                if (shift) { s_shifted++; break; }
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

} // namespace b200
