// What the correlator-driven decoders (ccsds_ldpc_decoder, ccsds_turbo_decoder, metop_dump_decoder) share: the frame records of the frame
// walk (k_ldpc_walk in ldpc.cuh, launched by frame_walk() in api_ldpc.cu; k_dump_walk in dump.cuh), the first-maximum reductions over
// correlator scores and rotate_soft. Device helpers and types only, so that more than one translation unit may include it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct LdpcFrameRec { long long off; int pos; float cor; int phase, swap, corr, pad; };
struct LdpcWalkOut { long long next; int nf, shifted; };

constexpr int WALK_SWAP_ONLY = -1; // k_ldpc_walk's `constellation` for the turbo correlator: its table index is the sign (swap), no phase

// (value, index) of a maximum, first index on ties: the order in which the correlator's strict '>' keeps its best
__device__ __forceinline__ void ldpc_best(float &v, int &i, float v2, int i2)
{
    if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}
__device__ __forceinline__ void ldpc_best_warp(float &v, int &i)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        ldpc_best(v, i, v2, i2);
    }
}

// first maximum of the scores over window [a, a + npos), by one warp: the partial blocks at both ends position by position, the
// complete blocks through their maxima
__device__ __forceinline__ void ldpc_window_max(const float *__restrict__ score, const float *__restrict__ bval, const int *__restrict__ bidx, long a,
                                int npos, float &v, int &vi)
{
    const int lane = threadIdx.x & 31;
    const long e = a + npos;
    const long b0 = (a + 31) >> 5, b1 = e >> 5;
    v = -INFINITY;
    vi = 0x7fffffff;
    const long h = a + lane;
    if (h < (b0 << 5) && h < e) ldpc_best(v, vi, score[h], (int)h);
    for (long b = b0 + lane; b < b1; b += 32) ldpc_best(v, vi, bval[b], bidx[b]);
    const long t = (b1 << 5) + lane;
    if (b1 >= b0 && t < e) ldpc_best(v, vi, score[t], (int)t);
    ldpc_best_warp(v, vi);
}

// soft byte k (0 .. F-1) of a frame after rotate_soft(phase, swap) (rotation.cpp:4-63)
__device__ __forceinline__ int ldpc_rot(const int8_t *__restrict__ f, int k, int phase, int swap)
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
