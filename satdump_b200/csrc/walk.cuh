// What the correlator-driven decoders (ccsds_ldpc_decoder, ccsds_turbo_decoder) share: the frame records of the frame walk (k_ldpc_walk in
// ldpc.cuh, launched by frame_walk() in api_ldpc.cu) and the first-maximum reductions over correlator scores. Device helpers and types
// only, so that more than one translation unit may include it.
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
