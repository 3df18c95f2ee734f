// Kernels of ccsds_turbo_decoder (module_ccsds_turbo_decoder.cpp:137-235, CCSDSTurbo::decode and the deepspace-turbo log-MAP BCJR).
// Included by api_turbo.cu only. The frame walk is k_ldpc_walk (ldpc.cuh), launched through frame_walk() of api_ldpc.cu.
//   k_turbo_corr    the module's correlator: |dot(soft[i .. i+ASM-1] / 127, asm table)| and its sign at every position + block maxima
//   k_turbo_gather  the frame as the module's buffer holds it (shift quirk), derand_ccsds_soft, / 127, sign fix, depuncturing, and the
//                   serial-to-parallel split into the upper and lower code streams; the a-priori values start at log(0.5)
//   k_turbo_rec     the backward and the forward recursion of convcode_extrinsic for one component code, stored per step
//   k_turbo_ext     the extrinsic values of every step (new a-priori values) and, in the last lower pass, the deinterleaved decisions
//   k_turbo_pack    the decided bits as bytes behind the ASM, the CRC-16 check
//   k_turbo_compact the CADUs whose CRC passes, in stream order
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

constexpr int TURBO_STATES = 16, TURBO_MEM = 4;  // 4 shift registers (backward connections "0011")
constexpr int TURBO_REC_THREADS = 128;           // 4 warps: 2 frames per warp, one direction per warp
constexpr int TURBO_EXT_THREADS = 128;
constexpr double TURBO_THRESHOLD = 1e10;         // convcode_extrinsic's `long int threshold = 1e10`

// One component code: trellis of convcode_initialize (libconvcodes.c:66-149), built on the host. out[s][u] bit j = component j's output
// bit on the branch (s, u); prev[s][n] / prev_u[s][n] = code.neighbors[s][n] (state, input) in the order the table holds them.
struct TurboCode
{
    int8_t next[TURBO_STATES][2];
    int8_t prev[TURBO_STATES][2], prev_u[TURBO_STATES][2];
    uint8_t out[TURBO_STATES][2];
};

// exp_sum (libconvcodes.c:544-548) as written: a when a > b, else b + log(1 + exp(-|a - b|)). Every operation rounded on its own.
// Below a - b = -40 the exp and log are skipped: exp(a - b) < 4.3e-18 is under half an ulp of 1, so 1 + exp(..) rounds to 1 and log(1)
// is 0 in any libm within an ulp, and the result is b + 0.0 either way. The first step of every fold (from -1e10) takes this path.
__device__ __forceinline__ double turbo_exp_sum(double a, double b)
{
    const double d = __dsub_rn(a, b);
    if (a > b)
        return a;
    if (d < -40.0)
        return __dadd_rn(b, 0.0);
    return __dadd_rn(b, log(__dadd_rn(1.0, exp(-d > 0 ? d : -d))));
}

// -g / (2 noise_variance) with g = sum over the components, in order, of pow(rho_j - (2 out_j - 1), 2); pow(x, 2) is x * x (a CPU test
// checks glibc on every value rho can take)
template <int C>
__device__ __forceinline__ double turbo_branch(const double (&rho)[C], unsigned out, double two_nv)
{
    double g = 0.0;
#pragma unroll
    for (int j = 0; j < C; j++) {
        const double x = __dsub_rn(rho[j], (out >> j) & 1 ? 1.0 : -1.0);
        g = __dadd_rn(g, __dmul_rn(x, x));
    }
    return __ddiv_rn(-g, two_nv);
}

// The normalisation's maximum over the 16 states of a half-warp: the value of the first state that reaches it (the reference keeps the
// first of equal values, which only matters for the sign of a zero)
__device__ __forceinline__ double turbo_max16(double v, int s)
{
    int i = s;
#pragma unroll
    for (int o = 8; o; o >>= 1) {
        const double v2 = __shfl_xor_sync(0xffffffffu, v, o, 16);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o, 16);
        if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
    }
    return v;
}

// Score of every position i < npos: the fp32 dot product of soft[i .. i+ASM-1] / 127 with the ASM table (+-1), summed left to right
// without contraction (the generic VOLK kernels). The module keeps a position when corr > best or -corr > best, so the score is |corr|
// and a negative corr means swapped. Block b's maximum over positions 32b .. 32b+31 (first index on ties) for every complete block.
template <int ASM>
__global__ void __launch_bounds__(256) k_turbo_corr(const int8_t *__restrict__ soft, long npos, const float *__restrict__ table,
                                                     float *__restrict__ score, unsigned char *__restrict__ swapped, float *__restrict__ bval,
                                                     int *__restrict__ bidx)
{
    __shared__ float x[256 + ASM];
    __shared__ float w[ASM];
    const long i0 = (long)blockIdx.x * 256;
    for (int k = threadIdx.x; k < 256 + ASM; k += 256) {
        const long j = i0 + k;
        x[k] = j < npos + ASM - 1 ? __fdiv_rn((float)soft[j], 127.0f) : 0.0f;
    }
    for (int k = threadIdx.x; k < ASM; k += 256)
        w[k] = table[k];
    __syncthreads();
    const long i = i0 + threadIdx.x;
    float acc = 0.0f;
#pragma unroll 16
    for (int k = 0; k < ASM; k++)
        acc = __fadd_rn(acc, __fmul_rn(x[threadIdx.x + k], w[k]));
    const float v0 = fabsf(acc);
    if (i < npos) {
        score[i] = v0;
        swapped[i] = acc < 0.0f;
    }
    float v = i < npos ? v0 : -INFINITY;
    int vi = (int)i;
    ldpc_best_warp(v, vi);
    const long b = i >> 5;
    if ((threadIdx.x & 31) == 0 && (b + 1) * 32 <= npos) {
        bval[b] = v;
        bidx[b] = vi;
    }
}

struct TurboGeom
{
    int F, asm_bits, cw;  // d_frame_size, d_asm_size, d_codeword_size
    int K, N;             // info bits (8 base), trellis steps K + 4
    int cu, cl;           // components of the upper / lower code
    int punct;            // rate 1/2: the lower code's output on odd blocks and the upper parity on even ones are sent
    long recv_stride;     // floats per frame: (cu + cl) N
};

// One CTA per frame. The module's buffer after a shift by pos (module :208-216: memmove(buf, buf + pos, pos), then pos new bytes at the
// end) holds stream byte o + pos + k at k < pos and k >= F - pos, and the stale o + k in between (o = the window start); for pos > F/2
// the memmove reads past the F-byte buffer (defined as zeros there), and those bytes are all overwritten by the new ones. Then
// derand_ccsds_soft over the codeword (~x where the sequence has a one), / 127, the sign flip when swapped, and CCSDSTurbo::decode's
// depuncturing (zeros at the punctured places) and turbo_decode's serial-to-parallel split: block b of cu + cl values feeds upper[b cu ..]
// and lower[b cl ..]. The a-priori values of the frame start at log(0.5).
__global__ void __launch_bounds__(256) k_turbo_gather(const int8_t *__restrict__ soft, const LdpcFrameRec *__restrict__ frames, TurboGeom G,
                                                       const unsigned char *__restrict__ pn, float *__restrict__ recv, double *__restrict__ msg,
                                                       double ln_half)
{
    const LdpcFrameRec r = frames[blockIdx.x];
    const int8_t *cur = soft + r.off, *stale = soft + (r.off - r.pos);
    float *up = recv + (size_t)blockIdx.x * G.recv_stride, *lo = up + (size_t)G.cu * G.N;
    auto in = [&](int c) { // codeword value c as the decoder reads it
        const int k = G.asm_bits + c;
        int v = (k < r.pos || k >= G.F - r.pos) ? cur[k] : stale[k];
        if (pn[c % 255])
            v = (int8_t)~v;
        const float x = __fdiv_rn((float)v, 127.0f);
        return r.swap ? -x : x;
    };
    const int cb = G.cu + G.cl;
    for (int b = threadIdx.x; b < G.N; b += blockDim.x) {
        if (G.punct) { // puncturing(): keep position 0 of every block of 3, position 1 on even blocks, position 2 on odd ones
            up[2 * b] = in(2 * b);
            const float p = in(2 * b + 1);
            up[2 * b + 1] = b & 1 ? 0.0f : p;
            lo[b] = b & 1 ? p : 0.0f;
        } else {
            for (int j = 0; j < G.cu; j++)
                up[b * G.cu + j] = in(b * cb + j);
            for (int j = 0; j < G.cl; j++)
                lo[b * G.cl + j] = in(b * cb + G.cu + j);
        }
    }
    double *m = msg + (size_t)blockIdx.x * 2 * G.K;
    for (int i = threadIdx.x; i < 2 * G.K; i += blockDim.x)
        m[i] = ln_half;
}

// a-priori value of input u at trellis step i: the frame's message (through the interleaver for the lower code), log(0.5) on the tail
__device__ __forceinline__ double turbo_app(const double *__restrict__ m, const int *__restrict__ perm, int K, int u, int i, double ln_half)
{
    return i < K ? m[(size_t)u * K + (perm ? perm[i] : i)] : ln_half;
}

// The two recursions of convcode_extrinsic (libconvcodes.c:380-467) for one component code with C outputs. Warp 2p of a CTA runs the
// backward recursion of frames 2p' and 2p'+1 (one per half-warp, lane = state), warp 2p+1 their forward recursion; the two are
// independent. Row i of each is normalised by its maximum and stored (met[frame][i][state]).
template <int C>
__global__ void __launch_bounds__(TURBO_REC_THREADS) k_turbo_rec(const float *__restrict__ recv, int stream_off, const double *__restrict__ msg,
                                                                 const int *__restrict__ perm, TurboGeom G, TurboCode code, double two_nv,
                                                                 double ln_half, double *__restrict__ bwd, double *__restrict__ fwd, int nf)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, s = lane & 15;
    const bool forward = warp & 1;
    const int f_raw = (warp >> 1) * 2 + (lane >> 4);
    if ((warp >> 1) * 2 >= nf)
        return; // (whole warp)
    const bool store = f_raw < nf;
    const int f = store ? f_raw : nf - 1;
    const float *rv = recv + (size_t)f * G.recv_stride + stream_off;
    const double *m = msg + (size_t)f * 2 * G.K;
    const int N = G.N, K = G.K;
    double *met = (forward ? fwd : bwd) + (size_t)f * N * TURBO_STATES;
    double cur = s == 0 ? 0.0 : -TURBO_THRESHOLD;
    const int first = forward ? 0 : N - 1;
    if (store)
        met[(size_t)first * TURBO_STATES + s] = cur;
    int br_st[2], br_u[2];
    unsigned br_out[2];
#pragma unroll
    for (int n = 0; n < 2; n++) {
        br_st[n] = forward ? code.prev[s][n] : code.next[s][n];
        br_u[n] = forward ? code.prev_u[s][n] : n;
        br_out[n] = forward ? code.out[code.prev[s][n]][code.prev_u[s][n]] : code.out[s][n];
    }
    // step t: the row computed from row t -/+ 1, whose received values and a-priori values are those of step t + 1 (backward) or
    // t - 1 (forward)
    auto load = [&](int t, double (&rho)[C], double &a0, double &a1) {
        const int q = forward ? t - 1 : t + 1;
#pragma unroll
        for (int j = 0; j < C; j++)
            rho[j] = (double)rv[(size_t)C * q + j];
        a0 = turbo_app(m, perm, K, 0, q, ln_half);
        a1 = turbo_app(m, perm, K, 1, q, ln_half);
    };
    double rho[C], a0, a1;
    int t = forward ? 1 : N - 2;
    const int step = forward ? 1 : -1;
    load(t, rho, a0, a1);
    for (int k = 1; k < N; k++, t += step) {
        double nrho[C], na0 = 0, na1 = 0;
        if (k + 1 < N)
            load(t + step, nrho, na0, na1);
        double acc = -TURBO_THRESHOLD;
#pragma unroll
        for (int n = 0; n < 2; n++) {
            const double other = __shfl_sync(0xffffffffu, cur, br_st[n], 16);
            const double a = br_u[n] ? a1 : a0;
            acc = turbo_exp_sum(acc, __dadd_rn(__dadd_rn(a, other), turbo_branch<C>(rho, br_out[n], two_nv)));
        }
        cur = __dsub_rn(acc, turbo_max16(acc, s));
        if (store)
            met[(size_t)t * TURBO_STATES + s] = cur;
#pragma unroll
        for (int j = 0; j < C; j++)
            rho[j] = nrho[j];
        a0 = na0;
        a1 = na1;
    }
}

// The extrinsic part of convcode_extrinsic (:469-521), one thread per (frame, step i): E_u = exp_sum over the states s = 0 .. 15 in order
// of forward[s][i] + backward[next(s, u)][i] - g / (2 noise_variance). It replaces the a-priori value of step i < K. In the last lower
// pass (`bits` != NULL) the decision one > zero (app + E) goes to the bit's deinterleaved place, and margins below 1e-9 are counted.
template <int C>
__global__ void __launch_bounds__(TURBO_EXT_THREADS) k_turbo_ext(const float *__restrict__ recv, int stream_off, double *__restrict__ msg,
                                                                 const int *__restrict__ perm, TurboGeom G, TurboCode code, double two_nv,
                                                                 double ln_half, const double *__restrict__ bwd, const double *__restrict__ fwd,
                                                                 unsigned char *__restrict__ bits, unsigned long long *__restrict__ near_ties)
{
    const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G.N)
        return;
    const int K = G.K;
    const float *rv = recv + (size_t)f * G.recv_stride + stream_off + (size_t)C * i;
    double rho[C];
#pragma unroll
    for (int j = 0; j < C; j++)
        rho[j] = (double)rv[j];
    const double *fr = fwd + ((size_t)f * G.N + i) * TURBO_STATES, *br = bwd + ((size_t)f * G.N + i) * TURBO_STATES;
    double e0 = -TURBO_THRESHOLD, e1 = -TURBO_THRESHOLD;
#pragma unroll 4
    for (int s = 0; s < TURBO_STATES; s++) {
        const double a = fr[s];
        e0 = turbo_exp_sum(e0, __dadd_rn(__dadd_rn(a, br[code.next[s][0]]), turbo_branch<C>(rho, code.out[s][0], two_nv)));
        e1 = turbo_exp_sum(e1, __dadd_rn(__dadd_rn(a, br[code.next[s][1]]), turbo_branch<C>(rho, code.out[s][1], two_nv)));
    }
    if (i >= K)
        return;
    double *m = msg + (size_t)f * 2 * K;
    const int at = perm ? perm[i] : i;
    const double app0 = m[at], app1 = m[(size_t)K + at];
    m[at] = e0;
    m[(size_t)K + at] = e1;
    if (bits) {
        const double one = __dadd_rn(app1, e1), zero = __dadd_rn(app0, e0);
        bits[(size_t)f * K + at] = one > zero;
        const double d = __dsub_rn(one, zero);
        if (fabs(d) < 1e-9)
            atomicAdd(near_ties, 1ull);
    }
}

// One CTA per frame: the K decided bits as base bytes behind 1A CF FC 1D, and GenericCRC(16, 0x1021, 0xFFFF, 0, false, false) over the
// first base - 2 of them against the last two (big endian). The result goes to the frame record's `corr` field (1 = the CRC passes).
__global__ void __launch_bounds__(256) k_turbo_pack(const unsigned char *__restrict__ bits, int base, LdpcFrameRec *__restrict__ frames,
                                                     uint8_t *__restrict__ cadu)
{
    extern __shared__ uint8_t sb[];
    const unsigned char *b = bits + (size_t)blockIdx.x * base * 8;
    uint8_t *o = cadu + (size_t)blockIdx.x * (base + 4);
    for (int t = threadIdx.x; t < base; t += blockDim.x) {
        uint8_t v = 0;
        for (int j = 0; j < 8; j++)
            v = (uint8_t)(v << 1 | b[8 * t + j]);
        sb[t] = v;
        o[4 + t] = v;
    }
    if (threadIdx.x < 4)
        o[threadIdx.x] = (uint8_t)(0x1acffc1du >> (8 * (3 - threadIdx.x)));
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned crc = 0xFFFF;
        for (int t = 0; t < base - 2; t++) {
            crc ^= (unsigned)sb[t] << 8;
            for (int k = 0; k < 8; k++)
                crc = crc & 0x8000 ? (crc << 1) ^ 0x1021 : crc << 1;
            crc &= 0xFFFF;
        }
        frames[blockIdx.x].corr = crc == ((unsigned)sb[base - 2] << 8 | sb[base - 1]);
    }
}

// One CTA per frame: a frame whose CRC passes goes to slot (frames before it that pass) of `out`
__global__ void __launch_bounds__(256) k_turbo_compact(const uint8_t *__restrict__ cadu, const LdpcFrameRec *__restrict__ frames, int bytes,
                                                        uint8_t *__restrict__ out)
{
    if (!frames[blockIdx.x].corr)
        return;
    __shared__ int s_dst;
    int n = 0;
    for (int k = threadIdx.x; k < (int)blockIdx.x; k += blockDim.x)
        n += frames[k].corr != 0;
    n = __reduce_add_sync(0xffffffffu, n);
    if (threadIdx.x == 0)
        s_dst = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && n)
        atomicAdd(&s_dst, n);
    __syncthreads();
    const uint8_t *src = cadu + (size_t)blockIdx.x * bytes;
    uint8_t *dst = out + (size_t)s_dst * bytes;
    for (int t = threadIdx.x; t < bytes; t += blockDim.x)
        dst[t] = src[t];
}
