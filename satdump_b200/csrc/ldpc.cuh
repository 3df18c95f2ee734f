// Kernels of ccsds_ldpc_decoder for the CCSDS C2 (8176, 7154) code (module_ccsds_ldpc_decoder.cpp:134-277, ldpc_rate "7/8").
// Included by api_ldpc.cu only.
//   k_ldpc_corr    CorrelatorGeneric::correlate's score (generic_correlator.cpp:176-231) at every soft position + the maxima of 32-position blocks
//   k_ldpc_walk    the module's frame walk: o_{k+1} = o_k + pos_k + F, pos_k = the window's first maximum if > 0, else 0
//   k_ldpc_gather  rotate_soft / OQPSK re-delay / derand_ccsds_soft of each frame -> the decoder's input with its 18 zero positions
//   k_ldpc_decode  LDPCDecoderGeneric::decode (ldpc_decoder_generic.cpp:69-194) on a level schedule, then the CADU repack
#pragma once
#include "walk.cuh"

constexpr int LDPC_ASM = 32;                 // syncword bits (d_ldpc_asm_size)
constexpr int LDPC_CW = 8160;                // code soft bytes per frame (d_ldpc_codeword_size)
constexpr int LDPC_F = LDPC_CW + LDPC_ASM;   // 8192 soft bytes per frame (d_ldpc_frame_size)
constexpr int LDPC_NPOS = LDPC_F - LDPC_ASM; // positions the correlator tries per window
constexpr int LDPC_VN = 8176, LDPC_ROWS = 1022, LDPC_DEG = 32, LDPC_SHORT = 18, LDPC_INFO_VN = LDPC_VN - LDPC_ROWS;
constexpr int LDPC_CADU = 1024;
constexpr int LDPC_WALK_WARPS = 32, LDPC_WALK_SPEC = 4 * LDPC_WALK_WARPS; // frames of the current lattice checked per round
constexpr int LDPC_DEC_THREADS = 1024;

struct LdpcSync { float w[4][LDPC_ASM]; }; // the correlator's syncword tables, built on the host (ldpc_syncwords)

// Score of every position i < npos: the best over the nsync tables of the fp32 dot product of soft[i .. i+31] / 63 with the table, summed
// left to right without contraction (the generic VOLK kernels), and the first table that reaches it. Block b's maximum over positions
// 32b .. 32b+31 (first index on ties) for every complete block.
__global__ void __launch_bounds__(256) k_ldpc_corr(const int8_t *__restrict__ soft, long npos, const LdpcSync sw, int nsync, float *__restrict__ score,
                                                    unsigned char *__restrict__ best_sync, float *__restrict__ bval, int *__restrict__ bidx)
{
    __shared__ float x[256 + LDPC_ASM];
    const long i0 = (long)blockIdx.x * 256;
    for (int k = threadIdx.x; k < 256 + LDPC_ASM; k += 256) {
        const long j = i0 + k;
        x[k] = j < npos + LDPC_ASM - 1 ? __fdiv_rn((float)soft[j], 63.0f) : 0.0f;
    }
    __syncthreads();
    const long i = i0 + threadIdx.x;
    float best = -INFINITY;
    int bs = 0;
#pragma unroll
    for (int s = 0; s < 4; s++) {
        if (s >= nsync)
            break;
        float acc = 0.0f;
#pragma unroll
        for (int k = 0; k < LDPC_ASM; k++)
            acc = __fadd_rn(acc, __fmul_rn(x[threadIdx.x + k], sw.w[s][k]));
        if (acc > best) { best = acc; bs = s; }
    }
    if (i < npos) {
        score[i] = best;
        best_sync[i] = (unsigned char)bs;
    }
    float v = i < npos ? best : -INFINITY;
    int vi = (int)i;
    ldpc_best_warp(v, vi);
    const long b = i >> 5;
    if ((threadIdx.x & 31) == 0 && (b + 1) * 32 <= npos) {
        bval[b] = v;
        bidx[b] = vi;
    }
}

// The frame walk over the `have` soft bytes of the FIFO, from offset 0, for frames of F soft bytes whose windows hold npos correlator
// positions. Each round checks up to LDPC_WALK_SPEC frames of the current lattice o + jF at once (one warp per frame): the frames up to
// and including the first one whose ASM is not at its window's start are exact, since their windows start where the module would read
// them; the walk then continues on the shifted lattice. Without signal every frame shifts, and each round takes one frame. A frame whose
// shifted start leaves fewer than F bytes waits for the next push. Offsets are < 2^31 (the FIFO is sized by max_soft).
// constellation WALK_SWAP_ONLY (the turbo correlator): the table index found is the frame's `swap`, its phase is 0.
__global__ void __launch_bounds__(1024) k_ldpc_walk(const float *__restrict__ score, const unsigned char *__restrict__ best_sync,
                                                     const float *__restrict__ bval, const int *__restrict__ bidx, long have, int F, int npos,
                                                     int constellation, LdpcFrameRec *__restrict__ frames, int max_frames,
                                                     LdpcWalkOut *__restrict__ out)
{
    __shared__ float s_v[LDPC_WALK_SPEC];
    __shared__ int s_i[LDPC_WALK_SPEC];
    __shared__ unsigned char s_bs[LDPC_WALK_SPEC];
    __shared__ long s_o;
    __shared__ int s_nf, s_shifted, s_done;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { s_o = 0; s_nf = 0; s_shifted = 0; s_done = 0; }
    __syncthreads();
    while (!s_done) {
        const long o = s_o;
        const long avail = have >= o + F ? (have - o - F) / F + 1 : 0;
        const int n = (int)min(min(avail, (long)LDPC_WALK_SPEC), (long)(max_frames - s_nf));
        for (int j = warp; j < n; j += LDPC_WALK_WARPS) {
            float v;
            int vi;
            ldpc_window_max(score, bval, bidx, o + (long)j * F, npos, v, vi);
            if (lane == 0) { s_v[j] = v; s_i[j] = vi; s_bs[j] = v > 0.0f ? best_sync[vi] : 0; }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long oo = o;
            int nf = s_nf, j = 0;
            bool stop = n == 0;
            for (; j < n; j++) {
                const float v = s_v[j];
                const int pos = v > 0.0f ? (int)(s_i[j] - oo) : 0;
                if (pos != 0 && oo + pos + F > have) { stop = true; break; }
                const int bs = s_bs[j];
                int phase, swap = 0; // generic_correlator.cpp:233-262
                if (constellation == WALK_SWAP_ONLY) { phase = 0; swap = bs; }
                else if (constellation == 0) phase = bs ? 2 : 0;
                else if (constellation == 1) phase = bs;
                else { phase = bs == 0 ? 1 : (bs == 1 ? 3 : (bs == 2 ? 0 : 2)); swap = bs >> 1; }
                LdpcFrameRec r;
                r.off = oo + pos;
                r.pos = pos;
                r.cor = v > 0.0f ? v : 0.0f;
                r.phase = phase;
                r.swap = swap;
                r.corr = 0;
                r.pad = 0;
                frames[nf++] = r;
                oo += pos + F;
                if (pos != 0) { s_shifted++; j++; break; }
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

// One CTA per frame: the decoder's input vn[0 .. 8175] = 18 zeros, then code soft bytes 0 .. 8157 of the frame after the phase fix
// (OQPSK: rotate_soft without swap, then on swap Q moves one symbol earlier and the frame's last Q is 0, module :159-173) and the
// derandomiser (~x where the sequence `pn`, one bit per entry, has a one; pn = NULL: "derandomize" off).
__global__ void __launch_bounds__(256) k_ldpc_gather(const int8_t *__restrict__ soft, const LdpcFrameRec *__restrict__ frames, int oqpsk,
                                                      const unsigned char *__restrict__ pn, int8_t *__restrict__ vn)
{
    const LdpcFrameRec r = frames[blockIdx.x];
    const int8_t *f = soft + r.off;
    int8_t *o = vn + (size_t)blockIdx.x * LDPC_VN;
    for (int t = threadIdx.x; t < LDPC_VN; t += blockDim.x) {
        if (t < LDPC_SHORT) { o[t] = 0; continue; }
        const int c = t - LDPC_SHORT, k = LDPC_ASM + c; // code soft byte c = frame byte k
        int v;
        if (oqpsk) {
            if (r.swap && (k & 1)) v = k + 2 < LDPC_F ? ldpc_rot(f, k + 2, r.phase, 0) : 0;
            else v = ldpc_rot(f, k, r.phase, 0);
        } else
            v = ldpc_rot(f, k, r.phase, r.swap);
        if (pn && pn[c % 255]) v = ~v;
        o[t] = (int8_t)v;
    }
}

// LDPCDecoderGeneric::decode on one codeword per CTA. The serial schedule (iterations x check rows 0..1021, each row reading and writing
// its 32 variable nodes) is cut into levels: a row instance's level is one more than the highest level of any earlier instance sharing a
// variable node with it. Rows of one level touch disjoint variable nodes, so they run at once (one warp per row, lane k = edge k) and the
// result is the serial one bit for bit. Each row keeps its last messages as min1, min2, the sign bits and the "equals min1" bits.
// Then the hard decisions (v >= 0), ldpc_corr, and the CADU: ASM 0x1ACFFC1D in host byte order, the 8158 decoded code bits and 2 zeros.
struct LdpcRowMsg { uint32_t sign, eq; uint16_t m1, m2; };

__global__ void __launch_bounds__(LDPC_DEC_THREADS) k_ldpc_decode(const int8_t *__restrict__ vn_in, const uint16_t *__restrict__ cols,
                                                                   const int *__restrict__ level_ptr, const uint16_t *__restrict__ level_rows,
                                                                   int nlevels, LdpcFrameRec *__restrict__ frames, uint8_t *__restrict__ cadu)
{
    extern __shared__ __align__(16) unsigned char smem[];
    int16_t *v = reinterpret_cast<int16_t *>(smem);
    LdpcRowMsg *msg = reinterpret_cast<LdpcRowMsg *>(smem + ((LDPC_VN * 2 + 15) & ~15));
    __shared__ int s_corr;
    const int8_t *in = vn_in + (size_t)blockIdx.x * LDPC_VN;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < LDPC_VN; i += blockDim.x)
        v[i] = in[i];
    for (int r = threadIdx.x; r < LDPC_ROWS; r += blockDim.x)
        msg[r] = LdpcRowMsg{0u, 0u, 0, 0};
    if (threadIdx.x == 0) s_corr = 0;
    __syncthreads();
    for (int L = 0; L < nlevels; L++) {
        const int a = level_ptr[L], b = level_ptr[L + 1];
        for (int q = a + warp; q < b; q += LDPC_DEC_THREADS / 32) {
            const int row = level_rows[q];
            const int col = cols[row * LDPC_DEG + lane];
            const LdpcRowMsg m = msg[row];
            const int old_mag = (m.eq >> lane) & 1 ? m.m2 : m.m1;
            const int old = (m.sign >> lane) & 1 ? -old_mag : old_mag;
            const int16_t x = (int16_t)(v[col] - old);
            const unsigned a_ = (unsigned)abs((int)x);
            const unsigned mn = __reduce_min_sync(0xffffffffu, a_);
            const unsigned at_min = __ballot_sync(0xffffffffu, a_ == mn);
            const unsigned second = __popc(at_min) > 1 ? mn : __reduce_min_sync(0xffffffffu, a_ == mn ? 0xffffffffu : a_);
            const unsigned min1 = min(mn, 255u), min2 = min(second, 255u);
            const unsigned negs = __ballot_sync(0xffffffffu, x < 0);
            const int sgn = (__popc(negs) & 1) ^ (x < 0);
            const bool eq = a_ == min1;
            const int mag = eq ? (int)min2 : (int)min1;
            const int nm = sgn ? -mag : mag;
            v[col] = (int16_t)(x + nm);
            const unsigned sb = __ballot_sync(0xffffffffu, sgn), eb = __ballot_sync(0xffffffffu, eq);
            if (lane == 0) msg[row] = LdpcRowMsg{sb, eb, (uint16_t)min1, (uint16_t)min2};
        }
        __syncthreads();
    }
    int corr = 0;
    for (int i = threadIdx.x; i < LDPC_INFO_VN; i += blockDim.x)
        corr += (v[i] >= 0) != (in[i] > 0);
    corr = __reduce_add_sync(0xffffffffu, corr);
    if (lane == 0 && corr) atomicAdd(&s_corr, corr);
    uint8_t *o = cadu + (size_t)blockIdx.x * LDPC_CADU;
    for (int t = threadIdx.x; t < LDPC_CADU; t += blockDim.x) {
        uint8_t byte;
        if (t < 4) byte = (uint8_t)(0x1acffc1du >> (8 * t)); // the uint32 as the host stores it (little endian)
        else {
            byte = 0;
            for (int k = 0; k < 8; k++) {
                const int i = LDPC_SHORT + 8 * (t - 4) + k;
                byte = (uint8_t)(byte << 1 | (i < LDPC_VN && v[i] >= 0));
            }
        }
        o[t] = byte;
    }
    __syncthreads();
    if (threadIdx.x == 0) frames[blockIdx.x].corr = s_corr;
}

// internal_stream: the first 7136 decoded bits of each of the nf codewords (bytes 4 .. 895 of its CADU as k_ldpc_decode wrote it) appended
// to the MSB-first bit FIFO behind its first bit0 bits, one thread per FIFO word (the bits in front of bit0 in the first word are kept)
constexpr int LDPC_INFO_BITS = 7136;
__global__ void __launch_bounds__(256) k_ldpc_append(const uint8_t *__restrict__ cadu, int nf, uint32_t *__restrict__ fifo, long bit0)
{
    const long nbits = (long)nf * LDPC_INFO_BITS, w0 = bit0 >> 5, w1 = (bit0 + nbits + 31) >> 5;
    for (long w = w0 + blockIdx.x * (long)blockDim.x + threadIdx.x; w < w1; w += (long)gridDim.x * blockDim.x) {
        const uint32_t old = w == w0 ? fifo[w] : 0u;
        uint32_t v = 0;
        for (int k = 0; k < 32; k++) {
            const long b = (w << 5) + k;
            unsigned bit;
            if (b < bit0) bit = (old >> (31 - k)) & 1u;
            else if (b >= bit0 + nbits) bit = 0;
            else {
                const long q = b - bit0, f = q / LDPC_INFO_BITS;
                const int i = (int)(q - f * LDPC_INFO_BITS);
                bit = (cadu[f * LDPC_CADU + 4 + (i >> 3)] >> (7 - (i & 7))) & 1u;
            }
            v |= bit << (31 - k);
        }
        fifo[w] = v;
    }
}
