// FEC kernels (sm_90a): int8 soft symbols -> Viterbi k=7 (r=1/2, MetOp-punctured 3/4) -> ASM deframer -> derandomiser
// -> RS(255,223|239) -> CADUs. All integer; results are bit-exact with the reference given the same soft bytes.
//
// Reference semantics being reproduced (SatDump tree):
//   rotate_soft                      src-core/common/codings/rotation.cpp:4-63
//   signed_soft_to_unsigned          src-core/common/codings/viterbi/utils.cpp:3-11
//   Viterbi3_4::depuncture (MetOp)   src-core/common/codings/viterbi/viterbi_3_4.cpp:84-104
//   ACS kernel                       src-core/common/codings/viterbi/volk_k7_r2_generic_fixed.h:80-163
//   CCDecoder chunk semantics        src-core/common/codings/viterbi/cc_decoder.cpp:159-209,228-302
//   lock machines / BER              viterbi_3_4.cpp:36-49,110-173 ; viterbi_1_2.cpp:36-116
//   NRZ-M                            src-core/common/codings/differential/nrzm.cpp:24-33
//   deframer                         src-core/common/codings/deframing/bpsk_ccsds_deframer.cpp:24-122
//   derandomiser                     src-core/common/codings/randomization.cpp:72-78
//   Reed-Solomon                     src-core/common/codings/reedsolomon/reedsolomon.cpp:53-116 + libs/correct/reed-solomon/decode.c
//
// Parallel formulation: one warp per Viterbi chunk (lane i owns butterfly i = states i, i+32; path metrics move with
// two __shfl_sync per step; the per-step renormalisation is a warp min; decisions are the two __ballot_sync words).
// A chunk depends on its predecessor only through a 6-bit start state, which k_vit_spec predicts from the tail of the
// previous chunk and the host verifies against the real chainback result. Lock search (rare) runs as a serial warp.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200
{

constexpr int VIT_TESTLEN = 2048; // TEST_BITS_LENGTH (viterbi_3_4.h:3)
constexpr int VIT_SPEC_STEPS_34 = 768;
constexpr int VIT_SPEC_STEPS_12 = 512;

struct VitGeom
{
    int rate34;   // 1: MetOp punctured 3/4, 0: rate 1/2
    int chunk;    // soft bytes per decoder call
    int F;        // decoded bits per chunk
    int dec_stride; // decision rows per chunk (F + 6 rounded up to 8)
    int bit_words;  // 32-bit words per chunk in the raw bit store
    // Viterbi_Depunc (viterbi_punc.cpp): the decoder windows read an already depunctured uint8 symbol stream (raw = 1; `chunk` symbols
    // per window, window q's symbols beyond chunk + tail_real[q] read as erasures), and the BER check re-encodes ber_bits bits and compares
    // ber_syms symbols (0: the defaults of the fixed-rate decoders)
    int raw;
    int ber_bits, ber_syms;
    const int *tail_real;
};

// Puncturing patterns of depunc.h as tables: input position ph of the period makes nout[ph] symbols, the data symbol at datapos[ph] of them
// (the other one is the erasure 128); cum[ph] = symbols made by positions 0..ph-1, cum[P] = Q symbols per period.
struct VitIdleState { int dec_start; /* -1 unbiased */ int enc_state; };
struct PuncTab
{
    int P, Q;
    float berscale;
    unsigned char nout[8], datapos[8], cum[9];
};

struct VitHyp { int swap, phase, shift; };

// soft byte k of the chunk after rotate_soft(swap, phase) and signed_soft_to_unsigned
#ifdef B200_DEFINE_KERNELS
__device__ __forceinline__ int soft_u8(const int8_t *__restrict__ c, int k, const VitHyp h)
{
    const int pair = k & ~1, isq = k & 1;
    int vi = c[pair], vq = c[pair + 1];
    if (vi == -128) vi = -127;
    if (vq == -128) vq = -127;
    if (h.swap) { int t = vi; vi = vq; vq = t; }
    int oi, oq;
    switch (h.phase) {
    case 1: oi = vq; oq = -vi; break;
    case 2: oi = -vi; oq = -vq; break;
    case 3: oi = -vq; oq = vi; break;
    default: oi = vi; oq = vq; break;
    }
    int u = (isq ? oq : oi) + 127;
    if (u == 128) u = 127;
    return u & 255;
}

// the two 8-bit symbols of trellis step t of a chunk: packed s0 | s1 << 8. `nsoft` = soft bytes that are real for this
// decoder call (chunk size, or TESTLEN for the lock test); beyond them the reference reads erasures (128) — or, for the
// r=3/4 lock test, never-written bytes that we take as `tail_fill`.
__device__ __forceinline__ int vit_symbols(const int8_t *__restrict__ c, int t, const VitGeom g, const VitHyp h, int nsoft, int tail_fill)
{
    int s0, s1;
    if (g.raw) { // depunctured uint8 stream
        const unsigned char *u = reinterpret_cast<const unsigned char *>(c);
        const int k0 = 2 * t;
        s0 = k0 < nsoft ? u[k0] : tail_fill;
        s1 = k0 + 1 < nsoft ? u[k0 + 1] : tail_fill;
        return s0 | (s1 << 8);
    }
    if (g.rate34) {
        const int grp = t / 3, r = t - 3 * grp, b = 4 * grp;
        if (b + 3 >= nsoft) return tail_fill | (tail_fill << 8);
        if (!h.shift) {
            if (r == 0) { s0 = soft_u8(c, b, h); s1 = soft_u8(c, b + 1, h); }
            else if (r == 1) { s0 = 128; s1 = soft_u8(c, b + 3, h); }
            else { s0 = soft_u8(c, b + 2, h); s1 = 128; }
        } else {
            if (r == 0) { s0 = 128; s1 = soft_u8(c, b + 1, h); }
            else if (r == 1) { s0 = soft_u8(c, b, h); s1 = 128; }
            else { s0 = soft_u8(c, b + 2, h); s1 = soft_u8(c, b + 3, h); }
        }
    } else {
        const int k0 = h.shift + 2 * t;
        s0 = k0 < nsoft ? soft_u8(c, k0, h) : tail_fill;
        s1 = k0 + 1 < nsoft ? soft_u8(c, k0 + 1, h) : tail_fill;
    }
    return s0 | (s1 << 8);
}

__device__ __forceinline__ int parity_u32(unsigned x) { return __popc(x) & 1; }
#endif // B200_DEFINE_KERNELS
struct AcsLane { int mask0, mask1; };
#ifdef B200_DEFINE_KERNELS
__device__ __forceinline__ AcsLane acs_lane_consts(int lane)
{
    // Branchtab[j*32+i] = parity((2i) & poly_j) ? 255 : 0, polys 79, 109 (cc_decoder.cpp:116-123)
    AcsLane a;
    a.mask0 = parity_u32((2u * lane) & 79u) ? 255 : 0;
    a.mask1 = parity_u32((2u * lane) & 109u) ? 255 : 0;
    return a;
}

__device__ __forceinline__ void acs_step(int sy, const AcsLane L, int lane, int &xl, int &xh, unsigned &D0, unsigned &D1)
{
    const int s0 = sy & 255, s1 = sy >> 8;
    const int m = (1 + (s0 ^ L.mask0) + (s1 ^ L.mask1)) >> 3; // ((sum >> 1) >> 2), volk_k7_r2_generic_fixed.h:99-104
    const int m0 = (xl + m) & 255, m1 = (xh + (63 - m)) & 255, m2 = (xl + (63 - m)) & 255, m3 = (xh + m) & 255;
    const bool d0 = m0 >= m1, d1 = m2 >= m3;
    int y0 = d0 ? m1 : m0, y1 = d1 ? m3 : m2;
    D0 = __ballot_sync(0xffffffffu, d0);
    D1 = __ballot_sync(0xffffffffu, d1);
    const unsigned mn = __reduce_min_sync(0xffffffffu, (unsigned)min(y0, y1));
    y0 -= mn;
    y1 -= mn;
    // new X[l] = Y[l] lives in lane l>>1 (y0 if l even), new X[l+32] = Y[l+32] in lane (l>>1)+16
    const int pk = y0 | (y1 << 16);
    const int a = __shfl_sync(0xffffffffu, pk, lane >> 1);
    const int b = __shfl_sync(0xffffffffu, pk, (lane >> 1) + 16);
    const int sh = (lane & 1) << 4;
    xl = (a >> sh) & 0xFFFF;
    xh = (b >> sh) & 0xFFFF;
}

// first-minimum end state over the 64 metrics (CCDecoder::find_endstate, cc_decoder.cpp:192-209)
__device__ __forceinline__ int acs_endstate(int xl, int xh, int lane)
{
    unsigned k0 = ((unsigned)xl << 6) | lane, k1 = ((unsigned)xh << 6) | (lane + 32);
    return (int)(__reduce_min_sync(0xffffffffu, min(k0, k1)) & 63);
}

__device__ __forceinline__ int tb_step(int state, unsigned D0, unsigned D1, int &bit)
{
    const unsigned w = (state & 1) ? D1 : D0;
    bit = (w >> (state >> 1)) & 1;
    return (state >> 1) | (bit << 5);
}

// ---------------------------------------------------------------- packed ACS core (production path)
// Same arithmetic as acs_step, two 16-bit fields per register: xl2 = X[i] | X[i]<<16, xh2 = X[i+32] | X[i+32]<<16.
// The per-step branch metric comes from a 4-entry table word (one byte per (Branchtab0, Branchtab1) combination) that the lane
// owning the step computed from the symbols and broadcast with one shuffle:
//   Sl = (xl2 + (m | 63-m << 16)) & 0x00FF00FF = m0 | m2<<16        (uint8 wrap of volk_k7_r2_generic_fixed.h:108-111)
//   Sh = (xh2 + (63-m | m << 16)) & 0x00FF00FF = m1 | m3<<16
//   Y  = min.u16x2(Sl, Sh) = Y[2i] | Y[2i+1]<<16 ; decision = (field of Y == field of Sh)  <=>  m0 >= m1 (ties pick m1, :112-115)
struct Acs2Lane { unsigned selA, selX; };
__device__ __forceinline__ Acs2Lane acs2_lane_consts(int lane)
{
    const unsigned idx = (parity_u32((2u * lane) & 79u) ? 2u : 0u) + (parity_u32((2u * lane) & 109u) ? 1u : 0u);
    Acs2Lane a;
    a.selA = idx | (4u << 4) | (idx << 8) | (4u << 12); // byte idx of the table word into both 16-bit fields
    a.selX = (lane & 1) ? 0x3232u : 0x1010u;            // after the shuffle: this lane's field of the source pair, duplicated
    return a;
}
__device__ __forceinline__ unsigned metric_table(int sy)
{
    const int s0 = sy & 255, s1 = sy >> 8;
    const unsigned m00 = (1 + s0 + s1) >> 3, m01 = (1 + s0 + (s1 ^ 255)) >> 3, m10 = (1 + (s0 ^ 255) + s1) >> 3,
                   m11 = (1 + (s0 ^ 255) + (s1 ^ 255)) >> 3;
    return m00 | (m01 << 8) | (m10 << 16) | (m11 << 24); // byte index = 2*[mask0 set] + [mask1 set]
}
__device__ __forceinline__ void acs2_step(unsigned w, const Acs2Lane L, int lane, unsigned &xl2, unsigned &xh2, unsigned &D0, unsigned &D1)
{
    const unsigned mm = __byte_perm(w, 0u, L.selA);
    const unsigned Sl = (xl2 + (mm ^ 0x003F0000u)) & 0x00FF00FFu;
    const unsigned Sh = (xh2 + (mm ^ 0x0000003Fu)) & 0x00FF00FFu;
    unsigned Y = __vminu2(Sl, Sh);
    const unsigned E = Y ^ Sh;
    D0 = __ballot_sync(0xffffffffu, (E << 16) == 0u);
    D1 = __ballot_sync(0xffffffffu, E < 0x10000u);
    const unsigned mn = __reduce_min_sync(0xffffffffu, min(Y & 0xFFFFu, Y >> 16));
    Y -= mn * 0x00010001u;
    const unsigned a = __shfl_sync(0xffffffffu, Y, lane >> 1);
    const unsigned b = __shfl_sync(0xffffffffu, Y, (lane >> 1) + 16);
    xl2 = __byte_perm(a, 0u, L.selX);
    xh2 = __byte_perm(b, 0u, L.selX);
}
__device__ __forceinline__ void acs2_init(int ss, int lane, unsigned &xl2, unsigned &xh2)
{
    // init_viterbi (63 everywhere, 0 at the start state) / init_viterbi_unbiased (31): cc_decoder.cpp:159-190
    const unsigned l = ss < 0 ? 31u : (lane == ss ? 0u : 63u), h = ss < 0 ? 31u : (lane + 32 == ss ? 0u : 63u);
    xl2 = l * 0x00010001u;
    xh2 = h * 0x00010001u;
}
__device__ __forceinline__ int acs2_endstate(unsigned xl2, unsigned xh2, int lane)
{
    const unsigned k0 = ((xl2 & 0xFFFFu) << 6) | lane, k1 = ((xh2 & 0xFFFFu) << 6) | (lane + 32);
    return (int)(__reduce_min_sync(0xffffffffu, min(k0, k1)) & 63);
}

// ---------------------------------------------------------------- start-state speculation
// For chunk index q (q = 1 .. n-1 of this launch's range): predict the decoder state at the end of chunk q-1's F bits
// by running the ACS over its last `spec` real steps + the 6 tail steps from all-equal metrics, then walking back 6.
__global__ void __launch_bounds__(128) k_vit_spec(const int8_t *__restrict__ soft, long chunk0, int nchunks, VitGeom g, VitHyp h, int spec,
                                                   int *__restrict__ start_state)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= nchunks - 1) return;
    const int8_t *c = soft + (chunk0 + w) * (long)g.chunk; // chunk w predicts the start of chunk w+1
    const int nlim = g.raw ? g.chunk + g.tail_real[w] : g.chunk;
    const Acs2Lane L = acs2_lane_consts(lane);
    unsigned xl2 = 0, xh2 = 0, D0 = 0, D1 = 0;
    for (int t0 = g.F - spec; t0 < g.F; t0 += 32) { // spec is a multiple of 32
        const unsigned mine = metric_table(vit_symbols(c, t0 + lane, g, h, nlim, 128));
#pragma unroll 8
        for (int j = 0; j < 32; j++)
            acs2_step(__shfl_sync(0xffffffffu, mine, j), L, lane, xl2, xh2, D0, D1);
    }
    unsigned d0h[6], d1h[6];
    const unsigned wt = metric_table(128 | (128 << 8)); // the six flush steps read erasures (d_veclen = frame + k - 1)
#pragma unroll
    for (int k = 0; k < 6; k++) {
        // (a depunctured window's flush steps read the next window's first symbols, or erasures where the stream ended)
        acs2_step(g.raw ? metric_table(vit_symbols(c, g.F + k, g, h, nlim, 128)) : wt, L, lane, xl2, xh2, D0, D1);
        d0h[k] = D0;
        d1h[k] = D1;
    }
    int st = acs2_endstate(xl2, xh2, lane), bit;
#pragma unroll
    for (int k = 5; k >= 0; k--)
        st = tb_step(st, d0h[k], d1h[k], bit);
    if (lane == 0) start_state[w + 1] = st;
}

#endif // B200_DEFINE_KERNELS
struct VitRec { int start_used, next_start, ber_errors, ber_total, enc_tail, end_state, pad1, pad2; };
#ifdef B200_DEFINE_KERNELS

// ---------------------------------------------------------------- main decode, part 1: ACS, DPX form (one warp per chunk)
// Same arithmetic as acs2_step with the metrics held as X << 8 in each 16-bit field (low byte 0): VIADD.16x2 adds per field modulo 2^16,
// which IS the reference's uint8 wrap (volk_k7_r2_generic_fixed.h:108-111), so no mask is needed; VIMNMX.U16x2 with predicate outputs
// returns the minima and both decisions in one instruction (min(Sh, Sl) prefers Sh on ties = the reference's "m0 >= m1 picks m1",
// :112-115); the per-step renormalisation is min over the two fields (PRMT + VIMNMX), one warp reduction and one subtraction. The
// branch-metric words come from the broadcast table byte by two IMADs on the FMA pipe: with mb = m << 8,
//   Ml = mb * (1 - 2^16) + (63 << 24) = m << 8 | (63 - m) << 24        (added to X[i]:    m0 | m2 << 16)
//   Mh = mb * (2^16 - 1) + (63 << 8)  = (63 - m) << 8 | m << 24        (added to X[i+32]: m1 | m3 << 16)
struct Acs3Lane { unsigned selM, selX; };
__device__ __forceinline__ Acs3Lane acs3_lane_consts(int lane)
{
    const unsigned idx = (parity_u32((2u * lane) & 79u) ? 2u : 0u) + (parity_u32((2u * lane) & 109u) ? 1u : 0u);
    Acs3Lane a;
    a.selM = 0x4404u | (idx << 4);                     // byte idx of the table word into byte 1, zeros elsewhere
    a.selX = (lane & 1) ? 0x3232u : 0x1010u;           // this lane's field of the shuffled pair, duplicated
    return a;
}
__device__ __forceinline__ void acs3_step(unsigned w, const Acs3Lane L, int lane, unsigned &xl2, unsigned &xh2, unsigned &D0, unsigned &D1)
{
    const unsigned mb = __byte_perm(w, 0u, L.selM);
    const unsigned Ml = mb * 0xFFFF0001u + 0x3F000000u;
    const unsigned Mh = mb * 0x0000FFFFu + 0x00003F00u;
    const unsigned Sl = __vadd2(xl2, Ml), Sh = __vadd2(xh2, Mh);
    bool p_hi, p_lo;
    unsigned Y = __vibmin_u16x2(Sh, Sl, &p_hi, &p_lo); // predicate = "the first operand (Sh) is the minimum" (ties included)
    D0 = __ballot_sync(0xffffffffu, p_lo);
    D1 = __ballot_sync(0xffffffffu, p_hi);
    const unsigned mn2 = __reduce_min_sync(0xffffffffu, __vminu2(Y, __byte_perm(Y, 0u, 0x1032u))); // min field, in both halves
    Y -= mn2;
    const unsigned a = __shfl_sync(0xffffffffu, Y, lane >> 1);
    const unsigned b = __shfl_sync(0xffffffffu, Y, (lane >> 1) + 16);
    xl2 = __byte_perm(a, 0u, L.selX);
    xh2 = __byte_perm(b, 0u, L.selX);
}
__device__ __forceinline__ void acs3_init(int ss, int lane, unsigned &xl2, unsigned &xh2)
{
    const unsigned l = ss < 0 ? 31u : (lane == ss ? 0u : 63u), h = ss < 0 ? 31u : (lane + 32 == ss ? 0u : 63u);
    xl2 = l * 0x01000100u;
    xh2 = h * 0x01000100u;
}
__device__ __forceinline__ int acs3_endstate(unsigned xl2, unsigned xh2, int lane)
{
    const unsigned k0 = ((xl2 & 0xFF00u) >> 2) | lane, k1 = ((xh2 & 0xFF00u) >> 2) | (lane + 32);
    return (int)(__reduce_min_sync(0xffffffffu, min(k0, k1)) & 63);
}

// start_state[q]: >= 0 biased start (63 everywhere, 0 at that state), -1: unbiased all-31 (first call ever). Writes the survivor
// decisions (two ballot words per trellis step) and the first-minimum end state. Per batch of 32 trellis steps: every lane prepares
// the metric table word of one step (next batch's symbol loads are issued one batch ahead), the 32 words are exchanged through shared
// memory (8 broadcast LDS.128 per lane instead of one SHFL per step: the kernel is bound by the SM's shuffle / vote / reduce port, not
// by the ALUs), and the two decision words of a step go to a per-warp shared-memory row (one STS by lane 0) that leaves as one
// coalesced 256-byte store per 32 steps.
__global__ void __launch_bounds__(128) k_vit_acs3(const int8_t *__restrict__ soft, long chunk0, int nchunks, VitGeom g, VitHyp h,
                                                   const int *__restrict__ start_state, uint2 *__restrict__ dec, VitRec *__restrict__ rec,
                                                   const int *__restrict__ qlist)
{
    __shared__ uint2 srow[4][2][32];
    __shared__ __align__(16) unsigned smet[4][2][32];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ql = blockIdx.x * 4 + wib;
    if (ql >= nchunks) return;
    const int q = qlist ? qlist[ql] : ql; // list mode: re-decode of the chunks whose speculated start state was wrong
    const int8_t *c = soft + (chunk0 + q) * (long)g.chunk;
    uint2 *d = dec + (long)q * g.dec_stride;
    const Acs3Lane L = acs3_lane_consts(lane);
    const int ss = start_state[q];
    unsigned xl2, xh2, D0, D1;
    acs3_init(ss, lane, xl2, xh2);
    const int steps = g.F + 6;
    const int nlim = g.raw ? g.chunk + g.tail_real[q] : g.chunk;
    int par = 0;
    unsigned next = lane < steps ? metric_table(vit_symbols(c, lane, g, h, nlim, 128)) : 0u;
    for (int t0 = 0; t0 < steps; t0 += 32, par ^= 1) {
        const unsigned mine = next;
        const int tn = t0 + 32 + lane;
        next = tn < steps ? metric_table(vit_symbols(c, tn, g, h, nlim, 128)) : 0u; // consumed one batch later
        uint2 *row = srow[wib][par];
        if (t0 + 32 <= steps) {
            unsigned w[32];
            smet[wib][par][lane] = mine;
            __syncwarp();
#pragma unroll
            for (int v = 0; v < 8; v++) {
                const uint4 u = reinterpret_cast<const uint4 *>(smet[wib][par])[v];
                w[4 * v] = u.x; w[4 * v + 1] = u.y; w[4 * v + 2] = u.z; w[4 * v + 3] = u.w;
            }
#pragma unroll
            for (int j = 0; j < 32; j++) {
                acs3_step(w[j], L, lane, xl2, xh2, D0, D1);
                if (lane == 0) row[j] = make_uint2(D0, D1);
            }
            __syncwarp();
            d[t0 + lane] = row[lane];
        } else {
            const int nn = steps - t0;
            for (int j = 0; j < nn; j++) {
                acs3_step(__shfl_sync(0xffffffffu, mine, j), L, lane, xl2, xh2, D0, D1);
                if (lane == 0) row[j] = make_uint2(D0, D1);
            }
            __syncwarp();
            if (lane < nn) d[t0 + lane] = row[lane];
        }
    }
    const int st = acs3_endstate(xl2, xh2, lane);
    if (lane == 0) {
        VitRec r = rec[q];
        r.start_used = ss;
        r.end_state = st;
        rec[q] = r;
    }
}

// ---------------------------------------------------------------- main decode, part 2: chainback, parallel blocks
// Rows F+5 .. 6 (cc_decoder.cpp:228-276): output bit i comes from row i+6; the state after the first six steps is the next
// call's start state. The walk is serial in the state, but survivor paths merge: a walk started TB_OVERLAP rows higher from an
// arbitrary state has joined the true path by the time it reaches its block. One thread per (chunk, block of TB_WORDS output
// words): block 0 starts from the true end state, block k>0 warms up over TB_OVERLAP rows and records the state it assumed at
// its top edge; k_vit_tb_check compares it with the state its upper neighbour really left there. If every edge agrees the
// result IS the serial chainback; chunks with a disagreeing edge are redone serially by k_vit_tb_serial (rare; counted).
#endif // B200_DEFINE_KERNELS
constexpr int TB_WORDS = 16;     // 512 output bits per block
constexpr int TB_OVERLAP = 256;  // warm-up rows (default; the host doubles it up to TB_OVERLAP_MAX when edges disagree often: low SNR)
constexpr int TB_OVERLAP_MAX = 2048;
struct TbEdge { unsigned char assumed, left; };
#ifdef B200_DEFINE_KERNELS
__device__ __forceinline__ int tb_walk_rows(const uint2 *__restrict__ rowbase, int nrows, int st)
{
    // walks rows rowbase[nrows-1] .. rowbase[0] without output (warm-up)
    int bit;
    for (int j = nrows - 1; j >= 0; j -= 8) {
        uint2 r[8];
#pragma unroll
        for (int k = 0; k < 8; k++) r[k] = (j - k >= 0) ? __ldg(rowbase + j - k) : make_uint2(0, 0);
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (j - k >= 0) st = tb_step(st, r[k].x, r[k].y, bit);
    }
    return st;
}

__global__ void __launch_bounds__(128) k_vit_tb(int nchunks, int nblocks, VitGeom g, const uint2 *__restrict__ dec, uint32_t *__restrict__ bits,
                                                 long out_chunk0, VitRec *__restrict__ rec, TbEdge *__restrict__ edges, const int *__restrict__ qlist, int overlap)
{
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long)nchunks * nblocks) return;
    const int ql = (int)(gid / nblocks), k = (int)(gid - (long)ql * nblocks);
    const int q = qlist ? qlist[ql] : ql;
    const uint2 *d = dec + (long)q * g.dec_stride;
    uint32_t *ob = bits + (out_chunk0 + q) * (long)g.bit_words;
    const int nwords = (g.F + 31) >> 5;
    const int w_hi = nwords - k * TB_WORDS;            // exclusive
    const int w_lo = max(0, w_hi - TB_WORDS);          // inclusive
    int st, bit, walked = 0, next_start = 0;
    if (k == 0)
        st = rec[q].end_state;
    else {
        // top edge of this block = row 6 + 32*w_hi (first row above it); warm up from TB_OVERLAP rows higher
        const int top = min(g.F, 32 * w_hi + overlap); // output index (exclusive) where the warm-up starts
        st = tb_walk_rows(d + 6 + 32 * w_hi, top - 32 * w_hi, 0);
        edges[(long)q * nblocks + k].assumed = (unsigned char)st;
    }
    for (int wv = w_hi - 1; wv >= w_lo; wv--) {
        const int i0 = wv << 5, nb = min(32, g.F - i0);
        const uint2 *row = d + 6 + i0;
        unsigned word = 0;
        for (int jb = ((nb - 1) >> 3) << 3; jb >= 0; jb -= 8) {
            uint2 r[8];
#pragma unroll
            for (int t = 0; t < 8; t++) r[t] = (jb + t < nb) ? __ldg(row + jb + t) : make_uint2(0, 0);
#pragma unroll
            for (int t = 7; t >= 0; t--)
                if (jb + t < nb) {
                    st = tb_step(st, r[t].x, r[t].y, bit);
                    word |= (unsigned)bit << (31 - (jb + t));
                    if (++walked == 6) next_start = st;
                }
        }
        ob[wv] = word;
    }
    if (k == 0) rec[q].next_start = next_start;
    edges[(long)q * nblocks + k].left = (unsigned char)st; // state handed to the block below (rows < 6 + 32*w_lo)
}

// flags chunks whose blocks disagree at an edge; list[0] = count, list[1..] = chunk indices
__global__ void k_vit_tb_check(int nchunks, int nblocks, const TbEdge *__restrict__ edges, int *__restrict__ list, int cap, const int *__restrict__ qlist)
{
    const int ql = blockIdx.x * blockDim.x + threadIdx.x;
    if (ql >= nchunks) return;
    const int q = qlist ? qlist[ql] : ql;
    bool bad = false;
    for (int k = 1; k < nblocks; k++)
        if (edges[(long)q * nblocks + k].assumed != edges[(long)q * nblocks + k - 1].left) bad = true;
    if (bad) {
        const int slot = atomicAdd(list, 1);
        if (slot < cap) list[1 + slot] = q;
    }
}

// serial chainback of the flagged chunks (one thread per chunk)
__global__ void __launch_bounds__(128) k_vit_tb_serial(const int *__restrict__ list, int cap, VitGeom g, const uint2 *__restrict__ dec,
                                                        uint32_t *__restrict__ bits, long out_chunk0, VitRec *__restrict__ rec)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(list[0], cap)) return;
    const int q = list[1 + i];
    const uint2 *d = dec + (long)q * g.dec_stride;
    uint32_t *ob = bits + (out_chunk0 + q) * (long)g.bit_words;
    int st = rec[q].end_state, bit, next_start = 0, walked = 0;
    for (int wv = (g.F - 1) >> 5; wv >= 0; wv--) {
        const int i0 = wv << 5, nb = min(32, g.F - i0);
        unsigned word = 0;
        for (int j = nb - 1; j >= 0; j--) {
            const uint2 r = d[6 + i0 + j];
            st = tb_step(st, r.x, r.y, bit);
            word |= (unsigned)bit << (31 - j);
            if (++walked == 6) next_start = st;
        }
        ob[wv] = word;
    }
    rec[q].next_start = next_start;
}

// BER pass (separate launch so every chunk's bits are complete): one warp per chunk.
__global__ void __launch_bounds__(128) k_vit_ber(const int8_t *__restrict__ soft, long chunk0, int nchunks, VitGeom g, VitHyp h,
                                                  const uint32_t *__restrict__ bits, long out_chunk0, int enc_state_in, VitRec *__restrict__ rec,
                                                  const int *__restrict__ qlist)
{
    const int ql = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (ql >= nchunks) return;
    const int q = qlist ? qlist[ql] : ql;
    const int8_t *c = soft + (chunk0 + q) * (long)g.chunk;
    const uint32_t *ob = bits + (out_chunk0 + q) * (long)g.bit_words;
    const int tb = g.ber_bits ? g.ber_bits : (g.rate34 ? VIT_TESTLEN * 3 / 4 : VIT_TESTLEN / 2); // bits re-encoded (the encoder register chains on)
    const int ns = g.ber_syms ? g.ber_syms : 2 * tb;                                            // symbols compared
    const int nlim = g.raw ? g.chunk + g.tail_real[q] : g.chunk;
    auto getbit = [&](const uint32_t *p, int k) { return (p[k >> 5] >> (31 - (k & 31))) & 1u; };
    unsigned init = (unsigned)enc_state_in & 63u;
    if (q > 0) {
        const uint32_t *pb = bits + (out_chunk0 + q - 1) * (long)g.bit_words;
        init = 0;
        for (int k = tb - 6; k < tb; k++) init = (init << 1) | getbit(pb, k);
    }
    int errors = 0, total = 0;
    for (int t = lane; 2 * t < ns; t += 32) {
        // encoder register after shifting in bit t: bits t-6..t, older bits from `init` when t < 6
        unsigned reg = 0;
        for (int k = 6; k >= 0; k--) {
            const int idx = t - k;
            const unsigned b = idx >= 0 ? getbit(ob, idx) : ((init >> (-idx - 1)) & 1u);
            reg = (reg << 1) | b;
        }
        const int e0 = parity_u32(reg & 79u), e1 = parity_u32(reg & 109u);
        const int sy = vit_symbols(c, t, g, h, nlim, 128);
        const int s0 = sy & 255, s1 = sy >> 8;
        if (s0 != 128) { errors += ((s0 > 127) != e0); total++; }
        if (2 * t + 1 < ns && s1 != 128) { errors += ((s1 > 127) != e1); total++; }
    }
    for (int off = 16; off; off >>= 1) {
        errors += __shfl_xor_sync(0xffffffffu, errors, off);
        total += __shfl_xor_sync(0xffffffffu, total, off);
    }
    if (lane == 0) {
        unsigned tail = 0;
        for (int k = tb - 6; k < tb; k++) tail = (tail << 1) | getbit(ob, k);
        rec[q].ber_errors = errors;
        rec[q].ber_total = total;
        rec[q].enc_tail = (int)tail;
    }
}

// ---------------------------------------------------------------- Viterbi_Depunc (rates 2/3, 3/4, 5/6, 7/8): viterbi_punc.cpp, depunc.h
// symbols made by the first m input positions of the pattern counted from position 0 of a period
__device__ __forceinline__ long punc_made(const PuncTab &P, long m) { return (m / P.P) * P.Q + P.cum[m % P.P]; }

// DepuncXX::depunc_cont over a run of consecutive module calls, in closed form: input symbol i of the run (pattern position (a0 + i) mod P)
// lands at out[lead + made(a0 + i) - made(a0)]; rotate_soft / signed_soft_to_unsigned applied on the way (soft_u8). `lead`: the run starts
// with the symbol the reference still holds in `buf` (set_shift's is_first after a late shift). The symbol a call keeps back when its
// count is odd stays in place in this stream: holding it back only delays WHEN a window can be decoded (host bookkeeping).
__global__ void k_punc_depunc(const int8_t *__restrict__ soft, long nsoft, VitHyp h, PuncTab P, int a0, int lead, int lead_value,
                              unsigned char *__restrict__ out)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && lead)
        out[0] = (unsigned char)lead_value;
    if (i >= nsoft)
        return;
    const long m = a0 + i;
    const int ph = (int)(m % P.P);
    const long o = lead + punc_made(P, m) - punc_made(P, a0);
    const unsigned char u = (unsigned char)soft_u8(soft, (int)i, h); // (pairs of a call stay pairs: the call size is even)
    if (P.nout[ph] == 1)
        out[o] = u;
    else {
        out[o + P.datapos[ph]] = u;
        out[o + 1 - P.datapos[ph]] = 128;
    }
}

// Lock search of Viterbi_Depunc::work (viterbi_punc.cpp:55-107), one warp, module call by module call until a hypothesis locks: for every
// (I/Q swap, phase, shift < 2 P) depunc_static of the first 2048 soft symbols into the PERSISTENT test buffer `bdep` (the reference's
// member array: the decoder always reads 4108 symbols of it, i.e. beyond the depunctured length whatever an earlier trial left there, or
// the zeros of a never written tail), decode 2048 bits with the chained test decoder, re-encode lenp/2 bits with the chained encoder,
// BER over lenp symbols with the rate's scale; lock on the lowest BER below the threshold. test_bit_len is the LAST trial's length.
#endif // B200_DEFINE_KERNELS
struct PuncIdleOut { int lock_call, swap, phase, shift, test_bit_len, pad; float ber; VitIdleState st; };
#ifdef B200_DEFINE_KERNELS
__global__ void __launch_bounds__(32) k_punc_idle(const int8_t *__restrict__ soft, long call0, int ncalls, int call_size, PuncTab P, int nswap, int nphases,
                                                   int ph0, int ph1, float thr, VitIdleState st_in, unsigned char *__restrict__ bdep,
                                                   uint2 *__restrict__ scratch_dec, PuncIdleOut *__restrict__ out)
{
    const int lane = threadIdx.x;
    const AcsLane L = acs_lane_consts(lane);
    const int F = VIT_TESTLEN, steps = F + 6;
    int dec_start = st_in.dec_start;
    unsigned enc = (unsigned)st_in.enc_state;
    __shared__ uint32_t tbits[VIT_TESTLEN / 32 + 2];
    float best = 10.f;
    int lock = -1, lswap = 0, lphase = 0, lshift = 0, tbl = 0;
    for (int q = 0; q < ncalls && lock < 0; q++) {
        const int8_t *c = soft + (call0 + q) * (long)call_size;
        best = 10.f;
        for (int s = 0; s < nswap; s++)
            for (int pi = 0; pi < nphases; pi++)
                for (int shift = 0; shift < 2 * P.P; shift++) {
                    const VitHyp h{s, pi == 0 ? ph0 : ph1, 0};
                    const int as = shift % P.P, lead = shift > P.P - 1 ? 1 : 0;
                    // depunc_static
                    if (lane == 0 && lead)
                        bdep[0] = 128;
                    for (int i = lane; i < VIT_TESTLEN; i += 32) {
                        const long m = as + i;
                        const int ph = (int)(m % P.P);
                        const long o = lead + punc_made(P, m) - punc_made(P, as);
                        const unsigned char u = (unsigned char)soft_u8(c, i, h);
                        if (P.nout[ph] == 1)
                            bdep[o] = u;
                        else {
                            bdep[o + P.datapos[ph]] = u;
                            bdep[o + 1 - P.datapos[ph]] = 128;
                        }
                    }
                    int lenp = lead + (int)(punc_made(P, as + VIT_TESTLEN) - punc_made(P, as));
                    if (lenp % 2)
                        lenp--;
                    tbl = lenp;
                    __syncwarp();
                    // the deprecated CCDecoder::work(in, out, size) ignores its size (cc_decoder.cpp:304-314): full 2048-bit frame
                    int xl, xh;
                    if (dec_start < 0) xl = xh = 31;
                    else { xl = (lane == dec_start) ? 0 : 63; xh = (lane + 32 == dec_start) ? 0 : 63; }
                    unsigned D0, D1;
                    for (int t0 = 0; t0 < steps; t0 += 32) {
                        const int tm = t0 + lane;
                        const int mine = tm < steps ? ((int)bdep[2 * tm] | ((int)bdep[2 * tm + 1] << 8)) : 0;
                        unsigned k0 = 0, k1 = 0;
                        const int nn = min(32, steps - t0);
                        for (int j = 0; j < nn; j++) {
                            const int sy = __shfl_sync(0xffffffffu, mine, j);
                            acs_step(sy, L, lane, xl, xh, D0, D1);
                            if (lane == j) { k0 = D0; k1 = D1; }
                        }
                        if (lane < nn) scratch_dec[t0 + lane] = make_uint2(k0, k1);
                    }
                    __syncwarp();
                    int st = acs_endstate(xl, xh, lane), bit;
                    for (int row = steps - 1, k = 0; row >= 6; row--, k++) {
                        const uint2 r = scratch_dec[row];
                        st = tb_step(st, r.x, r.y, bit);
                        if (k == 5) dec_start = st;
                        const int i = row - 6;
                        if (lane == 0) {
                            if ((i & 31) == 31 || i == F - 1) tbits[i >> 5] = 0; // first touch of this word (walking downwards)
                            tbits[i >> 5] |= (unsigned)bit << (31 - (i & 31));
                        }
                    }
                    __syncwarp();
                    // re-encode lenp / 2 bits with the chained encoder and count mismatches over lenp symbols
                    const int nb = lenp / 2;
                    int errors = 0, total = 0;
                    for (int t = lane; t < nb; t += 32) {
                        unsigned reg = 0;
                        for (int k = 6; k >= 0; k--) {
                            const int idx = t - k;
                            const unsigned b = idx >= 0 ? ((tbits[idx >> 5] >> (31 - (idx & 31))) & 1u) : ((enc >> (-idx - 1)) & 1u);
                            reg = (reg << 1) | b;
                        }
                        const int e0 = parity_u32(reg & 79u), e1 = parity_u32(reg & 109u);
                        const int s0 = bdep[2 * t], s1 = bdep[2 * t + 1];
                        if (s0 != 128) { errors += ((s0 > 127) != e0); total++; }
                        if (s1 != 128) { errors += ((s1 > 127) != e1); total++; }
                    }
                    for (int off = 16; off; off >>= 1) {
                        errors += __shfl_xor_sync(0xffffffffu, errors, off);
                        total += __shfl_xor_sync(0xffffffffu, total, off);
                    }
                    unsigned tail = 0;
                    for (int k = nb - 6; k < nb; k++) tail = (tail << 1) | ((tbits[k >> 5] >> (31 - (k & 31))) & 1u);
                    enc = tail;
                    const float b = ((float)errors / (float)total) * P.berscale;
                    if (b < thr && b < best) {
                        best = b; lock = q; lswap = s; lphase = h.phase; lshift = shift;
                    }
                    __syncwarp();
                }
    }
    if (lane == 0) {
        PuncIdleOut o;
        o.lock_call = lock; o.swap = lswap; o.phase = lphase; o.shift = lshift; o.test_bit_len = tbl; o.pad = 0; o.ber = best;
        o.st.dec_start = dec_start; o.st.enc_state = (int)enc;
        *out = o;
    }
}

// ---------------------------------------------------------------- lock search (IDLE state), one serial warp
// Replays Viterbi3_4::work / Viterbi1_2::work in the IDLE state chunk by chunk until a hypothesis locks
// (viterbi_3_4.cpp:112-144, viterbi_1_2.cpp:54-89), with the chained test decoder / encoder state.
#endif // B200_DEFINE_KERNELS
// head (M = 2 only): the first 16 bits the test decoder's last trial decoded, bit j at (head >> j) & 1
struct VitIdleOut { int lock_chunk, swap, phase, shift; float ber; float bers[16]; VitIdleState st; unsigned head; };
constexpr int VIT_IDLE_PLAIN = 0, VIT_IDLE_FY = 1, VIT_IDLE_R12_EXACT = 2; // the lock search's modes (k_vit_idle)

#ifdef B200_DEFINE_KERNELS
// M (the lock search's mode, VIT_IDLE_*):
//   FY (fengyun_ahrpt_decoder, Viterbi3_4 with fymode): hypothesis (s = 0, shift) runs as VitHyp{shift, 0, shift}; with the branch stream
//   stored by k_fy_split (fengyun.cuh) that is FengYun's depuncture through the MetOp one (the stored bers and lswap keep s = 0).
//   R12_EXACT (fengyun_mpt_decoder, r=1/2): the 12 symbols the test decoder reads past its 2048 test bytes are the first decoded bits (0 /
//   1) of the trial before it, carried in head (head_in: the last trial of the previous call), as Viterbi1_2's member layout gives them.
//   The other modes read them as 0.
template <int M = VIT_IDLE_PLAIN>
__global__ void __launch_bounds__(32) k_vit_idle(const int8_t *__restrict__ soft, long chunk0, int nchunks, VitGeom g, int nswap, int nphases,
                                                  int ph0, int ph1, float thr, VitIdleState st_in, uint2 *__restrict__ scratch_dec,
                                                  VitIdleOut *__restrict__ out, unsigned head_in)
{
    constexpr bool FY = M == VIT_IDLE_FY;
    unsigned head = head_in;
    const int lane = threadIdx.x;
    const AcsLane L = acs_lane_consts(lane);
    VitGeom tg = g;
    tg.F = g.rate34 ? VIT_TESTLEN * 3 / 4 : VIT_TESTLEN / 2;
    const int steps = tg.F + 6, nsym = g.rate34 ? VIT_TESTLEN * 3 / 2 : VIT_TESTLEN;
    int dec_start = st_in.dec_start;
    unsigned enc = (unsigned)st_in.enc_state;
    __shared__ uint32_t tbits[VIT_TESTLEN * 3 / 4 / 32 + 2];
    float best = 10.f;
    int lock = -1, lswap = 0, lphase = 0, lshift = 0;
    float bers[16];
    for (int i = 0; i < 16; i++) bers[i] = 10.f;
    for (int q = 0; q < nchunks && lock < 0; q++) {
        const int8_t *c = soft + (chunk0 + q) * (long)g.chunk;
        best = 10.f;
        for (int s = 0; s < nswap; s++)
            for (int pi = 0; pi < nphases; pi++)
                for (int shift = 0; shift < 2; shift++) {
                    VitHyp h{FY ? shift : s, pi == 0 ? ph0 : ph1, shift};
                    int xl, xh;
                    if (dec_start < 0) xl = xh = 31;
                    else { xl = (lane == dec_start) ? 0 : 63; xh = (lane + 32 == dec_start) ? 0 : 63; }
                    unsigned D0, D1;
                    for (int t0 = 0; t0 < steps; t0 += 32) {
                        const int tm = t0 + lane;
                        // r=1/2: the test decoder over-reads 12 bytes past the 2048 test bytes into the previous trial's decoded
                        // bits (viterbi_1_2.h:37-40); they only touch the last trellis steps. We feed erasure-neutral zeros/ones
                        // exactly like the reference layout would: previous decoded bits are 0/1 -> use 0.
                        int mine = tm < steps ? vit_symbols(c, tm, tg, h, VIT_TESTLEN, 0) : 0;
                        if (M == VIT_IDLE_R12_EXACT && tm < steps) { // (r=1/2: symbol k of the test buffer is byte k)
                            const int k0 = h.shift + 2 * tm - VIT_TESTLEN;
                            if (k0 >= 0) mine = (mine & ~255) | ((head >> k0) & 1);
                            if (k0 + 1 >= 0) mine = (mine & 255) | (((head >> (k0 + 1)) & 1) << 8);
                        }
                        unsigned k0 = 0, k1 = 0;
                        const int nn = min(32, steps - t0);
                        for (int j = 0; j < nn; j++) {
                            const int sy = __shfl_sync(0xffffffffu, mine, j);
                            acs_step(sy, L, lane, xl, xh, D0, D1);
                            if (lane == j) { k0 = D0; k1 = D1; }
                        }
                        if (lane < nn) scratch_dec[t0 + lane] = make_uint2(k0, k1);
                    }
                    __syncwarp();
                    int st = acs_endstate(xl, xh, lane), bit;
                    for (int row = steps - 1, k = 0; row >= 6; row--, k++) {
                        const uint2 r = scratch_dec[row];
                        st = tb_step(st, r.x, r.y, bit);
                        if (k == 5) dec_start = st;
                        const int i = row - 6;
                        if (lane == 0) {
                            if ((i & 31) == 31 || i == tg.F - 1) tbits[i >> 5] = 0; // first touch of this word (walking downwards)
                            tbits[i >> 5] |= (unsigned)bit << (31 - (i & 31));
                        }
                    }
                    __syncwarp();
                    // re-encode with the chained encoder and count mismatches
                    int errors = 0, total = 0;
                    for (int t = lane; t < tg.F; t += 32) {
                        unsigned reg = 0;
                        for (int k = 6; k >= 0; k--) {
                            const int idx = t - k;
                            const unsigned b = idx >= 0 ? ((tbits[idx >> 5] >> (31 - (idx & 31))) & 1u) : ((enc >> (-idx - 1)) & 1u);
                            reg = (reg << 1) | b;
                        }
                        const int e0 = parity_u32(reg & 79u), e1 = parity_u32(reg & 109u);
                        const int sy = vit_symbols(c, t, tg, h, VIT_TESTLEN, 0);
                        const int s0 = sy & 255, s1 = sy >> 8;
                        if (2 * t < nsym && s0 != 128) { errors += ((s0 > 127) != e0); total++; }
                        if (2 * t + 1 < nsym && s1 != 128) { errors += ((s1 > 127) != e1); total++; }
                    }
                    for (int off = 16; off; off >>= 1) {
                        errors += __shfl_xor_sync(0xffffffffu, errors, off);
                        total += __shfl_xor_sync(0xffffffffu, total, off);
                    }
                    unsigned tail = 0;
                    for (int k = tg.F - 6; k < tg.F; k++) tail = (tail << 1) | ((tbits[k >> 5] >> (31 - (k & 31))) & 1u);
                    enc = tail;
                    if (M == VIT_IDLE_R12_EXACT) // this trial's first bits: what the next trial's over-read sees
                        head = __brev(tbits[0]) & 0xffffu;
                    const float b = ((float)errors / (float)total) * (g.rate34 ? 5.0f : 2.5f);
                    bers[(s * 4 + h.phase) * 2 + shift] = b;
                    if ((best == 10.f && b < thr) || (best < 10.f && b < best)) {
                        best = b; lock = q; lswap = s; lphase = h.phase; lshift = shift;
                    }
                    __syncwarp();
                }
    }
    if (lane == 0) {
        VitIdleOut o;
        o.lock_chunk = lock; o.swap = lswap; o.phase = lphase; o.shift = lshift; o.ber = best;
        for (int i = 0; i < 16; i++) o.bers[i] = bers[i];
        o.st.dec_start = dec_start; o.st.enc_state = (int)enc; o.head = M == VIT_IDLE_R12_EXACT ? head : 0u;
        *out = o;
    }
}

// ---------------------------------------------------------------- lock search, parallel form
// The 4 (8 with the OQPSK I/Q-swap search) hypotheses of a chunk form a chain only through two 6-bit registers (the test decoder's
// start state and the BER encoder's register). One warp per hypothesis: pass A runs every ACS with a guessed start (hypothesis 0's is
// the exact carried one) to learn the chainback states; pass B re-runs hypotheses 1.. from their predecessor's pass-A state and does
// the full chainback; if every predecessor's pass-B state equals its pass-A state the chain is the serial one. Otherwise the kernel
// reports `fallback_chunk` and the host continues with the serial k_vit_idle from there.
#endif // B200_DEFINE_KERNELS
struct VitIdle2Out { VitIdleOut o; int fallback_chunk; int pad[3]; };
constexpr int VIT_IDLE_ROWS = VIT_TESTLEN * 3 / 4 + 6 + 2;           // decision rows per hypothesis (r=3/4 is the larger: 1542)
constexpr int VIT_IDLE_WARP_BYTES = VIT_IDLE_ROWS * 8 + 64 * 4;       // + 64 words of decoded bits
#ifdef B200_DEFINE_KERNELS
template <bool FY = false> // (as k_vit_idle; VIT_IDLE_R12_EXACT runs the serial kernel only)
__global__ void __launch_bounds__(256) k_vit_idle2(const int8_t *__restrict__ soft, long chunk0, int nchunks, VitGeom g, int nswap, int nphases, int ph0,
                                                    int ph1, float thr, VitIdleState st_in, VitIdle2Out *__restrict__ out)
{
    extern __shared__ __align__(16) unsigned char idle_smem[];
    __shared__ int rA[8], rB[8], errs[8], tots[8], tails[8];
    __shared__ int s_lock, s_dec, s_enc, s_fallback;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nh = nswap * nphases * 2;
    uint2 *dec = reinterpret_cast<uint2 *>(idle_smem + (size_t)w * VIT_IDLE_WARP_BYTES);
    uint32_t *tb = reinterpret_cast<uint32_t *>(idle_smem + (size_t)w * VIT_IDLE_WARP_BYTES + VIT_IDLE_ROWS * 8);
    const Acs2Lane L = acs2_lane_consts(lane);
    VitGeom tg = g;
    tg.F = g.rate34 ? VIT_TESTLEN * 3 / 4 : VIT_TESTLEN / 2;
    const int steps = tg.F + 6, nsym = g.rate34 ? VIT_TESTLEN * 3 / 2 : VIT_TESTLEN;
    // hypothesis w in the reference's loop order: swap-major, then phase, then shift
    const int hs = w / (nphases * 2), hp = (w / 2) % nphases, hshift = w & 1;
    const VitHyp h{FY ? hshift : hs, hp == 0 ? ph0 : ph1, hshift};
    if (threadIdx.x == 0) { s_lock = -1; s_dec = st_in.dec_start; s_enc = st_in.enc_state; s_fallback = -1; }
    __syncthreads();
    float bers[16];
    for (int i = 0; i < 16; i++) bers[i] = 10.f;
    float best = 10.f;
    int lswap = 0, lphase = 0, lshift = 0;
    for (int q = 0; q < nchunks; q++) {
        const int8_t *c = soft + (chunk0 + q) * (long)g.chunk;
        auto run_acs = [&](int start, bool keep) {
            unsigned xl2, xh2, D0, D1;
            acs2_init(start, lane, xl2, xh2);
            for (int t0 = 0; t0 < steps; t0 += 32) {
                const int tm = t0 + lane;
                const unsigned mine = tm < steps ? metric_table(vit_symbols(c, tm, tg, h, VIT_TESTLEN, 0)) : 0u;
                const int nn = min(32, steps - t0);
                for (int j = 0; j < nn; j++) {
                    acs2_step(__shfl_sync(0xffffffffu, mine, j), L, lane, xl2, xh2, D0, D1);
                    if (lane == 0 && (keep || t0 + j >= tg.F)) dec[t0 + j] = make_uint2(D0, D1);
                }
            }
            __syncwarp();
            return acs2_endstate(xl2, xh2, lane);
        };
        auto chain6 = [&](int st) { // state after the first six chainback steps = next call's start state
            int bit;
            for (int row = steps - 1; row >= steps - 6; row--) st = tb_step(st, dec[row].x, dec[row].y, bit);
            return st;
        };
        // ---- pass A
        if (w < nh) {
            const int e = run_acs(w == 0 ? s_dec : -1, w == 0);
            const int r = chain6(e);
            if (lane == 0) { rA[w] = r; if (w == 0) rB[0] = r; tails[w] = e; }
        }
        __syncthreads();
        // ---- pass B (hypothesis 0 already ran from its exact start)
        int endst = tails[w < nh ? w : 0];
        if (w > 0 && w < nh) {
            endst = run_acs(rA[w - 1], true);
            const int r = chain6(endst);
            if (lane == 0) rB[w] = r;
        }
        __syncthreads();
        bool ok = true;
        for (int k = 1; k < nh - 1; k++) ok &= (rB[k] == rA[k]); // rA[k] was the start handed to hypothesis k+1
        if (!ok) { // (uniform) the guesses did not reproduce the serial chain: hand this chunk to the serial kernel
            if (threadIdx.x == 0) s_fallback = q;
            break;
        }
        // ---- full chainback (lane 0 of each warp; rows in shared memory) + decoded bits, MSB first
        if (w < nh) {
            if (lane == 0) {
                int st = endst, bit;
                for (int i = 0; i < 64; i++) tb[i] = 0;
                for (int row = steps - 1; row >= 6; row--) {
                    st = tb_step(st, dec[row].x, dec[row].y, bit);
                    const int i = row - 6;
                    tb[i >> 5] |= (unsigned)bit << (31 - (i & 31));
                }
                unsigned tail = 0;
                for (int k = tg.F - 6; k < tg.F; k++) tail = (tail << 1) | ((tb[k >> 5] >> (31 - (k & 31))) & 1u);
                tails[w] = (int)tail;
            }
            __syncwarp();
        }
        __syncthreads();
        // ---- BER with the chained encoder register (previous hypothesis' last six decoded bits)
        if (w < nh) {
            const unsigned enc = (unsigned)(w == 0 ? s_enc : tails[w - 1]);
            int errors = 0, total = 0;
            for (int t = lane; t < tg.F; t += 32) {
                unsigned reg = 0;
                for (int k = 6; k >= 0; k--) {
                    const int idx = t - k;
                    const unsigned b = idx >= 0 ? ((tb[idx >> 5] >> (31 - (idx & 31))) & 1u) : ((enc >> (-idx - 1)) & 1u);
                    reg = (reg << 1) | b;
                }
                const int e0 = parity_u32(reg & 79u), e1 = parity_u32(reg & 109u);
                const int sy = vit_symbols(c, t, tg, h, VIT_TESTLEN, 0);
                const int s0 = sy & 255, s1 = sy >> 8;
                if (2 * t < nsym && s0 != 128) { errors += ((s0 > 127) != e0); total++; }
                if (2 * t + 1 < nsym && s1 != 128) { errors += ((s1 > 127) != e1); total++; }
            }
            for (int off = 16; off; off >>= 1) {
                errors += __shfl_xor_sync(0xffffffffu, errors, off);
                total += __shfl_xor_sync(0xffffffffu, total, off);
            }
            if (lane == 0) { errs[w] = errors; tots[w] = total; }
        }
        __syncthreads();
        // ---- the lock decision, in the reference's order (viterbi_3_4.cpp:130-141) — every thread evaluates it identically
        best = 10.f;
        int lock = -1;
        for (int k = 0; k < nh; k++) {
            const float b = ((float)errs[k] / (float)tots[k]) * (g.rate34 ? 5.0f : 2.5f);
            const int ks = k / (nphases * 2), kp = ((k / 2) % nphases) == 0 ? ph0 : ph1, ksh = k & 1;
            bers[(ks * 4 + kp) * 2 + ksh] = b;
            if ((best == 10.f && b < thr) || (best < 10.f && b < best)) { best = b; lock = q; lswap = ks; lphase = kp; lshift = ksh; }
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_dec = rB[nh - 1]; s_enc = tails[nh - 1]; s_lock = lock; }
        __syncthreads();
        if (lock >= 0) break;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        VitIdle2Out r;
        r.o.lock_chunk = s_lock; r.o.swap = lswap; r.o.phase = lphase; r.o.shift = lshift; r.o.ber = best;
        for (int i = 0; i < 16; i++) r.o.bers[i] = bers[i];
        r.o.st.dec_start = s_dec; r.o.st.enc_state = s_enc; r.o.head = 0;
        r.fallback_chunk = s_fallback; r.pad[0] = r.pad[1] = r.pad[2] = 0;
        *out = r;
    }
}

// ---------------------------------------------------------------- bit FIFO assembly (+ NRZ-M)
// Appends the F bits of each output chunk (chunk-local word stores) to the contiguous MSB-first bit FIFO at bit offset
// `fifo_bits0`. With nrzm, out[i] = b[i] ^ b[i-1] with the very first predecessor = last_bit (NRZMDiff::decode_bits).
__device__ __forceinline__ uint32_t stream_get32(const uint32_t *__restrict__ chunk_bits, long total, int F, int bit_words, long i, int last_bit)
{
    // bits [i, i+32) of the concatenated chunk bit stream; bit -1 = last_bit; bits >= total = 0
    if (i >= 0 && i + 32 <= total) {
        const long c = i / F;
        const int k = (int)(i - c * F);
        if (k + 32 <= F) {
            const uint32_t *p = chunk_bits + c * bit_words + (k >> 5);
            const int o = k & 31;
            return o ? ((p[0] << o) | (p[1] >> (32 - o))) : p[0];
        }
    }
    uint32_t v = 0;
    for (int b = 0; b < 32; b++) {
        const long j = i + b;
        unsigned bit = 0;
        if (j < 0) bit = (unsigned)last_bit & 1u;
        else if (j < total) {
            const long c = j / F;
            const int k = (int)(j - c * F);
            bit = (chunk_bits[c * bit_words + (k >> 5)] >> (31 - (k & 31))) & 1u;
        }
        v |= bit << (31 - b);
    }
    return v;
}

__global__ void k_bits_append(const uint32_t *__restrict__ chunk_bits, long nchunks, int F, int bit_words, int nrzm, int last_bit,
                              uint32_t *__restrict__ fifo, long fifo_bits0)
{
    const long total = nchunks * (long)F;
    const long w0 = fifo_bits0 >> 5, w1 = (fifo_bits0 + total + 31) >> 5;
    for (long w = w0 + (long)blockIdx.x * blockDim.x + threadIdx.x; w < w1; w += (long)gridDim.x * blockDim.x) {
        const long i = (w << 5) - fifo_bits0; // stream index of this word's MSB (may be negative in the first word)
        uint32_t v = stream_get32(chunk_bits, total, F, bit_words, i, last_bit);
        if (nrzm) v ^= stream_get32(chunk_bits, total, F, bit_words, i - 1, last_bit);
        uint32_t mask = 0xffffffffu;
        if (i < 0) mask &= 0xffffffffu >> (-i);                 // keep the old bits in front
        if (i + 32 > total) mask &= ~(0xffffffffu >> (total - i)); // nothing valid behind the end
        fifo[w] = (mask == 0xffffffffu) ? v : ((fifo[w] & ~mask) | (v & mask));
    }
}

__global__ void k_words_move(uint32_t *__restrict__ dst, const uint32_t *__restrict__ src, long n) // forward copy, dst < src, single CTA
{
    for (long base = 0; base < n; base += blockDim.x) {
        long i = base + threadIdx.x;
        uint32_t v = 0;
        if (i < n) v = src[i];
        __syncthreads();
        if (i < n) dst[i] = v;
        __syncthreads();
    }
}

__device__ __forceinline__ uint32_t fifo_window(const uint32_t *__restrict__ fifo, long first_bit)
{
    // 32 bits starting at bit index first_bit (MSB first)
    const long w = first_bit >> 5;
    const int o = (int)(first_bit & 31);
    const uint32_t a = fifo[w];
    if (o == 0) return a;
    return (a << o) | (fifo[w + 1] >> (32 - o));
}

// ---------------------------------------------------------------- hard decisions of ccsds_simple_psk_decoder (no convolutional code)
// One loop iteration of CCSDSSimplePSKDecoderModule::process (module_ccsds_simple_psk_decoder.cpp:144-262) takes `n` = cadu_size soft
// bytes and makes n bits out of them; here every thread makes one 32-bit word of one chunk's bit store (the chunk_bits layout
// k_bits_append reads). carry_in / carry_out: [0] = original I of the last symbol (the oqpsk_delay register), [1] = hard symbol of
// the last symbol (QPSKDiff's buffer) of the previous / this call.
//   BPSK              bitsB[k] = soft[k] > 0                                  (:151-158; NRZ-M is applied by k_bits_append)
//   QPSK, no NRZ-M    bitsA = (Q>0),(I>0) of the symbols as they are -> second deframer (:190-199); bitsB = the same after
//                     rotate_soft(PHASE_90): (I',Q') = (Q,-I)                 -> main deframer (:201-210)
//   QPSK, NRZ-M       QPSKDiff (differential/qpsk_diff.cpp:5-53) over the hard symbols 2*(Q>0)+(I>0): output i of the stream's very
//                     first chunk comes from symbols (i+1, i+2) and its last four bits are never written (left 0 here); afterwards
//                     output g comes from symbols (g-1, g)
struct SliceCfg { int n, bit_words, qpsk, nrzm, swap_iq, swap_diff, delay; };
__global__ void k_slice(const int8_t *__restrict__ soft, long nchunks, SliceCfg P, long first_global_chunk, const int *__restrict__ carry_in,
                        int *__restrict__ carry_out, uint32_t *__restrict__ bitsA, uint32_t *__restrict__ bitsB)
{
    const int wpc = (P.n + 31) >> 5; // words per chunk
    const long nw = nchunks * wpc;
    const long nsym_total = nchunks * (long)(P.n >> 1);
    auto sym_iq = [&](long g, int &I, int &Q) { // symbol g of this call after oqpsk_delay and qpsk_swap_iq
        int i0 = soft[2 * g], q0 = soft[2 * g + 1];
        if (P.delay)
            i0 = g > 0 ? soft[2 * (g - 1)] : carry_in[0];
        if (P.swap_iq) {
            const int t = i0;
            i0 = q0;
            q0 = t;
        }
        I = i0;
        Q = q0;
    };
    auto hard_sym = [&](long g) -> int { // constellation_t::soft_demod for QPSK: 2*(Q>0) + (I>0); g = -1: previous call's last
        if (g < 0)
            return carry_in[1];
        int I, Q;
        sym_iq(g, I, Q);
        return 2 * (Q > 0) + (I > 0);
    };
    for (long w = (long)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (long)gridDim.x * blockDim.x) {
        const long c = w / wpc;
        const int k0 = (int)(w - c * wpc) << 5;
        uint32_t a = 0, b = 0;
        for (int j = 0; j < 32 && k0 + j < P.n; j++) {
            const int k = k0 + j;
            unsigned ba = 0, bb = 0;
            if (!P.qpsk)
                bb = soft[c * P.n + k] > 0;
            else {
                const long g = c * (long)(P.n >> 1) + (k >> 1); // symbol of this call
                if (!P.nrzm) {
                    int I, Q;
                    sym_iq(g, I, Q);
                    ba = (k & 1) ? (I > 0) : (Q > 0);
                    bb = (k & 1) ? (Q > 0) : (I < 0);
                } else {
                    const bool first = first_global_chunk + c == 0;
                    long g0, g1; // the pair (older, newer)
                    if (first) {
                        g0 = g + 1;
                        g1 = g + 2;
                    } else {
                        g0 = g - 1;
                        g1 = g;
                    }
                    if (first && (k >> 1) >= (P.n >> 1) - 2)
                        bb = 0; // never written by the reference's first call
                    else {
                        const int s0 = hard_sym(g0), s1 = hard_sym(g1);
                        const int Xin_1 = s0 & 2, Yin_1 = s0 & 1, Xin = s1 & 2, Yin = s1 & 1;
                        int ou;
                        if (((Xin >> 1) ^ Yin) == 1) {
                            const int Xout = Yin_1 ^ Yin, Yout = Xin_1 ^ Xin;
                            ou = (Xout << 1) + (Yout >> 1);
                        } else {
                            const int Xout = Xin_1 ^ Xin, Yout = Yin_1 ^ Yin;
                            ou = Xout + Yout;
                        }
                        const int b0 = P.swap_diff ? (ou & 1) : (ou >> 1), b1 = P.swap_diff ? (ou >> 1) : (ou & 1);
                        bb = (k & 1) ? b1 : b0;
                    }
                }
            }
            a |= ba << (31 - j);
            b |= bb << (31 - j);
        }
        const long o = c * P.bit_words + (k0 >> 5);
        if (bitsA)
            bitsA[o] = a;
        bitsB[o] = b;
        if (w == nw - 1 && P.qpsk) {
            carry_out[0] = soft[2 * (nsym_total - 1)];
            carry_out[1] = hard_sym(nsym_total - 1);
        }
    }
}

// ---------------------------------------------------------------- deframer walk (one warp), frame level replay of the bit-serial machine
#endif // B200_DEFINE_KERNELS
struct DefrState
{
    int state;       // 2 NOSYNC, SYNCING value (6; FengYun 8), SYNCED value (12 / 18; FengYun 16): the numeric values double as thresholds
    int inversion, good, bad;
    long pos;        // FIFO bit index of the next bit the machine examines with its shifter (when not inside a frame)
    long frame_pay;  // >= 0: a frame is open, payload starts at this FIFO bit index (its ASM ended at frame_pay-1)
};
struct FrameRec { long pay_bit; int inversion; int pad; };
struct DefrEventDev { long pos; int state; int pad; };

// counters_out[0] = frames found, [1] = state-change events recorded (events[]: bit index at which the state changed)
#ifdef B200_DEFINE_KERNELS
__global__ void __launch_bounds__(32) k_deframe(const uint32_t *__restrict__ fifo, long nbits, int cadu_size, int st_syncing, int st_synced, uint32_t sync,
                                                 DefrState *__restrict__ st_io, FrameRec *__restrict__ frames, int max_frames,
                                                 DefrEventDev *__restrict__ events, int max_events, int *__restrict__ counters_out)
{
    const int lane = threadIdx.x;
    DefrState S = *st_io;
    int nf = 0, ne = 0;
    auto note = [&](long pos, int state) {
        if (lane == 0 && ne < max_events) events[ne] = DefrEventDev{pos, state, 0};
        ne++;
    };
    const long pay_bits = cadu_size - 32;
    bool stop = false;
    while (!stop) {
        if (S.frame_pay >= 0) {
            // open frame: complete once its last payload bit is present; the next shifter test is cadu_size bits after the ASM end
            if (S.frame_pay + pay_bits <= nbits) {
                if (lane == 0 && nf < max_frames) frames[nf] = FrameRec{S.frame_pay, S.inversion, 0};
                nf++;
                S.pos = S.frame_pay - 1 + cadu_size;
                S.frame_pay = -1;
            } else
                break;
            continue;
        }
        if (S.pos >= nbits) break;
        if (S.state == 2) {
            // bit-level search for an exact ASM / inverted ASM, 32 candidate end positions per iteration
            long p = S.pos;
            int found = -1, inv = 0;
            while (p < nbits) {
                const long e = p + lane;
                unsigned hit = 0;
                if (e < nbits) {
                    const uint32_t wv = fifo_window(fifo, e - 31);
                    hit = (wv == sync) ? 1u : ((wv == ~sync) ? 2u : 0u);
                }
                const unsigned any = __ballot_sync(0xffffffffu, hit != 0);
                if (any) {
                    const int l = __ffs(any) - 1;
                    found = l;
                    inv = __shfl_sync(0xffffffffu, (int)hit, l) == 2;
                    break;
                }
                p += 32;
            }
            if (found < 0) { S.pos = nbits; break; }
            const long e = p + found;
            S.inversion = inv;
            S.frame_pay = e + 1;
            S.state = st_syncing;
            S.good = S.bad = 0;
            note(e, st_syncing);
            continue;
        }
        if (S.state != st_syncing) {
            // SYNCED: 128 frames of lookahead per iteration (4 independent loads per lane, so their latencies overlap); lane l tests
            // the ASMs expected l, l+32, l+64, l+96 frames ahead. n = leading passes, m = how many of those are complete.
            constexpr int G = 4;
            unsigned pm[G], cm[G];
            const uint32_t want = S.inversion ? ~sync : sync;
#pragma unroll
            for (int gq = 0; gq < G; gq++) {
                const long e = S.pos + (long)(lane + 32 * gq) * cadu_size;
                bool pass = false;
                if (e < nbits)
                    pass = __popc(fifo_window(fifo, e - 31) ^ want) < st_synced;
                pm[gq] = __ballot_sync(0xffffffffu, pass);
                cm[gq] = __ballot_sync(0xffffffffu, pass && (e + 1 + pay_bits <= nbits));
            }
            int n = 0, m = 0;
            bool nrun = true, mrun = true;
#pragma unroll
            for (int gq = 0; gq < G; gq++) {
                if (nrun) {
                    const int k = (pm[gq] == 0xffffffffu) ? 32 : (__ffs(~pm[gq]) - 1);
                    n += k;
                    nrun = k == 32;
                }
                if (mrun) {
                    const int k = (cm[gq] == 0xffffffffu) ? 32 : (__ffs(~cm[gq]) - 1);
                    m += k;
                    mrun = k == 32;
                }
            }
            m = min(m, n);
#pragma unroll
            for (int gq = 0; gq < G; gq++) {
                const int f = lane + 32 * gq;
                if (f < m && nf + f < max_frames)
                    frames[nf + f] = FrameRec{S.pos + (long)f * cadu_size + 1, S.inversion, 0};
            }
            nf += m;
            const long e_m = S.pos + (long)m * cadu_size;
            if (m < n) { S.frame_pay = e_m + 1; S.pos = e_m; break; }                   // accepted, payload still arriving
            if (n == 32 * G) { S.pos = e_m; continue; }
            if (e_m >= nbits) { S.pos = e_m; break; }                                    // next ASM not here yet
            S.good = S.bad = 0; S.state = 2; S.pos = e_m + 1;                            // hard NOSYNC (bpsk_ccsds_deframer.cpp:98-102)
            note(e_m, 2);
            continue;
        }
        // SYNCING: single test at S.pos (bit index of the window's last bit)
        {
            const uint32_t wv = fifo_window(fifo, S.pos - 31);
            const int diff = __popc(wv ^ (S.inversion ? ~sync : sync));
            if (diff < st_syncing) {
                S.frame_pay = S.pos + 1;
                S.bad = 0;
                S.good++;
                if (S.good > 10) { S.state = st_synced; note(S.pos, st_synced); }
            } else {
                S.bad++;
                S.good = 0;
                if (S.bad > 2) { S.state = 2; note(S.pos, 2); }
                S.pos++;
            }
        }
    }
    if (lane == 0) {
        *st_io = S;
        counters_out[0] = nf;
        counters_out[1] = ne;
    }
}

// ---------------------------------------------------------------- frame extraction + derandomiser + Reed-Solomon
#endif // B200_DEFINE_KERNELS
struct RsTables
{
    uint8_t exp[512];
    uint8_t log[256];
    uint8_t to_dual[256];
    uint8_t from_dual[256];
    uint8_t pn[255];
    uint8_t pad;
};

struct FrameCfg
{
    int cadu_bytes, cadu_size; // bytes (ceil) and bits
    int derandomize, derand_after_rs, derand_start;
    int rs_i, rs_dual, rs_nroots, rs_fcr;
    uint32_t sync;
    int rs_row256; // rs_fill_bytes -1: the reference's (de)interleave runs one row past the codewords (see rs_decode_interleave)
};

// (the Reed-Solomon device code up to k_frames is also used by the MetOp dump decoder's frame kernel, dump.cuh)
__device__ __forceinline__ uint8_t gf_mul(const RsTables &T, uint8_t a, uint8_t b) { return (!a || !b) ? 0 : T.exp[T.log[a] + T.log[b]]; }
__device__ __forceinline__ uint8_t gf_div(const RsTables &T, uint8_t a, uint8_t b) { return (!a || !b) ? 0 : T.exp[255 + T.log[a] - T.log[b]]; }
__device__ __forceinline__ uint8_t gf_pow(const RsTables &T, uint8_t a, int p) { return T.exp[((int)T.log[a] * p) % 255]; }
__device__ __forceinline__ uint8_t log_mul(uint8_t a, uint8_t b) { unsigned r = (unsigned)a + b; return r > 255 ? r - 255 : r; }

// Sequential part of correct_reed_solomon_decode (decode.c:32-222,340-378) on one lane. r[] is the received polynomial
// (r[i] = codeword byte 254-i), syn[] its syndromes. Returns false when the locator does not factor (decode failure).
// libcorrect's decoder after the syndromes (decode.c:32-222), one warp per codeword, results identical to the serial code:
//   Berlekamp-Massey with its order bookkeeping (:32-118): lane 0 (a data-dependent recurrence over the 32 syndromes);
//   Chien search over all 256 field elements (:122-145): lane l tests elements 8l .. 8l+7, the roots are written in ascending order
//     (per-lane bit masks, prefix counts by shuffles) and accepted iff their number equals the locator's order;
//   error evaluator (polynomial.c: omega = lambda * syndromes mod x^nroots): lane k makes coefficient k;
//   Forney (:165-196) + the location search (:198-222): lane q handles root q. The reference finds the location by scanning j = 0..255
//     for j^11 == 1/root; that is j = (1/root)^(11^-1 mod 255), i.e. log j = 116 * log(1/root) mod 255 - except that its scan meets
//     j = 0 first, whose "power" reads exp[0] = 1: for 1/root == 1 the location is log[0] = 0 (checked against the scan for every value).
__device__ inline bool rs_correct_warp(const RsTables &T, uint8_t *r, const uint8_t *syn, int nroots, int fcr, uint8_t *lam, uint8_t *prev, uint8_t *lamlog,
                                uint8_t *roots, uint8_t *om, uint8_t *der, int lane)
{
    unsigned order = 0;
    if (lane == 0) {
        for (int i = 0; i < 66; i++) lam[i] = prev[i] = 0;
        lam[0] = prev[0] = 1;
        unsigned Lr = 0, prev_order = 0, delay = 1;
        uint8_t last_d = 1;
        for (unsigned i = 0; i < (unsigned)nroots; i++) {
            uint8_t d = syn[i];
            for (unsigned j = 1; j <= Lr; j++) d ^= gf_mul(T, lam[j], syn[i - j]);
            if (!d) { delay++; continue; }
            if (2 * Lr <= i) {
                for (int j = (int)prev_order; j >= 0; j--) prev[j + delay] = gf_div(T, gf_mul(T, prev[j], d), last_d);
                for (int j = (int)delay - 1; j >= 0; j--) prev[j] = 0;
                for (unsigned j = 0; j <= prev_order + delay; j++) { uint8_t t = lam[j]; lam[j] ^= prev[j]; prev[j] = t; }
                unsigned t = order; order = prev_order + delay; prev_order = t;
                Lr = i + 1 - Lr; last_d = d; delay = 1;
                continue;
            }
            for (int j = (int)prev_order; j >= 0; j--) lam[j + delay] ^= gf_div(T, gf_mul(T, prev[j], d), last_d);
            if (prev_order + delay > order) order = prev_order + delay;
            delay++;
        }
        for (unsigned i = 0; i <= order; i++) lamlog[i] = T.log[lam[i]];
    }
    order = __shfl_sync(0xffffffffu, order, 0);
    __syncwarp();
    // Chien: lambda at every field element
    unsigned mask = 0;
#pragma unroll 1
    for (int k = 0; k < 8; k++) {
        const int e = 8 * lane + k;
        uint8_t v;
        if (e == 0) v = lamlog[0] ? T.exp[lamlog[0]] : 0;
        else {
            const uint8_t el = T.log[e];
            uint8_t pw = T.log[1];
            v = 0;
            for (unsigned i = 0; i <= order; i++) { if (lamlog[i]) v ^= T.exp[lamlog[i] + pw]; pw = log_mul(pw, el); }
        }
        if (!v) mask |= 1u << k;
    }
    int pos = __popc(mask), nr;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, pos, off);
        if (lane >= off) pos += o;
    }
    nr = __shfl_sync(0xffffffffu, pos, 31);
    pos -= __popc(mask); // exclusive
    for (int k = 0; k < 8; k++)
        if (mask >> k & 1) {
            if (pos < 64) roots[pos] = (uint8_t)(8 * lane + k);
            pos++;
        }
    if ((unsigned)nr != order) return false;
    // omega and lambda' (nroots <= 32 coefficients: one per lane)
    if (lane < nroots) {
        uint8_t acc = 0;
        const unsigned top = min(order, (unsigned)lane);
        for (unsigned i = 0; i <= top; i++) acc ^= gf_mul(T, lam[i], syn[lane - i]);
        om[lane] = acc;
    }
    if ((unsigned)lane < order) der[lane] = ((lane + 1) % 2) ? lam[lane + 1] : 0;
    __syncwarp();
    const int gapinv = 116; // 11 * 116 = 5 * 255 + 1
    if ((unsigned)lane < order) {
        const uint8_t root = roots[lane];
        if (root != 0) {
            const uint8_t locv = gf_div(T, 1, root);
            const uint8_t loc = locv == 1 ? 0 : (uint8_t)(((int)T.log[locv] * gapinv) % 255);
            const uint8_t el = T.log[root];
            uint8_t pw = T.log[1], num = 0, den = 0;
            for (int i = 0; i < nroots; i++) { if (om[i]) num ^= T.exp[T.log[om[i]] + pw]; pw = log_mul(pw, el); }
            pw = T.log[1];
            for (unsigned i = 0; i + 1 <= order; i++) { if (der[i]) den ^= T.exp[T.log[der[i]] + pw]; pw = log_mul(pw, el); }
            r[loc] ^= gf_mul(T, gf_pow(T, root, fcr - 1), gf_div(T, num, den)); // (distinct roots -> distinct locations)
        }
    }
    __syncwarp();
    return true;
}

constexpr int RS_MAX_I = 8;

// decode_interlaved for interleave `warp` of the frame in shared memory, by one warp (`work`: its 704 bytes of scratch): deinterleave,
// dual basis -> conventional, syndromes, then rs_correct_warp. Writes the corrected message bytes back into the frame; returns -1 when
// the codeword does not decode, else the number of message bytes changed.
__device__ __forceinline__ int rs_decode_interleave(const RsTables &T, uint8_t *frame, const FrameCfg &fc, uint8_t *work, int warp, int lane)
{
    uint8_t *r = work, *syn = r + 256, *lam = syn + 64, *prev = lam + 66, *lamlog = prev + 66, *roots = lamlog + 66, *om = roots + 64,
            *der = om + 32;
    // deinterleave + dual->conventional + reverse: r[i] = cw[254-i]  (reedsolomon.cpp:145-149,73-77; decode.c:322-324)
    for (int i = lane; i < 255; i += 32) {
        uint8_t v = frame[4 + (254 - i) * fc.rs_i + warp];
        r[i] = fc.rs_dual ? T.from_dual[v] : v;
    }
    __syncwarp();
    // syndromes, lane j -> syndrome j (decode.c:12-28)
    uint8_t s = 0;
    if (lane < fc.rs_nroots) {
        const uint8_t rootlog = T.log[T.exp[(11 * (lane + fc.rs_fcr)) % 255]];
        uint8_t pw = T.log[1];
#pragma unroll 5
        for (int i = 0; i < 255; i++) {
            const uint8_t v = r[i];
            if (v) s ^= T.exp[T.log[v] + pw];
            pw = log_mul(pw, rootlog);
        }
        syn[lane] = s;
    }
    const unsigned nz = __ballot_sync(0xffffffffu, s != 0);
    __syncwarp();
    int err = 0;
    if (nz) {
        const int ok = rs_correct_warp(T, r, syn, fc.rs_nroots, fc.rs_fcr, lam, prev, lamlog, roots, om, der, lane) ? 1 : 0;
        if (!ok) err = -1;
        else {
            // copy back the message bytes only; parity stays as received (reedsolomon.cpp:96-104)
            const int k = 255 - fc.rs_nroots;
            int changed = 0;
            for (int i = lane; i < k; i += 32) {
                const uint8_t nv = r[254 - i];
                const int idx = 4 + i * fc.rs_i + warp;
                const uint8_t ov = fc.rs_dual ? T.from_dual[frame[idx]] : frame[idx];
                if (nv != ov) changed++;
                frame[idx] = fc.rs_dual ? T.to_dual[nv] : nv;
            }
            for (int off = 16; off; off >>= 1) changed += __shfl_xor_sync(0xffffffffu, changed, off);
            err = changed;
        }
    }
    // With rs_fill_bytes -1 the reference's (de)interleave loops run 256 rows (reedsolomon.cpp:145-155): byte 4 + 255*I + warp is read
    // into the slot one past its 255-byte codeword buffer, which is the first byte of its message buffer (reedsolomon.h:24-25), and is
    // written back from there: the corrected first message byte (conventional basis) when the word decodes, unchanged when it does not.
    // Here that byte is a spare byte of a CADU longer than 4 + 255*I; no other warp reads it. (When the CADU ends with the codewords the
    // reference writes the next frame of its module call instead; that is not restated.)
    const int spare = 4 + 255 * fc.rs_i + warp;
    if (fc.rs_row256 && err >= 0 && spare < fc.cadu_bytes && lane == 0) frame[spare] = r[254];
    return err;
}

#ifdef B200_DEFINE_KERNELS
// One CTA per frame; warp w decodes interleave w (up to 8 warps). Writes the frame (cadu_bytes) and rs_err[frame*rs_i + w].
__global__ void __launch_bounds__(256) k_frames(const uint32_t *__restrict__ fifo, const FrameRec *__restrict__ frames, int nframes, FrameCfg fc,
                                                 const RsTables *__restrict__ gtab, uint8_t *__restrict__ out, int *__restrict__ rs_err)
{
    extern __shared__ __align__(16) unsigned char fr_smem[];
    RsTables &T = *reinterpret_cast<RsTables *>(fr_smem);
    uint8_t *frame = fr_smem + sizeof(RsTables);                 // cadu_bytes (+pad)
    uint8_t *work = frame + ((fc.cadu_bytes + 15) & ~15);        // per warp: r[256] syn[64] lam[66] prev[66] lamlog[66] roots[64] om[32] der[66] = 680 -> 704
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < (int)sizeof(RsTables) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(&T)[i] = reinterpret_cast<const uint32_t *>(gtab)[i];
    for (int f = blockIdx.x; f < nframes; f += gridDim.x) {
        __syncthreads();
        const FrameRec fr = frames[f];
        // reset_frame + write_bit: ASM forced clean, payload bits XOR inversion (bpsk_ccsds_deframer.cpp:109-122). The derandomiser runs
        // from derand_start over the whole CADU, so with derand_start < 4 it also covers the (clean) ASM bytes
        const int pay_bytes = fc.cadu_bytes - 4;
        for (int i = t; i < fc.cadu_bytes; i += blockDim.x) {
            uint8_t b;
            if (i < 4) {
                b = (uint8_t)(fc.sync >> (24 - 8 * i));
                if (fc.derandomize && !fc.derand_after_rs && i >= fc.derand_start) b ^= T.pn[(i - fc.derand_start) % 255];
            } else {
                const long bit0 = fr.pay_bit + 8L * (i - 4);
                uint32_t wv = fifo_window(fifo, bit0);
                b = (uint8_t)(wv >> 24);
                if (fr.inversion) b = ~b;
                const int valid = fc.cadu_size - 8 * i; // bits of this byte that belong to the frame (padding case)
                if (valid < 8) b = (valid <= 0) ? 0 : (uint8_t)(b >> (8 - valid)); // write_bit shifts partial bytes in from the right
                if (fc.derandomize && !fc.derand_after_rs && i >= fc.derand_start) b ^= T.pn[(i - fc.derand_start) % 255];
            }
            frame[i] = b;
        }
        (void)pay_bytes;
        __syncthreads();
        if (warp < fc.rs_i) {
            const int err = rs_decode_interleave(T, frame, fc, work + warp * 704, warp, lane);
            if (lane == 0) rs_err[(long)f * fc.rs_i + warp] = err;
        }
        __syncthreads();
        for (int i = t; i < fc.cadu_bytes; i += blockDim.x) {
            uint8_t b = frame[i];
            if (fc.derandomize && fc.derand_after_rs && i >= fc.derand_start) b ^= T.pn[(i - fc.derand_start) % 255];
            out[(long)f * fc.cadu_bytes + i] = b;
        }
    }
}

// rs_usecheck: keep only frames whose interleaves all decoded (module_ccsds_conv_concat_decoder.cpp:183-195). k_frames_filter: single CTA,
// exclusive scan of the keep flags -> destination index of every frame (-1: dropped) and the number kept; k_frames_gather: one CTA per
// frame copies it (coalesced) to its place.
__global__ void __launch_bounds__(1024) k_frames_filter(const int *__restrict__ rs_err, int nframes, int rs_i, int *__restrict__ dst_index, int *__restrict__ nkept)
{
    __shared__ int wsum[32];
    __shared__ int run;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) run = 0;
    __syncthreads();
    for (int base = 0; base < nframes; base += 1024) {
        const int f = base + t;
        int ok = 0;
        if (f < nframes) {
            ok = 1;
            for (int j = 0; j < rs_i; j++)
                if (rs_err[(long)f * rs_i + j] == -1) ok = 0;
        }
        int v = ok;
        for (int off = 1; off < 32; off <<= 1) { int p = __shfl_up_sync(0xffffffffu, v, off); if (lane >= off) v += p; }
        if (lane == 31) wsum[warp] = v;
        __syncthreads();
        if (warp == 0) {
            int w = wsum[lane];
            for (int off = 1; off < 32; off <<= 1) { int p = __shfl_up_sync(0xffffffffu, w, off); if (lane >= off) w += p; }
            wsum[lane] = w;
        }
        __syncthreads();
        const int incl = run + v + (warp > 0 ? wsum[warp - 1] : 0);
        if (f < nframes) dst_index[f] = ok ? incl - 1 : -1;
        __syncthreads();
        if (t == 1023) run = incl;
        __syncthreads();
    }
    if (t == 0) *nkept = run;
}
__global__ void __launch_bounds__(256) k_frames_gather(const uint8_t *__restrict__ in, const int *__restrict__ dst_index, int nframes, int cadu_bytes,
                                                       uint8_t *__restrict__ out)
{
    for (int f = blockIdx.x; f < nframes; f += gridDim.x) {
        const int d = dst_index[f];
        if (d < 0) continue;
        const uint8_t *s = in + (long)f * cadu_bytes;
        uint8_t *o = out + (long)d * cadu_bytes;
        for (int i = threadIdx.x; i < cadu_bytes; i += blockDim.x) o[i] = s[i];
    }
}

#endif // B200_DEFINE_KERNELS
} // namespace b200
