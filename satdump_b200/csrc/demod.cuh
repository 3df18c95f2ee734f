// Demodulator kernels (sm_90a): raw IQ -> AGC -> 31-tap RRC FIR -> Costas -> [OQPSK delay] -> M&M -> int8 soft.
//
// Reference semantics being reproduced (SatDump tree):
//   sample conversion   src-core/common/dsp/io/baseband_interface.h:170-190
//   AGC                 src-core/common/dsp/utils/agc.cpp:25-39
//   RRC FIR             src-core/common/dsp/filter/fir.cpp:47-89, firdes.cpp:34-78
//   Costas loop         src-core/common/dsp/pll/costas_loop.cpp:23-65
//   OQPSK delay         src-core/common/dsp/demod/delay_one_imag.cpp:18-25
//   M&M clock recovery  src-core/common/dsp/clock_recovery/clock_recovery_mm.cpp:52-121
//   soft quantiser      src-core/pipeline/modules/demod/module_psk_demod.cpp:199-213
//   pm_demod / carrier mode: carrier PLL  src-core/common/dsp/pll/pll_carrier_tracking.cpp:25-70 (+ utils/fast_trig.cpp), PMToBPSK
//                       src-core/common/dsp/demod/pm_to_bpsk.cpp:10-35, FreqShiftBlock src-core/common/dsp/utils/freq_shift.cpp:16-50
//
// The reference runs every stage as a serial per-sample loop. Here:
//   * AGC: g' = g(1-r|x|) + r is an affine map -> per-tile composition (k_agc_compose), a scan over tiles
//     (k_tile_scan) and an in-tile block scan in fp64, then an 8-sample replay of the reference's float recurrence.
//   * FIR: data parallel, fused with conversion + AGC scale (k_agc_fir_w).
//   * Costas / M&M: contracting feedback loops -> one thread per stream segment, started W samples early
//     (warm-up) so it has converged onto the sequential trajectory at its first owned sample; the first segment
//     starts from the exact carried state. Costas segments converge up to a k*2pi/order rotation, which
//     k_costas_fix resolves as a prefix sum; k_mm applies it (exactly) to each input row it stages, since its TED
//     is not rotation invariant. Junction consistency is checked on the device and reported in the stats.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace b200
{

constexpr int FIR_NT = 31;           // taps
constexpr int FIR_TILE = 2048;       // samples (= outputs) per tile: 256 threads x 8
constexpr int FIR_THREADS = 256;
constexpr int FIR_BUF = FIR_TILE + 32;                   // smem tile with the 32-sample history in front
constexpr int FIR_BUF_F2 = FIR_BUF + 2 * (FIR_BUF / 8);  // padded (see xidx)
constexpr int RS_THREADS = 256;      // front-end resampler: outputs per CTA
constexpr int RS_MAX_TAPS = 160;     // taps per polyphase arm
constexpr int RS_SPAN = 2 * RS_THREADS + RS_MAX_TAPS + 8; // decimation < 2: at most 2 input samples per output
constexpr int SEG_THREADS = 128;     // threads (= stream segments) per CTA in the loop kernels
constexpr int MM_HIST = 16;       // inputs of the previous batch kept in the front pad (M&M reaches 7 back, Gardner up to 11)
constexpr int MM_BANK_STRIDE = 12; // floats per arm row in smem: 16-byte aligned rows (two 128-bit loads per arm), 8 bank groups
constexpr int MM_STAGE = 16;     // symbols per thread staged in smem between two coalesced copy-outs (one per 16-sample row)
// per CTA: the 64-sample rings, the bank, then per warp the staged symbols [MM_STAGE][32] and one int2 per thread for the copy-out
constexpr int MM_SMEM_BYTES = 64 * SEG_THREADS * 8 + 128 * MM_BANK_STRIDE * 4 + SEG_THREADS * (MM_STAGE + 1) * 8;

struct FirTaps { float h[32]; };

struct Affine { double a, b; };     // g -> a*g + b
struct Affine3 { double a, b, c; }; // g -> min(a*g + b, c): an AGC step with its max_gain clamp (agc.cpp:34-35); closed under composition
struct DcAff { double a, br, bi; };  // DC blocker: acc -> a*acc + (br, bi)
constexpr double AGC_NO_CLAMP = 1e30; // "c" of an Affine3 without a clamp (finite, so that a * c + b stays a number)

template <int FMT> struct RawBytes;
template <> struct RawBytes<0> { static constexpr int v = 8; };
template <> struct RawBytes<1> { static constexpr int v = 4; };
template <> struct RawBytes<2> { static constexpr int v = 2; };

// x / (2^B - 1) for an integer x of at most B bits, correctly rounded (= the generic VOLK converters' ((float)x) / scalar,
// SURVEY.md App. A.1) in two instructions. 1/(2^B-1) = 2^-B + 2^-2B + 2^-3B + ..., so with t = x*2^-B (exact) and
// c = 2^-2B + ... + 2^-mB (exact in a float), fma(x, c, t) is the single rounding of the series cut after m terms. The cut-off
// tail is below 2^-45 (cs16, m=3) / 2^-35 (cs8, m=5) of the quotient, and no rounding boundary can lie that close: a midpoint M
// with |x/(2^B-1) - M| that small would force x*2^k == odd*(2^B-1) with x*2^k even. tests/test_gpu_demod.py checks all 65 536 /
// 256 inputs bit for bit against the division.
__device__ __forceinline__ float cvt_s16(float x) { return fmaf(x, 0x1p-30f + 0x1p-45f, x * 0x1p-15f); }
__device__ __forceinline__ float cvt_s8(float x) { return fmaf(x, 0x1p-14f + 0x1p-21f + 0x1p-28f + 0x1p-35f, x * 0x1p-7f); }

// 8 consecutive complex samples: raw registers (so a tile's loads can be issued one tile ahead) and their conversion
#ifdef B200_DEFINE_KERNELS
template <int FMT> struct RawRegs;
template <> struct RawRegs<0> { float4 v[4]; };
template <> struct RawRegs<1> { int4 a, b; };
template <> struct RawRegs<2> { int4 a; };

// requires s0 + 8 <= n_valid; s0 a multiple of 8 relative to a 16-aligned base
template <int FMT> __device__ __forceinline__ void raw_fetch(const void *__restrict__ raw, long s0, RawRegs<FMT> &r)
{
    if constexpr (FMT == 1) {
        const int4 *p = reinterpret_cast<const int4 *>(reinterpret_cast<const int16_t *>(raw) + 2 * s0);
        r.a = __ldg(p);
        r.b = __ldg(p + 1);
    } else if constexpr (FMT == 2) {
        r.a = __ldg(reinterpret_cast<const int4 *>(reinterpret_cast<const int8_t *>(raw) + 2 * s0));
    } else {
        const float4 *p = reinterpret_cast<const float4 *>(reinterpret_cast<const float2 *>(raw) + s0);
#pragma unroll
        for (int i = 0; i < 4; i++)
            r.v[i] = __ldg(p + i);
    }
}

template <int FMT> __device__ __forceinline__ void raw_convert(const RawRegs<FMT> &r, float2 (&x)[8])
{
    if constexpr (FMT == 1) {
        const int w[8] = {r.a.x, r.a.y, r.a.z, r.a.w, r.b.x, r.b.y, r.b.z, r.b.w};
#pragma unroll
        for (int i = 0; i < 8; i++) {
            x[i].x = cvt_s16((float)(short)(w[i] & 0xFFFF));
            x[i].y = cvt_s16((float)(short)(w[i] >> 16));
        }
    } else if constexpr (FMT == 2) {
        const int w[4] = {r.a.x, r.a.y, r.a.z, r.a.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            x[2 * i].x = cvt_s8((float)(signed char)(w[i] & 0xFF));
            x[2 * i].y = cvt_s8((float)(signed char)((w[i] >> 8) & 0xFF));
            x[2 * i + 1].x = cvt_s8((float)(signed char)((w[i] >> 16) & 0xFF));
            x[2 * i + 1].y = cvt_s8((float)(signed char)((w[i] >> 24) & 0xFF));
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            x[2 * i] = make_float2(r.v[i].x, r.v[i].y);
            x[2 * i + 1] = make_float2(r.v[i].z, r.v[i].w);
        }
    }
}

// The same conversion with the power-of-two factor left out: x[i] = sample / S with S = 2^-15 (cs16), 2^-7 (cs8), 1 (cf32). Scaling by a
// power of two commutes with every rounding here (no subnormals in reach), so S * x[i] is bit for bit raw_convert's value; the fast
// path of k_agc_fir_w carries S in its per-sample gain (one multiply per sample instead of one per component).
template <int FMT> struct RawScale;
template <> struct RawScale<0> { static constexpr float v = 1.0f; };
template <> struct RawScale<1> { static constexpr float v = 0x1p-15f; };
template <> struct RawScale<2> { static constexpr float v = 0x1p-7f; };
__device__ __forceinline__ float cvt_s16_scaled(float x) { return fmaf(x, 0x1p-15f + 0x1p-30f, x); }
__device__ __forceinline__ float cvt_s8_scaled(float x) { return fmaf(x, 0x1p-7f + 0x1p-14f + 0x1p-21f + 0x1p-28f, x); }
template <int FMT> __device__ __forceinline__ void raw_convert_scaled(const RawRegs<FMT> &r, float2 (&x)[8])
{
    if constexpr (FMT == 1) {
        const int w[8] = {r.a.x, r.a.y, r.a.z, r.a.w, r.b.x, r.b.y, r.b.z, r.b.w};
#pragma unroll
        for (int i = 0; i < 8; i++) {
            x[i].x = cvt_s16_scaled((float)(short)(w[i] & 0xFFFF));
            x[i].y = cvt_s16_scaled((float)(short)(w[i] >> 16));
        }
    } else if constexpr (FMT == 2) {
        const int w[4] = {r.a.x, r.a.y, r.a.z, r.a.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            x[2 * i].x = cvt_s8_scaled((float)(signed char)(w[i] & 0xFF));
            x[2 * i].y = cvt_s8_scaled((float)(signed char)((w[i] >> 8) & 0xFF));
            x[2 * i + 1].x = cvt_s8_scaled((float)(signed char)((w[i] >> 16) & 0xFF));
            x[2 * i + 1].y = cvt_s8_scaled((float)(signed char)((w[i] >> 24) & 0xFF));
        }
    } else
        raw_convert<FMT>(r, x);
}

// samples beyond n_valid read as 0
template <int FMT> __device__ __forceinline__ void load8_ragged(const void *__restrict__ raw, long s0, long n_valid, float2 (&x)[8])
{
#pragma unroll
    for (int i = 0; i < 8; i++) {
        long s = s0 + i;
        float2 v = make_float2(0.f, 0.f);
        if (s < n_valid) {
            if (FMT == 1) {
                const int16_t *p = reinterpret_cast<const int16_t *>(raw) + 2 * s;
                v.x = cvt_s16((float)p[0]);
                v.y = cvt_s16((float)p[1]);
            } else if (FMT == 2) {
                const int8_t *p = reinterpret_cast<const int8_t *>(raw) + 2 * s;
                v.x = cvt_s8((float)p[0]);
                v.y = cvt_s8((float)p[1]);
            } else
                v = reinterpret_cast<const float2 *>(raw)[s];
        }
        x[i] = v;
    }
}

template <int FMT>
__device__ __forceinline__ void load8(const void *__restrict__ raw, long s0, long n_valid, float2 (&x)[8])
{
    if (s0 + 8 <= n_valid) {
        RawRegs<FMT> r;
        raw_fetch<FMT>(raw, s0, r);
        raw_convert<FMT>(r, x);
    } else
        load8_ragged<FMT>(raw, s0, n_valid, x);
}

// test hook: the conversion alone (8 samples per thread)
template <int FMT>
__global__ void k_convert_only(const void *__restrict__ raw, long N, float2 *__restrict__ out)
{
    const long s0 = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
    if (s0 >= N) return;
    float2 x[8];
    load8<FMT>(raw, s0, N, x);
    for (int i = 0; i < 8; i++)
        if (s0 + i < N) out[s0 + i] = x[i];
}

// ---------------------------------------------------------------- K0: front-end rational resampler (+ iq_swap)
// RationalResamplerBlock::process (resamp/rational_resampler.cpp:43-65) in closed form: with the carried counters (inc0, ctr0) of the
// batch, output j reads the ntaps-long window starting at buffer index inc0 + (ctr0 + j*D) / I with arm (ctr0 + j*D) % I of the
// polyphase bank, where buffer index b < ntaps-1 is the previous batch's tail and b >= ntaps-1 is input sample b - (ntaps-1).
// No feedback, so every output is independent: one thread per output, the CTA's input span staged (converted, optionally re<->im
// swapped: file_source.cpp:31-33) in shared memory. I = D = 1 with the one-tap bank {1} is the plain iq_swap pass.

template <int FMT> __device__ __forceinline__ float2 load1(const void *__restrict__ raw, long s)
{
    if (FMT == 1) {
        const short2 v = reinterpret_cast<const short2 *>(raw)[s];
        return make_float2(cvt_s16((float)v.x), cvt_s16((float)v.y));
    } else if (FMT == 2) {
        const char2 v = reinterpret_cast<const char2 *>(raw)[s];
        return make_float2(cvt_s8((float)v.x), cvt_s8((float)v.y));
    } else
        return reinterpret_cast<const float2 *>(raw)[s];
}

template <int FMT>
__global__ void __launch_bounds__(RS_THREADS) k_resample(const void *__restrict__ raw, long n_in, int iq_swap, const float2 *__restrict__ tail_in,
                                                         float2 *__restrict__ tail_out, const float *__restrict__ bank, int I, int D, int nt, long inc0,
                                                         long ctr0, long J, float2 *__restrict__ out)
{
    __shared__ float2 xs[RS_SPAN];
    const int t = threadIdx.x;
    const long j0 = (long)blockIdx.x * RS_THREADS;
    if (blockIdx.x == 0 && t < nt) { // new tail = buffer[n_in .. n_in + nt - 1) (memmove of rational_resampler.cpp:62)
        const long b = n_in + t;
        if (t < nt - 1) {
            float2 v = b < nt - 1 ? tail_in[b] : load1<FMT>(raw, b - (nt - 1));
            if (b >= nt - 1 && iq_swap)
                v = make_float2(v.y, v.x);
            tail_out[t] = v;
        }
    }
    if (j0 >= J)
        return;
    const long jl = min(j0 + RS_THREADS, J) - 1; // last output of this CTA
    const long b_first = inc0 + (ctr0 + j0 * D) / I, b_last = inc0 + (ctr0 + jl * D) / I + nt - 1;
    const int span = (int)(b_last - b_first + 1);
    for (int q = t; q < span; q += RS_THREADS) {
        const long b = b_first + q;
        float2 v;
        if (b < nt - 1)
            v = tail_in[b];
        else {
            v = load1<FMT>(raw, b - (nt - 1));
            if (iq_swap)
                v = make_float2(v.y, v.x);
        }
        xs[q] = v;
    }
    __syncthreads();
    const long j = j0 + t;
    if (j < J) {
        const long c = ctr0 + j * D;
        const int off = (int)(inc0 + c / I - b_first);
        const float *tp = bank + (long)(c % I) * nt;
        float re = 0.f, im = 0.f;
        for (int k = 0; k < nt; k++) {
            const float h = __ldg(tp + k);
            re = fmaf(xs[off + k].x, h, re);
            im = fmaf(xs[off + k].y, h, im);
        }
        out[j] = make_float2(re, im);
    }
}

// ---------------------------------------------------------------- K0'': power-of-two decimator stage (SmartResamplerBlock, ratio >= 2)
// One stage of PowerDecimatorBlock (resamp/power_decim.cpp:37-56) = DecimatingFIRBlock::process (filter/decimating_fir.cpp:46-87): output j
// is the ntaps-long dot product over the window ending at input sample inc0 + j * D, taps reversed so that taps_rev[0] meets the oldest
// sample; carried state = inc (phase of the decimation) and the last ntaps - 1 inputs. Buffer index b < nt - 1 is the previous batch's tail,
// b >= nt - 1 input sample b - (nt - 1), exactly the convention of k_resample (this IS the I = 1 case; a separate kernel because the
// windows of one CTA span D * 256 + nt samples, too many to stage for D up to 128). One thread per output, inputs through L1 / L2.
template <int FMT>
__global__ void __launch_bounds__(256) k_decim_fir(const void *__restrict__ raw, long n_in, int iq_swap, const float2 *__restrict__ tail_in,
                                                   float2 *__restrict__ tail_out, const float *__restrict__ taps_rev, int nt, int D, long inc0, long J,
                                                   float2 *__restrict__ out)
{
    const long j = (long)blockIdx.x * blockDim.x + threadIdx.x;
    auto at = [&](long b) {
        if (b < nt - 1)
            return tail_in[b];
        float2 v = load1<FMT>(raw, b - (nt - 1));
        return iq_swap ? make_float2(v.y, v.x) : v;
    };
    if (j < nt - 1) // new tail = buffer[n_in .. n_in + nt - 1)
        tail_out[j] = at(n_in + j);
    if (j >= J)
        return;
    const long b0 = inc0 + j * D;
    float re = 0.f, im = 0.f;
    for (int k = 0; k < nt; k++) {
        const float2 x = at(b0 + k);
        const float h = __ldg(taps_rev + k);
        re = fmaf(x.x, h, re);
        im = fmaf(x.y, h, im);
    }
    out[j] = make_float2(re, im);
}

// ---------------------------------------------------------------- affine recurrences scanned over 2048-sample tiles
// The DC blocker and the AGC's exact and clamp passes turn a serial recurrence into maps composed in fp64: per thread over its 8 samples,
// over the tile (tile_reduce), then across the tiles by one CTA (k_tile_scan) from the value carried over from the previous batch. Each
// map type has an identity, a composition compose(first, second) = second o first, a lane shuffle and its application to a seed.
__device__ __forceinline__ Affine compose(const Affine &first, const Affine &second)
{
    Affine r;
    r.a = second.a * first.a;
    r.b = fma(second.a, first.b, second.b);
    return r;
}
// (second o first)(g) = min(a2 min(a1 g + b1, c1) + b2, c2) = min(a2 a1 g + a2 b1 + b2, min(a2 c1 + b2, c2))   for a2 >= 0
__device__ __forceinline__ Affine3 compose(const Affine3 &first, const Affine3 &second)
{
    Affine3 r;
    r.a = second.a * first.a;
    r.b = fma(second.a, first.b, second.b);
    r.c = fmin(fma(second.a, first.c, second.b), second.c);
    return r;
}
__device__ __forceinline__ DcAff compose(const DcAff f, const DcAff s) { return DcAff{s.a * f.a, fma(s.a, f.br, s.br), fma(s.a, f.bi, s.bi)}; }

template <class M> __device__ __forceinline__ M ident();
template <> __device__ __forceinline__ Affine ident<Affine>() { return Affine{1.0, 0.0}; }
template <> __device__ __forceinline__ Affine3 ident<Affine3>() { return Affine3{1.0, 0.0, AGC_NO_CLAMP}; }
template <> __device__ __forceinline__ DcAff ident<DcAff>() { return DcAff{1.0, 0.0, 0.0}; }

__device__ __forceinline__ Affine shfl_up(const Affine &v, int off)
{
    return Affine{__shfl_up_sync(0xffffffffu, v.a, off), __shfl_up_sync(0xffffffffu, v.b, off)};
}
__device__ __forceinline__ Affine3 shfl_up(const Affine3 &v, int off)
{
    return Affine3{__shfl_up_sync(0xffffffffu, v.a, off), __shfl_up_sync(0xffffffffu, v.b, off), __shfl_up_sync(0xffffffffu, v.c, off)};
}
__device__ __forceinline__ DcAff shfl_up(const DcAff &v, int off)
{
    return DcAff{__shfl_up_sync(0xffffffffu, v.a, off), __shfl_up_sync(0xffffffffu, v.br, off), __shfl_up_sync(0xffffffffu, v.bi, off)};
}

// the map applied to a seed: an AGC gain, or the DC blocker's complex accumulator; widen = the carried float value as a seed
__device__ __forceinline__ double apply(const Affine &m, double g) { return fma(m.a, g, m.b); }
__device__ __forceinline__ double apply(const Affine3 &m, double g) { return fmin(fma(m.a, g, m.b), m.c); }
__device__ __forceinline__ double2 apply(const DcAff &m, double2 g) { return make_double2(fma(m.a, g.x, m.br), fma(m.a, g.y, m.bi)); }
__device__ __forceinline__ double widen(float g) { return (double)g; }
__device__ __forceinline__ double2 widen(float2 g) { return make_double2((double)g.x, (double)g.y); }

// inclusive scan over the lanes: lane i gets v_i o ... o v_0
template <class M> __device__ __forceinline__ M warp_scan(M v, int lane)
{
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const M p = shfl_up(v, off);
        if (lane >= off)
            v = compose(p, v);
    }
    return v;
}

// the composition of the FIR_THREADS threads' maps m (thread order) -> *out, written by thread 0
template <class M> __device__ __forceinline__ void tile_reduce(M m, M *out)
{
    __shared__ M wsum[FIR_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    m = warp_scan(m, lane);
    if (lane == 31)
        wsum[warp] = m;
    __syncthreads();
    if (t == 0) {
        M tot = wsum[0];
        for (int w = 1; w < FIR_THREADS / 32; w++)
            tot = compose(tot, wsum[w]);
        *out = tot;
    }
}

// seeds[k] = the value before tile k and seeds[ntiles] = after the batch, scanned from the carried value *in. Returns at once unless
// (*gate & mask) != 0 (gate = nullptr: always runs); count (may be nullptr) counts the runs.
template <class M, class S, class In>
__global__ void __launch_bounds__(1024) k_tile_scan(const M *__restrict__ tile_map, int ntiles, const In *__restrict__ in, const int *__restrict__ gate,
                                                   int mask, S *__restrict__ seeds, int *__restrict__ count)
{
    if (gate && (*gate & mask) == 0)
        return;
    if (count && threadIdx.x == 0)
        *count += 1;
    __shared__ M wsum[32];
    __shared__ S run;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0)
        run = widen(*in);
    __syncthreads();
    for (int base = 0; base < ntiles; base += 1024) {
        const int k = base + t;
        M m = ident<M>();
        if (k < ntiles)
            m = tile_map[k];
        const M inc = warp_scan(m, lane);
        if (lane == 31)
            wsum[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            const M w = warp_scan(wsum[lane], lane);
            wsum[lane] = w;
        }
        __syncthreads();
        M pre = ident<M>(); // composition of everything before this thread's tile in this round
        if (warp > 0)
            pre = wsum[warp - 1];
        const M e = shfl_up(inc, 1);
        const M excl = lane > 0 ? compose(pre, e) : pre;
        const S g0 = run;
        if (k < ntiles)
            seeds[k] = apply(excl, g0);
        __syncthreads();
        if (t == 1023)
            run = apply(compose(pre, inc), g0);
        __syncthreads();
    }
    if (t == 0)
        seeds[ntiles] = run;
}

// ---------------------------------------------------------------- K0': front-end DC blocker ("dc_block")
// CorrectIQBlock<complex_t>::work (utils/correct_iq.cpp:18-35): acc = acc*beta + x*alpha; y = x - acc, alpha = 1e-4, beta = 1 - alpha.
// A constant-coefficient linear recurrence: tiles of 2048 samples, each thread runs the reference's float recurrence over its 8
// samples from 0, the (beta^8, partial) maps are composed in fp64 (k_dc_tile -> k_tile_scan over tiles -> k_dc_apply), and every thread
// replays its 8 samples from its scanned accumulator. Output cf32 (what the reference hands to the resampler / AGC).
template <int FMT>
__device__ __forceinline__ DcAff dc_local(const void *__restrict__ raw, long s0, long N, int iq_swap, float alpha, float beta, float2 (&x)[8])
{
    load8<FMT>(raw, s0, N, x);
    float2 acc = make_float2(0.f, 0.f);
    double a = 1.0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (iq_swap)
            x[i] = make_float2(x[i].y, x[i].x);
        if (s0 + i < N) {
            acc.x = __fadd_rn(__fmul_rn(acc.x, beta), __fmul_rn(x[i].x, alpha));
            acc.y = __fadd_rn(__fmul_rn(acc.y, beta), __fmul_rn(x[i].y, alpha));
            a *= (double)beta;
        }
    }
    return DcAff{a, (double)acc.x, (double)acc.y};
}
template <int FMT>
__global__ void __launch_bounds__(FIR_THREADS) k_dc_tile(const void *__restrict__ raw, long N, int iq_swap, float alpha, float beta, DcAff *__restrict__ tile_map)
{
    float2 x[8];
    tile_reduce(dc_local<FMT>(raw, (long)blockIdx.x * FIR_TILE + 8 * threadIdx.x, N, iq_swap, alpha, beta, x), &tile_map[blockIdx.x]);
}
template <int FMT>
__global__ void __launch_bounds__(FIR_THREADS) k_dc_apply(const void *__restrict__ raw, long N, int iq_swap, float alpha, float beta,
                                                          const double2 *__restrict__ seeds, float2 *__restrict__ out, float2 *__restrict__ acc_out)
{
    __shared__ DcAff wsum[FIR_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const long s0 = (long)blockIdx.x * FIR_TILE + 8 * t;
    float2 x[8];
    const DcAff m = dc_local<FMT>(raw, s0, N, iq_swap, alpha, beta, x);
    const DcAff inc = warp_scan(m, lane);
    if (lane == 31)
        wsum[warp] = inc;
    __syncthreads();
    DcAff pre = ident<DcAff>();
    for (int w = 0; w < warp; w++)
        pre = compose(pre, wsum[w]);
    const DcAff e = shfl_up(inc, 1);
    const DcAff excl = lane > 0 ? compose(pre, e) : pre;
    const double2 g = apply(excl, seeds[blockIdx.x]);
    float2 acc = make_float2((float)g.x, (float)g.y);
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (s0 + i < N) {
            acc.x = __fadd_rn(__fmul_rn(acc.x, beta), __fmul_rn(x[i].x, alpha));
            acc.y = __fadd_rn(__fmul_rn(acc.y, beta), __fmul_rn(x[i].y, alpha));
            out[s0 + i] = make_float2(x[i].x - acc.x, x[i].y - acc.y);
            if (s0 + i == N - 1)
                *acc_out = acc;
        }
}

// sqrt(s2) as one MUFU.SQRT (sqrt.approx: ~1 ulp; sqrt(0) = 0, no guard needed)
__device__ __forceinline__ float fast_mag(float s2)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s2));
    return r;
}

// One AGC step (agc.cpp:30-33) for input x is the affine map g' = g*(1 - e) + rate with e = rate*|x| (exact while the clamp is
// not hit). Inside a tile a composed map is carried as the float pair (E, B): g -> g*(1 - E) + B. Keeping E = 1 - a rather than
// a keeps the *relative* precision of the decay for weak signals (e ~ 1e-5), so float is enough here: the composition depth on
// any path is ~20 and a seed error decays by (1 - e) per sample anyway. Across tiles the maps are composed in fp64.
// Strong input (cf32 above full scale, rate|x| ~ 0.1 per sample) is the opposite case: a composed decay 1 - E falls below the float
// resolution of E, and a gain far above the new level (the chunks right after a step up) would be weighted by a decay that is off by
// up to 6e-8 absolute, 1e-5 of the gain that follows. The decay is therefore also carried as the product a of the steps' (1 - e), which
// keeps its relative precision, and replaces 1 - E below AGC_A_SMALL. Inputs within full scale (rate|x| <= 0.0142, so a chunk decays by
// no less than 0.026 and a lane's prefix by more) never reach it, and their arithmetic is the (E, B) one alone.
struct EB { float E, B; };
constexpr float AGC_A_SMALL = 1.0f / 64;
constexpr float AGC_E_LANE = 0.12f; // a lane's E at most this: its decay >= 0.88, and 0.88^32 = 0.0167 > AGC_A_SMALL
__device__ __forceinline__ EB eb_compose(const EB first, const EB second)
{
    EB r;
    r.B = fmaf(-second.E, first.B, first.B + second.B);
    r.E = fmaf(-first.E, second.E, first.E + second.E);
    return r;
}
// second with first put in front when take is set (branch-free scan step)
__device__ __forceinline__ EB eb_compose_if(bool take, const EB first, const EB second)
{
    const EB c = eb_compose(first, second);
    EB r;
    r.E = take ? c.E : second.E;
    r.B = take ? c.B : second.B;
    return r;
}

struct EBC { float E, B, C; };            // g -> min(g*(1 - E) + B, C), the float form used inside a tile
__device__ __forceinline__ EBC ebc_compose(const EBC first, const EBC second)
{
    EBC r;
    r.B = fmaf(-second.E, first.B, first.B + second.B);
    r.E = fmaf(-first.E, second.E, first.E + second.E);
    r.C = fminf(fmaf(-second.E, first.C, first.C) + second.B, second.C);
    return r;
}

// smem index (float2 units): 8 samples + 16 B pad per group -> 16-byte aligned, conflict-free 128-bit accesses at a thread
// stride of 8 samples
__device__ __forceinline__ int xidx(int i) { return i + 2 * (i >> 3); }

// composed AGC map of 8 samples (all valid)
__device__ __forceinline__ EB agc_map8(const float2 (&x)[8], float rate, float (&e)[8])
{
    EB m{0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; i++) {
        e[i] = rate * fast_mag(fmaf(x[i].x, x[i].x, x[i].y * x[i].y));
        m.B = fmaf(-e[i], m.B, m.B + rate);
        m.E = fmaf(-m.E, e[i], m.E + e[i]);
    }
    return m;
}

// the decay of a lane's steps as a product (AGC_A_SMALL); e[q] = 0 for samples beyond the stream
__device__ __forceinline__ float decay8(const float (&e)[8])
{
    float a = 1.f;
#pragma unroll
    for (int q = 0; q < 8; q++)
        a = fmaf(-e[q], a, a);
    return a;
}

// Control block of the AGC seeding. need[epoch & 1] is raised by the fast pass when some range cannot prove its seed; the exact
// pass (k_agc_compose, k_agc_scan, k_agc_fir_w with seeded = 1) then runs, otherwise those launches return at once.
struct AgcCtl
{
    const double *seeds; // [ntiles + 1] gain before every tile (exact pass only)
    int *need;           // [2], indexed by launch parity; the fast pass clears the other one for the next batch
    unsigned epoch;
    int seeded;
    int warm_max;        // fast pass: how many tiles a range may walk back before giving up
    float max_gain;      // AGCBlock's max_gain: 65536 for BaseDemodModule's AGC (module_demod_base.cpp:207), 1000 for pm_demod's second one
};

// ---------------------------------------------------------------- K1: convert + AGC + 31-tap FIR, one WARP per range of tiles
// The AGC gain is a serial recurrence over the whole stream (agc.cpp:25-39). One step for input x is the affine map
// g' = g*(1 - e) + rate with e = rate*|x| (exact while the clamp is not hit), so maps compose and the recurrence becomes a scan.
// The stream is cut into ranges of R consecutive 2048-sample tiles; warp wg of the grid owns tiles [wg*R, (wg+1)*R) and walks them in
// chunks of 256 samples (8 per lane). A chunk needs one 5-step shuffle scan of the lanes' composed (E, B) maps, every lane then replays
// the reference's float recurrence over its 8 samples from its scanned seed, the gain chains from chunk to chunk in the warp's
// registers (fp64), and the AGC'd samples go to a WARP-PRIVATE shared-memory strip (32-sample history + 256 samples, the padded
// layout of xidx) from which the lanes run the 31-tap FFMA FIR. The warps of a CTA are independent: the only synchronisation is
// __syncwarp, so warps drift apart and the conversion / scan phases of some fill the issue slots the FIR phases of others leave.
// A chunk's composed decay stays above ~0.03 even for a full-scale input (E <= 0.97), so the float E keeps the relative precision
// of 1 - E that a 2048-sample tile loses when the gain falls from a large value (signal onset after silence).
// What a range needs from the past is its start gain. Because the loop is a contraction that gain is a function of the preceding
// samples only up to a weight A = prod(1 - rate|x|) on whatever came before: the warp walks backwards chunk by chunk composing the
// maps until A * max_gain is below float resolution of the seed (normally ~36 chunks, each a cheap map-only pass), which PROVES the
// seed to ~1e-9 without knowing anything older; if warm_max tiles do not suffice (very weak signal) it raises `need` and the exact
// pass (k_agc_compose -> k_agc_scan -> this kernel with seeded = 1) redoes the stage from scanned per-tile seeds. The chunk in front
// of the range is run without output to provide the 30-sample FIR history.
// gain_out: gain after the last sample; flags bit0 = the gain exceeded max_gain somewhere (silent input): the CLAMP instantiation
// then redoes the stage with the clamped step maps g -> min(g(1-e) + rate, 65536) composed as (E, B, C) triples and the clamp applied
// after every replayed step, seeded from the clamp-aware per-tile scan. Exact in the same sense as the unclamped passes.
constexpr int FW_CH = 256;                          // samples per chunk
constexpr int FW_WARPS = 4;                         // warps (= ranges) per CTA
constexpr int FW_BUF_F2 = ((32 + FW_CH) / 8) * 10;  // float2 slots of one warp's strip (xidx padding)

template <int FMT> struct FwState
{
    const void *__restrict__ raw;
    long N;
    float rate, maxg;  // AGC rate, max_gain
    double G;          // gain before the next chunk
    float2 *xs;        // the warp's strip
    const float2 *xrd; // this lane's FIR window: xidx(8 * lane + c) = 10 * lane + xidx(c)
    int lane, c_last;
};

// the 31-tap FIR of one chunk out of the warp's strip: lane -> outputs 8*lane .. 8*lane+7; y[n] = sum_j x[n-30+j] * h[30-j], oldest first
// (fir.cpp:74-83). One scalar FFMA per (re or im) x real tap MAC, the tap a broadcast register operand; the output pairs are packed into
// 64-bit words at the end so that each pair leaves as one 16-byte store.
__device__ __forceinline__ void fw_fir8(const float2 *xrd, const FirTaps &taps, ulonglong2 (&acc)[4])
{
    float2 a[8];
#pragma unroll
    for (int o = 0; o < 8; o++)
        a[o] = make_float2(0.f, 0.f);
#pragma unroll
    for (int pI = 0; pI < 19; pI++) {
        const float4 vv = *reinterpret_cast<const float4 *>(xrd + xidx(2 + 2 * pI));
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const float vr = h ? vv.z : vv.x, vi = h ? vv.w : vv.y;
            const int mI = 2 * pI + h;
#pragma unroll
            for (int o = 0; o < 8; o++) {
                const int j = mI - o; // tap position (0 = oldest)
                if (j >= 0 && j < FIR_NT) {
                    const float t = taps.h[FIR_NT - 1 - j];
                    a[o].x = fmaf(vr, t, a[o].x);
                    a[o].y = fmaf(vi, t, a[o].y);
                }
            }
        }
    }
#pragma unroll
    for (int o = 0; o < 4; o++)
        acc[o] = make_ulonglong2((unsigned long long)__float_as_uint(a[2 * o].y) << 32 | __float_as_uint(a[2 * o].x),
                                 (unsigned long long)__float_as_uint(a[2 * o + 1].y) << 32 | __float_as_uint(a[2 * o + 1].x));
}

// One chunk of k_agc_fir_w. FAST: every sample of the chunk exists, none belongs to the stream tail, output wanted, no dump, no clamp:
// no per-sample conditions, and the conversion's power-of-two factor S rides in the gain (raw_convert_scaled).
template <int FMT, bool DUMP, bool CLAMP, bool FAST>
__device__ __forceinline__ void fw_chunk(FwState<FMT> &st, RawRegs<FMT> &rr, int c, bool out, const FirTaps &taps, float2 *__restrict__ tail_out,
                                         float2 *__restrict__ fir_out, float2 *__restrict__ agc_dump, float *__restrict__ gain_out,
                                         int *__restrict__ flags)
{
    const int lane = st.lane;
    const long N = st.N;
    const float rate = st.rate;
    const long s0 = (long)c * FW_CH + 8 * lane;
    constexpr float S = FAST ? RawScale<FMT>::v : 1.0f;
    float2 x[8];
    if (FAST || s0 + 8 <= N) {
        if (FMT == 0) // cf32: 16 registers of raw data are too many to hold across a chunk
            raw_fetch<FMT>(st.raw, s0, rr);
        if (FAST)
            raw_convert_scaled<FMT>(rr, x);
        else
            raw_convert<FMT>(rr, x);
    } else
        load8_ragged<FMT>(st.raw, s0, N, x);
    if (FMT != 0 && c + 1 < st.c_last && s0 + FW_CH + 8 <= N) // the next chunk's loads fly under this chunk's arithmetic
        raw_fetch<FMT>(st.raw, s0 + FW_CH, rr);
    EB inc{0.f, 0.f};
    float incC = (float)AGC_NO_CLAMP;
    float e[8]; // rate * |sample|: the step map of sample q is g -> g * (1 - e[q]) + rate
    if (FAST) {
        const float rateS = rate * S;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            e[q] = rateS * fast_mag(fmaf(x[q].x, x[q].x, x[q].y * x[q].y));
            if (q == 0) { // the first step composed onto the identity, written out (the compiler keeps 0 + x and -0 * x otherwise)
                inc.B = rate;
                inc.E = e[0];
            } else {
                inc.B = fmaf(-e[q], inc.B, inc.B + rate);
                inc.E = fmaf(-inc.E, e[q], inc.E + e[q]);
            }
        }
    } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
            e[q] = 0.f;
            if (s0 + q < N) {
                e[q] = rate * fast_mag(fmaf(x[q].x, x[q].x, x[q].y * x[q].y));
                inc.B = fmaf(-e[q], inc.B, inc.B + rate);
                inc.E = fmaf(-inc.E, e[q], inc.E + e[q]);
                if (CLAMP)
                    incC = fminf(fmaf(-e[q], incC, incC) + rate, st.maxg);
            }
        }
    }
    const bool strong = inc.E > AGC_E_LANE; // (the lane's own map, before the scan)
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        EB p;
        p.E = __shfl_up_sync(0xffffffffu, inc.E, off);
        p.B = __shfl_up_sync(0xffffffffu, inc.B, off);
        if (CLAMP) {
            const float pC = __shfl_up_sync(0xffffffffu, incC, off);
            if (lane >= off)
                incC = fminf(fmaf(-inc.E, pC, pC) + inc.B, incC); // (p then inc), with inc's E, B before they are updated below
        }
        inc = eb_compose_if(lane >= off, p, inc);
    }
    const float totE = __shfl_sync(0xffffffffu, inc.E, 31), totB = __shfl_sync(0xffffffffu, inc.B, 31);
    EB excl;
    excl.E = __shfl_up_sync(0xffffffffu, inc.E, 1);
    excl.B = __shfl_up_sync(0xffffffffu, inc.B, 1);
    excl.E = lane > 0 ? excl.E : 0.f; // identity map in lane 0
    excl.B = lane > 0 ? excl.B : 0.f;
    // the decays as products (AGC_A_SMALL), scanned only when some lane's own E exceeds AGC_E_LANE: otherwise every prefix of the 32
    // lanes decays by more than AGC_A_SMALL and the (E, B) form is the one used anyway
    float exclA = 1.f, totA = 1.f;
    if (__any_sync(0xffffffffu, strong)) {
        float incA = decay8(e);
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const float pA = __shfl_up_sync(0xffffffffu, incA, off);
            incA = lane >= off ? pA * incA : incA;
        }
        totA = __shfl_sync(0xffffffffu, incA, 31);
        exclA = __shfl_up_sync(0xffffffffu, incA, 1);
        exclA = lane > 0 ? exclA : 1.f;
    }
    const float Gf = (float)st.G;
    float g = exclA < AGC_A_SMALL ? fmaf(exclA, Gf, excl.B) : fmaf(-excl.E, Gf, Gf) + excl.B;
    st.G = fma(totA < AGC_A_SMALL ? (double)totA : 1.0 - (double)totE, st.G, (double)totB);
    if (CLAMP) {
        const float totC = __shfl_sync(0xffffffffu, incC, 31);
        float exclC = __shfl_up_sync(0xffffffffu, incC, 1);
        exclC = lane > 0 ? exclC : (float)AGC_NO_CLAMP;
        g = fminf(g, exclC);
        st.G = fmin(st.G, (double)totC);
    }
    // per-sample gains from the scanned seed with the same step maps: g' = g*(1 - e) + rate is the reference's
    // gain += rate*(1 - |x*gain|) (agc.cpp:30-33) up to the rounding of one step (~1e-9 relative), two orders below the reference's
    // own accumulated float rounding noise in the gain that no parallel evaluation reproduces anyway (DESIGN.md 4.1).
    float gmax = g;
    if (FAST) {
        // the recurrence runs on gs = g * S (S a power of two: every product and sum rounds exactly as the unscaled one does), so that
        // (sample / S) * gs is the reference's sample * g without a multiply per sample for the scale
        const float rateS = rate * S;
        float gs = g * S, gprev = gs;
        gmax = gs;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            x[q] = make_float2(x[q].x * gs, x[q].y * gs);
            gs = fmaf(-e[q], gs, gs + rateS);
            if (q & 1)
                gmax = fmaxf(gmax, fmaxf(gprev, gs)); // (one three-input maximum per two samples)
            gprev = gs;
        }
    } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const long s = s0 + q;
            const float2 o = make_float2(x[q].x * g, x[q].y * g);
            if (s < N) {
                g = fmaf(-e[q], g, g + rate);
                gmax = fmaxf(gmax, g);
                g = fminf(g, st.maxg);
                if (out) {
                    if (DUMP)
                        agc_dump[s] = o;
                    if (s >= N - 32)
                        tail_out[s - (N - 32)] = o;
                    if (s == N - 1)
                        *gain_out = g;
                }
            }
            x[q] = o;
        }
    }
    if (!CLAMP && gmax > st.maxg * S)
        atomicOr(flags, 1);
    {
        float4 *dst = reinterpret_cast<float4 *>(&st.xs[10 * lane + 40]);
#pragma unroll
        for (int q = 0; q < 4; q++)
            dst[q] = make_float4(x[2 * q].x, x[2 * q].y, x[2 * q + 1].x, x[2 * q + 1].y);
    }
    __syncwarp();
    if (FAST || out) {
        ulonglong2 acc[4]; // (pairs of outputs: each pair leaves as one 16-byte store)
        fw_fir8(st.xrd, taps, acc);
        if (FAST || s0 + 8 <= N) {
            ulonglong2 *p = reinterpret_cast<ulonglong2 *>(fir_out + s0);
#pragma unroll
            for (int o = 0; o < 4; o++)
                p[o] = acc[o];
        } else {
#pragma unroll
            for (int o = 0; o < 8; o++)
                if (s0 + o < N)
                    *reinterpret_cast<unsigned long long *>(fir_out + s0 + o) = (o & 1) ? acc[o >> 1].y : acc[o >> 1].x;
        }
    }
    __syncwarp(); // every lane has read its window: the chunk's last 32 samples become the next chunk's history
    if (lane >= 28) {
        const float4 *src = reinterpret_cast<const float4 *>(&st.xs[10 * lane + 40]);
        float4 *dst = reinterpret_cast<float4 *>(&st.xs[10 * (lane - 28)]);
#pragma unroll
        for (int q = 0; q < 4; q++)
            dst[q] = src[q];
    }
}

template <int FMT, bool DUMP, bool CLAMP>
__global__ void __launch_bounds__(32 * FW_WARPS, 8) k_agc_fir_w(const void *__restrict__ raw, long N, float rate, const float *__restrict__ gain_in, int R,
                                                                  const AgcCtl ctl, const FirTaps taps, const float2 *__restrict__ tail_in,
                                                                  float2 *__restrict__ tail_out, float2 *__restrict__ fir_out,
                                                                  float2 *__restrict__ agc_dump, float *__restrict__ gain_out, int *__restrict__ flags)
{
    __shared__ __align__(16) float2 xs_all[FW_WARPS][FW_BUF_F2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2 *xs = xs_all[warp];
    int *need = ctl.need + (ctl.epoch & 1);
    if (CLAMP) {
        if ((*flags & 1) == 0)
            return;
    } else if (ctl.seeded) {
        if (*need == 0)
            return;
    } else if (blockIdx.x == 0 && threadIdx.x == 0)
        ctl.need[(ctl.epoch & 1) ^ 1] = 0;
    const int ntiles = (int)((N + FIR_TILE - 1) / FIR_TILE);
    const long first_t = ((long)blockIdx.x * FW_WARPS + warp) * R;
    if (first_t >= ntiles)
        return;
    const int last_t = (int)min(first_t + (long)R, (long)ntiles);
    const int nch = (int)((N + FW_CH - 1) / FW_CH);
    const int c_first = (int)first_t * (FIR_TILE / FW_CH), c_last = min(last_t * (FIR_TILE / FW_CH), nch);
    int c0 = c_first;
    double G; // gain before the next chunk to run
    if (first_t == 0) {
        G = (double)*gain_in;
        if (lane < 4) { // FIR history: the previous batch's last 32 AGC outputs
            float4 *dst = reinterpret_cast<float4 *>(&xs[10 * lane]);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float2 u = tail_in[8 * lane + 2 * i], v = tail_in[8 * lane + 2 * i + 1];
                dst[i] = make_float4(u.x, u.y, v.x, v.y);
            }
        }
    } else if (ctl.seeded || CLAMP) {
        c0 = ((int)first_t - 1) * (FIR_TILE / FW_CH); // the whole tile in front, from its scanned seed, without output
        G = ctl.seeds[first_t - 1];
    } else {
        c0 = c_first - 1;
        double A = 1.0, Bc = 0.0; // composition of the chunks walked so far: g(c0 start) = A * g(older) + Bc
        bool ok = false;
        for (int j = c0 - 1, w = 0;; j--, w++) {
            if (j < 0) { // reached the batch start: the carried gain is exact
                Bc = fma(A, (double)*gain_in, Bc);
                ok = true;
                break;
            }
            if (w >= ctl.warm_max * (FIR_TILE / FW_CH))
                break;
            float2 x[8];
            load8<FMT>(raw, (long)j * FW_CH + 8 * lane, N, x);
            float e[8];
            EB m = agc_map8(x, rate, e);
            const bool strong = __any_sync(0xffffffffu, m.E > AGC_E_LANE);
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) { // lane l <- groups [l, l + 2*off)
                EB o;
                o.E = __shfl_down_sync(0xffffffffu, m.E, off);
                o.B = __shfl_down_sync(0xffffffffu, m.B, off);
                if (lane + off < 32)
                    m = eb_compose(m, o);
            }
            const float tE = __shfl_sync(0xffffffffu, m.E, 0), tB = __shfl_sync(0xffffffffu, m.B, 0);
            double decay = 1.0 - (double)tE;
            if (strong) { // the chunk's decay as a product (AGC_A_SMALL)
                float a = decay8(e);
#pragma unroll
                for (int off = 1; off < 32; off <<= 1)
                    a *= __shfl_xor_sync(0xffffffffu, a, off);
                if (a < AGC_A_SMALL)
                    decay = (double)a;
            }
            Bc = fma(A, (double)tB, Bc);
            A *= decay;
            // anything older enters as A * gain with gain <= max_gain (2^16 for the demodulator's AGC): done once that is below float resolution of the seed
            if (A * (double)ctl.max_gain <= Bc * 0x1p-30) {
                ok = true;
                break;
            }
        }
        if (!ok) {
            if (lane == 0)
                atomicOr(need, 1);
            return;
        }
        G = Bc;
    }

    RawRegs<FMT> rr;
    if (FMT != 0 && (long)c0 * FW_CH + 8 * lane + 8 <= N)
        raw_fetch<FMT>(raw, (long)c0 * FW_CH + 8 * lane, rr);
    FwState<FMT> st{raw, N, rate, ctl.max_gain, G, xs, &xs[10 * lane], lane, c_last};
    // [c0, c_first): history only; [c_first, c_fast): every sample exists, none is in the stream tail -> the branch-free body;
    // the rest (the batch's last chunks; all of them in the dump / clamp instantiations): the general body
    int c = c0;
    for (; c < c_first; c++)
        fw_chunk<FMT, DUMP, CLAMP, false>(st, rr, c, false, taps, tail_out, fir_out, agc_dump, gain_out, flags);
    if (!DUMP && !CLAMP) {
        const int c_fast = (int)min((long)c_last, max(0L, (N - 32) / FW_CH)); // (c + 1) * FW_CH + 32 <= N
#pragma unroll 1
        for (; c < c_fast; c++)
            fw_chunk<FMT, false, false, true>(st, rr, c, true, taps, tail_out, fir_out, agc_dump, gain_out, flags);
    }
    for (; c < c_last; c++)
        fw_chunk<FMT, DUMP, CLAMP, false>(st, rr, c, true, taps, tail_out, fir_out, agc_dump, gain_out, flags);
}

// ---------------------------------------------------------------- exact and clamp passes: per-tile maps -> k_tile_scan -> seeds
// Per-tile composition of the AGC steps g -> (1 - rate|x|) g + rate: as Affine for the exact pass (weak signals), as Affine3 with the
// max_gain clamp for the clamp pass (the gain hit max_gain in this batch). Returns at once unless (*gate & mask) != 0: need[epoch & 1]
// for the exact pass, flags bit 0 for the clamp pass.
template <int FMT, class M>
__global__ void __launch_bounds__(FIR_THREADS) k_agc_compose(const void *__restrict__ raw, long N, float rate, double max_gain, const int *__restrict__ gate,
                                                             int mask, int ntiles, M *__restrict__ tile_map)
{
    if ((*gate & mask) == 0) // the usual case: a small grid that returns at once
        return;
    const int t = threadIdx.x;
    for (int k = blockIdx.x; k < ntiles; k += gridDim.x) {
        const long s0 = (long)k * FIR_TILE + 8 * t;
        M m = ident<M>();
        float2 x[8];
        load8<FMT>(raw, s0, N, x);
#pragma unroll
        for (int i = 0; i < 8; i++)
            if (s0 + i < N) {
                const float mag = fast_mag(fmaf(x[i].x, x[i].x, x[i].y * x[i].y));
                if constexpr (std::is_same<M, Affine3>::value)
                    m = compose(m, Affine3{1.0 - (double)rate * (double)mag, (double)rate, max_gain});
                else
                    m = compose(m, Affine{1.0 - (double)rate * (double)mag, (double)rate});
            }
        tile_reduce(m, &tile_map[k]);
        __syncthreads();
    }
}

// ---------------------------------------------------------------- test hook: the FIR alone (b200_demod_debug_run_stage)
// y[i] = sum_j x[i-30+j] * h[30-j] over a cf32 stream with zero history, oldest sample first (fir.cpp:74-83). STRICT evaluates it
// the way the generic VOLK dot product the oracle is built with does (separate multiply and add, left to right), so that fed the
// oracle's own AGC output the result must be BITWISE the oracle's FIR output; !STRICT uses one fma per tap in the same order, i.e.
// the arithmetic of k_agc_fir_w's FFMA loop.
template <bool STRICT> __global__ void __launch_bounds__(256) k_fir_only(const float2 *__restrict__ in, long N, const FirTaps taps, float2 *__restrict__ out)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N)
        return;
    float ar = 0.f, ai = 0.f;
#pragma unroll
    for (int j = 0; j < FIR_NT; j++) {
        const long s = i - (FIR_NT - 1) + j;
        const float2 x = s >= 0 ? in[s] : make_float2(0.f, 0.f);
        const float h = taps.h[FIR_NT - 1 - j];
        if (STRICT) {
            ar = __fadd_rn(ar, __fmul_rn(x.x, h));
            ai = __fadd_rn(ai, __fmul_rn(x.y, h));
        } else {
            ar = fmaf(x.x, h, ar);
            ai = fmaf(x.y, h, ai);
        }
    }
    out[i] = make_float2(ar, ai);
}

// ---------------------------------------------------------------- fsk_demod: quadrature demodulator, float DC blocker, float AGC, real RRC
// FSKDemodModule::init (module_fsk_demod.cpp:59-84) behind the complex AGC: QuadratureDemodBlock(agc, 1.0f) -> CorrectIQBlock<float> ->
// AGCBlock<float>(0.1, 0.5, 1.0, 65535) -> FIRBlock<float>(RRC) -> MMClockRecoveryBlock<float>. All stages work on 2048-sample tiles of
// 256 threads x 8 samples; the two recurrences are scanned like the complex DC blocker and AGC (k_tile_scan) and every thread then
// replays the reference's float recurrence over its 8 samples from its scanned seed.
constexpr float FSK_AGC_RATE = 0.1f, FSK_AGC_REF = 0.5f, FSK_AGC_MAX = 65535.0f;

// QuadratureDemodBlock::process (quadrature_demod.cpp:35-48): p = atan2f(im, re). p here is the correctly rounded float of the arctangent
// (evaluated in double, then rounded once; DESIGN §9), not CUDA's atan2f (up to 2 ulp).
__device__ __forceinline__ float quad_phase(float2 v) { return (float)atan2((double)v.y, (double)v.x); }
// d = p - phase; the wrap compares with the double M_PI and subtracts 2.0f * M_PI in double, rounded back to float; out = d * (1.0 / 1.0f)
__device__ __forceinline__ float quad_diff(float p, float prev)
{
    const double pi = 3.14159265358979323846;
    float d = __fsub_rn(p, prev);
    if ((double)d > pi)
        d = (float)((double)d - 2.0 * pi);
    else if ((double)d <= -pi)
        d = (float)((double)d + 2.0 * pi);
    return d;
}
// CorrectIQBlock<float> step: acc = acc * beta + x * alpha (correct_iq.cpp:29); the output is x - acc
__device__ __forceinline__ float dc_step(float acc, float x, float alpha, float beta) { return __fadd_rn(__fmul_rn(acc, beta), __fmul_rn(x, alpha)); }
// AGCBlock<float> step (agc.cpp:30-36): out = x * gain; gain += rate * (reference - |out|), clamped at max_gain
__device__ __forceinline__ float agc_step(float &g, float x)
{
    const float out = __fmul_rn(x, g);
    g = __fadd_rn(g, __fmul_rn(FSK_AGC_RATE, __fsub_rn(FSK_AGC_REF, fabsf(out))));
    if (g > FSK_AGC_MAX)
        g = FSK_AGC_MAX;
    return out;
}
// the same step as a map of the gain, for the scan: g -> min((1 - rate |x|) g + rate * reference, max_gain)
__device__ __forceinline__ Affine3 agc_map(float x)
{
    return Affine3{1.0 - (double)FSK_AGC_RATE * fabs((double)x), (double)FSK_AGC_RATE * (double)FSK_AGC_REF, (double)FSK_AGC_MAX};
}

// exclusive composition of the maps of the threads in front of this one in its tile (the block's threads in order)
template <class M> __device__ __forceinline__ M tile_exclusive(M m)
{
    __shared__ M wsum[FIR_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const M inc = warp_scan(m, lane);
    if (lane == 31)
        wsum[warp] = inc;
    __syncthreads();
    M pre = ident<M>();
    for (int w = 0; w < warp; w++)
        pre = compose(pre, wsum[w]);
    const M e = shfl_up(inc, 1);
    return lane > 0 ? compose(pre, e) : pre;
}

// the quadrature demodulator over the complex AGC output, and the DC blocker's per-tile maps (acc -> beta^8.. acc + local run from 0).
// phase_in: p of the sample in front of the batch (QuadratureDemodBlock::phase, 0 for a new stream); phase_out: p of the batch's last one.
__global__ void __launch_bounds__(FIR_THREADS) k_quad(const float2 *__restrict__ in, long N, const float *__restrict__ phase_in, float *__restrict__ phase_out,
                                                      float alpha, float beta, float *__restrict__ out, Affine *__restrict__ tile_map)
{
    const long s0 = (long)blockIdx.x * FIR_TILE + 8 * threadIdx.x;
    float prev = s0 == 0 ? *phase_in : (s0 - 1 < N ? quad_phase(in[s0 - 1]) : 0.f);
    float acc = 0.f;
    double a = 1.0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (s0 + i < N) {
            const float p = quad_phase(in[s0 + i]);
            const float d = quad_diff(p, prev);
            prev = p;
            out[s0 + i] = d;
            acc = dc_step(acc, d, alpha, beta);
            a *= (double)beta;
            if (s0 + i == N - 1)
                *phase_out = p;
        }
    tile_reduce(Affine{a, (double)acc}, &tile_map[blockIdx.x]);
}

// the DC blocker's output from the scanned seeds (acc before every tile), and the float AGC's per-tile maps over it (Affine3: clamp)
__global__ void __launch_bounds__(FIR_THREADS) k_fsk_dc(const float *__restrict__ in, long N, float alpha, float beta, const double *__restrict__ seeds,
                                                        float *__restrict__ out, float *__restrict__ acc_out, Affine3 *__restrict__ agc_tile_map)
{
    const long s0 = (long)blockIdx.x * FIR_TILE + 8 * threadIdx.x;
    float x[8];
    float acc = 0.f;
    double a = 1.0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        x[i] = s0 + i < N ? in[s0 + i] : 0.f;
        if (s0 + i < N) {
            acc = dc_step(acc, x[i], alpha, beta);
            a *= (double)beta;
        }
    }
    const Affine excl = tile_exclusive(Affine{a, (double)acc});
    acc = (float)apply(excl, seeds[blockIdx.x]);
    Affine3 m = ident<Affine3>();
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (s0 + i < N) {
            acc = dc_step(acc, x[i], alpha, beta);
            const float y = __fsub_rn(x[i], acc);
            out[s0 + i] = y;
            m = compose(m, agc_map(y));
            if (s0 + i == N - 1)
                *acc_out = acc;
        }
    __syncthreads(); // (tile_reduce's shared memory is its own; the barrier keeps the two reductions' phases apart)
    tile_reduce(m, &agc_tile_map[blockIdx.x]);
}

// the float AGC's output from the scanned seeds (gain before every tile)
__global__ void __launch_bounds__(FIR_THREADS) k_fsk_agc(const float *__restrict__ in, long N, const double *__restrict__ seeds, float *__restrict__ out,
                                                         float *__restrict__ gain_out)
{
    const long s0 = (long)blockIdx.x * FIR_TILE + 8 * threadIdx.x;
    float x[8];
    Affine3 m = ident<Affine3>();
#pragma unroll
    for (int i = 0; i < 8; i++) {
        x[i] = s0 + i < N ? in[s0 + i] : 0.f;
        if (s0 + i < N)
            m = compose(m, agc_map(x[i]));
    }
    const Affine3 excl = tile_exclusive(m);
    float g = (float)apply(excl, seeds[blockIdx.x]);
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (s0 + i < N) {
            out[s0 + i] = agc_step(g, x[i]);
            if (s0 + i == N - 1)
                *gain_out = g;
        }
}

// STRICT | SEQUENTIAL test hook: stage 0 the DC blocker, 1 the AGC, as ONE thread running the reference's recurrence from its initial state
__global__ void k_fsk_serial(int stage, const float *__restrict__ in, long N, float alpha, float beta, float *__restrict__ out)
{
    float acc = 0.f, g = 1.0f;
    for (long i = 0; i < N; i++) {
        if (stage == 0) {
            acc = dc_step(acc, in[i], alpha, beta);
            out[i] = __fsub_rn(in[i], acc);
        } else
            out[i] = agc_step(g, in[i]);
    }
}

// FIRBlock<float> (fir.cpp:57-67 with the generic VOLK dot product): y[i] = sum_j x[i-30+j] * h[30-j], oldest sample first, separate
// multiply and add, so it is bitwise the reference. in[-32 .. -1] holds the previous batch's last samples (zeros for a new stream).
// The output is the clock recovery's input (y, 0).
__global__ void __launch_bounds__(256) k_fir_real(const float *__restrict__ in, long N, const FirTaps taps, float2 *__restrict__ out)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N)
        return;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < FIR_NT; j++)
        acc = __fadd_rn(acc, __fmul_rn(in[i - (FIR_NT - 1) + j], taps.h[FIR_NT - 1 - j]));
    out[i] = make_float2(acc, 0.f);
}

// ---------------------------------------------------------------- cp.async helpers
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// ---------------------------------------------------------------- opt-in cycle counters of the loop kernels' main passes
// Built with -DB200_LOOP_CYCLES (tools/profile_loops.py --cycles), lane 0 of every warp of a main pass adds the clock64() cycles of
// each phase of its row loop to g_loop_cycles (b200_demod_debug_loop_cycles reads and clears them); mark(k) books the time since the
// previous mark to phase k. Without the flag every member is empty and the kernels are the production ones.
#endif // B200_DEFINE_KERNELS
enum { LC_COSTAS = 0, LC_MM = 5, LC_PHASES = 4, LC_SLOTS = 10 }; // per kernel: LC_PHASES phase totals, then the number of warps
#ifdef B200_DEFINE_KERNELS
#ifdef B200_LOOP_CYCLES
__device__ unsigned long long g_loop_cycles[LC_SLOTS];
struct LoopCycles
{
    long long c[LC_PHASES], t;
    static __device__ __forceinline__ long long now()
    {
        long long v;
        asm volatile("mov.u64 %0, %%clock64;" : "=l"(v));
        return v;
    }
    __device__ __forceinline__ LoopCycles() : c{0, 0, 0, 0}, t(now()) {}
    __device__ __forceinline__ void mark(int k)
    {
        const long long n = now();
        c[k] += n - t;
        t = n;
    }
    __device__ __forceinline__ void publish(int base, bool main_pass)
    {
        if (!main_pass || (threadIdx.x & 31))
            return;
        for (int k = 0; k < LC_PHASES; k++)
            atomicAdd(&g_loop_cycles[base + k], (unsigned long long)c[k]);
        atomicAdd(&g_loop_cycles[base + LC_PHASES], 1ull);
    }
};
#else
struct LoopCycles
{
    __device__ __forceinline__ void mark(int) {}
    __device__ __forceinline__ void publish(int, bool) {}
};
#endif

// ---------------------------------------------------------------- K2: Costas loop, one thread per segment
#endif // B200_DEFINE_KERNELS
struct CostasParams
{
    int order;          // 2, 4, 8
    float alpha, beta, fmin, fmax;
};
struct LoopRec { float ph_start, fr_start, ph_end, fr_end; };
// Repair checkpoints. The main pass of a loop kernel stores the loop state of every segment at its owned samples own0 + j * CKPT
// (j >= 1). A repair (the exact continuation of the predecessor) compares its own state with the stored one there: both loops are
// contracting, so the two runs approach each other, and once they agree within the junction tolerance everything the stored run
// produced from that sample on (outputs, end record) is as good a continuation as any accepted junction: the repair stops there
// instead of running the whole segment. A checkpoint that does not agree is overwritten, so the checkpoints always describe the
// outputs in memory; a repair that never agrees runs to the segment's end.
constexpr int CKPT = 512; // samples; a power of two and a multiple of the 16-sample row
struct LoopCkpt { float phase, freq; };
struct MMCkpt { int u, count; float mu, omega; }; // in front of the first symbol at or behind the checkpoint; count = slots filled so far
inline __host__ __device__ int ckpt_per_seg(int L) { return (L - 1) / CKPT; }
constexpr int MERGE_BUCKETS = 8; // histogram of repairs: [0] ran to the segment's end, [i] joined at checkpoint j, 2^(i-2) < j <= 2^(i-1)

#ifdef B200_DEFINE_KERNELS
__device__ __forceinline__ void count_repair(int *__restrict__ merge_hist, int joined_at)
{
    atomicAdd(&merge_hist[joined_at ? min(MERGE_BUCKETS - 1, 33 - __clz(joined_at - 1)) : 0], 1);
}

// Warp-cooperative staging shared by the two loop kernels. Every thread walks ITS OWN stretch of the stream, so a per-thread
// load touches 32 different cache lines per instruction (measured: the L1 wavefront rate, not the math, bounded the first version).
// Instead the warp moves whole 128-byte rows: in instruction i, lanes 8q..8q+7 copy the eight 16-byte chunks of the row of thread
// 4i+q -> 4 lines per instruction. In shared memory chunk p of thread T sits at 16-byte slot p*32 + (T ^ (p & 7)): the XOR makes both
// the copy-in (8 chunks of one thread) and the per-thread reads / transposed copy-out (one chunk of 8 consecutive threads) hit 8
// distinct bank groups, i.e. conflict free.
__device__ __forceinline__ int swz16(int p, int T) { return p * 32 + (T ^ (p & 7)); }

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem_src));
}

// copies row `row` (16 samples from sample index 16*row; may be negative for the history pad) of every lane's thread into that
// thread's ring of 32 chunk slots in dst (swizzled): chunk c of row r lands in slot (8r + 64 + c) mod 32. `base` must be 16-byte aligned
// at sample 0 and readable from the first requested sample on.
__device__ __forceinline__ void warp_load_rows(float4 *dst, const float2 *__restrict__ base, int row, bool row_valid, long limit, int lane)
{
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int T = 4 * i + (lane >> 3), c = lane & 7;
        const int r = __shfl_sync(0xffffffffu, row, T);
        const int ok = __shfl_sync(0xffffffffu, (int)row_valid, T);
        const long n0 = (long)r * 16 + 2 * c;
        const int pb = (r << 3) + 64; // the SOURCE thread's row decides the ring position
        if (ok && n0 < limit)
            cp_async16(&dst[swz16((pb + c) & 31, T)], base + n0);
    }
}

// The segment of this thread in the loop kernels: segment blockIdx.x * SEG_THREADS + threadIdx.x, or in repair mode
// (repair_list != nullptr) segment repair_list[i] for the i-th of the first min(*repair_count, 1024) threads. Repair mode re-runs a
// segment with NO warm-up, starting from the recorded end state of its predecessor, i.e. as the exact sequential continuation of that
// segment (used for junctions whose warm-up had not converged; the junction check runs again afterwards), up to the checkpoint at
// which it meets the segment's stored run (see CKPT). A thread without a segment gets active = false and s = 0.
__device__ __forceinline__ int loop_segment(int nseg, const int *__restrict__ repair_list, const int *__restrict__ repair_count, bool &active)
{
    int s = blockIdx.x * SEG_THREADS + threadIdx.x;
    active = true;
    if (repair_list) {
        if (s >= min(*repair_count, 1024))
            active = false;
        else
            s = repair_list[s];
    }
    if (s >= nseg)
        active = false;
    if (!active)
        s = 0;
    return s;
}

constexpr int COSTAS_SMEM_BYTES = (SEG_THREADS / 32) * (16 + 8) * 32 * 16; // per warp: 2 input rows + 1 output row of 8 chunks x 32 threads
// Gear shift: for the first G samples of a warm-up the loop runs first order (frequency held at the carried value) with 4x the phase
// gain: a warm-up that starts near an unstable lock point (a hang-up: the detector output is ~0 there) escapes four times faster, so
// the slow tail of the junction residuals disappears; the remaining W - G samples at the true gains bring the state from the wide
// loop's jitter down onto the sequential trajectory.

// the loop's state in registers: float phase / frequency exactly as the reference carries them, and (cs, sn) = cos / sin of the phase
struct CostasRegs { float phase, freq, cs, sn; };

// detector + branchless_clip(err, 1) (costas_loop.cpp:31-56)
template <int ORDER> __device__ __forceinline__ float costas_err(float vr, float vi)
{
    float err;
    if (ORDER == 4)
        err = (vr > 0.0f ? vi : -vi) - (vi > 0.0f ? vr : -vr); // sgn(0) = -1, and (+-1) * x is exact
    else if (ORDER == 2)
        err = vr * vi;
    else {
        const float K = 0.41421356237309515f; // sqrtf(2.0) - 1 rounded to float
        const float a = vr > 0.0f ? vi : -vi, b = vi > 0.0f ? vr : -vr;
        err = fabsf(vr) >= fabsf(vi) ? a - b * K : a * K - b;
    }
    return 0.5f * (fabsf(err + 1.0f) - fabsf(err - 1.0f));
}

// sin / cos of a loop phase (|x| <= 2 pi plus one step): three-term Cody-Waite reduction by pi/2 and the usual minimax polynomials on
// [-pi/4, pi/4]; max error 7e-8 over [-7, 7] (glibc's sinf / cosf, which the reference calls: 3e-8), no slow path to branch around.
__device__ __forceinline__ void sincos_loop_phase(float x, float &s, float &c)
{
    const float q = rintf(x * 0.636619772f);
    const int iq = (int)q;
    float t = fmaf(q, -1.57079601e+00f, x);
    t = fmaf(q, -3.13916473e-07f, t);
    t = fmaf(q, -5.39030253e-15f, t);
    const float t2 = t * t;
    const float sp = fmaf(fmaf(fmaf(-1.95152959e-4f, t2, 8.33216087e-3f), t2, -1.66666546e-1f), t2 * t, t);
    const float cp = fmaf(fmaf(fmaf(fmaf(2.44331571e-5f, t2, -1.38873163e-3f), t2, 4.16666457e-2f), t2, -0.5f), t2, 1.0f);
    const float ss = (iq & 1) ? cp : sp, cc = (iq & 1) ? sp : cp;
    s = (iq & 2) ? -ss : ss;
    c = ((iq + 1) & 2) ? -cc : cc;
}

// the rare part of a step, kept out of line (by value: a reference would pin the loop state to local memory): a wrap of the phase into
// (-2 pi, 2 pi) is due, or the step is too large for the small-angle rotation of (cs, sn). Returns (wrapped phase, flag, sin, cos): with
// the flag set, (cs, sn) were recomputed from the phase.
__device__ __noinline__ float4 costas_wrap(float phase, float d)
{
    bool refresh = fabsf(d) > 0.05f;
    // while (phase > 2*M_PI) in double == float compare against the largest float below 2*pi (0x40C90FDA)
    while (phase > 6.283185005f) {
        phase = (float)((double)phase - 6.283185307179586);
        refresh = true;
    }
    while (phase < -6.283185005f) {
        phase = (float)((double)phase + 6.283185307179586);
        refresh = true;
    }
    float sn = 0.f, cs = 0.f;
    if (refresh)
        sincos_loop_phase(phase, sn, cs);
    return make_float4(phase, refresh ? 1.0f : 0.0f, sn, cs);
}

// one sample of costas_loop.cpp:23-65. ANCHOR: (cs, sn) are recomputed from the float phase afterwards (every 4th sample: bounds the
// rotation's rounding drift to < 1e-6); otherwise they are rotated by the exact increment the float phase took.
template <int ORDER, bool ANCHOR>
__device__ __forceinline__ float2 costas_step(const float2 x, CostasRegs &r, float al, float be, float fmin, float fmax)
{
    // in * (cos(-phase) + j sin(-phase))  (costas_loop.cpp:26)
    const float vr = fmaf(x.y, r.sn, x.x * r.cs);
    const float vi = fmaf(-x.x, r.sn, x.y * r.cs);
    const float err = costas_err<ORDER>(vr, vi);
    r.freq = r.freq + be * err;
    const float prev = r.phase;
    r.phase = r.phase + (r.freq + al * err);
    const float d = r.phase - prev; // the increment the float phase really took (exact difference)
    r.freq = fminf(fmax, fmaxf(fmin, r.freq));
    const bool rare = fmaxf(fabsf(r.phase), fabsf(d) * 125.0f) > 6.25f; // a wrap is due or the step is too large to rotate by
    if (!ANCHOR) {
        // rotate (cs, sn) by the small increment d: Taylor sin/cos, |d| <= 0.05 -> truncation < 2e-10. Done before the (almost never
        // taken) branch below so that the branch's condition is long resolved when the rotation's last instruction issues.
        const float d2 = d * d;
        const float sd = d * fmaf(d2, fmaf(d2, 8.3333333e-3f, -0.16666667f), 1.0f);
        const float cd = fmaf(d2, fmaf(d2, 4.1666667e-2f, -0.5f), 1.0f);
        const float c2 = r.cs * cd - r.sn * sd;
        r.sn = r.sn * cd + r.cs * sd;
        r.cs = c2;
    }
    if (rare) {
        const float4 w = costas_wrap(r.phase, d);
        r.phase = w.x;
        if (w.y != 0.0f && !ANCHOR) {
            r.sn = w.z;
            r.cs = w.w;
        }
    }
    if (ANCHOR)
        sincos_loop_phase(r.phase, r.sn, r.cs);
    return make_float2(vr, vi);
}

// One thread per segment of a phase loop (k_costas, k_pll). in/out: N samples. Segment s owns samples [s*L, min((s+1)L, N)); its
// thread warms up from max(0, s*L - W), from phase 0 and the carried frequency. state_in = {phase, freq} carried from the previous batch
// (exact start of segment 0 and of any clipped warm-up). rec[s] = the loop state at the segment's first owned sample and at its end.
// Rows of 16 samples move between HBM and the warp's shared-memory strip cooperatively (see swz16): lanes 8q..8q+7 carry the eight
// 16-byte chunks of the row of thread 4i+q in their i-th copy; which row that is (its first row, row count, owned range) is
// exchanged ONCE before the loop, so a copy costs an add, a compare and the address, no shuffles.
// The loop policy supplies G, the length of the gear shift at the start of a warm-up (0: none); begin(phase, freq, gear_end): the start
// state, with samples below gear_end in the gear shift; row(mine, ring, slot, obuf, lane, b, own1): the loop over the staged row of
// samples b .. b+15 (those below own1; nothing unless mine) into obuf; and phase() / freq(), the state that goes into the record.
template <class Loop>
__device__ __forceinline__ void loop_segments(Loop &lp, unsigned char *smem, const float2 *__restrict__ in, long N, int L, int W, int nseg,
                                              const float *__restrict__ state_in, float2 *__restrict__ out, LoopRec *__restrict__ rec,
                                              const int *__restrict__ repair_list, const int *__restrict__ repair_count,
                                              LoopCkpt *__restrict__ ckpt, float tol_phase, float tol_freq, int *__restrict__ merge_hist)
{
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    float4 *ring = reinterpret_cast<float4 *>(smem) + warp * (24 * 32); // [16 chunk slots][32] in, then [8][32] out
    float4 *obuf = ring + 16 * 32;
    LoopCycles cyc;
    bool active;
    const int s = loop_segment(nseg, repair_list, repair_count, active);
    const long own0 = (long)s * L;
    const long own1 = active ? min(own0 + L, N) : own0;
    LoopCkpt *my_ck = ckpt + (long)s * ckpt_per_seg(L) - 1; // my_ck[j]: the state at sample own0 + j * CKPT, j >= 1
    const float lock_step = 6.283185307179586f / (float)lp.order();
    int joined_at = 0; // repair mode: the checkpoint at which this run met the stored one
    long start = own0 - W, gear_end = own0 - W + lp.G;
    float phase = 0.f, freq = state_in[1];
    if (repair_list && active) {
        // The predecessor's end state, moved by whole lock-point steps into the frame the stored run of this segment sits in (the loop
        // is the same loop in every frame, and k_costas_fix resolves the frame from ph_start): a stored tail it joins needs no rotation.
        start = own0;
        const int k = (int)rintf((rec[s].ph_start - rec[s - 1].ph_end) / lock_step) % lp.order();
        phase = rec[s - 1].ph_end + (float)k * lock_step;
        freq = rec[s - 1].fr_end;
        gear_end = 0;
    } else if (start <= 0) {
        start = 0;
        phase = state_in[0];
        gear_end = 0;
    }
    const int row0 = (int)(start >> 4), row1 = (int)((own1 + 15) >> 4); // rows of 16 samples, [row0, row1)
    int nrows = active ? row1 - row0 : 0;
    int maxrows = nrows;
#pragma unroll
    for (int off = 16; off; off >>= 1)
        maxrows = max(maxrows, __shfl_xor_sync(0xffffffffu, maxrows, off));
    lp.begin(phase, freq, gear_end);
    LoopRec lr;
    lr.ph_start = lp.phase();
    lr.fr_start = lp.freq();
    // what this lane needs to know about the threads whose rows it carries
    const int c = lane & 7;
    int src_row0[8], src_nrows[8], src_orow0[8], src_own1[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int T = 4 * i + (lane >> 3);
        src_row0[i] = __shfl_sync(0xffffffffu, row0, T);
        src_nrows[i] = __shfl_sync(0xffffffffu, nrows, T);
        src_orow0[i] = __shfl_sync(0xffffffffu, (int)(own0 >> 4), T); // first owned row
        src_own1[i] = __shfl_sync(0xffffffffu, (int)own1, T);
    }
    const float2 *in_c = in + 2 * c;
    auto load_row = [&](int it) { // row `it` of every thread -> input slot group it & 1
        const int pb = (it & 1) * 8;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int T = 4 * i + (lane >> 3);
            const int row = src_row0[i] + it;
            if (it < src_nrows[i] && (long)row * 16 + 2 * c < N)
                cp_async16(&ring[swz16(pb + c, T)], in_c + (long)row * 16);
        }
        cp_async_commit();
    };
    load_row(0);
    for (int it = 0; it < maxrows; it++) {
        if (repair_list && it > 0 && (it & (CKPT / 16 - 1)) == 0) {
            // every repair starts at its own0, so the whole warp is at a checkpoint: a thread whose state agrees with the stored
            // one (same frame, junction tolerances) owns no further rows, and the lanes that carry its rows learn that
            if (it < nrows) {
                LoopCkpt &ck = my_ck[it / (CKPT / 16)];
                const float d = lp.phase() - ck.phase, q = rintf(d / lock_step);
                if ((int)q % lp.order() == 0 && fabsf(d - q * lock_step) < tol_phase && fabsf(lp.freq() - ck.freq) < tol_freq) {
                    joined_at = it / (CKPT / 16);
                    nrows = it;
                } else
                    ck = LoopCkpt{lp.phase(), lp.freq()};
            }
            maxrows = nrows;
#pragma unroll
            for (int off = 16; off; off >>= 1)
                maxrows = max(maxrows, __shfl_xor_sync(0xffffffffu, maxrows, off));
#pragma unroll
            for (int i = 0; i < 8; i++)
                src_nrows[i] = __shfl_sync(0xffffffffu, nrows, 4 * i + (lane >> 3));
            if (it >= maxrows)
                break;
        }
        const int slot = (it & 1) * 8;
        load_row(it + 1);
        cp_async_wait<1>();
        __syncwarp();
        cyc.mark(0);
        const bool mine = it < nrows;
        const long b = (long)(row0 + it) << 4;
        // start / own0 are multiples of 16, so a row is entirely warm-up or entirely owned; only the batch's last row can be partial
        if (mine && b == own0) {
            lr.ph_start = lp.phase();
            lr.fr_start = lp.freq();
        }
        if (!repair_list && mine && b > own0 && ((int)(b - own0) & (CKPT - 1)) == 0)
            my_ck[(int)(b - own0) / CKPT] = LoopCkpt{lp.phase(), lp.freq()};
        lp.row(mine, ring, slot, obuf, lane, b, own1);
        __syncwarp();
        cyc.mark(1);
        // transposed copy-out: lanes 8q..8q+7 store the eight chunks of thread 4i+q's row (owned samples only)
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int T = 4 * i + (lane >> 3);
            const int row = src_row0[i] + it;
            const int n0 = row * 16 + 2 * c;
            if (it < src_nrows[i] && row >= src_orow0[i] && n0 < src_own1[i]) {
                const float4 v = obuf[swz16(c, T)];
                if (n0 + 1 < src_own1[i])
                    *reinterpret_cast<float4 *>(out + n0) = v;
                else
                    out[n0] = make_float2(v.x, v.y);
            }
        }
        __syncwarp();
        cyc.mark(2);
    }
    cp_async_wait<0>();
    cyc.mark(3);
    cyc.publish(LC_COSTAS, !repair_list);
    if (active) {
        if (joined_at) { // the stored run's end state stands, so the next junction is what it was
            lr.ph_end = rec[s].ph_end;
            lr.fr_end = rec[s].fr_end;
        } else {
            lr.ph_end = lp.phase();
            lr.fr_end = lp.freq();
        }
        rec[s] = lr;
        if (repair_list)
            count_repair(merge_hist, joined_at);
    }
}

// the Costas loop as the policy of loop_segments, with the gear shift over the first G samples of a warm-up
template <int ORDER> struct CostasLoop
{
    CostasParams P;
    int G;
    long gear_end;
    CostasRegs r;
    __device__ __forceinline__ float phase() const { return r.phase; }
    __device__ __forceinline__ float freq() const { return r.freq; }
    __device__ __forceinline__ int order() const { return ORDER; } // lock points per turn
    __device__ __forceinline__ void begin(float phase, float freq, long gear_until)
    {
        r.phase = phase;
        r.freq = freq;
        gear_end = gear_until;
        sincos_loop_phase(r.phase, r.sn, r.cs);
    }
    __device__ __forceinline__ void row(bool mine, const float4 *ring, int slot, float4 *obuf, int lane, long b, long own1)
    {
        const bool gear = b < gear_end;
        const float al = gear ? 4.0f * P.alpha : P.alpha, be = gear ? 0.0f : P.beta;
        if (mine && b + 16 <= own1) {
            // full row: 4 groups of 4 samples (the re-anchor pattern has period 4; a full 16-sample unroll stalls on instruction fetch)
#pragma unroll 1
            for (int p = 0; p < 8; p += 2) {
                const float4 v0 = ring[swz16(slot + p, lane)], v1 = ring[swz16(slot + p + 1, lane)];
                const float2 o0 = costas_step<ORDER, false>(make_float2(v0.x, v0.y), r, al, be, P.fmin, P.fmax);
                const float2 o1 = costas_step<ORDER, false>(make_float2(v0.z, v0.w), r, al, be, P.fmin, P.fmax);
                const float2 o2 = costas_step<ORDER, false>(make_float2(v1.x, v1.y), r, al, be, P.fmin, P.fmax);
                const float2 o3 = costas_step<ORDER, true>(make_float2(v1.z, v1.w), r, al, be, P.fmin, P.fmax);
                obuf[swz16(p, lane)] = make_float4(o0.x, o0.y, o1.x, o1.y);
                obuf[swz16(p + 1, lane)] = make_float4(o2.x, o2.y, o3.x, o3.y);
            }
        } else if (mine) {
            const int nvalid = (int)min(16L, own1 - b);
#pragma unroll 1
            for (int p = 0; p < 8; p++) {
                const float4 v = ring[swz16(slot + p, lane)];
                float2 o0 = make_float2(0.f, 0.f), o1 = o0;
                if (2 * p < nvalid)
                    o0 = costas_step<ORDER, false>(make_float2(v.x, v.y), r, al, be, P.fmin, P.fmax);
                if (2 * p + 1 < nvalid) {
                    if (p & 1)
                        o1 = costas_step<ORDER, true>(make_float2(v.z, v.w), r, al, be, P.fmin, P.fmax);
                    else
                        o1 = costas_step<ORDER, false>(make_float2(v.z, v.w), r, al, be, P.fmin, P.fmax);
                }
                obuf[swz16(p, lane)] = make_float4(o0.x, o0.y, o1.x, o1.y);
            }
        }
    }
};

template <int ORDER>
__global__ void __launch_bounds__(SEG_THREADS) k_costas(const float2 *__restrict__ in, long N, int L, int W, int G, int nseg, CostasParams P,
                                                         const float *__restrict__ state_in, float2 *__restrict__ out, LoopRec *__restrict__ rec,
                                                         const int *__restrict__ repair_list, const int *__restrict__ repair_count,
                                                         LoopCkpt *__restrict__ ckpt, float tol_phase, float tol_freq, int *__restrict__ merge_hist)
{
    extern __shared__ __align__(16) unsigned char cs_smem[];
    CostasLoop<ORDER> lp{P, G};
    loop_segments(lp, cs_smem, in, N, L, W, nseg, state_in, out, rec, repair_list, repair_count, ckpt, tol_phase, tol_freq, merge_hist);
}

// ---------------------------------------------------------------- K2b: resolve per-segment rotation (prefix sum mod order)
// quad[s] = number of 2pi/order steps segment s's phase runs AHEAD of the sequential loop. Also publishes the true
// carried loop state. unconv counts junctions whose residual exceeds tol.
// repair_list / repair_count: junctions (segment indices) that failed the check in THIS call (count is reset here).
__global__ void __launch_bounds__(1024) k_costas_fix(const LoopRec *__restrict__ rec, int nseg, int order, float tol_phase, float tol_freq,
                                                    uint8_t *__restrict__ quad, float *__restrict__ state_out, int *__restrict__ unconv,
                                                    int *__restrict__ repair_list, int *__restrict__ repair_count, int round, int *__restrict__ repairs_total)
{
    __shared__ int wsum[32];
    __shared__ int run;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (round > 0) { // repair round: nothing was re-run since the last pass unless junctions had been flagged
        const int pending = *repair_count;
        if (pending == 0)
            return;
        __syncthreads(); // everyone has read the count before thread 0 resets it below
        if (t == 0)
            *repairs_total += min(pending, 1024);
    }
    const float step = 6.283185307179586f / (float)order;
    if (t == 0) {
        run = 0;
        *repair_count = 0;
    }
    __syncthreads();
    for (int base = 0; base < nseg; base += 1024) {
        int s = base + t, k = 0;
        if (s > 0 && s < nseg) {
            float d = rec[s].ph_start - rec[s - 1].ph_end;
            float q = rintf(d / step);
            float resid = fabsf(d - q * step);
            k = ((int)q % order + order) % order;
            if (resid > tol_phase || fabsf(rec[s].fr_start - rec[s - 1].fr_end) > tol_freq) {
                const int slot = atomicAdd(repair_count, 1);
                if (slot < 1024)
                    repair_list[slot] = s;
            }
        }
        int v = k;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            int p = __shfl_up_sync(0xffffffffu, v, off);
            if (lane >= off)
                v += p;
        }
        if (lane == 31)
            wsum[warp] = v;
        __syncthreads();
        if (warp == 0) {
            int w = wsum[lane];
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                int p = __shfl_up_sync(0xffffffffu, w, off);
                if (lane >= off)
                    w += p;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        int tot = run + v + (warp > 0 ? wsum[warp - 1] : 0);
        if (s < nseg)
            quad[s] = (uint8_t)(tot % order);
        __syncthreads();
        if (t == 1023)
            run = tot % order;
        __syncthreads();
    }
    __syncthreads();
    if (t == 0) {
        *unconv = *repair_count; // junctions still failing after this pass
        int q = quad[nseg - 1];
        float ph = (float)((double)rec[nseg - 1].ph_end - (double)q * (6.283185307179586 / order));
        while (ph > 6.283185307179586)
            ph = (float)((double)ph - 6.283185307179586);
        while (ph < -6.283185307179586)
            ph = (float)((double)ph + 6.283185307179586);
        state_out[0] = ph;
        state_out[1] = rec[nseg - 1].fr_end;
    }
}

// ---------------------------------------------------------------- pm_demod: carrier PLL (one thread per segment) and the rotator
// PLLCarrierTrackingBlock (common/dsp/pll/pll_carrier_tracking.cpp:25-70): a second-order loop whose detector is the phase of the
// INPUT sample minus the loop phase (table-driven fast_atan2f), i.e. linear up to its wrap into (-pi, pi] and the frequency clamp: two
// copies started from different states approach each other geometrically whatever the noise, so the stream is cut into segments exactly
// like the Costas loop's (warm-up of W samples from phase 0 and the carried frequency, junction check and repair rounds by
// k_costas_fix with order 1). The arithmetic is the reference's, operation by operation (separate multiplies and adds, the
// polynomials of fast_cos / fast_sin in double, the wraps compared and stepped in double): a segment that continues its predecessor
// exactly (segment 0, repairs) is bit for bit the reference's output; the others inherit the junction tolerance.
#endif // B200_DEFINE_KERNELS
struct PllParams
{
    float alpha, beta, fmin, fmax;
};
#ifdef B200_DEFINE_KERNELS
// fast_trig.cpp:158-180: powers in float, Horner sums in double, one rounding on return
__device__ __forceinline__ float pll_fast_cos(float x)
{
    const float x2 = __fmul_rn(x, x), x4 = __fmul_rn(x2, x2), x8 = __fmul_rn(x4, x4);
    const double d2 = x2, d4 = x4, d8 = x8;
    const double a = __dadd_rn(__dmul_rn(-2.7236370439787708e-7, d2), 2.4799852696610628e-5);
    const double b = __dadd_rn(__dmul_rn(-1.3888885054799695e-3, d2), 4.1666666636943683e-2);
    const double c = __dadd_rn(__dmul_rn(-4.9999999999963024e-1, d2), 1.0);
    return (float)__dadd_rn(__dadd_rn(__dmul_rn(a, d8), __dmul_rn(b, d4)), c);
}
__device__ __forceinline__ float pll_fast_sin(float x)
{
    const float x2 = __fmul_rn(x, x), x4 = __fmul_rn(x2, x2);
    const double d2 = x2, d4 = x4, dx = x;
    const double a = __dadd_rn(__dmul_rn(2.7181216275479732e-6, d2), -1.9839312269456257e-4);
    const double b = __dadd_rn(__dmul_rn(8.3333293048425631e-3, d2), -1.6666666640797048e-1);
    const double in = __dadd_rn(__dmul_rn(a, d4), b);
    return (float)__dadd_rn(__dmul_rn(__dmul_rn(in, d2), dx), dx);
}
// fast_trig.cpp:80-154; tab = the 257-entry arctangent table (host-generated: atan(k / 255) through seven significant digits)
__device__ __forceinline__ float pll_fast_atan2f(float y, float x, const float *__restrict__ tab)
{
    const float ya = fabsf(y), xa = fabsf(x);
    if (!(ya > 0.0f || xa > 0.0f))
        return 0.0f;
    const float z = ya < xa ? __fdiv_rn(ya, xa) : __fdiv_rn(xa, ya);
    float base;
    if ((double)z < 0.003921569)
        base = z;
    else {
        float a = __fmul_rn(z, 255.0f);
        const int idx = ((int)a) & 0xff;
        a = __fsub_rn(a, (float)idx);
        const float t0 = tab[idx], t1 = tab[idx + 1];
        base = __fadd_rn(t0, __fmul_rn(__fsub_rn(t1, t0), a));
    }
    const float PI_F = 3.14159274101257324f, HPI_F = 1.57079637050628662f; // (float)M_PI, (float)M_PI_2
    if (xa > ya) {
        if (x >= 0.0f)
            return y >= 0.0f ? base : -base;
        return y >= 0.0f ? __fsub_rn(PI_F, base) : __fsub_rn(base, PI_F);
    }
    if (y >= 0.0f)
        return x >= 0.0f ? __fsub_rn(HPI_F, base) : __fadd_rn(HPI_F, base);
    return x >= 0.0f ? __fadd_rn(-HPI_F, base) : __fsub_rn(-HPI_F, base);
}
// while (v < -M_PI) v += 2 M_PI; while (v > M_PI) v -= 2 M_PI, compared and stepped in double, stored as float (:45-48, :59-62)
__device__ __forceinline__ float pll_wrap(float v)
{
    while ((double)v < -3.14159265358979323846)
        v = (float)((double)v + 6.28318530717958647692);
    while ((double)v > 3.14159265358979323846)
        v = (float)((double)v - 6.28318530717958647692);
    return v;
}
__device__ __forceinline__ float2 pll_step(const float2 x, float &phase, float &freq, const PllParams &P, const float *__restrict__ tab)
{
    const float vr = pll_fast_cos(phase), vi = -pll_fast_sin(phase);
    const float2 o = make_float2(__fsub_rn(__fmul_rn(x.x, vr), __fmul_rn(x.y, vi)), __fadd_rn(__fmul_rn(x.y, vr), __fmul_rn(x.x, vi)));
    const float err = pll_wrap(__fsub_rn(pll_fast_atan2f(x.y, x.x, tab), phase));
    freq = __fadd_rn(freq, __fmul_rn(P.beta, err));
    if (freq > P.fmax)
        freq = P.fmax;
    else if (freq < P.fmin)
        freq = P.fmin;
    phase = pll_wrap(__fadd_rn(__fadd_rn(phase, freq), __fmul_rn(P.alpha, err)));
    return o;
}

// the carrier PLL as the policy of loop_segments (no gear shift)
struct PllLoop
{
    PllParams P;
    const float *tab;
    static constexpr int G = 0; // no gear shift
    float ph, fr;
    __device__ __forceinline__ float phase() const { return ph; }
    __device__ __forceinline__ float freq() const { return fr; }
    __device__ __forceinline__ int order() const { return 1; } // the lock point is unique
    __device__ __forceinline__ void begin(float phase, float freq, long)
    {
        ph = phase;
        fr = freq;
    }
    __device__ __forceinline__ void row(bool mine, const float4 *ring, int slot, float4 *obuf, int lane, long b, long own1)
    {
        if (!mine)
            return;
        const int nvalid = (int)min(16L, own1 - b);
#pragma unroll 1
        for (int p = 0; p < 8; p++) {
            const float4 v = ring[swz16(slot + p, lane)];
            float2 o0 = make_float2(0.f, 0.f), o1 = o0;
            if (2 * p < nvalid)
                o0 = pll_step(make_float2(v.x, v.y), ph, fr, P, tab);
            if (2 * p + 1 < nvalid)
                o1 = pll_step(make_float2(v.z, v.w), ph, fr, P, tab);
            obuf[swz16(p, lane)] = make_float4(o0.x, o0.y, o1.x, o1.y);
        }
    }
};

// Same staging as k_costas (loop_segments). Dynamic shared memory: COSTAS_SMEM_BYTES of strips + the 257-entry table.
constexpr int PLL_SMEM_BYTES = COSTAS_SMEM_BYTES + 260 * 4;
__global__ void __launch_bounds__(SEG_THREADS) k_pll(const float2 *__restrict__ in, long N, int L, int W, int nseg, PllParams P,
                                                      const float *__restrict__ state_in, const float *__restrict__ atan_tab, float2 *__restrict__ out,
                                                      LoopRec *__restrict__ rec, const int *__restrict__ repair_list, const int *__restrict__ repair_count,
                                                      LoopCkpt *__restrict__ ckpt, float tol_phase, float tol_freq, int *__restrict__ merge_hist)
{
    extern __shared__ __align__(16) unsigned char pl_smem[];
    float *tab = reinterpret_cast<float *>(pl_smem + COSTAS_SMEM_BYTES);
    for (int i = threadIdx.x; i < 257; i += SEG_THREADS)
        tab[i] = atan_tab[i];
    __syncthreads();
    PllLoop lp{P, tab};
    loop_segments(lp, pl_smem, in, N, L, W, nseg, state_in, out, rec, repair_list, repair_count, ckpt, tol_phase, tol_freq, merge_hist);
}

// The VOLK rotator behind FreqShiftBlock (freq_shift.cpp:16-50) and PMToBPSK (pm_to_bpsk.cpp:10-35): out[n] = in[n] * e^{j n delta}
// with delta the angle of the float pair (cos, sin)(2 pi f / fs) the reference multiplies by. The reference advances its phasor by one
// rounded complex multiplication per sample (renormalised every 512 samples): a serial recurrence whose angle follows n * delta up to a
// rounding walk that depends on the VOLK flavour. Here the phasor of sample n comes in closed form from a 64-bit fixed-point count of
// turns (pos * dturn mod 2^64: exact for any stream position), evaluated in double and rounded once. imag_only: PMToBPSK first
// reduces its input to (0, imag) (pm_to_bpsk.cpp:24-25). iq_swap / FMT: the reader's conversion when the rotator is the first stage.
template <int FMT>
__global__ void __launch_bounds__(256) k_rotator(const void *__restrict__ raw, long N, int iq_swap, int imag_only, unsigned long long turn0,
                                                 unsigned long long dturn, float2 *__restrict__ out)
{
    const long s0 = ((long)blockIdx.x * 256 + threadIdx.x) * 8;
    if (s0 >= N)
        return;
    float2 x[8];
    load8<FMT>(raw, s0, N, x);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (s0 + i < N) {
            float2 v = x[i];
            if (iq_swap)
                v = make_float2(v.y, v.x);
            if (imag_only)
                v.x = 0.0f;
            const unsigned long long turn = turn0 + (unsigned long long)(s0 + i) * dturn; // fraction of a turn, 0.64 fixed point
            double sn, cs;
            sincospi((double)(long long)turn * 0x1p-63, &sn, &cs); // signed: [-1, 1) half turns
            const float pr = (float)cs, pi = (float)sn;
            out[s0 + i] = make_float2(__fsub_rn(__fmul_rn(v.x, pr), __fmul_rn(v.y, pi)), __fadd_rn(__fmul_rn(v.x, pi), __fmul_rn(v.y, pr)));
        }
    }
}

__device__ __forceinline__ float2 rot_steps(float2 v, int q, int order)
{
    // multiply by e^{+j q 2pi/order}
    if (order == 4) {
        if (q == 1) return make_float2(-v.y, v.x);
        if (q == 2) return make_float2(-v.x, -v.y);
        if (q == 3) return make_float2(v.y, -v.x);
        return v;
    } else if (order == 2) {
        return q ? make_float2(-v.x, -v.y) : v;
    } else {
        if (q == 0) return v;
        float sn, cs;
        sincospif(2.0f * (float)q / (float)order, &sn, &cs);
        return make_float2(v.x * cs - v.y * sn, v.y * cs + v.x * sn);
    }
}

// k quarter turns (multiply by j^k) as rot_steps computes them for orders 2 and 4, without a branch: swap = k & 1, then the real
// part's sign flips for k = 1, 2 and the imaginary part's for k = 2, 3 (neg_* = 0x80000000 or 0: an exact negation)
__device__ __forceinline__ float2 rot_quarter(float2 v, bool swap, unsigned neg_re, unsigned neg_im)
{
    const float re = swap ? v.y : v.x, im = swap ? v.x : v.y;
    return make_float2(__uint_as_float(__float_as_uint(re) ^ neg_re), __uint_as_float(__float_as_uint(im) ^ neg_im));
}

// ---------------------------------------------------------------- K2c: apply rotation (+ OQPSK delay) -> M&M input
// mmin has a 16-sample front pad: mmin[16 + n]; mmin[0..15] = last MM_HIST inputs of the previous batch (hist_in).
// `src` is the Costas output (or, with order == 0, the FIR output passed straight through).
__global__ void k_rotate(const float2 *__restrict__ src, long N, int L, int order, int oqpsk, const uint8_t *__restrict__ quad,
                         const float2 *__restrict__ hist_in /*MM_HIST: true pre-delay values*/, float2 *__restrict__ hist_out,
                         float2 *__restrict__ mmin)
{
    const long stride = (long)gridDim.x * blockDim.x;
    if (!oqpsk) {
        // two samples per thread, 16-byte accesses (src and mmin + 16 are 128-byte aligned; L is a multiple of 16, so a pair never
        // straddles two Costas segments)
        const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x;
        if (tid < MM_HIST) {
            const float2 h = hist_in[tid];
            mmin[16 - MM_HIST + tid] = h;
        }
        for (long p = tid; 2 * p < N; p += stride) {
            const long n = 2 * p;
            if (n + 1 < N) {
                float4 v = *reinterpret_cast<const float4 *>(src + n);
                float2 a = make_float2(v.x, v.y), b = make_float2(v.z, v.w);
                if (order) {
                    const int q = quad[n / L];
                    a = rot_steps(a, q, order);
                    b = rot_steps(b, q, order);
                }
                *reinterpret_cast<float4 *>(mmin + 16 + n) = make_float4(a.x, a.y, b.x, b.y);
                if (n >= N - MM_HIST)
                    hist_out[n - (N - MM_HIST)] = a;
                if (n + 1 >= N - MM_HIST)
                    hist_out[n + 1 - (N - MM_HIST)] = b;
            } else {
                float2 a = src[n];
                if (order)
                    a = rot_steps(a, quad[n / L], order);
                mmin[16 + n] = a;
                hist_out[n - (N - MM_HIST)] = a;
            }
        }
        return;
    }
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x - MM_HIST; n < N; n += stride) {
        float2 cur, prev;
        if (n >= 0) {
            cur = src[n];
            if (order)
                cur = rot_steps(cur, quad[n / L], order);
        } else
            cur = hist_in[MM_HIST + n];
        if (n >= N - MM_HIST && n >= 0) // (the host rejects batches below 64 samples)
            hist_out[n - (N - MM_HIST)] = cur;
        float2 v = cur;
        if (n - 1 >= 0) {
            prev = src[n - 1];
            if (order)
                prev = rot_steps(prev, quad[(n - 1) / L], order);
        } else if (n - 1 >= -MM_HIST)
            prev = hist_in[MM_HIST + n - 1];
        else
            prev = make_float2(0.f, 0.f);
        v.y = prev.y;
        mmin[16 + n] = v;
    }
}

// Fused path (k_mm applies the rotation itself): only the 8-sample history moves. src has a 16-sample front pad: src[16 + n].
__global__ void k_mm_prep(float2 *__restrict__ src, long N, int L, int order, const uint8_t *__restrict__ quad, const float2 *__restrict__ hist_in,
                          float2 *__restrict__ hist_out)
{
    const int t = threadIdx.x;
    if (t >= MM_HIST)
        return;
    src[16 - MM_HIST + t] = hist_in[t]; // the previous batch's last inputs, already in their final orientation (segment 0 never rotates)
    const long n = N - MM_HIST + t;
    float2 v = src[16 + n];
    if (order)
        v = rot_steps(v, quad[n / L], order);
    hist_out[t] = v;
}

// ---------------------------------------------------------------- K3: Mueller & Mueller clock recovery, one thread per segment
#endif // B200_DEFINE_KERNELS
struct MMParams
{
    float omega_mid, omega_limit, omega_gain, mu_gain;
};
struct MMState // carried between batches (exact for segment 0)
{
    float mu, omega;
    float2 p0, p1, p2, c0, c1, c2;
    int inc; // window start of the next symbol, relative to the batch start, in buffer coordinates
    int pad;
};
// per-segment record: the thread also emits the symbols of a short candidate zone BEFORE its segment (u >= own0 - MM_ZONE) and
// records the sampling instants of its first emitted symbols; k_mm_scan stitches neighbours by matching real-valued instants
// u + mu (so a symbol whose window start falls within the loops' ~1e-4 disagreement of a segment boundary is neither lost nor doubled).
constexpr int MM_ZONE = 6;
struct MMRec { int u_final, count, skip, pad; float mu_final, omega_final; int head_u[4]; float head_mu[4]; float2 p0, p1, p2, c0, c1, c2; };

#ifdef B200_DEFINE_KERNELS
// STRICT (test hook, b200_demod_debug_run_stage): the reference's operation order, separate multiplies and adds, left to right
// (volk_32fc_32f_dot_prod_32fc generic; clock_recovery_mm.cpp:103-114 compiled without FMA contraction) -> run as ONE sequential
// segment on the oracle's own M&M input the symbols must come out BITWISE the oracle's. The production instantiation keeps the
// two-chain FMA interpolator.
// GARDNER: dsp::GardnerClockRecoveryBlock<complex_t>::work (clock_recovery_gardner.cpp:33-131, SURVEY row G) instead of the M&M
// detector: same interpolator bank, omega / mu updates, history and segmentation; the error is zc * (last - sample) with a second
// interpolation half a symbol back (window u - offzc - 7 .. u - offzc); `p1` after the delay-line shift is last_sample.
// FIX: fused input fix-up (rot_order != 0 or oqpsk): mmin is then the Costas loop's raw output, and every thread applies the exact
// rotation by its row's quad[] entry (and the OQPSK one-sample delay of the imaginary rail, delay_one_imag.cpp:18-25) to each 16-sample
// row of its ring right after the row has landed, instead of a separate pass over the whole stream (k_rotate). Its state (quadrant,
// masks, OQPSK carry) would stay live through the symbol loop, which runs at 128 registers: the instantiation without FIX, for input
// that needs no fix-up, carries none of it.
// 8 consecutive samples n0 .. n0+7 of this thread's ring (sample n sits in 16-byte chunk slot (n >> 1) & 31 of the swizzled strip): five
// 128-bit loads and a select per value on the parity of n0, instead of eight 64-bit loads with their own address arithmetic.
__device__ __forceinline__ void mm_fetch8(const float4 *__restrict__ ring, int n0, int lane, float2 (&x)[8])
{
    const int p0 = n0 >> 1;
    const bool odd = n0 & 1;
    float4 v[5];
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const int pp = (p0 + j) & 31;
        v[j] = ring[pp * 32 + (lane ^ (pp & 7))];
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const float4 a = v[k >> 1], b = v[(k + 1) >> 1];
        const float2 ev = (k & 1) ? make_float2(a.z, a.w) : make_float2(a.x, a.y);       // start even: sample k = chunk k/2, half k%2
        const float2 od = ((k + 1) & 1) ? make_float2(b.z, b.w) : make_float2(b.x, b.y); // start odd: chunk (k+1)/2, half (k+1)%2
        x[k] = make_float2(odd ? od.x : ev.x, odd ? od.y : ev.y);
    }
}

template <bool STRICT, bool GARDNER, bool FIX, bool REAL = false>
__global__ void __launch_bounds__(SEG_THREADS) k_mm(const float2 *__restrict__ mmin /* 16-sample front pad */, long N, int L, int W, int G, int nseg,
                                                     MMParams P, const MMState *__restrict__ st_in, MMState *__restrict__ st_out,
                                                     const float *__restrict__ bank /*128x8*/, float2 *__restrict__ slots, int cap,
                                                     MMRec *__restrict__ rec, const int *__restrict__ repair_list, const int *__restrict__ repair_count,
                                                     const uint8_t *__restrict__ quad, int rot_order, int oqpsk, MMCkpt *__restrict__ ckpt, float tol_t,
                                                     float tol_omega, int *__restrict__ merge_hist)
{
    extern __shared__ __align__(16) unsigned char mm_smem[];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // per warp: ring of 64 samples = 32 chunk slots x 32 threads x 16 B (swizzled, see warp_load_rows); then the interpolator bank
    float4 *ring = reinterpret_cast<float4 *>(mm_smem) + warp * (32 * 32);
    float *sbank = reinterpret_cast<float *>(mm_smem + 64 * SEG_THREADS * sizeof(float2)); // [128][MM_BANK_STRIDE]
    // the symbols a thread emits in one row iteration: its j-th at stage[j * 32 + (lane ^ j)], so that the lanes storing their j-th
    // symbols and the copy-out's half-warps (lanes 8q..8q+7 read symbols 0..7 of thread i + 8q) are free of bank conflicts;
    // pub[lane] = (slot of the first, how many) for the copy-out
    float2 *stage = reinterpret_cast<float2 *>(sbank + 128 * MM_BANK_STRIDE) + warp * 32 * (MM_STAGE + 1);
    int2 *pub = reinterpret_cast<int2 *>(stage + 32 * MM_STAGE);
    LoopCycles cyc;
    for (int i = t; i < 128 * 8; i += SEG_THREADS)
        sbank[(i >> 3) * MM_BANK_STRIDE + (i & 7)] = bank[i];
    __syncthreads();
    bool active;
    const int s = loop_segment(nseg, repair_list, repair_count, active); // repair mode: exact sequential continuation of segment s-1
    const long own0 = (long)s * L, own1 = active ? min(own0 + L, N) : own0;
    // buffer coordinate u: window = input samples u-7 .. u
    long u;
    float mu, omega;
    float2 p0, p1, p2, c0, c1, c2;
    long ustart = own0 - W, gear_end = own0 - W + G; // gear shift as in k_costas: omega held, 4x the mu gain for the first G samples
    // Repair mode: the symbols go to the slots from `count` = the stored run's skip on (k_mm_scan: its candidate-zone symbols in
    // front of the junction), where the stored run has its own first kept symbol; the slots below stay skipped (placeholder heads in
    // front of the junction). A stored tail the repair joins is then already in place behind the repaired symbols.
    int count = 0;
    MMRec mr;
#pragma unroll
    for (int i = 0; i < 4; i++) { mr.head_u[i] = 0; mr.head_mu[i] = 0.f; }
    if (repair_list && active) {
        gear_end = 0;
        const MMRec pr = rec[s - 1];
        count = rec[s].skip & 3;
#pragma unroll
        for (int i = 0; i < 3; i++)
            if (i < count)
                mr.head_u[i] = pr.u_final - 4 * (count - i);
        mu = pr.mu_final; omega = pr.omega_final; p0 = pr.p0; p1 = pr.p1; p2 = pr.p2; c0 = pr.c0; c1 = pr.c1; c2 = pr.c2;
        u = pr.u_final;
    } else if (ustart <= 0) {
        MMState st = *st_in;
        mu = st.mu; omega = st.omega; p0 = st.p0; p1 = st.p1; p2 = st.p2; c0 = st.c0; c1 = st.c1; c2 = st.c2;
        u = st.inc;
        gear_end = 0;
    } else {
        mu = 0.5f; omega = st_in->omega;
        p0 = p1 = p2 = c0 = c1 = c2 = make_float2(0.f, 0.f);
        u = ustart;
    }
    // rows of 16 samples; sample n lives in chunk slot ((n + 64) >> 1) & 31; the first window's oldest sample is u-7 (>= -8)
    int r0;
    {
        const long a = u - 7 - (GARDNER ? 4 : 0); // (the zero-crossing window reaches floor(omega / 2) + 1 <= 3 samples further back)
        r0 = (int)((a >= 0) ? (a >> 4) : -((-a + 15) >> 4));
    }
    if (oqpsk && r0 > -1)
        r0 -= 1; // one more row in front: its last sample's imaginary part is the delay register of the first row that is used
                 // (row -1 is the front pad: nothing lies in front of it, and its first samples are never read)
    const int rend = (int)((own1 + 15) >> 4); // exclusive: samples < own1 <= N are ever needed
    // iteration `it` makes row r0+it+1 the newest complete row; symbols with u < 16*(r0+it+2) can then be produced
    int nit = active ? max(0, rend - r0) : 0, maxit = nit;
#pragma unroll
    for (int off = 16; off; off >>= 1)
        maxit = max(maxit, __shfl_xor_sync(0xffffffffu, maxit, off));
    const float2 *base = mmin + 16; // sample 0
    auto load = [&](int row, bool ok) { warp_load_rows(ring, base, row, ok && row < rend, N, lane); cp_async_commit(); };
    load(r0, active);
    load(r0 + 1, active);
    float carry_im = 0.f; // OQPSK: imaginary part (after rotation) of the sample in front of the next row
    // quadrant of the segment holding the first sample of the last row fixed, and the first row whose first sample lies in a later
    // segment: rows are fixed in increasing order, so quad[] is read once per segment the thread's rows enter (normally s-1 and s)
    // instead of once per row, where the global load waited behind the whole SM's row copies and symbol stores. Rows in front of
    // sample 0 (the front pad) keep q = 0: they come first, before any load.
    // For orders 2 and 4 the rotation is q * 4 / order quarter turns, applied as a swap and two sign flips chosen once per quadrant
    // (rot_quarter): the lanes of a warp hold different segments, and rot_steps' branch on q ran the lanes of each quadrant one
    // after the other for every sample. Order 8 keeps rot_steps (its odd steps multiply).
    int q = 0, qrow_next = 0;
    const bool quarter = rot_order == 2 || rot_order == 4;
    bool qswap = false;
    unsigned qneg_re = 0, qneg_im = 0;
    auto fixrow = [&](int row) {
        if (!FIX || !active || row >= rend || (!rot_order && !oqpsk))
            return;
        if (rot_order && row >= qrow_next) {
            const int sq = (16 * row) / L;
            q = quad[sq];
            qrow_next = (int)(((long)(sq + 1) * L + 15) >> 4);
            const int k = quarter ? q * (4 / rot_order) : 0;
            qswap = k & 1;
            qneg_re = ((k + 1) & 2) ? 0x80000000u : 0u;
            qneg_im = (k & 2) ? 0x80000000u : 0u;
        }
        if (q == 0 && !oqpsk)
            return;
        const int sb = (row << 3) + 64;
        float4 v[8]; // the whole row in registers first, so that the eight loads are in flight together
#pragma unroll
        for (int c = 0; c < 8; c++)
            v[c] = ring[swz16((sb + c) & 31, lane)];
#pragma unroll
        for (int c = 0; c < 8; c++) {
            float2 a = make_float2(v[c].x, v[c].y), b = make_float2(v[c].z, v[c].w);
            if (quarter) {
                a = rot_quarter(a, qswap, qneg_re, qneg_im);
                b = rot_quarter(b, qswap, qneg_re, qneg_im);
            } else if (q) {
                a = rot_steps(a, q, rot_order);
                b = rot_steps(b, q, rot_order);
            }
            if (oqpsk) {
                const float ta = a.y, tb = b.y;
                a.y = carry_im;
                b.y = ta;
                carry_im = tb;
            }
            v[c] = make_float4(a.x, a.y, b.x, b.y);
        }
#pragma unroll
        for (int c = 0; c < 8; c++)
            ring[swz16((sb + c) & 31, lane)] = v[c];
    };
    const long emit0 = (s == 0 || repair_list) ? min(own0, u) : own0 - MM_ZONE;
    float2 *my = slots + (long)s * cap;
    // the symbol loop runs on 32-bit offsets from the thread's start: ur = u - ubase (a segment plus its warm-up is far below 2^31)
    const long ubase = u;
    int ur = 0;
    const int emit32 = (int)max(-0x40000000L, min(0x40000000L, emit0 - ubase)), gear32 = (int)max(-0x40000000L, min(0x40000000L, gear_end - ubase));
    const int uring = (int)(ubase & 63) + 64; // ring sample index of sample n is (n + 64) mod 64 taken over chunk slots: only (n >> 1) & 31 and n & 1 matter
    bool done = !active;
    MMCkpt *my_ck = ckpt + (long)s * ckpt_per_seg(L) - 1; // my_ck[j]: in front of the first symbol with u >= own0 + j * CKPT, j >= 1
    const int orow0 = (int)(own0 >> 4);
    int joined_at = 0; // repair mode: the checkpoint at which this run met the stored one
    // the copy-out's view of the threads whose symbols this lane writes (lanes 8q..8q+7 carry thread i + 8q in step i)
    long src_slots[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
        src_slots[i] = (long)__shfl_sync(0xffffffffu, s, i + 8 * (lane >> 3)) * cap;
    int nst = 0, cfirst = 0; // symbols staged in this row iteration, slot of the first
    for (int it = 0; it < maxit; it++) {
        const int rr = r0 + 1 + it;
        load(rr + 1, active);
        cp_async_wait<1>(); // rows <= rr complete
        __syncwarp();
        cyc.mark(0);
        if (it == 0)
            fixrow(r0);
        fixrow(rr);
        cyc.mark(1);
        if (!done) {
            const long lim = min((long)(rr + 1) << 4, own1);
            const int lim32 = (int)(lim - ubase);
            while (ur < lim32) {
                const bool emit = ur >= emit32;
                if (emit && count < 4) {
                    if (count == 0) { mr.head_u[0] = (int)(ubase + ur); mr.head_mu[0] = mu; }
                    else if (count == 1) { mr.head_u[1] = (int)(ubase + ur); mr.head_mu[1] = mu; }
                    else if (count == 2) { mr.head_u[2] = (int)(ubase + ur); mr.head_mu[2] = mu; }
                    else { mr.head_u[3] = (int)(ubase + ur); mr.head_mu[3] = mu; }
                }
                p2 = p1; p1 = p0; c2 = c1; c1 = c0;
                int imu = __float2int_rn(mu * 128.0f); // (int)rint(mu * 128)
                imu = max(0, min(127, imu));
                const float4 *tp4 = reinterpret_cast<const float4 *>(&sbank[imu * MM_BANK_STRIDE]);
                const float4 ta = tp4[0], tb = tp4[1];
                const float tp[8] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
                float zr = 0.f, zi = 0.f;
                if (GARDNER) { // zero-crossing sample (clock_recovery_gardner.cpp:49-63,88)
                    const float muz = (float)((double)mu - (double)omega / 2.0);
                    int offzc = (int)floor((double)omega / 2.0);
                    float mupos = (float)fmod((double)__fadd_rn(muz, (float)offzc), 1.0);
                    if (mupos < 0.f) {
                        mupos = __fadd_rn(1.0f, mupos);
                        offzc += 1;
                    }
                    int imuz = (int)rintf(__fmul_rn(mupos, 128.0f));
                    imuz = max(0, min(127, imuz));
                    const float *tz = &sbank[imuz * MM_BANK_STRIDE];
                    float2 xz[8];
                    mm_fetch8(ring, uring + ur - offzc - 7, lane, xz);
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        if (STRICT) {
                            zr = __fadd_rn(zr, __fmul_rn(xz[k].x, tz[k]));
                            zi = __fadd_rn(zi, __fmul_rn(xz[k].y, tz[k]));
                        } else {
                            zr = fmaf(xz[k].x, tz[k], zr);
                            zi = fmaf(xz[k].y, tz[k], zi);
                        }
                    }
                }
                float2 xw[8];
                mm_fetch8(ring, uring + ur - 7, lane, xw); // ring index of sample u - 7 (>= 56)
                float ar = 0.f, ai = 0.f;
                if (STRICT) {
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        ar = __fadd_rn(ar, __fmul_rn(xw[k].x, tp[k]));
                        ai = __fadd_rn(ai, __fmul_rn(xw[k].y, tp[k]));
                    }
                } else {
                    float br = 0.f, bi = 0.f; // two chains (taps 0-3 / 4-7) to halve the dependent-FMA depth
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        ar = fmaf(xw[k].x, tp[k], ar);
                        ai = fmaf(xw[k].y, tp[k], ai);
                        br = fmaf(xw[k + 4].x, tp[k + 4], br);
                        bi = fmaf(xw[k + 4].y, tp[k + 4], bi);
                    }
                    ar += br;
                    ai += bi;
                }
                p0 = make_float2(ar, ai);
                float pe;
                if (GARDNER) { // zc * (last - sample), last = the previous output (p1 after the shift above); exact clip (:98-100)
                    pe = STRICT ? __fadd_rn(__fmul_rn(zr, __fsub_rn(p1.x, ar)), __fmul_rn(zi, __fsub_rn(p1.y, ai))) : zr * (p1.x - ar) + zi * (p1.y - ai);
                } else if (REAL) { // MMClockRecoveryBlock<float> (clock_recovery_mm.cpp:70-82): sgn(last) * sample - sgn(sample) * last, sgn(0) = +1
                    const float last = p1.x; // last_sample: the previous output (p1 after the shift above)
                    pe = __fsub_rn(last < 0.0f ? -ar : ar, ar < 0.0f ? -last : last);
                } else {
                    c0 = make_float2(ar > 0.0f ? 1.0f : 0.0f, ai > 0.0f ? 1.0f : 0.0f);
                    // Re[(p0-p2) conj(c1) - (c0-c2) conj(p1)]  (clock_recovery_mm.cpp:103)
                    float xr = (p0.x - p2.x) * c1.x + (p0.y - p2.y) * c1.y;
                    float yr = (c0.x - c2.x) * p1.x + (c0.y - c2.y) * p1.y;
                    pe = xr - yr;
                }
                pe = fminf(1.0f, fmaxf(-1.0f, pe));
                if (emit) {
                    if (nst < MM_STAGE) { // (only a loop taking steps below one sample could fill the stage within a row)
                        if (nst == 0)
                            cfirst = count;
                        stage[nst * 32 + (lane ^ nst)] = p0;
                        nst++;
                    } else if (count < cap)
                        my[count] = p0;
                    count++;
                }
                if (ur < gear32)
                    mu = (mu + omega) + 4.0f * P.mu_gain * pe;
                else {
                    omega = STRICT ? __fadd_rn(omega, __fmul_rn(P.omega_gain, pe)) : omega + P.omega_gain * pe;
                    float dev = omega - P.omega_mid;
                    if (GARDNER) // BRANCHLESS_CLIP with float operands (block.h:10): the two sums in float, the rest in double (:109)
                        omega = (float)((double)P.omega_mid + 0.5 * (double)__fsub_rn(fabsf(__fadd_rn(dev, P.omega_limit)), fabsf(__fsub_rn(dev, P.omega_limit))));
                    else {
                        dev = fminf(P.omega_limit, fmaxf(-P.omega_limit, dev));
                        omega = P.omega_mid + dev;
                    }
                    mu = STRICT ? __fadd_rn(__fadd_rn(mu, omega), __fmul_rn(P.mu_gain, pe)) : (mu + omega) + P.mu_gain * pe;
                }
                const float fl = floorf(mu);
                ur += (int)fl;
                mu -= fl;
            }
            if (ubase + ur >= own1)
                done = true;
            // the row ended on a checkpoint: the main pass stores the state there; a repair stops when it has filled the same slots as
            // the stored run and sits on the same sampling instant and omega (the stored symbols from here on follow in place)
            const int rel = rr + 1 - orow0;
            if (!done && rel > 0 && (rel & (CKPT / 16 - 1)) == 0) {
                MMCkpt &ck = my_ck[rel / (CKPT / 16)];
                const int un = (int)(ubase + ur);
                if (repair_list && ck.count == count && fabsf((float)(un - ck.u) + (mu - ck.mu)) < tol_t && fabsf(omega - ck.omega) < tol_omega) {
                    joined_at = rel / (CKPT / 16);
                    done = true;
                } else
                    ck = MMCkpt{un, count, mu, omega};
            }
        }
        cyc.mark(2);
        // copy-out of this iteration's symbols: each thread's are consecutive slots, so a store instruction writes four short runs
        // instead of 32 scattered symbols
        pub[lane] = make_int2(cfirst, nst);
        __syncwarp();
        {
            const int c = lane & 7;
            const bool more = __any_sync(0xffffffffu, nst > 8);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int T = i + 8 * (lane >> 3);
                const int2 pb = pub[T];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int j = c + 8 * h;
                    if ((h == 0 || more) && j < pb.y && pb.x + j < cap)
                        slots[src_slots[i] + pb.x + j] = stage[j * 32 + (T ^ j)];
                }
            }
        }
        nst = 0;
        cyc.mark(3);
        __syncwarp(); // the next iteration's copy overwrites the oldest row of the ring, its symbols the stage
        if (repair_list && __all_sync(0xffffffffu, done))
            break;
    }
    cp_async_wait<0>();
    cyc.publish(LC_MM, !repair_list);
    if (!active)
        return;
    if (repair_list)
        count_repair(merge_hist, joined_at);
    if (joined_at) { // the stored run's symbols behind the checkpoint, its count and its end state stand
#pragma unroll
        for (int i = 0; i < 4; i++) {
            rec[s].head_u[i] = mr.head_u[i];
            rec[s].head_mu[i] = mr.head_mu[i];
        }
        return;
    }
    u = ubase + ur;
    mr.u_final = (int)u;
    mr.mu_final = mu;
    mr.omega_final = omega;
    mr.count = count;
    mr.skip = 0;
    mr.pad = 0;
    mr.p0 = p0; mr.p1 = p1; mr.p2 = p2; mr.c0 = c0; mr.c1 = c1; mr.c2 = c2;
    rec[s] = mr;
    if (s == nseg - 1) {
        MMState st;
        st.mu = mu; st.omega = omega; st.p0 = p0; st.p1 = p1; st.p2 = p2; st.c0 = c0; st.c1 = c1; st.c2 = c2;
        st.inc = (int)(u - N);
        st.pad = 0;
        *st_out = st;
    }
}

// ---------------------------------------------------------------- K3b: symbol offsets (exclusive scan) + junction check
__global__ void __launch_bounds__(1024) k_mm_scan(MMRec *__restrict__ rec, int nseg, float tol_t, long *__restrict__ offs /*nseg+1*/,
                                                 int *__restrict__ unconv, int cap, int *__restrict__ flags, int *__restrict__ repair_list,
                                                 int *__restrict__ repair_count, int round, int *__restrict__ repairs_total)
{
    __shared__ long wsum[32];
    __shared__ long run;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (round > 0) {
        const int pending = *repair_count;
        if (pending == 0)
            return;
        __syncthreads();
        if (t == 0)
            *repairs_total += min(pending, 1024);
    }
    if (t == 0) {
        run = 0;
        *repair_count = 0;
    }
    __syncthreads();
    int bad = 0, over = 0;
    for (int base = 0; base < nseg; base += 1024) {
        int s = base + t;
        long c = 0;
        if (s < nseg) {
            MMRec b = rec[s];
            c = b.count;
            if (c > cap)
                over = 1;
            int skip = 0;
            if (s > 0) {
                // instant of the symbol that follows segment s-1's last one, as seen by its own thread
                const MMRec a = rec[s - 1];
                const double tref = (double)a.u_final + (double)a.mu_final;
                const int nh = (int)min(4L, c);
                while (skip < nh && (double)b.head_u[skip] + (double)b.head_mu[skip] < tref - 0.5)
                    skip++;
                // the first kept symbol must be that very symbol
                double tk = (skip < nh) ? (double)b.head_u[skip] + (double)b.head_mu[skip] : (double)b.u_final + (double)b.mu_final;
                if (skip >= 4 || fabs(tk - tref) > tol_t) {
                    bad++;
                    const int slot = atomicAdd(repair_count, 1);
                    if (slot < 1024)
                        repair_list[slot] = s;
                }
            }
            rec[s].skip = skip;
            c -= skip;
        }
        long v = c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            long p = __shfl_up_sync(0xffffffffu, v, off);
            if (lane >= off)
                v += p;
        }
        if (lane == 31)
            wsum[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long w = wsum[lane];
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                long p = __shfl_up_sync(0xffffffffu, w, off);
                if (lane >= off)
                    w += p;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        long incl = run + v + (warp > 0 ? wsum[warp - 1] : 0);
        if (s < nseg)
            offs[s] = incl - c;
        __syncthreads();
        if (t == 1023)
            run = incl;
        __syncthreads();
    }
    for (int off = 16; off; off >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, off);
        over |= __shfl_xor_sync(0xffffffffu, over, off);
    }
    (void)bad;
    if (lane == 0 && over)
        atomicOr(flags, 2);
    __syncthreads();
    if (t == 0) {
        offs[nseg] = run;
        *unconv = *repair_count; // junctions still failing after this pass
    }
}

// module_demod_base.h:106-113 (clamp) applied to re*scale / im*scale
__device__ __forceinline__ int8_t soft_quant(float x)
{
    if (x < -128.0f) return -127;
    if (x > 127.0f) return 127;
    return (int8_t)(int)x;
}

// ---------------------------------------------------------------- K3c: compact per-segment symbol slots -> contiguous symbols + int8 soft
constexpr int SNR_WINDOW = 1024 * 64; // symbols at the end of a batch that k_snr_m2m4 reads (one CTA, 64 per thread)
// all_symbols == 0: only the last SNR_WINDOW symbols go to sym_out (the soft stream is the batch's only consumer-visible output, and the
// SNR estimate needs no more), which saves 8 of the 18 bytes per symbol this pass moves. Each thread loads MC_UNROLL slots before it
// stores anything, so enough loads are in flight to keep HBM busy.
constexpr int MC_UNROLL = 4;
__global__ void __launch_bounds__(256) k_mm_compact(const float2 *__restrict__ slots, int cap, const MMRec *__restrict__ rec,
                                                   const long *__restrict__ offs, int nseg, int bpsk, int all_symbols,
                                                   float2 *__restrict__ sym_out, int8_t *__restrict__ soft_out)
{
    // symbols from here on are written to sym_out (fsk_demod, bpsk 3: one float each, and its SNR estimate reads them as pairs)
    const long keep0 = all_symbols ? 0 : offs[nseg] - (bpsk == 3 ? 2 * SNR_WINDOW + 1 : SNR_WINDOW);
    for (int s = blockIdx.x; s < nseg; s += gridDim.x) {
        const int sk = rec[s].skip;
        const int c = min(rec[s].count, cap) - sk;
        const long o = offs[s];
        const float2 *src = slots + (long)s * cap + sk;
        for (int i0 = threadIdx.x; i0 < c; i0 += MC_UNROLL * blockDim.x) {
            float2 v[MC_UNROLL];
#pragma unroll
            for (int j = 0; j < MC_UNROLL; j++) {
                const int i = i0 + j * blockDim.x;
                if (i < c)
                    v[j] = src[i];
            }
#pragma unroll
            for (int j = 0; j < MC_UNROLL; j++) {
                const int i = i0 + j * blockDim.x;
                if (i >= c)
                    break;
                if (o + i >= keep0) {
                    if (bpsk == 3)
                        reinterpret_cast<float *>(sym_out)[o + i] = v[j].x;
                    else
                        sym_out[o + i] = v[j];
                }
                // 1: psk_demod's BPSK, real * 50 (module_psk_demod.cpp:199-205); 2: pm_demod, real * 100 (module_pm_demod.cpp:141-144);
                // 3: fsk_demod, real * 50 (module_fsk_demod.cpp:133-134)
                if (bpsk)
                    soft_out[o + i] = soft_quant(v[j].x * (bpsk == 2 ? 100.0f : 50.0f));
                else {
                    char2 q;
                    q.x = soft_quant(v[j].x * 100.0f);
                    q.y = soft_quant(v[j].y * 100.0f);
                    reinterpret_cast<char2 *>(soft_out)[o + i] = q;
                }
            }
        }
    }
}

// ---------------------------------------------------------------- M2M4 SNR estimate over the recovered symbols
// M2M4SNREstimator::update (common/dsp/utils/snr_estimator.cpp:16-39): two exponential averages y <- alpha * m + beta * y of |s|^2 and
// |s|^4 over the symbol stream (alpha = 0.001: a memory of ~1000 symbols). Linear with constant coefficients, so the end value of a batch
// is sum_i beta^(n-1-i) alpha m_i + beta^n y_in; terms older than 2^16 symbols weigh below e^-65 and are left out. One CTA: every thread
// runs the recurrence over 64 consecutive symbols (fp64), the partial results are combined with their powers of beta.
// pairs = 1 (fsk_demod): sym holds *total floats, estimated as *total / 2 complex pairs (module_fsk_demod.cpp:127).
__global__ void __launch_bounds__(1024) k_snr_m2m4(const float2 *__restrict__ sym, const long *__restrict__ total, int pairs, float alpha,
                                                  const float *__restrict__ yin, float *__restrict__ yout)
{
    __shared__ double red[2][32];
    const long n = *total >> pairs;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int RUN = SNR_WINDOW / 1024;
    const long M = min(n, (long)SNR_WINDOW), base = n - M;
    const double beta = (double)(float)(1.0 - (double)alpha), al = (double)alpha;
    const long i0 = (long)t * RUN, i1 = min(M, i0 + RUN);
    double a1 = 0.0, a2 = 0.0;
    for (long i = i0; i < i1; i++) {
        const float2 v = sym[base + i];
        const float ab = hypotf(v.x, v.y);
        const float m2 = ab * ab, m4 = ab * ab * ab * ab;
        a1 = fma(a1, beta, al * (double)m2);
        a2 = fma(a2, beta, al * (double)m4);
    }
    const double w = i1 > i0 ? pow(beta, (double)(M - i1)) : 0.0;
    a1 *= w;
    a2 *= w;
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        a1 += __shfl_xor_sync(0xffffffffu, a1, off);
        a2 += __shfl_xor_sync(0xffffffffu, a2, off);
    }
    if (lane == 0) { red[0][warp] = a1; red[1][warp] = a2; }
    __syncthreads();
    if (t == 0) {
        double s1 = 0.0, s2 = 0.0;
        for (int k = 0; k < 32; k++) { s1 += red[0][k]; s2 += red[1][k]; }
        const double carry = n > 0 ? pow(beta, (double)n) : 1.0;
        float y1 = (float)(s1 + carry * (double)yin[0]), y2 = (float)(s2 + carry * (double)yin[1]);
        if (y1 != y1) y1 = 0.f; // snr_estimator.cpp:27-30
        if (y2 != y2) y2 = 0.f;
        yout[0] = y1;
        yout[1] = y2;
    }
}

#endif // B200_DEFINE_KERNELS
} // namespace b200
