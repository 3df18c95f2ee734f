/*
 * TEST INFRASTRUCTURE ONLY — see oracle.h. CPU restatement ("port") of the reference's
 * baseband -> CADU path. Plain C, scalar, single thread. Float code must be built WITHOUT FMA
 * contraction (-ffp-contract=off, no -march) so that it reproduces the reference's x86-64 baseline
 * arithmetic bit for bit (the oracle of record is the generic/scalar VOLK flavour, SURVEY.md §8c).
 */
#include "oracle.h"
#include <stdio.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define STREAM_MAX 1000000 /* dsp::STREAM_BUFFER_SIZE, src-core/common/dsp/buffer.cpp:7 */

/* ======================================================================= filter design */

/* firdes::root_raised_cosine — src-core/common/dsp/filter/firdes.cpp:34-78 (all double, odd tap count, unit DC gain) */
int orc_rrc_taps(double gain, double fs, double rs, double alpha, int ntaps, float *out)
{
    ntaps |= 1;
    double spb = fs / rs, scale = 0;
    for (int i = 0; i < ntaps; i++) {
        double xi = i - ntaps / 2;
        double x1 = M_PI * xi / spb, x2 = 4 * alpha * xi / spb, x3 = x2 * x2 - 1, num, den;
        if (fabs(x3) >= 0.000001) {
            if (i != ntaps / 2)
                num = cos((1 + alpha) * x1) + sin((1 - alpha) * x1) / (4 * alpha * xi / spb);
            else
                num = cos((1 + alpha) * x1) + (1 - alpha) * M_PI / (4 * alpha);
            den = x3 * M_PI;
        } else {
            if (alpha == 1) {
                out[i] = -1;
                scale += out[i];
                continue;
            }
            x3 = (1 - alpha) * x1;
            x2 = (1 + alpha) * x1;
            num = (sin(x2) * (1 + alpha) * M_PI - cos(x3) * ((1 - alpha) * M_PI * spb) / (4 * alpha * xi) +
                   sin(x3) * spb * spb / (4 * alpha * xi * xi));
            den = -32 * M_PI * alpha * alpha * xi / spb;
        }
        out[i] = 4 * alpha * num / den; /* stored as float before the normalisation sum, like the reference */
        scale += out[i];
    }
    for (int i = 0; i < ntaps; i++)
        out[i] = out[i] * gain / scale;
    return ntaps;
}

/* windowed_sinc(1024, 2*pi*0.5/128, nuttall, 128) rearranged into 128 arms x 8 taps —
 * src-core/common/dsp/window/window.cpp:9-50, src-core/common/dsp/resamp/polyphase_bank.cpp:6-39 */
void orc_mm_bank(float *out)
{
    const int nfilt = 128, ntaps = 8, count = nfilt * ntaps;
    const double coefs[4] = {0.355768, 0.487396, 0.144232, 0.012604};
    double omega = 2.0 * M_PI * ((0.5 / (double)nfilt) / 1.0);
    double half = count / 2.0, corr = nfilt * omega / M_PI;
    for (int i = 0; i < count; i++) {
        double t = (double)i - half + 0.5;
        double x = t * omega;
        double sinc = (x == 0.0) ? 1.0 : sin(x) / x;
        double win = 0, sign = 1;
        for (int c = 0; c < 4; c++) {
            win += sign * coefs[c] * cos((double)c * 2.0 * M_PI * (t - half) / count);
            sign = -sign;
        }
        float tap = sinc * win * corr;
        out[((nfilt - 1) - (i % nfilt)) * ntaps + i / nfilt] = tap;
    }
}

/* ======================================================================= front-end resampler of BaseDemodModule
 * SmartResamplerBlock (resamp/smart_resampler.cpp:8-61) = optional power-of-two decimator (PowerDecimatorBlock, resamp/power_decim.cpp: a
 * cascade of DecimatingFIRBlocks, filter/decimating_fir.cpp) + RationalResamplerBlock. The decimator's tap tables are numeric data of the
 * reference (resamp/power_decim/\*.h), shared with the CUDA path through satdump_b200/csrc/power_decim_taps.inc (generated). */
#include "../satdump_b200/csrc/power_decim_taps.inc"

static double izero(double x) /* firdes.cpp:357-373 */
{
    double sum, u, halfx, temp;
    int n;
    sum = u = n = 1;
    halfx = x / 2.0;
    do {
        temp = halfx / (double)n;
        n += 1;
        temp *= temp;
        u *= temp;
        sum += u;
    } while (u >= 1E-21 * sum);
    return sum;
}

/* firdes::design_resampler_filter_float (firdes.cpp:276-301) -> low_pass (:80-120) with window::kaiser (:453-478); returns ntaps */
static int design_resampler(unsigned interpolation, unsigned decimation, float fractional_bw, float **out)
{
    float beta = 7.0, halfband = 0.5, rate = (float)interpolation / (float)decimation, trans_width, mid;
    if (rate >= 1.0) { trans_width = halfband - fractional_bw; mid = halfband - trans_width / 2.0; }
    else { trans_width = rate * (halfband - fractional_bw); mid = rate * halfband - trans_width / 2.0; }
    double gain = interpolation, fs = interpolation, cutoff = mid, tw = trans_width, b = beta;
    double a = b / 0.1102 + 8.7; /* window::max_attenuation(WIN_KAISER) */
    int ntaps = (int)(a * fs / (22.0 * tw));
    if ((ntaps & 1) == 0) ntaps++;
    float *taps = malloc(sizeof(float) * ntaps), *w = malloc(sizeof(float) * ntaps);
    {
        double IBeta = 1.0 / izero(b), inm1 = 1.0 / ((double)(ntaps - 1)), temp;
        w[0] = IBeta;
        for (int i = 1; i < ntaps - 1; i++) { temp = 2 * i * inm1 - 1; w[i] = izero(b * sqrt(1.0 - temp * temp)) * IBeta; }
        w[ntaps - 1] = IBeta;
    }
    int M = (ntaps - 1) / 2;
    double fwT0 = 2 * M_PI * cutoff / fs;
    for (int n = -M; n <= M; n++) {
        if (n == 0) taps[n + M] = fwT0 / M_PI * w[n + M];
        else taps[n + M] = sin(n * fwT0) / (n * M_PI) * w[n + M];
    }
    double fmax = taps[0 + M];
    for (int n = 1; n <= M; n++) fmax += 2 * taps[n + M];
    gain /= fmax;
    for (int i = 0; i < ntaps; i++) taps[i] *= gain;
    free(w);
    *out = taps;
    return ntaps;
}

static unsigned gcd_u(unsigned a, unsigned b) { while (b) { unsigned t = a % b; a = b; b = t; } return a; }

typedef struct /* DecimatingFIRBlock<complex_t> (filter/decimating_fir.cpp:12-87) */
{
    int D, nt, inc;
    const float *taps; /* as designed; applied reversed (decimating_fir.cpp:30) */
    float *buffer;     /* re,im pairs: nt history + the call's input */
} orc_decim;

typedef struct
{
    int active, interp, decim, ntaps, ctr, inc; /* RationalResamplerBlock: d_interpolation, d_decimation, pfb.ntaps, d_ctr, inc */
    float *bank;                                /* [interp][ntaps] */
    float *buffer;                              /* re,im pairs */
    int nstages;                                /* PowerDecimatorBlock in front (0 = none), smart_resampler.cpp:22-29 */
    orc_decim st[4];
    float *tmp;
} orc_resamp;

/* DecimatingFIRBlock::process: out[k] = sum_j buffer[inc + 1 + j] * taps[nt - 1 - j], inc += D; generic dot product, left to right */
static int decim_run(orc_decim *d, const float *in, int nsamples, float *out)
{
    memcpy(&d->buffer[2 * d->nt], in, (size_t)nsamples * 2 * sizeof(float));
    int outc = 0;
    for (; d->inc < nsamples; d->inc += d->D) {
        const float *x = &d->buffer[2 * (d->inc + 1)];
        float re = 0, im = 0;
        for (int j = 0; j < d->nt; j++) { float h = d->taps[d->nt - 1 - j]; re += x[2 * j] * h; im += x[2 * j + 1] * h; }
        out[2 * outc] = re; out[2 * outc + 1] = im; outc++;
    }
    d->inc -= nsamples;
    memmove(&d->buffer[0], &d->buffer[2 * nsamples], (size_t)d->nt * 2 * sizeof(float));
    return outc;
}

/* SmartResamplerBlock ctor (smart_resampler.cpp:8-61) */
static int resamp_init(orc_resamp *r, unsigned interpolation, unsigned decimation, int max_in)
{
    memset(r, 0, sizeof(*r));
    if (decimation == interpolation) return 1;
    double rsamp_in = decimation, fout = interpolation;
    if (decimation > interpolation) {
        int best_power = floor(log2(decimation / interpolation)); /* integer division, as in the reference */
        if (best_power > 0) {
            int best_decim = 1 << best_power;
            if (best_decim > (1 << PD_NPLANS)) best_decim = 1 << PD_NPLANS;
            rsamp_in = (double)decimation / (double)best_decim;
            const PdPlan *plan = &PD_PLANS[(int)log2(best_decim) - 1]; /* power_decim.cpp:15-29 */
            r->nstages = plan->nstages;
            for (int i = 0; i < plan->nstages; i++) {
                r->st[i].D = plan->stages[i].decimation; r->st[i].nt = plan->stages[i].ntaps; r->st[i].taps = PD_TAPS + plan->stages[i].offset;
                r->st[i].buffer = calloc((size_t)2 * (max_in + r->st[i].nt + 16), sizeof(float));
            }
            r->tmp = calloc((size_t)2 * (max_in + 16), sizeof(float));
            r->active = 1; r->interp = r->decim = 1; /* (the rational part below may replace these) */
        }
        if (rsamp_in == fout) { r->ntaps = 0; return 1; }
        double t;
        while (modf(rsamp_in, &t) != 0 || modf(fout, &t) != 0) { rsamp_in *= 10; fout *= 10; }
    }
    unsigned I = (unsigned)fout, D = (unsigned)rsamp_in, g = gcd_u(I, D); /* rational_resampler.cpp:27-41 */
    I /= g; D /= g;
    float *rt;
    int n = design_resampler(I, D, 0.4, &rt);
    /* PolyphaseBank::init(rtaps, nfilt = I) — polyphase_bank.cpp:6-39 */
    int nt = (n + I - 1) / I;
    if (fmod((double)n / (double)I, 1.0) > 0.0) nt++;
    r->bank = calloc((size_t)I * nt, sizeof(float));
    for (int i = 0; i < (int)I * nt; i++) r->bank[((I - 1) - (i % I)) * nt + i / I] = i < n ? rt[i] : 0;
    free(rt);
    r->active = 1; r->interp = I; r->decim = D; r->ntaps = nt;
    r->buffer = calloc((size_t)2 * (max_in + nt + 16), sizeof(float));
    return 1;
}

/* RationalResamplerBlock::process (rational_resampler.cpp:43-65); generic volk_32fc_32f_dot_prod_32fc: left to right, mul then add */
static int resamp_run(orc_resamp *r, const float *in, int nsamples, float *out)
{
    if (r->nstages) { /* SmartResamplerBlock::process: decimator, then (in place) the rational resampler */
        float *cur = r->tmp;
        for (int i = 0; i < r->nstages; i++) {
            nsamples = decim_run(&r->st[i], in, nsamples, r->ntaps == 0 && i == r->nstages - 1 ? out : cur);
            in = cur;
        }
        if (r->ntaps == 0) return nsamples;
    }
    memcpy(&r->buffer[2 * (r->ntaps - 1)], in, nsamples * 2 * sizeof(float));
    int outc = 0;
    while (r->inc < nsamples) {
        const float *x = &r->buffer[2 * r->inc], *t = &r->bank[(size_t)r->ctr * r->ntaps];
        float re = 0, im = 0;
        for (int k = 0; k < r->ntaps; k++) { re += x[2 * k] * t[k]; im += x[2 * k + 1] * t[k]; }
        out[2 * outc] = re; out[2 * outc + 1] = im; outc++;
        r->ctr += r->decim;
        r->inc += r->ctr / r->interp;
        r->ctr = r->ctr % r->interp;
    }
    r->inc -= nsamples;
    memmove(&r->buffer[0], &r->buffer[2 * nsamples], r->ntaps * 2 * sizeof(float));
    return outc;
}

int orc_resampler_taps(unsigned interpolation, unsigned decimation, float *out, int cap, int *nfilt)
{
    orc_resamp r;
    /* RationalResamplerBlock(nullptr, interpolation, decimation) directly (no SmartResampler pre-scaling) */
    unsigned g = gcd_u(interpolation, decimation), I = interpolation / g, D = decimation / g;
    float *rt;
    int n = design_resampler(I, D, 0.4, &rt);
    int nt = (n + I - 1) / I;
    if (fmod((double)n / (double)I, 1.0) > 0.0) nt++;
    *nfilt = I;
    if ((long)I * nt > cap) { free(rt); return -1; }
    memset(out, 0, sizeof(float) * I * nt);
    for (int i = 0; i < (int)I * nt; i++) out[((I - 1) - (i % I)) * nt + i / I] = i < n ? rt[i] : 0;
    free(rt);
    (void)r;
    return nt;
}

/* ======================================================================= demodulator chain */

typedef struct { float re, im; } cf_t;

typedef struct
{
    orc_demod_cfg cfg;
    int buffer_size, ntaps, order;
    float sps;
    /* AGC (utils/agc.cpp:16-43) */
    float agc_rate, agc_ref, agc_gain, agc_max;
    /* FIR (filter/fir.cpp:13-89) */
    float taps[512];
    cf_t *fir_buf;
    /* Costas (pll/costas_loop.cpp:5-69) */
    float phase, freq, alpha, beta, fmin, fmax;
    /* OQPSK delay (demod/delay_one_imag.cpp:10-30) */
    float last_imag;
    /* M&M (clock_recovery/clock_recovery_mm.cpp:10-137) */
    float bank[128 * 8];
    float mu, omega, omega_gain, mu_gain, omega_mid, omega_limit;
    cf_t p0, p1, p2, c0, c1, c2;
    int inc;
    cf_t *mm_buf;
    cf_t *w0, *w1, *w2; /* per-buffer scratch */
    orc_resamp rs;      /* front-end resampler (module_demod_base.cpp:203-204) */
    long last_front;    /* samples that entered the AGC in the last orc_demod_run call */
    cf_t dc_acc;        /* CorrectIQBlock::acc (front) */
    cf_t dc_acc2;       /* CorrectIQBlock::acc (behind the Costas loop) */
    cf_t *rs_in;
    /* pm_demod (module_pm_demod.cpp:61-88) and freq_shift (module_demod_base.cpp:122-123) */
    int rs_after;            /* the resampler sits behind PMToBPSK ("resample_after_pll") */
    float pll_state[2];      /* PLLCarrierTrackingBlock: d_phase, d_freq */
    float pm_inc[2], pm_phase[2], fs_inc[2], fs_phase[2]; /* rotator steps / phasors of PMToBPSK and FreqShiftBlock */
    float agc2_gain;         /* AGCBlock(resampler out, 0.001, 1.0, 1.0, 1000.0) (module_pm_demod.cpp:73-74) */
    cf_t dc_acc3;            /* CorrectIQBlock::acc behind the carrier PLL (has_carrier, module_psk_demod.cpp:112) */
    long pm_pos;
    float *pll_dump, *pm_dump;
} orc_demod;

static float clip_branchless(float x, float c) { return 0.5 * (fabsf(x + c) - fabsf(x - c)); } /* block.cpp:5 */
static float clip_branched(float x, float c) { return x < -c ? -c : (x > c ? c : x); }           /* block.cpp:7-15 */

void *orc_demod_create(const orc_demod_cfg *c)
{
    orc_demod *d = calloc(1, sizeof(*d));
    d->cfg = *c;
    long fs = (long)c->samplerate, rs = (long)c->symbolrate;
    /* module_demod_base.cpp:25 */
    int def = fs / 200 > 8193 ? (int)(fs / 200) : 8193;
    if (def > STREAM_MAX) def = STREAM_MAX;
    d->buffer_size = c->buffer_size > 0 ? c->buffer_size : def;
    float final_fs = c->final_samplerate > 0 ? (float)c->final_samplerate : (float)fs; /* float final_samplerate, module_demod_base.h:58 */
    d->sps = final_fs / (float)rs;     /* module_demod_base.cpp:81 */
    if (c->pm) { /* PMToBPSK(pll out, d_resample_after_pll ? d_samplerate : final_samplerate, subcarrier == 0 ? d_symbolrate : subcarrier), float args */
        const float rate = c->pm_resample_after_pll ? (float)fs : final_fs;
        const unsigned long sub = (unsigned long)c->pm_subcarrier_offset;
        const float f = sub == 0 ? (float)rs : (float)sub;
        orc_rotator_inc(-(double)f, (double)rate, d->pm_inc); /* pm_to_bpsk.cpp:12 */
        d->pm_phase[0] = 1.0f;
        d->agc2_gain = 1.0f;
        d->rs_after = c->pm_resample_after_pll;
    }
    if (c->freq_shift != 0) { /* FreqShiftBlock(input, d_samplerate, d_frequency_shift): long parameters (module_demod_base.cpp:122-123) */
        orc_rotator_inc((double)(long)c->freq_shift, (double)fs, d->fs_inc);
        d->fs_phase[0] = 1.0f;
    }
    if (c->final_samplerate > 0 && (long)c->final_samplerate != fs) {
        float decimation_factor = fs / final_fs; /* module_demod_base.cpp:84-87 */
        d->buffer_size *= ceil(decimation_factor);
        if (d->buffer_size > 8192 * 20) d->buffer_size = 8192 * 20;
        /* SmartResamplerBlock(input, final_samplerate, d_samplerate): (unsigned interpolation, unsigned decimation) */
        if (!resamp_init(&d->rs, (unsigned)final_fs, (unsigned)fs, d->buffer_size)) { free(d); return NULL; }
        d->rs_in = malloc(sizeof(cf_t) * d->buffer_size);
    }
    d->agc_rate = c->agc_rate; d->agc_ref = 1.0f; d->agc_gain = 1.0f; d->agc_max = 65536; /* module_demod_base.cpp:207 */
    d->ntaps = orc_rrc_taps(1, final_fs, (int)rs, c->rrc_alpha, c->rrc_taps, d->taps);      /* module_psk_demod.cpp:91 */
    d->fir_buf = calloc(2 * STREAM_MAX, sizeof(cf_t));
    d->order = c->constellation == 0 ? 2 : (c->constellation == 3 ? 8 : (c->constellation == 4 ? 0 : 4));
    if (c->pm) d->order = 2;
    {   /* costas_loop.cpp:5-12 */
        float damping = sqrtf(2.0f) / 2.0f;
        float denom = (1.0 + 2.0 * damping * c->pll_bw + c->pll_bw * c->pll_bw);
        d->alpha = (4 * damping * c->pll_bw) / denom;
        d->beta = (4 * c->pll_bw * c->pll_bw) / denom;
        d->fmin = -c->costas_max_offset; d->fmax = c->costas_max_offset;
        if (c->pm) { d->fmin = -1.0f; d->fmax = 1.0f; } /* CostasLoopBlock(rrc out, d_loop_bw, 2): freq_limit defaults to 1.0 (module_pm_demod.cpp:84) */
    }
    orc_mm_bank(d->bank);
    d->mu = c->clock_mu; d->omega = d->sps; d->omega_gain = c->clock_gain_omega; d->mu_gain = c->clock_gain_mu;
    d->omega_mid = d->sps; d->omega_limit = c->clock_omega_limit * d->sps; /* clock_recovery_mm.cpp:14-15 */
    d->mm_buf = calloc(STREAM_MAX + 64, sizeof(cf_t)); /* (+ 8 / 28 samples of history in front: M&M / Gardner) */
    /* the resampler may interpolate: up to ceil(n * I / D) + 1 outputs per input buffer */
    size_t wn = d->rs.active ? (size_t)((double)d->buffer_size * d->rs.interp / d->rs.decim) + 16 : (size_t)d->buffer_size;
    if (wn < (size_t)d->buffer_size) wn = d->buffer_size;
    d->w0 = malloc(sizeof(cf_t) * wn);
    d->w1 = malloc(sizeof(cf_t) * wn);
    d->w2 = malloc(sizeof(cf_t) * wn);
    return d;
}

void orc_demod_destroy(void *h)
{
    orc_demod *d = h;
    free(d->fir_buf); free(d->mm_buf); free(d->w0); free(d->w1); free(d->w2); free(d->rs.bank); free(d->rs.buffer); free(d->rs_in);
    for (int i = 0; i < d->rs.nstages; i++) free(d->rs.st[i].buffer);
    free(d->rs.tmp); free(d);
}
float orc_demod_sps(void *h) { return ((orc_demod *)h)->sps; }

void orc_demod_state(void *h, float *o)
{
    orc_demod *d = h;
    o[0] = d->agc_gain; o[1] = d->phase; o[2] = d->freq; o[3] = d->mu; o[4] = d->omega; o[5] = d->inc; o[6] = d->alpha; o[7] = d->beta;
}

/* baseband_interface.h:170-190 with the generic VOLK converters (divide by the scale) */
static void convert_in(const orc_demod_cfg *c, const void *raw, long off, int n, cf_t *dst)
{
    float *o = (float *)dst;
    if (c->format == 0) memcpy(dst, (const cf_t *)raw + off, n * sizeof(cf_t));
    else if (c->format == 1) { const int16_t *s = (const int16_t *)raw + off * 2; for (int i = 0; i < 2 * n; i++) o[i] = ((float)s[i]) / 32767.0f; }
    else { const int8_t *s = (const int8_t *)raw + off * 2; for (int i = 0; i < 2 * n; i++) o[i] = ((float)s[i]) / 127.0f; }
    if (c->iq_swap) /* file_source.cpp:31-33 */
        for (int i = 0; i < n; i++) { float t = dst[i].re; dst[i].re = dst[i].im; dst[i].im = t; }
}

/* reader + optional CorrectIQBlock<complex_t>::work (utils/correct_iq.cpp:18-35; alpha = 1e-4 member default, beta = 1 - alpha) */
void orc_rotator(const float *in, long n, long call, float inc_re, float inc_im, int imag_only, float *phase, float *out);
static void front_in(orc_demod *d, const void *raw, long off, int n, cf_t *dst)
{
    convert_in(&d->cfg, raw, off, n, dst);
    if (d->cfg.dc_block) {
        const float alpha = 0.0001, beta = 1.0f - alpha;
        for (int i = 0; i < n; i++) {
            d->dc_acc.re = d->dc_acc.re * beta + dst[i].re * alpha;
            d->dc_acc.im = d->dc_acc.im * beta + dst[i].im * alpha;
            dst[i].re = dst[i].re - d->dc_acc.re;
            dst[i].im = dst[i].im - d->dc_acc.im;
        }
    }
    if (d->cfg.freq_shift != 0 && n > 0) /* one rotator call per buffer (freq_shift.cpp:16-37); in place: sample k is read before it is written */
        orc_rotator((const float *)dst, n, n, d->fs_inc[0], d->fs_inc[1], 0, d->fs_phase, (float *)dst);
}

/* AGCBlock<complex_t>::work — agc.cpp:25-39. The magnitude goes through ::sqrt(double). */
static void agc_unit(const cf_t *in, cf_t *out, int n, float rate, float ref, float max_gain, float *gain)
{
    float g = *gain;
    for (int i = 0; i < n; i++) {
        cf_t o = {in[i].re * g, in[i].im * g};
        g += rate * (ref - sqrt(o.re * o.re + o.im * o.im));
        if (max_gain > 0.0 && g > max_gain) g = max_gain;
        out[i] = o;
    }
    *gain = g;
}
static void agc_run(orc_demod *d, const cf_t *in, cf_t *out, int n) { agc_unit(in, out, n, d->agc_rate, d->agc_ref, d->agc_max, &d->agc_gain); }

/* ================================================================== pm_demod / freq_shift blocks
 * fast_atan2f: 256-interval table of atan over [0, 1] with linear interpolation (common/dsp/utils/fast_trig.cpp:16-154). The table is
 * the arctangent of k/255 printed with seven significant digits (the reference lists those literals, taken from GNU Radio); it is
 * regenerated here from atan() through the same decimal rounding and pinned entry by entry through the function's outputs
 * (tests/test_oracle.py). Entry 256 repeats entry 255. */
static float fat_tab[257];
static int fat_ready;
static void fat_build(void)
{
    char buf[40];
    for (int k = 0; k < 256; k++) {
        snprintf(buf, sizeof buf, "%.6e", atan((double)k / 255.0));
        fat_tab[k] = (float)strtod(buf, NULL);
    }
    fat_tab[256] = fat_tab[255];
    fat_ready = 1;
}
const float *orc_fast_atan_table(void)
{
    if (!fat_ready)
        fat_build();
    return fat_tab;
}

float orc_fast_atan2f(float y, float x)
{
    if (!fat_ready)
        fat_build();
    const float ya = fabsf(y), xa = fabsf(x);
    if (!(ya > 0.0f || xa > 0.0f)) /* fast_trig.cpp:90-91 */
        return 0.0f;
    const float z = ya < xa ? ya / xa : xa / ya; /* :93-96 */
    float base;
    if ((double)z < 0.003921569) /* :100-101: below the table resolution the angle is the ratio itself */
        base = z;
    else { /* :104-111 */
        float a = z * 255.0f;
        const int idx = ((int)a) & 0xff;
        a -= (float)idx;
        base = fat_tab[idx];
        base += (fat_tab[idx + 1] - fat_tab[idx]) * a;
    }
    float ang;
    if (xa > ya) { /* :114-131 */
        if (x >= 0.0f)
            ang = y >= 0.0f ? base : -base;
        else {
            ang = (float)3.14159265358979323846;
            if (y >= 0.0f)
                ang -= base;
            else
                ang = base - ang;
        }
    } else { /* :132-151 */
        if (y >= 0.0f) {
            ang = (float)1.57079632679489661923;
            if (x >= 0.0f)
                ang -= base;
            else
                ang += base;
        } else {
            ang = (float)-1.57079632679489661923;
            if (x >= 0.0f)
                ang += base;
            else
                ang -= base;
        }
    }
    return ang;
}

/* even / odd minimax polynomials, the powers in float, the Horner sums in double, rounded once on return (fast_trig.cpp:158-180) */
float orc_fast_cos(float x)
{
    const float x2 = x * x, x4 = x2 * x2, x8 = x4 * x4;
    return (float)((-2.7236370439787708e-7 * x2 + 2.4799852696610628e-5) * x8 + (-1.3888885054799695e-3 * x2 + 4.1666666636943683e-2) * x4 +
                   (-4.9999999999963024e-1 * x2 + 1.0000000000000000e+0));
}
float orc_fast_sin(float x)
{
    const float x2 = x * x, x4 = x2 * x2;
    return (float)(((2.7181216275479732e-6 * x2 - 1.9839312269456257e-4) * x4 + (8.3333293048425631e-3 * x2 - 1.6666666640797048e-1)) * x2 * x + x);
}

void orc_pll_carrier(const float *in, long n, float loop_bw, float max_freq, float min_freq, float *state, float *out)
{
    /* gains: pll_carrier_tracking.cpp:17-21 (damping sqrt(2)/2, the same second-order design as the Costas loop) */
    const float damping = sqrtf(2.0f) / 2.0f;
    const float denom = (float)(1.0 + 2.0 * damping * loop_bw + loop_bw * loop_bw);
    const float alpha = (4 * damping * loop_bw) / denom, beta = (4 * loop_bw * loop_bw) / denom;
    float phase = state[0], freq = state[1];
    for (long i = 0; i < n; i++) {
        const float re = in[2 * i], im = in[2 * i + 1];
        const float vr = orc_fast_cos(phase), vi = -orc_fast_sin(phase); /* :38 */
        out[2 * i] = re * vr - im * vi;                                 /* :41, complex.h:68-72 */
        out[2 * i + 1] = im * vr + re * vi;
        float err = orc_fast_atan2f(im, re) - phase; /* :44 */
        while ((double)err < -M_PI)                   /* :45-48: compared and stepped in double, stored as float */
            err = (float)((double)err + 2 * M_PI);
        while ((double)err > M_PI)
            err = (float)((double)err - 2 * M_PI);
        freq = freq + beta * err; /* :51-55 */
        if (freq > max_freq)
            freq = max_freq;
        else if (freq < min_freq)
            freq = min_freq;
        phase = phase + freq + alpha * err; /* :58-62 */
        while ((double)phase < -M_PI)
            phase = (float)((double)phase + 2 * M_PI);
        while ((double)phase > M_PI)
            phase = (float)((double)phase - 2 * M_PI);
    }
    state[0] = phase;
    state[1] = freq;
}

void orc_rotator_inc(double freq, double samplerate, float *inc2)
{
    const double w = 2.0 * M_PI * (freq / samplerate); /* hz_to_rad, common/dsp/block.cpp:17 */
    inc2[0] = (float)cos(w);
    inc2[1] = (float)sin(w);
}

/* VOLK's rotator (system library, not vendored by the reference; generic flavour of 2.x / 3.x as published): the phasor advances by
 * one complex multiplication per sample and is brought back to unit length after every 512 samples of a call and at the end of a call
 * that is not a multiple of 512. Same arithmetic as oracle/shim/volk/volk.h, which the compiled reference blocks call. */
void orc_rotator(const float *in, long n, long call, float inc_re, float inc_im, int imag_only, float *phase, float *out)
{
    float pr = phase[0], pi = phase[1];
    for (long pos = 0; pos < n; pos += call) {
        const long m = n - pos < call ? n - pos : call;
        int since = 0;
        for (long k = pos; k < pos + m; k++) {
            const float a = imag_only ? 0.0f : in[2 * k], b = in[2 * k + 1];
            out[2 * k] = a * pr - b * pi;
            out[2 * k + 1] = a * pi + b * pr;
            const float nr = pr * inc_re - pi * inc_im, ni = pr * inc_im + pi * inc_re;
            pr = nr;
            pi = ni;
            if (++since == 512) {
                const float mag = hypotf(pr, pi);
                pr /= mag;
                pi /= mag;
                since = 0;
            }
        }
        if (since) {
            const float mag = hypotf(pr, pi);
            pr /= mag;
            pi /= mag;
        }
    }
    phase[0] = pr;
    phase[1] = pi;
}

/* The same recurrence evaluated in double precision (gain, product and magnitude): what agc.cpp:25-39 computes before its float
 * rounding. The distance of the reference's float output from this is the reference's own rounding noise (a random walk of the gain
 * with the loop's memory of ~100 * gain samples): the floor no other evaluation of the recurrence can get under. Test use only. */
void orc_agc_exact(const float *in, long n, double rate, double ref, double max_gain, float *out)
{
    double g = 1.0;
    for (long i = 0; i < n; i++) {
        const double re = (double)in[2 * i] * g, im = (double)in[2 * i + 1] * g;
        out[2 * i] = (float)re;
        out[2 * i + 1] = (float)im;
        g += rate * (ref - sqrt(re * re + im * im));
        if (max_gain > 0.0 && g > max_gain) g = max_gain;
    }
}

/* FIRBlock<complex_t>::work — fir.cpp:47-89; y[i] = sum_j buf[i+1+j] * taps[ntaps-1-j], oldest sample first */
static void fir_run(orc_demod *d, const cf_t *in, cf_t *out, int n)
{
    int nt = d->ntaps;
    memcpy(&d->fir_buf[nt], in, n * sizeof(cf_t));
    for (int i = 0; i < n; i++) {
        const cf_t *x = &d->fir_buf[i + 1];
        float ar = 0.0f, ai = 0.0f;
        for (int j = 0; j < nt; j++) {
            float h = d->taps[nt - 1 - j];
            ar += x[j].re * h;
            ai += x[j].im * h;
        }
        out[i].re = ar; out[i].im = ai;
    }
    memmove(&d->fir_buf[0], &d->fir_buf[n], nt * sizeof(cf_t));
}

/* CostasLoopBlock::work — costas_loop.cpp:23-65 */
static void costas_run(orc_demod *d, const cf_t *in, cf_t *out, int n)
{
    float phase = d->phase, freq = d->freq, err = 0;
    for (int i = 0; i < n; i++) {
        float cr = cosf(-phase), ci = sinf(-phase);
        cf_t v = {in[i].re * cr - in[i].im * ci, in[i].im * cr + in[i].re * ci};
        out[i] = v;
        if (d->order == 2) err = v.re * v.im;
        else if (d->order == 4) err = (v.re > 0.0f ? 1.0f : -1.0f) * v.im - (v.im > 0.0f ? 1.0f : -1.0f) * v.re;
        else {
            const float K = (sqrtf(2.0) - 1);
            if (fabsf(v.re) >= fabsf(v.im)) err = ((v.re > 0.0f ? 1.0f : -1.0f) * v.im - (v.im > 0.0f ? 1.0f : -1.0f) * v.re * K);
            else err = ((v.re > 0.0f ? 1.0f : -1.0f) * v.im * K - (v.im > 0.0f ? 1.0f : -1.0f) * v.re);
        }
        err = clip_branchless(err, 1.0);
        freq += d->beta * err;
        phase += freq + d->alpha * err;
        while (phase > (2 * M_PI)) phase -= 2 * M_PI;
        while (phase < (-2 * M_PI)) phase += 2 * M_PI;
        if (freq > d->fmax) freq = d->fmax;
        if (freq < d->fmin) freq = d->fmin;
    }
    d->phase = phase; d->freq = freq;
}

/* DelayOneImagBlock::work — delay_one_imag.cpp:18-25 (in place is fine going backwards) */
static void delay_run(orc_demod *d, cf_t *x, int n)
{
    float carry = x[n - 1].im;
    for (int i = n - 1; i > 0; i--) x[i].im = x[i - 1].im;
    x[0].im = d->last_imag;
    d->last_imag = carry;
}

/* MMClockRecoveryBlock<complex_t>::work — clock_recovery_mm.cpp:35-137 */
static int mm_run(orc_demod *d, const cf_t *in, cf_t *out, int n)
{
    cf_t *buf = d->mm_buf;
    memcpy(&buf[7], in, n * sizeof(cf_t));
    int ouc = 0, inc = d->inc;
    float mu = d->mu, omega = d->omega;
    for (; inc < n && ouc < STREAM_MAX;) {
        d->p2 = d->p1; d->p1 = d->p0; d->c2 = d->c1; d->c1 = d->c0;
        int imu = (int)rint(mu * 128);
        if (imu < 0) imu = 0;
        if (imu >= 128) imu = 127;
        const float *tp = &d->bank[imu * 8];
        float ar = 0.0f, ai = 0.0f;
        for (int k = 0; k < 8; k++) { ar += buf[inc + k].re * tp[k]; ai += buf[inc + k].im * tp[k]; }
        d->p0.re = ar; d->p0.im = ai;
        d->c0.re = ar > 0.0f ? 1.0f : 0.0f; d->c0.im = ai > 0.0f ? 1.0f : 0.0f;
        /* ((p0-p2)*conj(c1) - (c0-c2)*conj(p1)).real with complex_t float arithmetic (complex.h:74-78) */
        float a_r = d->p0.re - d->p2.re, a_i = d->p0.im - d->p2.im, b_i = -d->c1.im;
        float c_r = d->c0.re - d->c2.re, c_i = d->c0.im - d->c2.im, e_i = -d->p1.im;
        float x = (a_r * d->c1.re) - (a_i * b_i);
        float y = (c_r * d->p1.re) - (c_i * e_i);
        float pe = clip_branched(x - y, 1.0);
        out[ouc++] = d->p0;
        omega = omega + d->omega_gain * pe;
        omega = d->omega_mid + clip_branched((omega - d->omega_mid), d->omega_limit);
        mu = mu + omega + d->mu_gain * pe;
        inc += (int)floor(mu);
        mu -= floor(mu);
        if (inc < 0) inc = 0;
    }
    inc -= n;
    if (inc < 0) inc = 0;
    memmove(&buf[0], &buf[n], 8 * sizeof(cf_t));
    d->inc = inc; d->mu = mu; d->omega = omega;
    return ouc;
}

/* GardnerClockRecoveryBlock<complex_t>::work — clock_recovery_gardner.cpp:33-131. Same interpolator bank, omega / mu updates as M&M;
   the error is zc * (last - sample) with a second interpolation half a symbol back. History: ntaps - 1 + bufs (= 27) samples.
   BRANCHLESS_CLIP (block.h:10) is 0.5 * (abs(x + c) - abs(x - c)): with the double constant 1.0 the error clip is evaluated in double
   (exact), the omega clip in float for the two sums, double for the rest. */
static int gardner_run(orc_demod *d, const cf_t *in, cf_t *out, int n)
{
    const int bufs = 20;
    cf_t *buf = d->mm_buf;
    memcpy(&buf[7 + bufs], in, n * sizeof(cf_t));
    int ouc = 0, inc = d->inc;
    float mu = d->mu, omega = d->omega;
    for (; inc < n && ouc < STREAM_MAX;) {
        float muz = mu - (omega / 2.0);
        int offzc = floor(omega / 2.0);
        float mupos = fmod(muz + offzc, 1.0);
        if (mupos < 0) { mupos = 1 + mupos; offzc += 1; }
        int imuz = (int)rint(mupos * 128);
        if (imuz < 0) imuz = 0;
        if (imuz >= 128) imuz = 127;
        int imu = (int)rint(mu * 128);
        if (imu < 0) imu = 0;
        if (imu >= 128) imu = 127;
        const float *tz = &d->bank[imuz * 8], *tp = &d->bank[imu * 8];
        const cf_t *xz = &buf[inc - offzc + bufs], *xs = &buf[inc + bufs];
        float zr = 0.0f, zi = 0.0f, sr = 0.0f, si = 0.0f;
        for (int k = 0; k < 8; k++) { zr += xz[k].re * tz[k]; zi += xz[k].im * tz[k]; }
        for (int k = 0; k < 8; k++) { sr += xs[k].re * tp[k]; si += xs[k].im * tp[k]; }
        float pe = zr * (d->p0.re - sr) + zi * (d->p0.im - si); /* p0 = last_sample */
        pe = 0.5 * (fabs(pe + 1.0) - fabs(pe - 1.0));
        d->p0.re = sr; d->p0.im = si;
        out[ouc].re = sr; out[ouc].im = si; ouc++;
        omega = omega + d->omega_gain * pe;
        { float x = omega - d->omega_mid; omega = d->omega_mid + 0.5 * (fabsf(x + d->omega_limit) - fabsf(x - d->omega_limit)); }
        mu = mu + omega + d->mu_gain * pe;
        inc += (int)floor(mu);
        mu -= floor(mu);
        if (inc < 0) inc = 0;
    }
    inc -= n;
    if (inc < 0) inc = 0;
    memmove(&buf[0], &buf[n], (8 + bufs) * sizeof(cf_t));
    d->inc = inc; d->mu = mu; d->omega = omega;
    return ouc;
}

/* module_demod_base.h:106-113 */
static int8_t soft_clamp(float x)
{
    if (x < -128.0) return -127;
    if (x > 127.0) return 127;
    return (int8_t)x;
}

long orc_demod_run(void *h, const void *raw, long nsamples, float *agc_out, float *fir_out, float *costas_out, float *mm_out,
                   int8_t *soft_out, long sym_cap)
{
    orc_demod *d = h;
    long nsym = 0, pos = 0; /* pos: samples after the (optional) resampler so far in this call */
    d->pm_pos = 0;
    for (long off = 0; off < nsamples; off += d->buffer_size) {
        int n = (int)(nsamples - off < d->buffer_size ? nsamples - off : d->buffer_size);
        if (d->rs.active && !d->rs_after) {
            front_in(d, raw, off, n, d->rs_in);
            n = resamp_run(&d->rs, (const float *)d->rs_in, n, (float *)d->w0);
            if (n <= 0) continue;
        } else
            front_in(d, raw, off, n, d->w0);
        agc_run(d, d->w0, d->w1, n);
        if (agc_out) memcpy(agc_out + (d->cfg.pm ? d->pm_pos : pos) * 2, d->w1, n * sizeof(cf_t));
        if (d->cfg.pm) { /* module_pm_demod.cpp:65-74 */
            orc_pll_carrier((const float *)d->w1, n, d->cfg.pm_pll_bw, d->cfg.pm_pll_max_offset, -d->cfg.pm_pll_max_offset, d->pll_state, (float *)d->w0);
            if (d->pll_dump) memcpy(d->pll_dump + d->pm_pos * 2, d->w0, n * sizeof(cf_t));
            orc_rotator((const float *)d->w0, n, n, d->pm_inc[0], d->pm_inc[1], 1, d->pm_phase, (float *)d->w1); /* PMToBPSK: one call per buffer */
            if (d->pm_dump) memcpy(d->pm_dump + d->pm_pos * 2, d->w1, n * sizeof(cf_t));
            d->pm_pos += n;
            if (d->rs_after) {
                if (d->rs.active) {
                    memcpy(d->rs_in, d->w1, n * sizeof(cf_t));
                    n = resamp_run(&d->rs, (const float *)d->rs_in, n, (float *)d->w0);
                    if (n <= 0) continue;
                } else
                    memcpy(d->w0, d->w1, n * sizeof(cf_t));
                agc_unit(d->w0, d->w1, n, 0.001f, 1.0f, 1000.0f, &d->agc2_gain);
            }
        }
        fir_run(d, d->w1, d->w0, n);
        if (fir_out) memcpy(fir_out + pos * 2, d->w0, n * sizeof(cf_t));
        cf_t *cur = d->w0;
        if (d->order && d->cfg.has_carrier) { /* module_psk_demod.cpp:109-112: carrier PLL, then CorrectIQBlock, in front of the Costas loop */
            orc_pll_carrier((const float *)d->w0, n, d->cfg.carrier_pll_bw, d->cfg.carrier_pll_max_offset, -d->cfg.carrier_pll_max_offset, d->pll_state, (float *)d->w1);
            if (d->pll_dump) memcpy(d->pll_dump + pos * 2, d->w1, n * sizeof(cf_t));
            const float alpha = 0.0001, beta = 1.0f - alpha;
            for (int i = 0; i < n; i++) {
                d->dc_acc3.re = d->dc_acc3.re * beta + d->w1[i].re * alpha;
                d->dc_acc3.im = d->dc_acc3.im * beta + d->w1[i].im * alpha;
                d->w0[i].re = d->w1[i].re - d->dc_acc3.re;
                d->w0[i].im = d->w1[i].im - d->dc_acc3.im;
            }
            if (d->pm_dump) memcpy(d->pm_dump + pos * 2, d->w0, n * sizeof(cf_t));
        }
        if (d->order) {
            costas_run(d, d->w0, d->w1, n);
            cur = d->w1;
            if (d->cfg.post_costas_dc) { /* module_psk_demod.cpp:127-128, correct_iq.cpp:18-35 */
                const float alpha = 0.0001, beta = 1.0f - alpha;
                for (int i = 0; i < n; i++) {
                    d->dc_acc2.re = d->dc_acc2.re * beta + cur[i].re * alpha;
                    d->dc_acc2.im = d->dc_acc2.im * beta + cur[i].im * alpha;
                    cur[i].re = cur[i].re - d->dc_acc2.re;
                    cur[i].im = cur[i].im - d->dc_acc2.im;
                }
            }
            if (d->cfg.constellation == 2) delay_run(d, cur, n);
            if (costas_out) memcpy(costas_out + pos * 2, cur, n * sizeof(cf_t));
        }
        pos += n;
        int m = d->cfg.clock_recovery == 1 ? gardner_run(d, cur, d->w2, n) : mm_run(d, cur, d->w2, n);
        if (nsym + m > sym_cap) m = (int)(sym_cap - nsym);
        if (mm_out) memcpy(mm_out + nsym * 2, d->w2, m * sizeof(cf_t));
        if (soft_out) { /* module_psk_demod.cpp:199-213 */
            if (d->cfg.pm) /* module_pm_demod.cpp:141-144 */
                for (int i = 0; i < m; i++) soft_out[nsym + i] = soft_clamp(d->w2[i].re * 100);
            else if (d->cfg.constellation == 0)
                for (int i = 0; i < m; i++) soft_out[nsym + i] = soft_clamp(d->w2[i].re * 50);
            else
                for (int i = 0; i < m; i++) {
                    soft_out[(nsym + i) * 2] = soft_clamp(d->w2[i].re * 100);
                    soft_out[(nsym + i) * 2 + 1] = soft_clamp(d->w2[i].im * 100);
                }
        }
        nsym += m;
    }
    d->last_front = pos;
    return nsym;
}
long orc_demod_last_front(void *h) { return ((orc_demod *)h)->last_front; }
void orc_demod_pm_dumps(void *h, float *pll_out, float *pm_out) { orc_demod *d = h; d->pll_dump = pll_out; d->pm_dump = pm_out; }
void orc_demod_pm_state(void *h, float *o) { orc_demod *d = h; o[0] = d->pll_state[0]; o[1] = d->pll_state[1]; o[2] = d->cfg.pm && d->rs_after ? d->agc2_gain : 0; o[3] = 0; }
/* ONE stage of the chain on a caller-supplied cf32 input, in reference-sized buffers (stage-isolated parity tests): 1 = FIR,
   2 = Costas loop (+ post-Costas DC blocker / OQPSK delay: what the clock recovery reads), 5 = M&M. Returns the output count. */
long orc_demod_run_stage(void *h, int stage, const float *in, long nsamples, float *out, long cap)
{
    orc_demod *d = h;
    long pos = 0;
    if (stage == 2 && !d->order) return -1;
    for (long off = 0; off < nsamples; off += d->buffer_size) {
        int n = (int)(nsamples - off < d->buffer_size ? nsamples - off : d->buffer_size), m = n;
        memcpy(d->w0, in + off * 2, n * sizeof(cf_t));
        cf_t *res = d->w1;
        if (stage == 0)
            agc_run(d, d->w0, d->w1, n);
        else if (stage == 1)
            fir_run(d, d->w0, d->w1, n);
        else if (stage == 2) {
            costas_run(d, d->w0, d->w1, n);
            if (d->cfg.post_costas_dc) {
                const float alpha = 0.0001, beta = 1.0f - alpha;
                for (int i = 0; i < n; i++) {
                    d->dc_acc2.re = d->dc_acc2.re * beta + d->w1[i].re * alpha;
                    d->dc_acc2.im = d->dc_acc2.im * beta + d->w1[i].im * alpha;
                    d->w1[i].re = d->w1[i].re - d->dc_acc2.re;
                    d->w1[i].im = d->w1[i].im - d->dc_acc2.im;
                }
            }
            if (d->cfg.constellation == 2) delay_run(d, d->w1, n);
        } else {
            m = d->cfg.clock_recovery == 1 ? gardner_run(d, d->w0, d->w2, n) : mm_run(d, d->w0, d->w2, n);
            res = d->w2;
        }
        if (pos + m > cap) m = (int)(cap - pos);
        memcpy(out + pos * 2, res, m * sizeof(cf_t));
        pos += m;
    }
    return pos;
}


long orc_resample(const orc_demod_cfg *c, const void *raw, long nsamples, float *out, long cap)
{
    orc_demod *d = orc_demod_create(c);
    if (!d) return -1;
    long pos = 0;
    cf_t *in = malloc(sizeof(cf_t) * d->buffer_size);
    for (long off = 0; off < nsamples; off += d->buffer_size) {
        int n = (int)(nsamples - off < d->buffer_size ? nsamples - off : d->buffer_size);
        front_in(d, raw, off, n, in);
        int m = n;
        const float *src = (const float *)in;
        if (d->rs.active) { m = resamp_run(&d->rs, (const float *)in, n, (float *)d->w0); src = (const float *)d->w0; }
        if (pos + m > cap) m = (int)(cap - pos);
        memcpy(out + pos * 2, src, m * sizeof(cf_t));
        pos += m;
    }
    free(in);
    orc_demod_destroy(d);
    return pos;
}

/* ======================================================================= convolutional code k=7 r=1/2 */

static int parity32(unsigned x) { x ^= x >> 16; x ^= x >> 8; x ^= x >> 4; x ^= x >> 2; x ^= x >> 1; return x & 1; }

typedef struct
{
    int frame;            /* decoded bits per call */
    uint8_t branch[64];   /* cc_decoder.cpp:116-123: [j*32+i] = parity(2i & poly_j) ? 255 : 0 */
    uint8_t metric[2][64];
    uint32_t *dec;        /* (frame+6) x 2 words, bit s of row t = survivor choice of new state s */
} orc_ccdec;

static void ccdec_init(orc_ccdec *v, int frame)
{
    static const int polys[2] = {79, 109};
    v->frame = frame;
    for (int i = 0; i < 32; i++)
        for (int j = 0; j < 2; j++) v->branch[j * 32 + i] = parity32((2 * i) & polys[j]) ? 255 : 0;
    memset(v->metric[0], 31, 64); /* init_viterbi_unbiased, cc_decoder.cpp:177-190 */
    v->dec = malloc(sizeof(uint32_t) * 2 * (frame + 6));
}

/* CCDecoder::work(in,out) — cc_decoder.cpp:295-302 with the vendored generic ACS (volk_k7_r2_generic_fixed.h:80-163),
 * find_endstate :192-209, chainback_viterbi :228-276, init_viterbi :159-175. */
static void ccdec_work(orc_ccdec *v, const uint8_t *syms, uint8_t *out)
{
    int steps = v->frame + 6;
    uint8_t *X = v->metric[0], *Y = v->metric[1];
    memset(v->dec, 0, sizeof(uint32_t) * 2 * steps);
    for (int s = 0; s < steps; s++) {
        for (int i = 0; i < 32; i++) {
            unsigned sum = 1 + (v->branch[i] ^ syms[2 * s]) + (v->branch[32 + i] ^ syms[2 * s + 1]);
            uint8_t m = (sum >> 1) >> 2, mx = 63;
            uint8_t m0 = X[i] + m, m1 = X[i + 32] + (mx - m), m2 = X[i] + (mx - m), m3 = X[i + 32] + m;
            unsigned d0 = ((int)m0 - (int)m1) >= 0, d1 = ((int)m2 - (int)m3) >= 0;
            Y[2 * i] = d0 ? m1 : m0;
            Y[2 * i + 1] = d1 ? m3 : m2;
            v->dec[2 * s + i / 16] |= (d0 | d1 << 1) << ((2 * i) & 31);
        }
        uint8_t mn = Y[0];
        for (int i = 1; i < 64; i++) if (Y[i] < mn) mn = Y[i];
        for (int i = 0; i < 64; i++) Y[i] -= mn;
        uint8_t *t = X; X = Y; Y = t;
    }
    /* steps is even for every frame size on the path, so the newest metrics are back in metric[0] (= "old_metrics") */
    const uint8_t *met = (steps % 2 == 0) ? v->metric[0] : v->metric[1];
    int state = 0;
    for (int i = 1; i < 64; i++) if (met[i] < met[state]) state = i;
    int next_start = 0;
    for (int row = steps - 1, k = 0; row >= 6; row--, k++) {
        int bit = (v->dec[2 * row + state / 32] >> (state % 32)) & 1;
        state = (state >> 1) | (bit << 5);
        out[row - 6] = bit;
        if (k == 5) next_start = state;
    }
    memset(v->metric[0], 63, 64);
    v->metric[0][next_start & 63] = 0;
}

typedef struct { unsigned state; } orc_ccenc;
/* CCEncoder::work — cc_encoder.cpp:92-104 (register carried across calls) */
static void ccenc_work(orc_ccenc *e, const uint8_t *in, int n, uint8_t *out)
{
    unsigned st = e->state;
    for (int i = 0; i < n; i++) {
        st = (st << 1) | (in[i] & 1);
        out[2 * i] = parity32(st & 79);
        out[2 * i + 1] = parity32(st & 109);
    }
    e->state = st;
}

void orc_cc_decode(const uint8_t *syms, int frame, int ncalls, uint8_t *out_bits)
{
    orc_ccdec v; ccdec_init(&v, frame);
    for (int c = 0; c < ncalls; c++) ccdec_work(&v, syms + (long)c * 2 * frame, out_bits + (long)c * frame);
    free(v.dec);
}
void orc_cc_encode(const uint8_t *bits, int n, uint8_t *out) { orc_ccenc e = {0}; ccenc_work(&e, bits, n, out); }

/* rotate_soft — common/codings/rotation.cpp:4-63 */
void orc_rotate_soft(int8_t *s, int size, int phase, int iqswap)
{
    for (int i = 0; i < size; i++) if (s[i] == -128) s[i] = -127;
    if (iqswap) for (int i = 0; i + 1 < size + 1 && i < size; i += 2) { int8_t t = s[i + 1]; s[i + 1] = s[i]; s[i] = t; }
    if (phase == 1) for (int i = 0; i < size; i += 2) { int8_t t = s[i]; s[i] = s[i + 1]; s[i + 1] = -t; }
    else if (phase == 2) for (int i = 0; i < size; i++) s[i] = -s[i];
    else if (phase == 3) for (int i = 0; i < size; i += 2) { int8_t t = s[i]; s[i] = -s[i + 1]; s[i + 1] = t; }
}
/* signed_soft_to_unsigned — common/codings/viterbi/utils.cpp:3-11 */
static void soft_to_u8(const int8_t *in, uint8_t *out, int n)
{
    for (int i = 0; i < n; i++) { out[i] = in[i] + 127; if (out[i] == 128) out[i] = 127; }
}
/* Viterbi3_4::depuncture, MetOp branch — viterbi_3_4.cpp:84-104 */
static int depunc34(const uint8_t *in, uint8_t *out, int size, int shift)
{
    int o = 0;
    for (int i = 0; i < size / 2; i++) {
        if (shift ^ (i % 2 == 0)) { out[o++] = in[2 * i]; out[o++] = in[2 * i + 1]; }
        else { out[o++] = 128; out[o++] = in[2 * i + 1]; out[o++] = in[2 * i]; out[o++] = 128; }
    }
    return o;
}
/* get_ber — viterbi_3_4.cpp:36-49 / viterbi_1_2.cpp:36-49 */
static float ber_of(const uint8_t *raw, const uint8_t *renc, int len, float k)
{
    float errors = 0, total = 0;
    for (int i = 0; i < len; i++) if (raw[i] != 128) { errors += (raw[i] > 127) != renc[i]; total++; }
    return (errors / total) * k;
}

#define TESTLEN 2048 /* TEST_BITS_LENGTH, viterbi_3_4.h:3 */

typedef struct
{
    int rate34, size, state, phase, shift, swap, invalid, outsync, check_swap, nphases, phases[4];
    float thr, ber, bers[2][4][2];
    orc_ccdec dec_ber, dec_main;
    orc_ccenc enc_ber;
    /* BER scratch laid out like the reference members so that the r=1/2 tail over-read lands in the decoded buffer
     * (viterbi_1_2.h:37-40); the r=3/4 tail bytes are never written in the reference (viterbi_3_4.h:38) -> zeros here */
    int8_t test[TESTLEN];
    uint8_t bsoft[TESTLEN], bdecoded[TESTLEN * 2], bencoded[TESTLEN * 2], bdepunc[TESTLEN * 2];
    uint8_t *soft, *depunc;
} orc_vit;

static void vit_init(orc_vit *v, int rate34, float thr, int outsync, int size, const int *phases, int nphases, int check_swap)
{
    memset(v, 0, sizeof(*v));
    v->rate34 = rate34; v->thr = thr; v->outsync = outsync; v->size = size; v->check_swap = check_swap;
    v->nphases = nphases; memcpy(v->phases, phases, sizeof(int) * nphases);
    ccdec_init(&v->dec_ber, rate34 ? TESTLEN * 3 / 4 : TESTLEN / 2);
    ccdec_init(&v->dec_main, rate34 ? size * 3 / 4 : size / 2);
    v->soft = malloc(size * 2); v->depunc = malloc(size * 2);
    for (int s = 0; s < 2; s++) for (int p = 0; p < 4; p++) for (int o = 0; o < 2; o++) v->bers[s][p][o] = 10;
}
static void vit_free(orc_vit *v) { free(v->dec_ber.dec); free(v->dec_main.dec); free(v->soft); free(v->depunc); }

static float vit_ber(const orc_vit *v)
{
    if (v->state) return v->ber;
    float b = 10;
    for (int s = 0; s < (v->check_swap ? 2 : 1); s++)
        for (int pi = 0; pi < v->nphases; pi++)
            for (int o = 0; o < 2; o++) if (b > v->bers[s][v->phases[pi]][o]) b = v->bers[s][v->phases[pi]][o];
    return b;
}

/* Viterbi3_4::work — viterbi_3_4.cpp:110-173 ; Viterbi1_2::work — viterbi_1_2.cpp:52-116. `in` is modified in place. */
static int vit_work(orc_vit *v, int8_t *in, uint8_t *out)
{
    int size = v->size;
    if (!v->state) {
        v->ber = 10;
        for (int s = 0; s < (v->check_swap ? 2 : 1); s++)
            for (int pi = 0; pi < v->nphases; pi++) {
                int ph = v->phases[pi];
                memcpy(v->test, in, TESTLEN);
                if (!v->rate34) orc_rotate_soft(v->test, TESTLEN, 0, s);
                orc_rotate_soft(v->test, TESTLEN, ph, 0);
                soft_to_u8(v->test, v->bsoft, TESTLEN);
                for (int shift = 0; shift < 2; shift++) {
                    float b;
                    if (v->rate34) {
                        depunc34(v->bsoft, v->bdepunc, TESTLEN, shift);
                        ccdec_work(&v->dec_ber, v->bdepunc, v->bdecoded);
                        ccenc_work(&v->enc_ber, v->bdecoded, TESTLEN * 3 / 4, v->bencoded);
                        b = ber_of(v->bdepunc, v->bencoded, TESTLEN * 3 / 2, 5);
                    } else {
                        ccdec_work(&v->dec_ber, v->bsoft + shift, v->bdecoded);
                        ccenc_work(&v->enc_ber, v->bdecoded, TESTLEN / 2, v->bencoded);
                        b = ber_of(v->bsoft + shift, v->bencoded, TESTLEN, 2.5);
                    }
                    v->bers[s][ph][shift] = b;
                    if ((v->ber == 10 && b < v->thr) || (v->ber < 10 && b < v->ber)) {
                        v->ber = b; v->swap = s; v->state = 1; v->phase = ph; v->shift = shift; v->invalid = 0;
                        memset(v->soft, 128, size * 2);
                        if (v->rate34) memset(v->depunc, 128, size * 2);
                    }
                }
            }
    }
    int out_n = 0;
    if (v->state) {
        if (!v->rate34) orc_rotate_soft(in, size, 0, v->swap);
        orc_rotate_soft(in, size, v->phase, 0);
        soft_to_u8(in, v->soft, size);
        if (v->rate34) {
            depunc34(v->soft, v->depunc, size, v->shift);
            ccdec_work(&v->dec_main, v->depunc, out);
            out_n = (size * 1.5) / 2;
            ccenc_work(&v->enc_ber, out, TESTLEN * 3 / 4, v->bencoded);
            v->ber = ber_of(v->depunc, v->bencoded, TESTLEN * 3 / 2, 5);
        } else {
            ccdec_work(&v->dec_main, v->soft + v->shift, out);
            out_n = size / 2;
            ccenc_work(&v->enc_ber, out, TESTLEN / 2, v->bencoded);
            v->ber = ber_of(v->soft + v->shift, v->bencoded, TESTLEN, 2.5);
        }
        if (v->ber > v->thr) { v->invalid++; if (v->invalid > v->outsync) v->state = 0; }
        else v->invalid = 0;
    }
    return out_n;
}

/* ======================================================================= Viterbi_Depunc (rates 2/3, 3/4, 5/6, 7/8)
 * viterbi_punc.cpp:53-145 + depunc.h. One table per rate: for every input position of the puncturing period, how many symbols it
 * makes (1 or 2) and where the data symbol sits among them (the other one is the erasure 128). */
typedef struct { int period, numstates; float berscale; uint8_t nout[8], datapos[8]; } orc_punc;
static const orc_punc PUNC_23 = {3, 3, 3.5f, {1, 2, 1}, {0, 0, 0}};
static const orc_punc PUNC_34 = {4, 4, 5.0f, {1, 2, 1, 2}, {0, 0, 0, 0}};
static const orc_punc PUNC_56 = {6, 6, 8.0f, {1, 2, 1, 2, 2, 2}, {0, 0, 0, 0, 1, 0}};
static const orc_punc PUNC_78 = {8, 8, 10.0f, {1, 2, 2, 2, 1, 2, 2, 2}, {0, 0, 0, 0, 0, 0, 1, 0}};

static int punc_emit(const orc_punc *p, int phase, uint8_t v, uint8_t *out, int oo)
{
    if (p->nout[phase] == 1) out[oo++] = v;
    else if (p->datapos[phase] == 0) { out[oo++] = v; out[oo++] = 128; }
    else { out[oo++] = 128; out[oo++] = v; }
    return oo;
}
/* DepuncXX::depunc_static */
static int punc_static(const orc_punc *p, const uint8_t *in, uint8_t *out, int size, int shift)
{
    int oo = 0, a = shift % p->period;
    if (shift > p->period - 1) out[oo++] = 128;
    for (int i = 0; i < size; i++) oo = punc_emit(p, (i + a) % p->period, in[i], out, oo);
    return oo;
}
typedef struct
{
    const orc_punc *p;
    int is_first, changing_shift, got_extra; /* DepuncXX members */
    uint8_t buf;
    int size, vit_bufsize, in_buffer, state, phase, shift, swap, invalid, outsync, check_swap, nphases, phases[4], test_bit_len;
    float thr, ber;
    orc_ccdec dec_ber, dec_main;
    orc_ccenc enc_ber;
    int8_t test[TESTLEN];
    uint8_t bsoft[TESTLEN], bdepunc[TESTLEN * 4], bdecoded[TESTLEN * 4], bencoded[TESTLEN * 4]; /* (zeroed: the oracle's pin of reads before writes) */
    uint8_t *soft, *depunc, *vitbuf;
} orc_vitp;

static void vitp_init(orc_vitp *v, int conv_rate, float thr, int outsync, int size, const int *phases, int nphases, int check_swap)
{
    memset(v, 0, sizeof(*v));
    v->p = conv_rate == 2 ? &PUNC_23 : (conv_rate == 3 ? &PUNC_34 : (conv_rate == 5 ? &PUNC_56 : &PUNC_78));
    v->buf = 128;
    v->thr = thr; v->outsync = outsync; v->size = size; v->vit_bufsize = size; v->check_swap = check_swap;
    v->nphases = nphases; memcpy(v->phases, phases, sizeof(int) * nphases);
    ccdec_init(&v->dec_ber, TESTLEN);
    ccdec_init(&v->dec_main, size / 2);
    v->soft = malloc((size_t)size * 8); v->depunc = malloc((size_t)size * 8); v->vitbuf = calloc((size_t)size * 4, 1);
}
static void vitp_free(orc_vitp *v) { free(v->dec_ber.dec); free(v->dec_main.dec); free(v->soft); free(v->depunc); free(v->vitbuf); }

/* DepuncXX::depunc_cont */
static int punc_cont(orc_vitp *v, const uint8_t *in, uint8_t *out, int size)
{
    int oo = 0;
    if (v->is_first || v->got_extra) { out[oo++] = v->buf; v->is_first = 0; v->got_extra = 0; }
    v->changing_shift %= v->p->period;
    for (int i = 0; i < size; i++) { oo = punc_emit(v->p, v->changing_shift % v->p->period, in[i], out, oo); v->changing_shift++; }
    if (oo % 2 == 1) { v->buf = out[oo - 1]; oo -= 1; v->got_extra = 1; }
    return oo;
}

/* Viterbi_Depunc::work. `in` is modified in place. The deprecated CCDecoder::work(in, out, size) the lock search calls ignores its
 * size (cc_decoder.cpp:304-314): it decodes the full TEST_BITS_LENGTH frame from 2 * 2054 symbols of the test buffer. */
static int vitp_work(orc_vitp *v, int8_t *in, uint8_t *out)
{
    int size = v->size;
    if (!v->state) {
        v->ber = 10;
        for (int s = 0; s < (v->check_swap ? 2 : 1); s++)
            for (int pi = 0; pi < v->nphases; pi++) {
                int ph = v->phases[pi];
                memcpy(v->test, in, TESTLEN);
                orc_rotate_soft(v->test, TESTLEN, 0, s);
                orc_rotate_soft(v->test, TESTLEN, ph, 0);
                soft_to_u8(v->test, v->bsoft, TESTLEN);
                for (int shift = 0; shift < v->p->numstates * 2; shift++) {
                    int lenp = punc_static(v->p, v->bsoft, v->bdepunc, TESTLEN, shift);
                    if (lenp % 2) lenp--;
                    ccdec_work(&v->dec_ber, v->bdepunc, v->bdecoded);
                    ccenc_work(&v->enc_ber, v->bdecoded, lenp / 2, v->bencoded);
                    v->test_bit_len = lenp;
                    float b = ber_of(v->bdepunc, v->bencoded, lenp, v->p->berscale);
                    if (b < v->thr && b < v->ber) {
                        v->ber = b; v->swap = s; v->state = 1; v->phase = ph; v->shift = shift; v->invalid = 0;
                        v->changing_shift = shift; v->is_first = shift > v->p->period - 1; /* set_shift */
                        memset(v->soft, 128, (size_t)size * 4);
                        memset(v->depunc, 128, (size_t)size * 4);
                    }
                }
            }
    }
    int out_n = 0;
    if (v->state) {
        orc_rotate_soft(in, size, 0, v->swap);
        orc_rotate_soft(in, size, v->phase, 0);
        soft_to_u8(in, v->soft, size);
        int sz = punc_cont(v, v->soft, v->depunc, size);
        memcpy(&v->vitbuf[v->in_buffer], v->depunc, sz); /* ViterbiSlidingBuffer::add */
        v->in_buffer += sz;
        while (v->in_buffer > v->vit_bufsize) {
            ccdec_work(&v->dec_main, v->vitbuf, out + out_n);
            ccenc_work(&v->enc_ber, out + out_n, TESTLEN, v->bencoded);
            v->ber = ber_of(v->vitbuf, v->bencoded, v->test_bit_len, 5);
            out_n += v->vit_bufsize / 2;
            int len = v->vit_bufsize; /* ViterbiSlidingBuffer::del */
            memmove(v->vitbuf, v->vitbuf + len, v->in_buffer - len);
            v->in_buffer -= len;
            memset(v->vitbuf + v->in_buffer, 128, len > 100 ? 100 : len);
        }
        if (v->ber > v->thr) { v->invalid++; if (v->invalid > v->outsync) v->state = 0; }
        else v->invalid = 0;
    }
    return out_n;
}

/* ======================================================================= deframer */

typedef struct
{
    uint32_t sync, sync_inv, shifter;
    int cadu_size, pad, st_nosync, st_syncing, st_synced;
    int state, in_frame, inversion, bit_of_frame, bad, good;
    uint8_t *frame;
} orc_deframer;

static void defr_init(orc_deframer *f, int cadu_size, uint32_t sync)
{
    memset(f, 0, sizeof(*f));
    f->sync = sync; f->sync_inv = ~sync; f->cadu_size = cadu_size;
    f->st_nosync = 2; f->st_syncing = 6; f->st_synced = 12; /* bpsk_ccsds_deframer.h:34-36 */
    f->state = 2;
    f->frame = calloc(cadu_size + 64, 1); /* the reference sizes it in bits-as-bytes, .cpp:11 */
}
static int popc32(uint32_t v) { int c = 0; for (; v; c++) v &= v - 1; return c; }
static void defr_new_frame(orc_deframer *f)
{
    memset(f->frame, 0, (f->cadu_size + f->pad) / 8);
    f->frame[0] = f->sync >> 24; f->frame[1] = f->sync >> 16; f->frame[2] = f->sync >> 8; f->frame[3] = f->sync;
    f->bit_of_frame = 32; f->in_frame = 1;
}
/* BPSK_CCSDS_Deframer::work — bpsk_ccsds_deframer.cpp:24-107 */
static int defr_work(orc_deframer *f, const uint8_t *in, int n, uint8_t *out)
{
    int nfr = 0, fbytes = (f->cadu_size + f->pad) / 8;
    for (int i = 0; i < n; i++) {
        f->shifter = f->shifter << 1 | in[i];
        if (f->in_frame) {
            int b = in[i] ^ f->inversion;
            f->frame[f->bit_of_frame / 8] = f->frame[f->bit_of_frame / 8] << 1 | b;
            f->bit_of_frame++;
            if (f->bit_of_frame == f->cadu_size) memcpy(out + (size_t)(nfr++) * fbytes, f->frame, fbytes);
            else if (f->bit_of_frame == f->cadu_size + 32 - 1) f->in_frame = 0;
            continue;
        }
        if (f->state == f->st_nosync) {
            int hit = f->shifter == f->sync ? 1 : (f->shifter == f->sync_inv ? 2 : 0);
            if (hit) { f->inversion = hit == 2; defr_new_frame(f); f->state = f->st_syncing; f->good = f->bad = 0; }
        } else if (f->state == f->st_syncing) {
            if (popc32(f->shifter ^ (f->inversion ? f->sync_inv : f->sync)) < f->state) {
                defr_new_frame(f); f->bad = 0; f->good++;
                if (f->good > 10) f->state = f->st_synced;
            } else { f->bad++; f->good = 0; if (f->bad > 2) f->state = f->st_nosync; }
        } else if (f->state == f->st_synced) {
            if (popc32(f->shifter ^ (f->inversion ? f->sync_inv : f->sync)) < f->state) defr_new_frame(f);
            else { f->good = f->bad = 0; f->state = f->st_nosync; }
        }
    }
    return nfr;
}

int orc_deframe(const uint8_t *bits, int nbits, int cadu_size, int state_synced, uint8_t *out)
{
    orc_deframer f; defr_init(&f, cadu_size, 0x1ACFFC1D); f.st_synced = state_synced;
    int total = 0;
    for (int off = 0; off < nbits; off += 8192) {
        int n = nbits - off < 8192 ? nbits - off : 8192;
        total += defr_work(&f, bits + off, n, out + (size_t)total * (cadu_size / 8));
    }
    free(f.frame);
    return total;
}

/* ======================================================================= CCSDS randomiser */

static uint8_t g_pn[255];
static void pn_init(void)
{   /* h(x) = x^8+x^7+x^5+x^3+1 from all ones; byte table equals ccsds_pn[] of randomization.cpp:4-36 */
    if (g_pn[0]) return;
    uint8_t r = 0xFF;
    for (int i = 0; i < 255; i++) {
        uint8_t b = 0;
        for (int k = 0; k < 8; k++) {
            b = (b << 1) | (r >> 7);
            uint8_t nb = ((r >> 7) ^ (r >> 4) ^ (r >> 2) ^ r) & 1;
            r = (r << 1) | nb;
        }
        g_pn[i] = b;
    }
}
/* derand_ccsds — randomization.cpp:72-78 */
void orc_derand(uint8_t *data, int len) { pn_init(); for (int i = 0; i < len; i++) data[i] ^= g_pn[i % 255]; }

/* ======================================================================= Reed-Solomon (libcorrect semantics) */

static uint8_t gexp[512], glog[256], to_dual[256], from_dual[256];
static int gf_ready;
static void gf_init(void)
{   /* field_create — libs/correct/reed-solomon/field.h:26-62: log[1] ends up 255, log[0] = 0 sentinel */
    if (gf_ready) return;
    unsigned e = 1;
    gexp[0] = 1; glog[0] = 0;
    for (int i = 1; i < 512; i++) {
        e <<= 1;
        if (e > 255) e ^= 0x187;
        gexp[i] = e;
        if (i < 256) glog[e] = i;
    }
    /* CCSDS dual basis <-> conventional: GF(2)-linear, images of the unit vectors (tables reedsolomon.cpp:6-28) */
    static const uint8_t img[8] = {0x7B, 0xAF, 0x99, 0xFA, 0x86, 0xEC, 0xEF, 0x8D};
    for (int v = 0; v < 256; v++) {
        uint8_t r = 0;
        for (int b = 0; b < 8; b++) if (v >> b & 1) r ^= img[b];
        to_dual[v] = r;
    }
    for (int v = 0; v < 256; v++) from_dual[to_dual[v]] = v;
    gf_ready = 1;
}
static uint8_t gmul(uint8_t a, uint8_t b) { return (!a || !b) ? 0 : gexp[glog[a] + glog[b]]; }
static uint8_t gdiv(uint8_t a, uint8_t b) { return (!a || !b) ? 0 : gexp[255 + glog[a] - glog[b]]; }
static uint8_t gpow(uint8_t a, int p) { int m = (glog[a] * p) % 255; if (m < 0) m += 255; return gexp[m]; }
static uint8_t logmul(uint8_t a, uint8_t b) { unsigned r = a + b; return r > 255 ? r - 255 : r; } /* field_mul_log */

/* correct_reed_solomon_decode — libs/correct/reed-solomon/decode.c:299-379 for (255, 255-nroots), fcr, gap 11.
 * Returns -1 on failure, else 0 with the corrected message in msg[0..k). */
static int rs_decode_block(const uint8_t *enc, int nroots, int fcr, uint8_t *msg)
{
    const int gap = 11, k = 255 - nroots;
    uint8_t r[255], syn[64], lam[66], prev[66], lamlog[66];
    for (int i = 0; i < 255; i++) r[i] = enc[254 - i];
    /* syndromes: decode.c:12-28 with generator_root_exp from polynomial_build_exp_lut (polynomial.c:159-171) */
    int allz = 1;
    for (int j = 0; j < nroots; j++) {
        uint8_t rootlog = glog[gexp[(gap * (j + fcr)) % 255]], pw = glog[1], s = 0;
        for (int i = 0; i < 255; i++) {
            if (r[i]) s ^= gexp[glog[r[i]] + pw];
            pw = logmul(pw, rootlog);
        }
        syn[j] = s;
        if (s) allz = 0;
    }
    if (allz) { for (int i = 0; i < k; i++) msg[i] = r[254 - i]; return 0; }
    /* Berlekamp-Massey: decode.c:32-118 */
    memset(lam, 0, sizeof(lam)); memset(prev, 0, sizeof(prev));
    lam[0] = prev[0] = 1;
    unsigned L = 0, order = 0, prev_order = 0, delay = 1;
    uint8_t last_d = 1;
    for (unsigned i = 0; i < (unsigned)nroots; i++) {
        uint8_t d = syn[i];
        for (unsigned j = 1; j <= L; j++) d ^= gmul(lam[j], syn[i - j]);
        if (!d) { delay++; continue; }
        if (2 * L <= i) {
            for (int j = prev_order; j >= 0; j--) prev[j + delay] = gdiv(gmul(prev[j], d), last_d);
            for (int j = delay - 1; j >= 0; j--) prev[j] = 0;
            for (unsigned j = 0; j <= prev_order + delay; j++) { uint8_t t = lam[j]; lam[j] ^= prev[j]; prev[j] = t; }
            unsigned t = order; order = prev_order + delay; prev_order = t;
            L = i + 1 - L; last_d = d; delay = 1;
            continue;
        }
        for (int j = prev_order; j >= 0; j--) lam[j + delay] ^= gdiv(gmul(prev[j], d), last_d);
        if (prev_order + delay > order) order = prev_order + delay;
        delay++;
    }
    /* Chien search over all 256 elements: decode.c:122-145, polynomial_eval_log_lut (polynomial.c:137-157) */
    for (unsigned i = 0; i <= order; i++) lamlog[i] = glog[lam[i]];
    uint8_t roots[64]; unsigned nr = 0;
    for (int e = 0; e < 256; e++) {
        uint8_t v;
        if (e == 0) v = lamlog[0] ? gexp[lamlog[0]] : 0;
        else {
            uint8_t el = glog[e], pw = glog[1];
            v = 0;
            for (unsigned i = 0; i <= order; i++) { if (lamlog[i]) v ^= gexp[lamlog[i] + pw]; pw = logmul(pw, el); }
        }
        if (!v) { if (nr < 64) roots[nr] = e; nr++; }
    }
    if (nr != order) return -1;
    /* error evaluator / derivative / Forney: decode.c:149-196 ; locations: decode.c:198-222 */
    uint8_t om[32], der[66];
    memset(om, 0, sizeof(om));
    for (unsigned i = 0; i <= order; i++) {
        if (i > (unsigned)nroots - 1) continue;
        unsigned jl = nroots - 1 - i;
        for (unsigned j = 0; j <= jl; j++) om[i + j] ^= gmul(lam[i], syn[j]);
    }
    for (unsigned i = 0; i + 1 <= order; i++) der[i] = ((i + 1) % 2) ? lam[i + 1] : 0;
    for (unsigned q = 0; q < order; q++) {
        uint8_t root = roots[q];
        if (root == 0) continue;
        uint8_t locv = gdiv(1, root), loc = 0;
        for (int j = 0; j < 256; j++) if (gpow(j, gap) == locv) { loc = glog[j]; break; }
        uint8_t el = glog[root], pw = glog[1], num = 0, den = 0;
        for (int i = 0; i < nroots; i++) { if (om[i]) num ^= gexp[glog[om[i]] + pw]; pw = logmul(pw, el); }
        pw = glog[1];
        for (unsigned i = 0; i + 1 <= order; i++) { if (der[i]) den ^= gexp[glog[der[i]] + pw]; pw = logmul(pw, el); }
        r[loc] ^= gmul(gpow(root, fcr - 1), gdiv(num, den));
    }
    for (int i = 0; i < k; i++) msg[i] = r[254 - i];
    return 0;
}

/* ReedSolomon::decode — common/codings/reedsolomon/reedsolomon.cpp:63-116 (fill_bytes <= 0 only: no shortening). *odata0: the first
 * byte of the decoder's message buffer, which the decoder overwrites with the corrected first message byte (conventional basis) when
 * the word decodes and leaves alone when it does not (decode.c:337-339,361,375) */
static int rs_decode_cw(uint8_t *data, int dual, int rs_type, uint8_t *odata0)
{
    gf_init();
    int nroots = rs_type == 1 ? 16 : 32, fcr = rs_type == 1 ? 120 : 112, k = 255 - nroots;
    uint8_t msg[255];
    if (dual) for (int i = 0; i < 255; i++) data[i] = from_dual[data[i]];
    int rc = rs_decode_block(data, nroots, fcr, msg), err = -1;
    if (rc == 0) {
        err = 0;
        for (int i = 0; i < k; i++) if (data[i] != msg[i]) err++;
        memcpy(data, msg, k); /* only the message bytes are replaced; parity stays as received */
        *odata0 = msg[0];
    }
    if (dual) for (int i = 0; i < 255; i++) data[i] = to_dual[data[i]];
    return err;
}
/* ReedSolomon::decode_interlaved — reedsolomon.cpp:53-61,145-155. The (de)interleave loops run 255 - fill_bytes rows: with fill_bytes
 * -1 (the decoder modules' default) that is 256, one row past the codewords. The extra byte of codeword b, data[255 * interleave + b],
 * lands one past the 255-byte deinterleave buffer, in the first byte of the message buffer that follows it (reedsolomon.h:24-25), and is
 * written back from there after the decode: the corrected first message byte when the word decodes, the byte as read when it does not.
 * Callers keep `interleave` bytes of room behind the codewords. */
void orc_rs_decode_interleaved(uint8_t *data, int dual, int interleave, int rs_type, int fill_bytes, int *errors)
{
    uint8_t cw[255];
    for (int b = 0; b < interleave; b++) {
        for (int i = 0; i < 255; i++) cw[i] = data[i * interleave + b];
        uint8_t odata0 = fill_bytes == -1 ? data[255 * interleave + b] : 0;
        errors[b] = rs_decode_cw(cw, dual, rs_type, &odata0);
        for (int i = 0; i < 255; i++) data[i * interleave + b] = cw[i];
        if (fill_bytes == -1) data[255 * interleave + b] = odata0;
    }
}

/* ======================================================================= decoder modules */

typedef struct
{
    orc_fec_cfg cfg;
    int chunk, cadu_bytes, nosync_runs, errors[16];
    orc_vit vit;
    orc_vitp vitp; /* conv_rate != 0: Viterbi_Depunc instead of Viterbi1_2 */
    orc_deframer defr, defr_qpsk; /* defr_qpsk: the second deframer of ccsds_simple_psk_decoder (QPSK without NRZ-M) */
    uint8_t nrzm_last;
    uint8_t *vout, *frames;
    int8_t *soft;
    /* ccsds_simple_psk_decoder: oqpsk_delay register, QPSKDiff state (differential/qpsk_diff.h: buffer[2], inBuf) */
    int8_t last_q_oqpsk;
    uint8_t qd_buf[2];
    int qd_in;
} orc_fec;

void *orc_fec_create(const orc_fec_cfg *c)
{
    orc_fec *f = calloc(1, sizeof(*f));
    f->cfg = *c;
    if (c->kind == 0) { /* module_metop_ahrpt_decoder.cpp:17-25 */
        int ph[2] = {0, 1};
        f->chunk = 16384; f->cadu_bytes = 1024;
        vit_init(&f->vit, 1, c->ber_thresold, c->outsync_after, f->chunk, ph, 2, 0);
        defr_init(&f->defr, 8192, 0x1ACFFC1D);
        f->defr.st_synced = 18;
    } else if (c->kind == 2) { /* module_ccsds_simple_psk_decoder.cpp:19-98 */
        f->chunk = c->cadu_size;
        f->cadu_bytes = (c->cadu_size + 7) / 8;
        defr_init(&f->defr, c->cadu_size, c->asm_sync);
        defr_init(&f->defr_qpsk, c->cadu_size, c->asm_sync);
        f->defr.pad = f->defr_qpsk.pad = c->cadu_size % 8;
        f->vout = calloc(1, f->chunk * 8); f->frames = malloc(f->chunk * 8 + 10240); f->soft = malloc(f->chunk);
        return f;
    } else { /* module_ccsds_conv_concat_decoder.cpp:16-131 */
        int ph[2] = {0, 1}, n = 2;
        if (c->constellation == 0) { ph[0] = 0; n = 1; }
        else if (c->constellation == 5) { ph[0] = 1; n = 1; }
        f->chunk = c->cadu_size > 8192 ? c->cadu_size : 8192;
        f->cadu_bytes = (c->cadu_size + 7) / 8;
        if (c->conv_rate) vitp_init(&f->vitp, c->conv_rate, c->ber_thresold, c->outsync_after, f->chunk, ph, n, c->constellation == 2);
        else vit_init(&f->vit, 0, c->ber_thresold, c->outsync_after, f->chunk, ph, n, c->constellation == 2);
        defr_init(&f->defr, c->cadu_size, c->asm_sync);
        f->defr.pad = c->cadu_size % 8;
    }
    f->vout = malloc(f->chunk * 8); f->frames = malloc(f->chunk * 8 + 10240); f->soft = malloc(f->chunk);
    return f;
}
void orc_fec_destroy(void *h)
{
    orc_fec *f = h;
    if (f->cfg.kind == 1 && f->cfg.conv_rate) vitp_free(&f->vitp);
    else if (f->cfg.kind != 2) vit_free(&f->vit);
    free(f->defr.frame); free(f->defr_qpsk.frame); free(f->vout); free(f->frames); free(f->soft); free(f);
}

/* QPSKDiff::work — differential/qpsk_diff.cpp:5-53 (2 output bits per decoded symbol; the first two symbols only fill the buffer) */
static int qpsk_diff_work(orc_fec *f, const uint8_t *in, int len, uint8_t *out, int swap)
{
    int oo = 0;
    for (int ii = 0; ii < len; ii++) {
        f->qd_buf[0] = f->qd_buf[1];
        f->qd_buf[1] = in[ii];
        if (f->qd_in < 2) { f->qd_in++; continue; }
        uint8_t Xin_1 = f->qd_buf[0] & 0x02, Yin_1 = f->qd_buf[0] & 0x01, Xin = f->qd_buf[1] & 0x02, Yin = f->qd_buf[1] & 0x01, Xout, Yout, ou;
        if (((Xin >> 1) ^ Yin) == 1) { Xout = (Yin_1 ^ Yin); Yout = (Xin_1 ^ Xin); ou = (Xout << 1) + (Yout >> 1); }
        else { Xout = (Xin_1 ^ Xin); Yout = (Yin_1 ^ Yin); ou = (Xout + Yout); }
        if (swap) { out[oo * 2 + 0] = ou & 1; out[oo * 2 + 1] = ou >> 1; }
        else { out[oo * 2 + 0] = ou >> 1; out[oo * 2 + 1] = ou & 1; }
        oo++;
    }
    return oo;
}

/* one iteration of CCSDSSimplePSKDecoderModule::process — module_ccsds_simple_psk_decoder.cpp:144-262 (oqpsk_method2/3 not restated);
 * leaves the bits for the main deframer in f->vout, returns the frames the second deframer already put into f->frames */
static int simple_bits(orc_fec *f)
{
    const orc_fec_cfg *k = &f->cfg;
    const int n = f->chunk;
    int8_t *sb = f->soft;
    uint8_t *bits = f->vout;
    int frames = 0;
    if (k->constellation == 0) {
        for (int i = 0; i < n; i++) bits[i] = sb[i] > 0;
        if (k->nrzm)
            for (int i = 0; i < n; i++) { uint8_t cur = bits[i]; bits[i] = cur ^ f->nrzm_last; f->nrzm_last = cur; }
        return 0;
    }
    if (k->oqpsk_delay)
        for (int i = 0; i < n / 2; i++) { int8_t back = sb[i * 2]; sb[i * 2] = f->last_q_oqpsk; f->last_q_oqpsk = back; }
    if (k->qpsk_swap_iq) orc_rotate_soft(sb, n, 0, 1);
    if (k->nrzm) {
        uint8_t *syms = f->frames + f->chunk * 4; /* scratch behind the frame area */
        for (int i = 0; i < n / 2; i++) syms[i] = 2 * (sb[i * 2 + 1] > 0) + (sb[i * 2] > 0); /* constellation_t::soft_demod, QPSK */
        qpsk_diff_work(f, syms, n / 2, bits, k->qpsk_swap_diff);
    } else {
        for (int i = 0; i < n / 2; i++) { bits[i * 2] = sb[i * 2 + 1] > 0; bits[i * 2 + 1] = sb[i * 2] > 0; }
        frames += defr_work(&f->defr_qpsk, bits, n, f->frames);
        orc_rotate_soft(sb, n, 1, 0);
        for (int i = 0; i < n / 2; i++) { bits[i * 2] = sb[i * 2 + 1] > 0; bits[i * 2 + 1] = sb[i * 2] > 0; }
    }
    return frames;
}
int orc_fec_chunk_size(void *h) { return ((orc_fec *)h)->chunk; }
int orc_fec_cadu_bytes(void *h) { return ((orc_fec *)h)->cadu_bytes; }

/* MetOpAHRPTDecoderModule::process (module_metop_ahrpt_decoder.cpp:34-90) and
 * CCSDSConvConcatDecoderModule::process (module_ccsds_conv_concat_decoder.cpp:140-200), one chunk per iteration */
long orc_fec_run(void *h, const int8_t *soft, long nsoft, uint8_t *cadu_out, long cadu_cap, int *vit_state, float *vit_b,
                 int *defr_state, uint8_t *bits_out, long *nbits, int *rs_err, long *nframes_seen)
{
    orc_fec *f = h;
    const orc_fec_cfg *k = &f->cfg;
    long outp = 0, bitp = 0, seen = 0;
    for (long c = 0; c < nsoft / f->chunk; c++) {
        memcpy(f->soft, soft + c * f->chunk, f->chunk);
        if (k->kind == 2) {
            int nf = simple_bits(f);
            if (bits_out) memcpy(bits_out + bitp, f->vout, f->chunk);
            bitp += f->chunk;
            nf += defr_work(&f->defr, f->vout, f->chunk, f->frames + nf * f->cadu_bytes);
            for (int i = 0; i < nf; i++) {
                uint8_t *cadu = f->frames + i * f->cadu_bytes;
                if (k->derandomize && !k->derand_after_rs) orc_derand(cadu + k->derand_start, f->cadu_bytes - k->derand_start);
                if (k->rs_i) orc_rs_decode_interleaved(cadu + 4, k->rs_dualbasis, k->rs_i, k->rs_type, k->rs_fill_bytes, f->errors);
                int valid = 1;
                for (int j = 0; j < k->rs_i; j++) if (f->errors[j] == -1) valid = 0;
                if (k->derandomize && k->derand_after_rs) orc_derand(cadu + k->derand_start, f->cadu_bytes - k->derand_start);
                if (rs_err) memcpy(rs_err + seen * k->rs_i, f->errors, sizeof(int) * k->rs_i);
                seen++;
                if ((!k->rs_usecheck || valid) && outp + f->cadu_bytes <= cadu_cap) { memcpy(cadu_out + outp, cadu, f->cadu_bytes); outp += f->cadu_bytes; }
            }
            if (vit_state) vit_state[c] = f->defr_qpsk.state;
            if (defr_state) defr_state[c] = f->defr.state;
            continue;
        }
        if (k->kind == 1 && (k->constellation == 5 || k->iq_invert)) orc_rotate_soft(f->soft, f->chunk, 0, 1);
        const int punc = k->kind == 1 && k->conv_rate;
        int vout = punc ? vitp_work(&f->vitp, f->soft, f->vout) : vit_work(&f->vit, f->soft, f->vout);
        if (vit_state) vit_state[c] = punc ? f->vitp.state : f->vit.state;
        if (vit_b) vit_b[c] = punc ? f->vitp.ber : vit_ber(&f->vit);
        if (k->kind == 0) {
            if (vout > 0) {
                if (bits_out) memcpy(bits_out + bitp, f->vout, vout);
                bitp += vout;
                int nf = defr_work(&f->defr, f->vout, vout, f->frames);
                if (f->defr.state == f->defr.st_nosync) { if (++f->nosync_runs >= 10) { f->vit.state = 0; f->nosync_runs = 0; } }
                else f->nosync_runs = 0;
                for (int i = 0; i < nf; i++) {
                    uint8_t *cadu = f->frames + i * 1024;
                    orc_derand(cadu + 4, 1020);
                    orc_rs_decode_interleaved(cadu + 4, 1, 4, 0, 0, f->errors);
                    if (rs_err) memcpy(rs_err + seen * 4, f->errors, 16);
                    seen++;
                    if (outp + 1024 <= cadu_cap) { memcpy(cadu_out + outp, cadu, 1024); outp += 1024; }
                }
            }
        } else {
            if (k->nrzm) /* NRZMDiff::decode_bits — differential/nrzm.cpp:24-33 */
                for (int i = 0; i < vout; i++) { uint8_t cur = f->vout[i]; f->vout[i] = cur ^ f->nrzm_last; f->nrzm_last = cur; }
            if (bits_out && vout > 0) memcpy(bits_out + bitp, f->vout, vout);
            bitp += vout;
            int nf = defr_work(&f->defr, f->vout, vout, f->frames);
            for (int i = 0; i < nf; i++) {
                uint8_t *cadu = f->frames + i * f->cadu_bytes;
                if (k->derandomize && !k->derand_after_rs) orc_derand(cadu + k->derand_start, f->cadu_bytes - k->derand_start);
                if (k->rs_i) orc_rs_decode_interleaved(cadu + 4, k->rs_dualbasis, k->rs_i, k->rs_type, k->rs_fill_bytes, f->errors);
                int valid = 1;
                for (int j = 0; j < k->rs_i; j++) if (f->errors[j] == -1) valid = 0;
                if (k->derandomize && k->derand_after_rs) orc_derand(cadu + k->derand_start, f->cadu_bytes - k->derand_start);
                if (rs_err) memcpy(rs_err + seen * k->rs_i, f->errors, sizeof(int) * k->rs_i);
                seen++;
                if ((!k->rs_usecheck || valid) && outp + f->cadu_bytes <= cadu_cap) { memcpy(cadu_out + outp, cadu, f->cadu_bytes); outp += f->cadu_bytes; }
            }
        }
        if (defr_state) defr_state[c] = f->defr.state;
    }
    if (nbits) *nbits = bitp;
    if (nframes_seen) *nframes_seen = seen;
    return outp;
}

/* Single-thread end to end: demod buffers feed the decoder chunk by chunk (the reference joins the two modules with a
 * byte FIFO, pipeline_run.cpp:72-104; results do not depend on the FIFO granularity). */
long orc_pipeline_run(const orc_demod_cfg *dc, const orc_fec_cfg *fc, const void *raw, long nsamples, uint8_t *cadu_out, long cadu_cap)
{
    orc_demod *d = orc_demod_create(dc);
    orc_fec *f = orc_fec_create(fc);
    int bps = dc->constellation == 0 ? 1 : 2;
    long cap = (long)(d->buffer_size) * bps + f->chunk + 64, have = 0, outp = 0;
    int8_t *fifo = malloc(cap);
    for (long off = 0; off < nsamples; off += d->buffer_size) {
        long n = nsamples - off < d->buffer_size ? nsamples - off : d->buffer_size;
        const char *p = (const char *)raw + off * (dc->format == 0 ? 8 : (dc->format == 1 ? 4 : 2));
        long m = orc_demod_run(d, p, n, 0, 0, 0, 0, fifo + have, (cap - have) / bps);
        have += m * bps;
        long used = have / f->chunk * f->chunk;
        if (used) {
            outp += orc_fec_run(f, fifo, used, cadu_out + outp, cadu_cap - outp, 0, 0, 0, 0, 0, 0, 0);
            memmove(fifo, fifo + used, have - used);
            have -= used;
        }
    }
    free(fifo);
    orc_demod_destroy(d);
    orc_fec_destroy(f);
    return outp;
}


/* ================================================================== CADU -> CCSDS space packets
 * ccsds::ccsds_aos::Demuxer::work (common/ccsds/ccsds_aos/demuxer.cpp:64-199), one instance per virtual channel, with all of its
 * behaviour on inconsistent frames: the packet under construction keeps its bytes until it is pushed or aborted (readPacket does not
 * clear them, :26-33), the continuation is cut at first_header_pointer + 1 (:101), a continuation in a frame without a header may take
 * more than what remains (:109) and then never completes, a frame whose pointer lies outside the data zone is skipped whole (:71-74). */
typedef struct
{
    int used;
    uint8_t hdr[6];  /* currentCCSDSPacket.header.raw */
    uint8_t *pay;    /* currentCCSDSPacket.payload */
    long npay, cappay;
    int cpl, tpl, rem; /* currentPacketPayloadLength, totalPacketLength, remainingPacketLength */
    int working, in_header, ihb;
    uint8_t hb[6];
} orc_dmx_vc;
typedef struct
{
    int mpdu, insert, insert_size, sec_ext;
    orc_dmx_vc vc[64];
    /* output cursor of the running call */
    uint8_t *out;
    long cap_bytes, nb, np, cap_recs;
    int *recs;
    long frame;
    int vcid, overflow;
} orc_dmx;

void *orc_demux_create(int mpdu_data_size, int has_insert_zone, int insert_zone_size, int secondary_header_extends)
{
    orc_dmx *d = calloc(1, sizeof(*d));
    d->mpdu = mpdu_data_size; d->insert = has_insert_zone; d->insert_size = insert_zone_size; d->sec_ext = secondary_header_extends;
    return d;
}
void orc_demux_destroy(void *h)
{
    orc_dmx *d = h;
    for (int i = 0; i < 64; i++) free(d->vc[i].pay);
    free(d);
}
static void dmx_read_packet(orc_dmx *d, orc_dmx_vc *v, const uint8_t *h) /* demuxer.cpp:26-33, ccsds.cpp:11-22 */
{
    v->working = 1;
    memcpy(v->hdr, h, 6);
    const int packet_length = h[4] << 8 | h[5], sec = (h[0] >> 3) & 1;
    v->cpl = packet_length + 1 + (d->sec_ext ? (sec ? 8 : 0) : 0);
    v->tpl = v->cpl + 6;
    v->rem = v->cpl;
}
static void dmx_push_payload(orc_dmx_vc *v, const uint8_t *data, int len) /* :47-53 (a negative length adds nothing but is still subtracted) */
{
    if (len > 0) {
        if (v->npay + len > v->cappay) { v->cappay = (v->npay + len) * 2 + 1024; v->pay = realloc(v->pay, v->cappay); }
        memcpy(v->pay + v->npay, data, len);
        v->npay += len;
    }
    v->rem -= len;
}
static void dmx_clear(orc_dmx_vc *v) { v->working = 0; v->npay = 0; v->cpl = 0; v->rem = 0; } /* abortPacket :56-62 / the tail of pushPacket */
static void dmx_push_packet(orc_dmx *d, orc_dmx_vc *v) /* :36-44 */
{
    if (d->np >= d->cap_recs || d->nb + 6 + v->npay > d->cap_bytes)
        d->overflow = 1;
    else {
        memcpy(d->out + d->nb, v->hdr, 6);
        memcpy(d->out + d->nb + 6, v->pay, v->npay);
        d->recs[4 * d->np + 0] = (int)d->frame;
        d->recs[4 * d->np + 1] = d->vcid;
        d->recs[4 * d->np + 2] = (int)v->npay;
        d->recs[4 * d->np + 3] = (v->hdr[0] & 7) << 8 | v->hdr[1];
        d->nb += 6 + v->npay;
        d->np++;
    }
    dmx_clear(v);
}
static void dmx_work(orc_dmx *d, orc_dmx_vc *v, const uint8_t *cadu)
{
    const int M = d->mpdu, base = d->insert ? 10 + d->insert_size : 10;
    const int fhp = (cadu[base] & 7) << 8 | cadu[base + 1]; /* mpdu.cpp:11 */
    const uint8_t *data = cadu + base + 2;
    if (fhp < 2047 && fhp >= M) /* :71-74 */
        return;
    int offset = 0;
    if (v->in_header) { /* :81-92 */
        v->in_header = 0;
        memcpy(v->hb + v->ihb, data, 6 - v->ihb);
        offset = 6 - v->ihb;
        v->ihb = 6;
        dmx_read_packet(d, v, v->hb);
    }
    if (v->rem > 0 && v->working) { /* :95-112 */
        if (fhp < 2047) {
            const int n = (v->rem + offset) > fhp + 1 ? (fhp + 1) - offset : v->rem;
            dmx_push_payload(v, data + offset, n);
            v->rem = 0;
        } else {
            const int n = (v->rem + offset) > M - offset ? M - offset : v->rem;
            dmx_push_payload(v, data + offset, n);
        }
    }
    if (v->rem == 0 && v->working) /* :115-118 */
        dmx_push_packet(d, v);
    if (fhp < 2047) { /* :121-195 */
        if (fhp + 6 < M) {
            dmx_read_packet(d, v, data + fhp);
            if (M > fhp + v->tpl) {
                dmx_push_payload(v, data + fhp + 6, v->cpl); /* (fhp + tpl < M always holds here) */
                dmx_push_packet(d, v);
                int next = fhp + v->tpl;
                while (next < M) {
                    if (next + 6 < M) {
                        dmx_read_packet(d, v, data + next);
                        const int room = M - (next + 6);
                        dmx_push_payload(v, data + next + 6, v->rem > room ? room : v->rem);
                    } else {
                        v->in_header = 1;
                        memcpy(v->hb, data + next, M - next);
                        v->ihb = M - next;
                        break;
                    }
                    if (v->rem == 0 && v->working)
                        dmx_push_packet(d, v);
                    next += v->tpl;
                }
            } else if (v->working) {
                const int room = M - (fhp + 6);
                dmx_push_payload(v, data + fhp + 6, v->rem > room ? room : v->rem);
            }
        } else if (fhp < M) {
            v->in_header = 1;
            memcpy(v->hb, data + fhp, M - fhp);
            v->ihb = M - fhp;
        }
    }
}
long orc_demux_run(void *h, const uint8_t *frames, long nframes, int cadu_size, unsigned long long vcid_mask, long frame0, uint8_t *out, long cap_bytes,
                   long *nbytes, int *recs, long cap_recs)
{
    orc_dmx *d = h;
    d->out = out; d->cap_bytes = cap_bytes; d->nb = 0; d->np = 0; d->cap_recs = cap_recs; d->recs = recs; d->overflow = 0;
    for (long f = 0; f < nframes; f++) {
        const uint8_t *cadu = frames + f * cadu_size;
        const int vcid = cadu[5] & 63; /* vcdu.cpp:14 */
        if (!((vcid_mask >> vcid) & 1ull)) continue;
        d->frame = frame0 + f;
        d->vcid = vcid;
        dmx_work(d, &d->vc[vcid], cadu);
        if (d->overflow) return -1;
    }
    *nbytes = d->nb;
    return d->np;
}
