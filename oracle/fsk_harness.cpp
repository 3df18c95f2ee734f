/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref/libsatref_fsk.so harness: wires the UNMODIFIED reference blocks of fsk_demod (compiled from the reference tree by
 * oracle/Makefile) the way FSKDemodModule does, behind BaseDemodModule's AGC:
 *   FSKDemodModule::init / process    src-core/pipeline/modules/demod/module_fsk_demod.cpp:59-158
 *   BaseDemodModule::initb (AGC)      src-core/pipeline/modules/demod/module_demod_base.cpp:207
 * and exposes every stage's output, the symbols, the soft bytes and the per-read SNR through a small C ABI.
 *
 * The library is linked with -Wl,--wrap=atan2f: QuadratureDemodBlock's atan2f lands in __wrap_atan2f, which returns glibc's atan2f
 * (ref_fsk_atan2_mode(0), what SatDump runs) or the correctly rounded (float)atan2((double)y, (double)x) (mode 1, the default; the
 * GPU computes that one: DESIGN §9).
 *
 * No reference source is copied here: this file only *calls* the reference classes.
 */
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>
#include <volk/volk.h>
#include "logger.h"
#define protected public
#define private public
#include "common/dsp/block.h"
#include "common/dsp/utils/agc.h"
#include "common/dsp/utils/correct_iq.h"
#include "common/dsp/utils/snr_estimator.h"
#include "common/dsp/filter/fir.h"
#include "common/dsp/filter/firdes.h"
#include "common/dsp/demod/quadrature_demod.h"
#include "common/dsp/clock_recovery/clock_recovery_mm.h"
#undef private
#undef protected

std::shared_ptr<slog::Logger> logger = std::make_shared<slog::Logger>();

static int g_atan2_mode = 1;
extern "C" float __real_atan2f(float y, float x);
extern "C" float __wrap_atan2f(float y, float x) { return g_atan2_mode ? (float)atan2((double)y, (double)x) : __real_atan2f(y, x); }

namespace
{
struct RefFsk
{
    int buffer_size;
    std::shared_ptr<dsp::stream<complex_t>> in;
    std::shared_ptr<dsp::AGCBlock<complex_t>> agc;
    std::shared_ptr<dsp::QuadratureDemodBlock> qua;
    std::shared_ptr<dsp::CorrectIQBlock<float>> dcb2;
    std::shared_ptr<dsp::AGCBlock<float>> agc2;
    std::shared_ptr<dsp::FIRBlock<float>> rrc;
    std::shared_ptr<dsp::MMClockRecoveryBlock<float>> rec;
    M2M4SNREstimator snr_estimator;
    float snr = 0, peak_snr = 0;
};

// BaseDemodModule::clamp (module_demod_base.h:105-112), a protected member of the module there
int8_t clamp(float x)
{
    if (x < -128.0)
        return -127;
    if (x > 127.0)
        return 127;
    return x;
}

// appends what a stream holds to out (as floats) and flushes it
template <class T> void take(const std::shared_ptr<dsp::stream<T>> &s, float *out, long cap, long &pos)
{
    const int m = s->getDataSize();
    const long per = sizeof(T) / sizeof(float);
    if (out && pos + m <= cap)
        memcpy(out + pos * per, s->readBuf, m * sizeof(T));
    pos += m;
}
} // namespace

extern "C"
{
    void ref_fsk_atan2_mode(int cr) { g_atan2_mode = cr; }
    float ref_fsk_atan2f(float y, float x) { return __wrap_atan2f(y, x); }

    /* the module's chain at the working rate final_samplerate (module_demod_base.cpp:89: final_sps = final_samplerate / (float)symbolrate) */
    void *ref_fsk_create(float final_samplerate, int symbolrate, float rrc_alpha, int rrc_taps, float agc_rate, float gain_omega, float mu, float gain_mu,
                         float omega_limit, int buffer_size)
    {
        RefFsk *d = new RefFsk;
        d->buffer_size = buffer_size;
        d->in = std::make_shared<dsp::stream<complex_t>>();
        d->agc = std::make_shared<dsp::AGCBlock<complex_t>>(d->in, agc_rate, 1.0f, 1.0f, 65536);
        d->qua = std::make_shared<dsp::QuadratureDemodBlock>(d->agc->output_stream, 1.0f);
        d->dcb2 = std::make_shared<dsp::CorrectIQBlock<float>>(d->qua->output_stream);
        d->agc2 = std::make_shared<dsp::AGCBlock<float>>(d->dcb2->output_stream, 0.1f, 0.5f, 1.0f, 65535.0f);
        std::vector<float> taps = dsp::firdes::root_raised_cosine(1, final_samplerate, symbolrate, rrc_alpha, rrc_taps);
        d->rrc = std::make_shared<dsp::FIRBlock<float>>(d->agc2->output_stream, taps);
        const float final_sps = final_samplerate / (float)symbolrate;
        d->rec = std::make_shared<dsp::MMClockRecoveryBlock<float>>(d->rrc->output_stream, final_sps, gain_omega, mu, gain_mu, omega_limit);
        d->rec->last_sample = 0; // never initialised by the block (clock_recovery_mm.h:30): a new stream starts from 0, as on the GPU
        d->rec->sample = 0;
        return d;
    }
    void ref_fsk_destroy(void *h) { delete (RefFsk *)h; }

    /* Runs n cf32 samples (what the reader hands the AGC) through the chain in reads of buffer_size. Every stage output pointer may be
       NULL; counts[0..6] = samples of agc (complex) / quad / dc2 / agc2 / fir, symbols, and the reads. snr_out[r] = the module's snr after
       read r (cap_reads of them); stats[0..1] = snr, peak_snr after the call. Returns 0, or -1 when an output did not fit. */
    int ref_fsk_run(void *h, const float *iq, long n, float *agc, float *quad, float *dc2, float *agc2, float *fir, long cap, float *sym, int8_t *soft,
                    long cap_sym, float *snr_out, long cap_reads, long *counts, float *stats)
    {
        RefFsk *d = (RefFsk *)h;
        long pa = 0, pq = 0, pd = 0, pg = 0, pf = 0, ps = 0, reads = 0;
        for (long off = 0; off < n; off += d->buffer_size)
        {
            const int m = (int)std::min<long>(d->buffer_size, n - off);
            memcpy(d->in->writeBuf, iq + 2 * off, m * sizeof(complex_t));
            d->in->swap(m);
            d->agc->work();
            take(d->agc->output_stream, agc, cap, pa);
            d->qua->work();
            take(d->qua->output_stream, quad, cap, pq);
            d->dcb2->work();
            take(d->dcb2->output_stream, dc2, cap, pd);
            d->agc2->work();
            take(d->agc2->output_stream, agc2, cap, pg);
            d->rrc->work();
            take(d->rrc->output_stream, fir, cap, pf);
            d->rec->work();
            const int dat_size = d->rec->output_stream->getDataSize();
            if (dat_size > 0) // module_fsk_demod.cpp:112-134
            {
                const float *buf = d->rec->output_stream->readBuf;
                d->snr_estimator.update((complex_t *)buf, dat_size / 2);
                d->snr = d->snr_estimator.snr();
                if (d->snr > d->peak_snr)
                    d->peak_snr = d->snr;
                if (ps + dat_size <= cap_sym)
                    for (int i = 0; i < dat_size; i++)
                    {
                        if (sym)
                            sym[ps + i] = buf[i];
                        if (soft)
                            soft[ps + i] = clamp(buf[i] * 50);
                    }
                ps += dat_size;
            }
            if (snr_out && reads < cap_reads)
                snr_out[reads] = d->snr;
            reads++;
            d->rec->output_stream->flush();
            d->agc->output_stream->flush();
            d->qua->output_stream->flush();
            d->dcb2->output_stream->flush();
            d->agc2->output_stream->flush();
            d->rrc->output_stream->flush();
        }
        counts[0] = pa;
        counts[1] = pq;
        counts[2] = pd;
        counts[3] = pg;
        counts[4] = pf;
        counts[5] = ps;
        counts[6] = reads;
        stats[0] = d->snr;
        stats[1] = d->peak_snr;
        return (pa > cap || ps > cap_sym) ? -1 : 0;
    }

    /* ONE block of a fresh chain on a caller-supplied input written straight into the stream it reads, in reads of buffer_size:
       stage 8 QuadratureDemodBlock (complex input), 9 CorrectIQBlock<float>, 10 AGCBlock<float>, 1 FIRBlock<float>, 5
       MMClockRecoveryBlock<float> (float inputs). Returns the number of float outputs (<= cap), or -1 for an unknown stage. */
    long ref_fsk_run_stage(void *h, int stage, const float *in, long n, float *out, long cap)
    {
        RefFsk *d = (RefFsk *)h;
        long pos = 0;
        for (long off = 0; off < n; off += d->buffer_size)
        {
            const int m = (int)std::min<long>(d->buffer_size, n - off);
            if (stage == 8)
            {
                memcpy(d->agc->output_stream->writeBuf, in + 2 * off, m * sizeof(complex_t));
                d->agc->output_stream->swap(m);
                d->qua->work();
                take(d->qua->output_stream, out, cap, pos);
                d->qua->output_stream->flush();
                continue;
            }
            std::shared_ptr<dsp::stream<float>> src = stage == 9 ? d->qua->output_stream
                                                      : (stage == 10 ? d->dcb2->output_stream : (stage == 1 ? d->agc2->output_stream : d->rrc->output_stream));
            std::shared_ptr<dsp::stream<float>> dst;
            memcpy(src->writeBuf, in + off, m * sizeof(float));
            src->swap(m);
            if (stage == 9)
                d->dcb2->work(), dst = d->dcb2->output_stream;
            else if (stage == 10)
                d->agc2->work(), dst = d->agc2->output_stream;
            else if (stage == 1)
                d->rrc->work(), dst = d->rrc->output_stream;
            else if (stage == 5)
                d->rec->work(), dst = d->rec->output_stream;
            else
                return -1;
            take(dst, out, cap, pos);
            dst->flush();
        }
        return std::min(pos, cap);
    }

    /* M2M4SNREstimator fed the way the module feeds it (module_fsk_demod.cpp:127): block b of the float symbols `sym` (sizes[b] of them) as
       sizes[b] / 2 complex pairs in one update; out[b] = snr() after it */
    void ref_fsk_snr(const float *sym, const long *sizes, int nblocks, float *out)
    {
        M2M4SNREstimator est;
        for (int b = 0; b < nblocks; b++)
        {
            est.update((complex_t *)sym, (int)(sizes[b] / 2));
            out[b] = est.snr();
            sym += sizes[b];
        }
    }

    /* RRC taps and the clock recovery's starting omega (final_sps) as the module designs them */
    int ref_fsk_taps(void *h, float *out, int cap, float *omega)
    {
        RefFsk *d = (RefFsk *)h;
        const int nt = d->rrc->ntaps;
        for (int j = 0; j < nt && j < cap; j++)
            out[j] = d->rrc->taps[0][(nt - 1) - j]; // (stored reversed, fir.cpp:30)
        *omega = d->rec->omega;
        return nt;
    }
}
