/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref GAC / DMSP harness: wires the UNMODIFIED reference deframers deframing::BPSK_CCSDS_Deframer
 * (src-core/common/codings/deframing/bpsk_ccsds_deframer.cpp) and dmsp::DMSP_Deframer (plugins/dmsp_support/dmsp/dmsp_deframer.cpp),
 * compiled from the reference tree by oracle/Makefile, the way
 *   noaa::NOAAGACDecoderModule::process   plugins/noaa_metop_support/noaa/module_noaa_gac_decoder.cpp:30-133
 *   dmsp::DMSPRTDDecoderModule::process   plugins/dmsp_support/dmsp/module_dmsp_rtd_decoder.cpp:34-70
 * run them, and exposes them through a small C ABI for the Python tests (oracle/gac.py). The module files pull in ImGui and the pipeline
 * base, so their loops are restated here as wiring. The PN table is the reference's own noaa/gac_pn.h, included at compile time.
 *
 * Definitions made here:
 *   - Reads: both modules read 8192 soft bytes at a time from the start of the stream. run() collects the bytes it is given and runs the
 *     loop body once per complete 8192-byte read; a partial read waits for the next run() (a stream reader blocks the same way).
 *   - GAC frames come out in decode order, after the backward reversal and the PN; the reversal of the frame ORDER that the module
 *     applies to its file at the end of a backward run is left to the caller.
 *   - DMSP: with start_timestamp != -1 each frame's "_timestamps.txt" value is returned as a double.
 *
 * No reference source is copied here: this file only *calls* the reference code (and includes its PN table header).
 */
#include <cstdint>
#include <cstring>
#include <vector>
#include "common/codings/deframing/bpsk_ccsds_deframer.h"
#include "dmsp/dmsp_deframer.h"

namespace refgac
{
#include "noaa/gac_pn.h"
}

namespace
{
    constexpr int BUFSIZE = 8192, GAC_BYTES = 4159, DMSP_BYTES = 19;

    struct RefGac
    {
        int dmsp = 0, backward = 0;
        double start_timestamp = -1;
        deframing::BPSK_CCSDS_Deframer *gac = nullptr;
        dmsp::DMSP_Deframer *def = nullptr;
        uint8_t gac_pn[GAC_BYTES];
        std::vector<int8_t> pending; // bytes of the read not yet complete
        long frame_count = 0;        // GAC: frames so far (the module's frame_count before its / 11090)
        size_t accumulated = 0;      // DMSP: accumulated_samples
    };
}

extern "C"
{
    /* the reference's gac_rand_bits as 0 / 1 bytes (1023 entries) */
    void ref_gac_pn_table(uint8_t *out)
    {
        for (int i = 0; i < 1023; i++)
            out[i] = refgac::gac_rand_bits[i];
    }

    /* dmsp 0: noaa_gac_decoder with `backward`; dmsp 1: dmsp_rtd_decoder with start_timestamp (-1: none) */
    void *ref_gac_create(int dmsp, int backward, double start_timestamp)
    {
        RefGac *r = new RefGac();
        r->dmsp = dmsp;
        r->backward = backward;
        r->start_timestamp = start_timestamp;
        if (dmsp) {
            r->def = new dmsp::DMSP_Deframer(150, 2);
        } else {
            r->gac = new deframing::BPSK_CCSDS_Deframer(33270, backward ? 0x33c3e4a6 : 0xA116FD71);
            r->gac->CADU_PADDING = 33270 % 8;
            memset(r->gac_pn, 0, GAC_BYTES); // module_noaa_gac_decoder.cpp:55-63
            for (int i = 0; i < GAC_BYTES * 8 - 60; i++) {
                int real_bit = i + 60;
                r->gac_pn[real_bit / 8] = r->gac_pn[real_bit / 8] << 1 | refgac::gac_rand_bits[i % 1023];
            }
        }
        return r;
    }
    void ref_gac_destroy(void *h)
    {
        RefGac *r = (RefGac *)h;
        delete r->gac;
        delete r->def;
        delete r;
    }

    /* Appends n soft bytes to the stream and runs the module loop over every complete read. Writes the frames (4159 / 19 bytes) to out
       (cap bytes, *nbytes written); DMSP with a start timestamp: one value per frame to ts (at most tcap, *nts written). stats[0] = frames
       so far, stats[1] = getState(). Returns 0, or -1 when a buffer is too small. */
    int ref_gac_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap, long *nbytes, double *ts, long tcap, long *nts, long *stats)
    {
        RefGac *r = (RefGac *)h;
        r->pending.insert(r->pending.end(), soft, soft + n);
        long nb = 0, nt = 0;
        size_t at = 0;
        uint8_t bits[BUFSIZE];
        std::vector<uint8_t> frames(GAC_BYTES * 10 > BUFSIZE ? GAC_BYTES * 10 : BUFSIZE);
        for (; at + BUFSIZE <= r->pending.size(); at += BUFSIZE) {
            const int8_t *buf = r->pending.data() + at;
            for (int i = 0; i < BUFSIZE; i++)
                bits[i] = buf[i] > 0;
            if (r->dmsp) {
                const int nf = r->def->work(bits, BUFSIZE, frames.data());
                if (nf > 0) {
                    if (nb + (long)nf * DMSP_BYTES > cap)
                        return -1;
                    memcpy(out + nb, frames.data(), (size_t)nf * DMSP_BYTES);
                    nb += (long)nf * DMSP_BYTES;
                    r->accumulated += BUFSIZE;
                    if (r->start_timestamp != -1)
                        for (int i = 0; i < nf; i++) {
                            if (nt >= tcap)
                                return -1;
                            ts[nt++] = r->start_timestamp + double(r->accumulated) / 1.024e6;
                        }
                }
                r->frame_count += nf;
            } else {
                const int nf = r->gac->work(bits, BUFSIZE, frames.data());
                r->frame_count += nf;
                for (int i = 0; i < nf; i++) {
                    uint8_t *frm = &frames[i * GAC_BYTES];
                    if (r->backward) { // module :84-95
                        uint8_t invert_buf[GAC_BYTES];
                        memcpy(invert_buf, frm, GAC_BYTES);
                        memset(frm, 0, GAC_BYTES);
                        for (int ii = 0; ii < 33270; ii++) {
                            int inv = (33270 - 1) - ii;
                            frm[ii / 8] = frm[ii / 8] << 1 | ((invert_buf[inv / 8] >> (7 - (inv % 8))) & 1);
                        }
                    }
                    for (int k = 0; k < GAC_BYTES; k++)
                        frm[k] ^= r->gac_pn[k];
                    if (nb + GAC_BYTES > cap)
                        return -1;
                    memcpy(out + nb, frm, GAC_BYTES);
                    nb += GAC_BYTES;
                }
            }
        }
        r->pending.erase(r->pending.begin(), r->pending.begin() + at);
        *nbytes = nb;
        *nts = nt;
        stats[0] = r->frame_count;
        stats[1] = r->dmsp ? r->def->getState() : r->gac->getState();
        return 0;
    }
}
