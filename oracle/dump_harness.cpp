/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref MetOp dump harness: wires the UNMODIFIED reference translation units of the MetOp X-band dump decoder's parts
 * (correlator32.cpp, rotation.cpp, randomization.cpp, reedsolomon.cpp and libcorrect's Reed-Solomon, compiled from the reference tree by
 * oracle/Makefile) the way
 *   metop::MetOpDumpDecoderModule::process   plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:27-83
 * runs them, and exposes them through a small C ABI for the Python tests (oracle/dump.py).
 *
 * Two reads of the module are defined here:
 *   - The module's memmove(buffer, &buffer[pos], pos) reads past its F-byte buffer when pos > F / 2. Here the buffer has 2F bytes and the
 *     F bytes behind the frame stay zero.
 *   - Correlator32::correlate scans 8184 bytes of its 160 KiB hard_buf, of which only the first 1024 are ever written. The rest is what
 *     a fresh new[] returns: in the module's process, with its small heap, glibc serves a request above the 128 KiB mmap threshold with
 *     fresh zero pages. In a test process (Python with numpy) the same request can be served from a large free chunk of recycled heap,
 *     whatever the threshold (glibc only maps when the top chunk is too small), so create() writes the zeros the module sees.
 *
 * No reference source is copied here: this file only *calls* the reference code. Correlator32's hard_buf is private; the harness reads it.
 */
#include <cstring>
#include <memory>
#include <vector>
#define private public
#include "common/codings/correlator32.h"
#undef private
#include "common/codings/randomization.h"
#include "common/codings/reedsolomon/reedsolomon.h"
#include "common/codings/rotation.h"

namespace
{
    constexpr int F = 8192, FRAME = 1024, HARD_BUF = 8192 * 20;

    struct RefDump
    {
        std::unique_ptr<Correlator32> correlator;
        std::unique_ptr<reedsolomon::ReedSolomon> rs;
        std::vector<int8_t> pend;   // soft bytes not consumed yet (the module's blocking read waits for them)
        long base_off = 0;          // stream offset of pend[0]
        std::vector<int8_t> buffer; // 2F bytes, the second half zero
    };
}

extern "C"
{
    /* A decoder as MetOpDumpDecoderModule::process sets it up (:30-33) */
    void *ref_dump_create(void)
    {
        RefDump *r = new RefDump();
        r->correlator = std::make_unique<Correlator32>(QPSK, 0x1acffc1d);
        memset(r->correlator->hard_buf, 0, HARD_BUF);
        r->rs = std::make_unique<reedsolomon::ReedSolomon>(reedsolomon::RS223);
        r->buffer.assign(2 * F, 0);
        return r;
    }
    void ref_dump_destroy(void *h) { delete (RefDump *)h; }

    /* Appends n soft bytes to the stream and runs the module loop (:41-79) over every frame they complete. Writes the frames the module
       writes (1A CF FC 1D + 1020 bytes) to out (*nbytes of at most cap_bytes) and one record of 9 int64 per frame: stream offset of the
       frame (window start + the shift), pos, cor, phase, swap, errors[0..3] of decode_interlaved. Returns the number of frames, or -1 when a
       capacity is too small. */
    long ref_dump_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
    {
        RefDump *r = (RefDump *)h;
        r->pend.insert(r->pend.end(), soft, soft + n);
        const long size = (long)r->pend.size();
        long o = 0, nf = 0, nb = 0;
        int8_t *buf = r->buffer.data();
        uint8_t frame[FRAME];
        while (size - o >= F)
        {
            memcpy(buf, &r->pend[o], F);
            phase_t phase;
            bool swap;
            int cor = 0, errors[4] = {0, 0, 0, 0};
            const int pos = r->correlator->correlate(buf, phase, swap, cor, F);
            const bool shift = pos != 0 && pos < F;
            if (shift)
            {
                if (o + pos + F > size)
                    break; // the module's read of the pos missing bytes waits for the next push
                std::memmove(buf, &buf[pos], pos);
                memcpy(&buf[F - pos], &r->pend[o + F], pos);
            }
            if (nf >= cap_frames || nb + FRAME > cap_bytes)
                return -1;
            rotate_soft(buf, F, phase, swap);
            memset(frame, 0, FRAME);
            for (int i = 0; i < FRAME; i++)
            {
                for (int y = 0; y < 8; y++)
                    frame[i] = frame[i] << 1 | (buf[i * 8 + y] > 0);
                frame[i] ^= 0xFF;
            }
            derand_ccsds(&frame[4], FRAME - 4);
            r->rs->decode_interlaved(&frame[4], true, 4, errors);
            const uint8_t sync[4] = {0x1a, 0xcf, 0xfc, 0x1d};
            memcpy(out + nb, sync, 4);
            memcpy(out + nb + 4, &frame[4], FRAME - 4);
            nb += FRAME;
            long long *rec = recs + 9 * nf;
            rec[0] = r->base_off + o + (shift ? pos : 0);
            rec[1] = pos;
            rec[2] = cor;
            rec[3] = phase;
            rec[4] = swap;
            for (int i = 0; i < 4; i++)
                rec[5 + i] = errors[i];
            nf++;
            o += F + (shift ? pos : 0);
        }
        r->pend.erase(r->pend.begin(), r->pend.begin() + o);
        r->base_off += o;
        *nbytes = nb;
        return nf;
    }
}
