/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref EOS harness: wires the UNMODIFIED reference blocks dsp::constellation_t (QPSK soft_demod), diff::NRZMDiff,
 * deframing::BPSK_CCSDS_Deframer, derand_ccsds and reedsolomon::ReedSolomon, compiled from the reference tree by oracle/Makefile, the way
 *   aqua::AquaDBDecoderModule::process  plugins/eos_support/aqua/module_aqua_db_decoder.cpp:27-83
 * runs them: 65 536-byte reads, the deframer with STATE_SYNCING 6 and STATE_SYNCED 10, every frame derandomised, RS-decoded and written.
 * The module file pulls in ImGui and the pipeline base, so its loop is restated here as wiring. The stream reader hands the loop whole
 * reads: a run() call that leaves less than one read keeps those bytes for the next call.
 *
 * No reference source is copied here: this file only *calls* the reference code.
 */
#include <cstring>
#include <vector>
#include "common/codings/deframing/bpsk_ccsds_deframer.h"
#include "common/codings/differential/nrzm.h"
#include "common/codings/randomization.h"
#include "common/codings/reedsolomon/reedsolomon.h"
#include "common/dsp/demod/constellation.h"

namespace
{
    constexpr int BUFFER_SIZE = 1024 * 8 * 8, FRAME_SIZE = 1024;

    struct RefAqua
    {
        dsp::constellation_t constellation{dsp::QPSK};
        reedsolomon::ReedSolomon rs{reedsolomon::RS223};
        diff::NRZMDiff diff1, diff2;
        deframing::BPSK_CCSDS_Deframer deframer{8192};
        std::vector<uint8_t> pending;
        long frames = 0, corrected = 0, failed = 0;
        RefAqua()
        {
            deframer.STATE_SYNCING = 6;
            deframer.STATE_SYNCED = 10;
        }
    };
}

extern "C"
{
    void *ref_aqua_create() { return new RefAqua(); }
    void ref_aqua_destroy(void *h) { delete (RefAqua *)h; }

    /* Appends n soft bytes to the stream and runs the module loop over every whole read. Writes the CADUs to out (cap bytes, *nbytes
       written) and each frame's four RS results (errors[]) to rs_out (rs_cap ints). stats: [0] frames written so far, [1] getState(),
       [2] bytes corrected so far, [3] codewords that failed so far, [4] soft bytes kept for the next read. Returns 0, or -1 when a buffer
       is too small. */
    int ref_aqua_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap, long *nbytes, int *rs_out, long rs_cap, long *stats)
    {
        RefAqua *r = (RefAqua *)h;
        r->pending.insert(r->pending.end(), (const uint8_t *)soft, (const uint8_t *)soft + n);
        std::vector<uint8_t> bufI(BUFFER_SIZE / 2), bufQ(BUFFER_SIZE / 2), final_buf(BUFFER_SIZE), frame_buffer(FRAME_SIZE * 100);
        long nb = 0, nrs = 0, used = 0;
        int ok = 0;
        while ((long)r->pending.size() - used >= BUFFER_SIZE) {
            uint8_t *buffer = r->pending.data() + used;
            used += BUFFER_SIZE;
            for (int i = 0; i < BUFFER_SIZE / 2; i++) {
                uint8_t demod = r->constellation.soft_demod((int8_t *)&buffer[i * 2]);
                bufI[i] = demod >> 1;
                bufQ[i] = demod & 1;
            }
            r->diff1.decode_bits(bufI.data(), BUFFER_SIZE / 2);
            r->diff2.decode_bits(bufQ.data(), BUFFER_SIZE / 2);
            for (int i = 0; i < BUFFER_SIZE / 2; i++) {
                final_buf[i * 2 + 0] = bufI[i];
                final_buf[i * 2 + 1] = bufQ[i];
            }
            const int frames = r->deframer.work(final_buf.data(), BUFFER_SIZE, frame_buffer.data());
            for (int i = 0; i < frames; i++) {
                uint8_t *cadu = &frame_buffer[i * FRAME_SIZE];
                int errors[4];
                derand_ccsds(&cadu[4], FRAME_SIZE - 4);
                r->rs.decode_interlaved(&cadu[4], true, 4, errors);
                if (nb + FRAME_SIZE > cap || nrs + 4 > rs_cap) {
                    ok = -1;
                    continue;
                }
                std::memcpy(out + nb, cadu, FRAME_SIZE);
                nb += FRAME_SIZE;
                for (int k = 0; k < 4; k++) {
                    rs_out[nrs++] = errors[k];
                    if (errors[k] < 0)
                        r->failed++;
                    else
                        r->corrected += errors[k];
                }
                r->frames++;
            }
        }
        r->pending.erase(r->pending.begin(), r->pending.begin() + used);
        *nbytes = nb;
        stats[0] = r->frames;
        stats[1] = r->deframer.getState();
        stats[2] = r->corrected;
        stats[3] = r->failed;
        stats[4] = (long)r->pending.size();
        return ok;
    }
}
