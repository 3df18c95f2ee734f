/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref METEOR LRPT harness: wires the UNMODIFIED reference translation units of the METEOR-M LRPT decoder's parts (correlator.cpp,
 * viterbi27.cpp with cc_decoder.cpp / cc_encoder.cpp, viterbi_1_2.cpp, nrzm.cpp, rotation.cpp, randomization.cpp, bpsk_ccsds_deframer.cpp,
 * reedsolomon.cpp and libcorrect's Reed-Solomon, compiled from the reference tree by oracle/Makefile) the way
 *   meteor::METEORLRPTDecoderModule::process   plugins/meteor_support/meteor/module_meteor_lrpt_decoder.cpp:101-262
 * runs them in its two working modes (m2x_mode false: :198-262; m2x_mode without "interleaved": :103-197), and exposes them through a
 * small C ABI for the Python tests (oracle/meteor.py). The module file itself pulls in ImGui and the pipeline base, so its two loops are
 * restated here as wiring.
 *
 * Two reads of the module are defined here:
 *   - The module reads its input with a blocking read. A push that ends inside a frame (or inside the pos bytes a shift reads) leaves that
 *     frame for the next push; the statistics are those of the last frame completed.
 *   - decode_interlaved with fill_bytes -1 runs 256 rows, so it reads and writes the 4 bytes behind the module's 1024-byte frameBuffer.
 *     Here the frame buffer has 16 spare bytes; they never reach the output.
 *
 * No reference source is copied here: this file only *calls* the reference code.
 */
#include <cstring>
#include <memory>
#include <vector>
#include "common/codings/correlator.h"
#include "common/codings/deframing/bpsk_ccsds_deframer.h"
#include "common/codings/differential/nrzm.h"
#include "common/codings/randomization.h"
#include "common/codings/reedsolomon/reedsolomon.h"
#include "common/codings/rotation.h"
#include "common/codings/viterbi/viterbi27.h"
#include "common/codings/viterbi/viterbi_1_2.h"

namespace
{
    constexpr int F = 1024 * 8 * 2, FRAME = 1024, BUFFER_SIZE = 8192;

    struct RefMeteor
    {
        bool diff_decode = false;
        std::unique_ptr<Correlator> correlator;
        std::unique_ptr<viterbi::Viterbi27> viterbi;
        std::unique_ptr<reedsolomon::ReedSolomon> rs;
        diff::NRZMDiff diff;
        std::vector<int8_t> pend;   // soft bytes not consumed yet (the module's blocking read waits for them)
        long base_off = 0;          // stream offset of pend[0]
        std::vector<int8_t> buffer; // F bytes
        bool locked = false;
        int errors[4] = {0, 0, 0, 0};
    };

    struct RefMeteorM2x
    {
        bool diff_decode = false;
        std::unique_ptr<viterbi::Viterbi1_2> viterbin;
        std::unique_ptr<deframing::BPSK_CCSDS_Deframer> deframer;
        std::unique_ptr<reedsolomon::ReedSolomon> rs;
        diff::NRZMDiff diff;
        std::vector<int8_t> pend;
        std::vector<uint8_t> viterbi_out, frame_buffer;
        float viterbi_ber = 0;
        int viterbi_lock = 0;
        int errors[4] = {0, 0, 0, 0};
    };
}

extern "C"
{
    /* m2x_mode false: the decoder as the module sets it up (:22-27, :46, :200-213) */
    void *ref_meteor_create(int diff_decode)
    {
        RefMeteor *r = new RefMeteor();
        r->diff_decode = diff_decode != 0;
        r->correlator = std::make_unique<Correlator>(QPSK, r->diff_decode ? 0xfc4ef4fd0cc2df89 : 0xfca2b63db00d9794);
        r->viterbi = std::make_unique<viterbi::Viterbi27>(F / 2, viterbi::CCSDS_R2_K7_POLYS);
        r->rs = std::make_unique<reedsolomon::ReedSolomon>(reedsolomon::RS223);
        r->buffer.assign(F, 0);
        return r;
    }
    void ref_meteor_destroy(void *h) { delete (RefMeteor *)h; }

    /* Appends n soft bytes to the stream and runs the module loop (:215-260) over every frame they complete. Writes the frames the module
       writes (1D CF FC 1D + 1020 bytes) to out (*nbytes of at most cap_bytes) and one record of 10 int64 per frame: stream offset of the
       frame (window start + the shift), pos, cor, phase, swap, errors[0..3] of decode_interlaved, Viterbi27's ber() as float32 bits.
       stats[3]: correlator_lock, viterbi_ber (float32 bits), rs_avg (:282-287). Returns the number of frames, or -1 when a capacity is too
       small. */
    long ref_meteor_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames,
                        long long *stats)
    {
        RefMeteor *r = (RefMeteor *)h;
        r->pend.insert(r->pend.end(), soft, soft + n);
        const long size = (long)r->pend.size();
        long o = 0, nf = 0, nb = 0;
        int8_t *buf = r->buffer.data();
        uint8_t frameBuffer[FRAME + 16];
        while (size - o >= F)
        {
            memcpy(buf, &r->pend[o], F);
            phase_t phase;
            bool swap;
            int cor = 0;
            const int pos = r->correlator->correlate(buf, phase, swap, cor, F);
            const bool shift = pos != 0 && pos < F;
            if (shift)
            {
                if (o + F + pos > size)
                    break; // the module's read of the pos missing bytes waits for the next push
                std::memmove(buf, &buf[pos], F - pos);
                memcpy(&buf[F - pos], &r->pend[o + F], pos);
            }
            if (nf >= cap_frames)
                return -1;
            r->locked = pos == 0;
            rotate_soft(buf, F, phase, swap);
            memset(frameBuffer, 0, sizeof(frameBuffer));
            r->viterbi->work(buf, frameBuffer);
            if (r->diff_decode)
                r->diff.decode(frameBuffer, FRAME);
            derand_ccsds(&frameBuffer[4], FRAME - 4);
            if (frameBuffer[9] == 0xFF)
                for (int i = 0; i < FRAME; i++)
                    frameBuffer[i] ^= 0xFF;
            r->rs->decode_interlaved(&frameBuffer[4], false, 4, r->errors);
            if (r->errors[0] >= 0 && r->errors[1] >= 0 && r->errors[2] >= 0 && r->errors[3] >= 0)
            {
                if (nb + FRAME > cap_bytes)
                    return -1;
                const uint8_t sync[4] = {0x1d, 0xcf, 0xfc, 0x1d};
                memcpy(out + nb, sync, 4);
                memcpy(out + nb + 4, &frameBuffer[4], FRAME - 4);
                nb += FRAME;
            }
            long long *rec = recs + 10 * nf;
            rec[0] = r->base_off + o + (shift ? pos : 0);
            rec[1] = pos;
            rec[2] = cor;
            rec[3] = phase;
            rec[4] = swap;
            for (int i = 0; i < 4; i++)
                rec[5 + i] = r->errors[i];
            float ber = r->viterbi->ber();
            uint32_t bb;
            memcpy(&bb, &ber, 4);
            rec[9] = bb;
            nf++;
            o += F + (shift ? pos : 0);
        }
        r->pend.erase(r->pend.begin(), r->pend.begin() + o);
        r->base_off += o;
        *nbytes = nb;
        float ber = r->viterbi->ber();
        uint32_t bb;
        memcpy(&bb, &ber, 4);
        stats[0] = r->locked;
        stats[1] = bb;
        stats[2] = (r->errors[0] + r->errors[1] + r->errors[2] + r->errors[3]) / 4;
        return nf;
    }

    /* m2x_mode without "interleaved": the decoder as the module sets it up (:29-36, :115-120) */
    void *ref_meteor_m2x_create(int diff_decode, float ber_thresold, int outsync_after)
    {
        RefMeteorM2x *r = new RefMeteorM2x();
        r->diff_decode = diff_decode != 0;
        std::vector<phase_t> phases = {PHASE_0, PHASE_90};
        r->viterbin = std::make_unique<viterbi::Viterbi1_2>(ber_thresold, outsync_after, BUFFER_SIZE, phases, true);
        r->deframer = std::make_unique<deframing::BPSK_CCSDS_Deframer>(8192);
        r->rs = std::make_unique<reedsolomon::ReedSolomon>(reedsolomon::RS223);
        r->viterbi_out.assign(BUFFER_SIZE * 2, 0);
        r->frame_buffer.assign(BUFFER_SIZE * 2 + 16, 0);
        return r;
    }
    void ref_meteor_m2x_destroy(void *h) { delete (RefMeteorM2x *)h; }

    /* Appends n soft bytes and runs the loop (:130-192) over every complete call of 8192 soft bytes. Writes the frames the module writes
       (1024 bytes each) to out. stats[5]: deframer state (2 / 6 / 12), viterbi_ber (float32 bits), viterbi_lock, rs_avg, frames written so far
       by this call. Returns the number of frames written, or -1 when cap_bytes is too small. */
    long ref_meteor_m2x_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long long *stats)
    {
        RefMeteorM2x *r = (RefMeteorM2x *)h;
        r->pend.insert(r->pend.end(), soft, soft + n);
        const long size = (long)r->pend.size();
        long o = 0, nb = 0, nf = 0;
        std::vector<int8_t> buffer(BUFFER_SIZE);
        while (size - o >= BUFFER_SIZE)
        {
            memcpy(buffer.data(), &r->pend[o], BUFFER_SIZE);
            o += BUFFER_SIZE;
            const int vitout = r->viterbin->work(buffer.data(), BUFFER_SIZE, r->viterbi_out.data());
            r->viterbi_ber = r->viterbin->ber();
            r->viterbi_lock = r->viterbin->getState();
            if (r->diff_decode)
                r->diff.decode_bits(r->viterbi_out.data(), vitout);
            const int frames = r->deframer->work(r->viterbi_out.data(), vitout, r->frame_buffer.data());
            for (int i = 0; i < frames; i++)
            {
                uint8_t *cadu = &r->frame_buffer[i * 1024];
                derand_ccsds(&cadu[4], 1020);
                r->rs->decode_interlaved(&cadu[4], false, 4, r->errors);
                if (r->errors[0] >= 0 && r->errors[1] >= 0 && r->errors[2] >= 0 && r->errors[3] >= 0)
                {
                    if (nb + 1024 > cap_bytes)
                        return -1;
                    memcpy(out + nb, cadu, 1024);
                    nb += 1024;
                    nf++;
                }
            }
        }
        r->pend.erase(r->pend.begin(), r->pend.begin() + o);
        float ber = r->viterbi_ber;
        uint32_t bb;
        memcpy(&bb, &ber, 4);
        stats[0] = r->deframer->getState();
        stats[1] = bb;
        stats[2] = r->viterbi_lock;
        stats[3] = (r->errors[0] + r->errors[1] + r->errors[2] + r->errors[3]) / 4;
        stats[4] = nf;
        return nf;
    }
}
