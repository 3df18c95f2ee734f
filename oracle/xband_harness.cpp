/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref METEOR X-band harness: wires the UNMODIFIED reference blocks meteor::MTVZA_ExtDeframer and meteor::KMSS_BPSK_ExtDeframer
 * (plugins/meteor_support/meteor/meteor_rec_deframer.h, with meteor_rec_deframer.cpp), diff::NRZMDiff (common/codings/differential/nrzm.cpp),
 * RepackBitsByte (common/repack_bits_byte.cpp) and def::SimpleDeframer (common/simple_deframer.h), compiled from the reference tree by
 * oracle/Makefile, the way
 *   meteor::MeteorXBandDecoderModule::process   plugins/meteor_support/meteor/module_meteor_xband_decoder.cpp:62-212
 * runs them ("mtvza" and "kmss_bpsk"), and exposes them through a small C ABI for the Python tests (oracle/xband.py). The module file
 * pulls in ImGui and the pipeline base, so its loop is restated here as wiring.
 *
 * Definitions made here:
 *   - Reads: the module reads 8192 soft bytes at a time from the start of the stream. run() collects the bytes it is given and runs the
 *     loop body once per complete read; a partial read waits for the next run() (a stream reader blocks the same way).
 *   - The record deframers' shift buffers come from new[] and are left uninitialised; this library's operator new[] returns zeroed
 *     storage, so they start at 0, as the GPU decoder defines them.
 *
 * No reference source is copied here: this file only *calls* the reference code.
 */
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>
#include "common/codings/differential/nrzm.h"
#include "common/repack_bits_byte.h"
#include "common/simple_deframer.h"
#include "meteor/meteor_rec_deframer.h"

void *operator new[](size_t n)
{
    void *p = calloc(n ? n : 1, 1);
    if (!p)
        throw std::bad_alloc();
    return p;
}
void operator delete[](void *p) noexcept { free(p); }
void operator delete[](void *p, size_t) noexcept { free(p); }

namespace
{
    constexpr int BUFFER_SIZE = 8192;

    struct RefXBand
    {
        int kmss = 0;
        diff::NRZMDiff nrzm;
        RepackBitsByte repack;
        meteor::MTVZA_ExtDeframer mtvza_recdef;
        meteor::KMSS_BPSK_ExtDeframer kmssbpsk_def;
        def::SimpleDeframer mtvza_deframer{0x38fb456a, 32, 3040, 0, false};
        def::SimpleDeframer kmss1{0xaf5fff50aa5aa0, 56, 481280, 0, false};
        def::SimpleDeframer kmss2{0xae5eec61bb7982, 56, 481280, 0, false};
        def::SimpleDeframer kmss3{0xab5bb394eed628, 56, 481280, 0, false};
        std::vector<uint8_t> pending;
        long frame_count = 0;
        // the module's buffers (rfrm / rpkt: 12288 * 4 bytes for kmss_bpsk, BUFFER_SIZE for mtvza)
        std::vector<int8_t> soft_buffer = std::vector<int8_t>(BUFFER_SIZE);
        std::vector<uint8_t> bit_buffer = std::vector<uint8_t>(BUFFER_SIZE), rfrm, rpkt;
    };

    void kmss_frame(std::vector<uint8_t> &kfrm, uint8_t (*ff)[4][15040]) // kmssFrameProcessor (module :44-53), restated as wiring
    {
        for (size_t u = 0; u < kfrm.size(); u++)
            kfrm[u] ^= 0xF0;
        for (int o = 0; o < 4; o++)
            for (int c = 0; c < 15040; c++) {
                uint8_t v = 0;
                for (int i = 0; i < 4; i++)
                    v = (uint8_t)(v << 2 | ((kfrm[c * 4 + i] >> (7 - o)) & 1) << 1 | ((kfrm[c * 4 + i] >> (3 - o)) & 1));
                (*ff)[o][c] = v;
            }
    }
}

extern "C"
{
    void *ref_xb_create(int kmss)
    {
        RefXBand *r = new RefXBand();
        r->kmss = kmss;
        r->rfrm.resize(kmss ? 12288 * 4 : BUFFER_SIZE);
        r->rpkt.resize(kmss ? 12288 * 4 : BUFFER_SIZE);
        return r;
    }
    void ref_xb_destroy(void *h) { delete (RefXBand *)h; }

    /* Appends n soft bytes and runs the module loop over every whole read: the frames it writes go to out (cap bytes, *nbytes written).
       stats: [0] frame_count so far, [1] soft bytes waiting for the next read. Returns 0, or -1 when out is too small. */
    int ref_xb_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap, long *nbytes, long *stats)
    {
        RefXBand *r = (RefXBand *)h;
        r->pending.insert(r->pending.end(), (const uint8_t *)soft, (const uint8_t *)soft + n);
        long nb = 0, used = 0;
        int ok = 0;
        auto put = [&](const uint8_t *p, long len) {
            if (nb + len > cap) {
                ok = -1;
                return;
            }
            memcpy(out + nb, p, len);
            nb += len;
        };
        static uint8_t final_frames[4][15040];
        while ((long)r->pending.size() - used >= BUFFER_SIZE) {
            memcpy(r->soft_buffer.data(), r->pending.data() + used, BUFFER_SIZE);
            used += BUFFER_SIZE;
            uint8_t *bits = r->bit_buffer.data();
            for (int i = 0; i < BUFFER_SIZE; i++)
                bits[i] = r->soft_buffer[i] > 0;
            r->nrzm.decode_bits(bits, BUFFER_SIZE);
            int rpktpos = 0;
            if (!r->kmss) {
                int nfrm = r->mtvza_recdef.work(bits, BUFFER_SIZE, r->rfrm.data());
                for (int i = 0; i < nfrm; i++)
                    for (int k = 0; k < 8; k++) {
                        memcpy(&r->rpkt[rpktpos], &r->rfrm[i * 384] + 2 + 48 * k, 46);
                        rpktpos += 46;
                    }
                for (int i = 0; i < rpktpos; i++)
                    r->rpkt[i] ^= 0xAA;
                auto frames = r->mtvza_deframer.work(r->rpkt.data(), rpktpos);
                r->frame_count += frames.size();
                for (auto &f : frames)
                    put(f.data(), 380);
            } else {
                int nbytes_in = r->repack.work(bits, BUFFER_SIZE, bits);
                int nfrm = r->kmssbpsk_def.work(bits, nbytes_in, r->rfrm.data());
                for (int i = 0; i < nfrm; i++)
                    for (int k = 0; k < 8; k++) {
                        memcpy(&r->rpkt[rpktpos], &r->rfrm[i * 1536] + 2 + 192 * k, 188);
                        rpktpos += 188;
                    }
                auto d1 = r->kmss1.work(r->rpkt.data(), rpktpos);
                auto d2 = r->kmss2.work(r->rpkt.data(), rpktpos);
                auto d3 = r->kmss3.work(r->rpkt.data(), rpktpos);
                r->frame_count += d1.size() + d2.size() + d3.size();
                for (int d = 0; d < 3; d++)
                    for (auto &kfrm : (d == 0 ? d1 : (d == 1 ? d2 : d3))) {
                        kmss_frame(kfrm, &final_frames);
                        if (d == 1) {
                            memmove(&final_frames[2][1], &final_frames[2][0], 15040 - 1);
                            memmove(&final_frames[3][1], &final_frames[3][0], 15040 - 1);
                        } else if (d == 2) {
                            memmove(&final_frames[0][1], &final_frames[0][0], 15040 - 1);
                            memmove(&final_frames[1][1], &final_frames[1][0], 15040 - 1);
                        }
                        put(&final_frames[0][0], 4 * 15040);
                    }
            }
        }
        r->pending.erase(r->pending.begin(), r->pending.begin() + used);
        *nbytes = nb;
        stats[0] = r->frame_count;
        stats[1] = (long)r->pending.size();
        return ok;
    }
}
