/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref turbo harness: wires the UNMODIFIED reference translation units of the CCSDS turbo decoder (ccsds_turbo.cpp, the
 * deepspace-turbo library, crc_generic.cpp and randomization.cpp, compiled from the reference tree by oracle/Makefile, with oracle/shim
 * standing in for VOLK) the way
 *   CCSDSTurboDecoderModule::process   src-core/pipeline/modules/ccsds/module_ccsds_turbo_decoder.cpp:137-235
 * runs them, and exposes them through a small C ABI for the Python tests (oracle/turbo.py).
 *
 * The module reads past its F-byte buffer when the correlator's position is above F / 2 (memmove(buf, buf + pos, pos)). Here the buffer
 * has 2F bytes and the F bytes behind the frame are zeros, which defines that read.
 *
 * No reference source is copied here: this file only *calls* the reference code. CCSDSTurbo's members are private; the harness reads
 * the interleaver and the component codes through them.
 */
#include <cstring>
#include <memory>
#include <vector>
#include <volk/volk.h>
#define private public
#include "common/codings/turbo/ccsds_turbo.h"
#undef private
#include "common/codings/crc/crc_generic.h"
#include "common/codings/randomization.h"

namespace
{
    using codings::turbo::CCSDSTurbo;

    // the ASM of each rate (module :38-117), MSB first
    const char *asm_hex(int rate)
    {
        switch (rate)
        {
        case 2: return "034776C7272895B0";
        case 3: return "25D5C0CE8990F6C9461BF79C";
        case 4: return "034776C7272895B0FCB88938D8D76A4F";
        default: return "25D5C0CE8990F6C9461BF79CDA2A3F31766F0936B9E40863";
        }
    }
    codings::turbo::turbo_rate_t rate_of(int rate)
    {
        return rate == 2 ? codings::turbo::RATE_1_2 : (rate == 3 ? codings::turbo::RATE_1_3 : (rate == 4 ? codings::turbo::RATE_1_4 : codings::turbo::RATE_1_6));
    }
    int codeword_size(int rate, int base)
    {
        const int n = 8 * base + 4;
        return rate == 2 ? 2 * n : (rate == 3 ? 3 * n : (rate == 4 ? 4 * n : 6 * n));
    }

    struct RefTurbo
    {
        int rate, base, iters, asm_size, cw, F;
        std::vector<float> asm_softs;
        std::unique_ptr<CCSDSTurbo> dec;
        std::unique_ptr<codings::crc::GenericCRC> crc;
        std::vector<int8_t> pend;       // soft bytes not consumed yet (the module's blocking FIFO read waits for them)
        long base_off = 0;              // stream offset of pend[0]
        std::vector<int8_t> buffer_soft; // 2F bytes, the second half zero
        std::vector<float> buffer_floats;
    };
}

extern "C"
{
    /* rate 2, 3, 4, 6 ("1/2" ... "1/6"), base 223 / 446 / 892 / 1115, iterations >= 1 */
    void *ref_turbo_create(int rate, int base, int iters)
    {
        RefTurbo *r = new RefTurbo();
        r->rate = rate;
        r->base = base;
        r->iters = iters;
        r->asm_size = rate == 2 ? 64 : (rate == 3 ? 96 : (rate == 4 ? 128 : 192));
        const char *hex = asm_hex(rate);
        for (int i = 0; i < r->asm_size; i++)
        {
            const char h = hex[i / 4];
            const int nib = h <= '9' ? h - '0' : h - 'A' + 10;
            r->asm_softs.push_back((nib >> (3 - i % 4)) & 1 ? 1.0f : -1.0f);
        }
        r->cw = codeword_size(rate, base);
        r->F = r->cw + r->asm_size;
        r->dec = std::make_unique<CCSDSTurbo>((codings::turbo::turbo_base_t)base, rate_of(rate));
        r->crc = std::make_unique<codings::crc::GenericCRC>(16, 0x1021, 0xFFFF, 0x0, false, false);
        r->buffer_soft.assign(2 * r->F, 0);
        r->buffer_floats.assign(r->F, 0.f);
        return r;
    }
    void ref_turbo_destroy(void *h) { delete (RefTurbo *)h; }
    int ref_turbo_frame_size(void *h) { return ((RefTurbo *)h)->F; }

    /* Appends n soft bytes to the stream and runs the module loop (:170-252) over every frame they complete. Writes the frames the module
       writes (1A CF FC 1D + base bytes, CRC passed) to out (*nbytes of at most cap_bytes) and one record of 6 int64 per frame: stream
       offset of the frame (window start + pos), pos, cor (float bits), swapped, crc_ok, locked. Returns the number of frames, or -1 when a
       capacity is too small. */
    long ref_turbo_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
    {
        RefTurbo *r = (RefTurbo *)h;
        r->pend.insert(r->pend.end(), soft, soft + n);
        const long size = (long)r->pend.size();
        const int F = r->F, A = r->asm_size;
        long o = 0, nf = 0, nb = 0;
        int8_t *buf = r->buffer_soft.data();
        float *fl = r->buffer_floats.data();
        uint8_t frame[1115 + 4];
        while (size - o >= F)
        {
            memcpy(buf, &r->pend[o], F);
            volk_8i_s32f_convert_32f(fl, buf, 127, F);
            int best_pos = 0;
            float best_cor = 0, corr_value = 0;
            bool best_swapped = false;
            for (int pos = 0; pos < F - A; pos++)
            {
                volk_32f_x2_dot_prod_32f(&corr_value, &fl[pos], r->asm_softs.data(), A);
                if (corr_value > best_cor)
                {
                    best_cor = corr_value;
                    best_pos = pos;
                    best_swapped = false;
                }
                if (-corr_value > best_cor)
                {
                    best_cor = -corr_value;
                    best_pos = pos;
                    best_swapped = true;
                }
            }
            if (best_pos != 0)
            {
                if (o + best_pos + F > size)
                    break; // the module's read of the pos missing bytes waits for the next push
                std::memmove(buf, &buf[best_pos], best_pos);
                memcpy(&buf[F - best_pos], &r->pend[o + F], best_pos);
            }
            if (nf >= cap_frames)
                return -1;
            derand_ccsds_soft(&buf[A], r->cw);
            volk_8i_s32f_convert_32f(fl, buf, 127.0, F);
            if (best_swapped)
                for (int i = 0; i < F; i++)
                    fl[i] = -fl[i];
            r->dec->decode(&fl[A], &frame[4], r->iters);
            frame[0] = 0x1a;
            frame[1] = 0xcf;
            frame[2] = 0xfc;
            frame[3] = 0x1d;
            const uint16_t compu = r->crc->compute(&frame[4], r->base - 2);
            const uint16_t local = frame[(r->base + 4) - 2] << 8 | frame[(r->base + 4) - 1];
            const bool ok = compu == local;
            if (ok)
            {
                if (nb + r->base + 4 > cap_bytes)
                    return -1;
                memcpy(out + nb, frame, r->base + 4);
                nb += r->base + 4;
            }
            long long *rec = recs + 6 * nf;
            uint32_t cbits;
            memcpy(&cbits, &best_cor, 4);
            rec[0] = r->base_off + o + best_pos;
            rec[1] = best_pos;
            rec[2] = cbits;
            rec[3] = best_swapped;
            rec[4] = ok;
            rec[5] = best_pos == 0;
            nf++;
            o += best_pos + F;
        }
        r->pend.erase(r->pend.begin(), r->pend.begin() + o);
        r->base_off += o;
        *nbytes = nb;
        return nf;
    }

    /* CCSDSTurbo::encode: base information bytes -> the codeword, packed MSB first (codeword bits / 8 bytes). Returns the byte count. */
    int ref_turbo_encode(int rate, int base, const uint8_t *info, uint8_t *codeword)
    {
        CCSDSTurbo t((codings::turbo::turbo_base_t)base, rate_of(rate));
        std::vector<uint8_t> in(info, info + base);
        t.encode(in.data(), codeword);
        return t.codeword_length() / 8;
    }

    /* The interleaver of CCSDSTurbo (8 base entries) */
    int ref_turbo_perm(int base, int *out)
    {
        CCSDSTurbo t((codings::turbo::turbo_base_t)base, codings::turbo::RATE_1_3);
        memcpy(out, t.d_pi, sizeof(int) * t.d_info_length);
        return t.d_info_length;
    }

    /* One convcode_extrinsic call (libconvcodes.c:355-542) of the upper (lower = 0) or lower code of (rate, base) on `stream` (components x
       (8 base + 4) values) with the a-priori arrays app0 / app1 (8 base values each, replaced by the extrinsic ones) and noise variance
       d_sigma * d_sigma. decision != 0: the decisions go to `decoded` (8 base ints). */
    void ref_turbo_half(int rate, int base, int lower, const double *stream, double *app0, double *app1, int decision, int *decoded)
    {
        CCSDSTurbo t((codings::turbo::turbo_base_t)base, rate_of(rate));
        t_convcode code = lower ? t.d_code2 : t.d_code1;
        const int K = 8 * base, len = code.components * (K + code.memory);
        std::vector<double> s(stream, stream + len);
        double *m[2] = {app0, app1};
        double **mp = m;
        int *d = convcode_extrinsic(s.data(), len, &mp, code, t.d_sigma * t.d_sigma, decision);
        if (d)
        {
            memcpy(decoded, d, sizeof(int) * K);
            free(d);
        }
    }
}
