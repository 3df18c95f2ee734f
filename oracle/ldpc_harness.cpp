/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref LDPC harness: wires the UNMODIFIED reference translation units of the CCSDS LDPC decoder (compiled from the reference
 * tree by oracle/Makefile, with oracle/ldpc_shim + oracle/shim standing in for VOLK and the logger) the way
 *   CCSDSLDPCDecoderModule::process   src-core/pipeline/modules/ccsds/module_ccsds_ldpc_decoder.cpp:134-277 (ldpc_rate "7/8", with and
 *                                     without internal_stream)
 * runs them, and exposes them through a small C ABI for the Python tests (oracle/ldpc.py).
 *
 * The decoder comes from the reference's own get_best_ldpc_decoder (ldpc_decoder.cpp:20-36): no SIMD plugin registers on the empty
 * event bus defined here and the VOLK stand-in names no SIMD extension, so it returns LDPCDecoderGeneric.
 *
 * No reference source is copied here: this file only *calls* the reference classes.
 */
#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>
#include <volk/volk.h>
#include "logger.h"
#include "core/plugin.h"
#include "common/codings/deframing/bpsk_ccsds_deframer.h"
#include "common/codings/generic_correlator.h"
#include "common/codings/ldpc/ccsds_ldpc.h"
#include "common/codings/ldpc/make_ccsds.h"
#include "common/codings/randomization.h"
#include "common/codings/rotation.h"
#include "utils/binary.h"

std::shared_ptr<slog::Logger> logger = std::make_shared<slog::Logger>();
namespace satdump
{
    std::shared_ptr<EventBus> eventBus = std::make_shared<EventBus>();
}

namespace
{
    constexpr int ASM_BITS = 32, CW = 8160, F = CW + ASM_BITS; // d_ldpc_asm_size, d_ldpc_codeword_size, d_ldpc_frame_size (:84-91)

    struct RefLdpc
    {
        int constellation, iterations, derandomize;
        int cadu_bytes = 1024;
        std::unique_ptr<deframing::BPSK_CCSDS_Deframer> deframer; // internal_stream (:100-113)
        std::unique_ptr<CorrelatorGeneric> correlator;
        std::unique_ptr<codings::ldpc::CCSDSLDPC> dec;
        std::vector<int8_t> pend;           // soft bytes not consumed yet (the module's blocking read_data waits for them)
        long base = 0;                      // stream offset of pend[0]
        std::vector<int8_t> soft_buffer;    // :115
        std::vector<uint8_t> ldpc_output;   // :118, value-initialised here: bits 8158 / 8159 of every frame are never written
        std::vector<uint8_t> deframer_buffer;
    };

    dsp::constellation_type_t cons_of(int c) { return c == 0 ? dsp::BPSK : (c == 1 ? dsp::QPSK : dsp::OQPSK); }
}

extern "C"
{
    /* constellation 0 bpsk, 1 qpsk, 2 oqpsk ("constellation"); iterations ("ldpc_iterations"); derandomize ("derandomize");
       internal_cadu_size > 0: "internal_stream" with that "internal_cadu_size" (a multiple of 8) and "internal_asm" */
    void *ref_ldpc_create(int constellation, int iterations, int derandomize, int internal_cadu_size, unsigned internal_asm)
    {
        RefLdpc *r = new RefLdpc();
        r->constellation = constellation;
        r->iterations = iterations;
        r->derandomize = derandomize;
        r->dec = std::make_unique<codings::ldpc::CCSDSLDPC>(codings::ldpc::RATE_7_8, 0);
        r->correlator = std::make_unique<CorrelatorGeneric>(cons_of(constellation), satdump::unsigned_to_bitvec<uint32_t>(0x1acffc1d), F);
        r->soft_buffer.resize(F);
        r->ldpc_output.assign(CW * r->dec->simd(), 0);
        r->deframer_buffer.assign(F * 64, 0);
        if (internal_cadu_size > 0)
        {
            r->deframer = std::make_unique<deframing::BPSK_CCSDS_Deframer>(internal_cadu_size, internal_asm);
            r->cadu_bytes = internal_cadu_size / 8;
        }
        return r;
    }
    void ref_ldpc_destroy(void *h) { delete (RefLdpc *)h; }

    /* Appends n soft bytes to the stream and runs the module loop over every LDPC frame they complete. Writes what the module writes (the
       1024-byte CADUs, or with internal_stream the inner frames of the deframer) to out (*nbytes of at most cap_bytes) and one record of
       8 int64 per LDPC frame: stream offset of the frame (window start + pos), pos, correlator_corr (float bits), phase, swap, ldpc_corr,
       correlator_locked, the deframer's state after the frame's info bits (internal_stream, else 0). Returns the number of LDPC frames, or
       -1 when a capacity is too small. */
    long ref_ldpc_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
    {
        RefLdpc *r = (RefLdpc *)h;
        r->pend.insert(r->pend.end(), soft, soft + n);
        const long size = (long)r->pend.size();
        long o = 0, nf = 0, nb = 0;
        int8_t *sb = r->soft_buffer.data();
        while (size - o >= F)
        {
            phase_t phase;
            bool swap;
            float cor;
            memcpy(sb, &r->pend[o], F);
            int pos = r->correlator->correlate(sb, phase, swap, cor, F);
            if (pos != 0)
            {
                if (o + pos + F > size)
                    break; // the module's read_data of the pos missing bytes waits for the next push
                memmove(sb, &sb[pos], F - pos);
                memcpy(&sb[F - pos], &r->pend[o + F], pos);
            }
            if (nf >= cap_frames)
                return -1;
            if (r->constellation == 2)
            {
                rotate_soft(sb, F, phase, false);
                if (swap)
                {
                    int8_t last_q_oqpsk = 0;
                    for (int i = (F / 2) - 1; i >= 0; i--)
                    {
                        int8_t back = sb[i * 2 + 1];
                        sb[i * 2 + 1] = last_q_oqpsk;
                        last_q_oqpsk = back;
                    }
                }
            }
            else
                rotate_soft(sb, F, phase, swap);
            if (r->derandomize)
                derand_ccsds_soft(&sb[ASM_BITS], CW);
            const int corr = r->dec->decode(&sb[ASM_BITS], r->ldpc_output.data(), r->iterations);
            uint8_t *db = r->deframer_buffer.data();
            int defr_state = 0;
            if (r->deframer)
            {
                const int frames = r->deframer->work(r->ldpc_output.data(), r->dec->data_length(), db); // (:233-242)
                if (nb + (long)frames * r->cadu_bytes > cap_bytes)
                    return -1;
                memcpy(out + nb, db, (size_t)frames * r->cadu_bytes);
                nb += (long)frames * r->cadu_bytes;
                defr_state = r->deframer->getState();
            }
            else
            {
                for (int i = 0; i < CW; i++)
                    db[i / 8] = db[i / 8] << 1 | r->ldpc_output[i];
                const uint32_t sync = 0x1acffc1d;
                if (nb + 1024 > cap_bytes)
                    return -1;
                memcpy(out + nb, &sync, 4);
                memcpy(out + nb + 4, db, CW / 8);
                nb += 1024;
            }
            long long *rec = recs + 8 * nf;
            uint32_t cbits;
            memcpy(&cbits, &cor, 4);
            rec[0] = r->base + o + pos;
            rec[1] = pos;
            rec[2] = cbits;
            rec[3] = phase;
            rec[4] = swap;
            rec[5] = corr;
            rec[6] = pos == 0;
            rec[7] = defr_state;
            nf++;
            o += pos + F;
        }
        r->pend.erase(r->pend.begin(), r->pend.begin() + o);
        r->base += o;
        *nbytes = nb;
        return nf;
    }

    /* CCSDSLDPC::decode alone (ccsds_ldpc.cpp:76-123): 8160 soft bytes in (8158 used), 8160 bytes out (the first 8158 written). */
    int ref_ldpc_decode(void *h, const int8_t *codeword, uint8_t *out, int iterations)
    {
        RefLdpc *r = (RefLdpc *)h;
        std::vector<int8_t> in(codeword, codeword + CW);
        return r->dec->decode(in.data(), out, iterations);
    }

    /* The parity-check matrix make_r78_code() builds (make_ccsds.cpp:394-433): the column indices of rows 0..1021, 32 per row, ascending
       within a row. Returns the number of rows. */
    int ref_ldpc_matrix(int *cols, int cap_rows)
    {
        codings::ldpc::Sparse_matrix H = codings::ldpc::ccsds_78::make_r78_code();
        const int rows = (int)H.get_n_rows();
        if (rows > cap_rows)
            return -1;
        for (int row = 0; row < rows; row++)
        {
            std::vector<uint32_t> c = H.get_cols_from_row(row);
            std::sort(c.begin(), c.end());
            if (c.size() != 32)
                return -2;
            for (int k = 0; k < 32; k++)
                cols[row * 32 + k] = (int)c[k];
        }
        return rows;
    }
}
