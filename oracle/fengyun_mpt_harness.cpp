/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref FengYun-3 MPT harness: wires the UNMODIFIED reference blocks viterbi::Viterbi1_2 (common/codings/viterbi/viterbi_1_2.cpp
 * with cc_decoder.cpp, cc_encoder.cpp, utils.cpp), rotate_soft (common/codings/rotation.cpp), fengyun3::FengyunDiff
 * (plugins/fengyun3_support/fengyun3/diff.cpp), deframing::BPSK_CCSDS_Deframer, derand_ccsds and reedsolomon::ReedSolomon (RS223,
 * libcorrect), compiled from the reference tree by oracle/fengyun_mpt.mk, the way
 *   fengyun3::FengyunMPTDecoderModule::process   plugins/fengyun3_support/fengyun3/module_fengyun_mpt_decoder.cpp:42-135
 * runs them, and exposes them through a small C ABI for the Python tests (oracle/fengyun_mpt.py). The module file pulls in ImGui and the
 * pipeline base, so its loop is restated here as wiring.
 *
 * Definitions made here (as in fengyun_harness.cpp):
 *   - Reads: the module reads 16384 soft bytes at a time from the start of the stream. run() collects the bytes it is given and runs the
 *     loop body once per complete read; a partial read waits for the next run(). A short last read is never decoded.
 *   - With shift = 1 the split reads soft_buffer[16384] and [16385], past the module's 16384-byte new[]: this harness's buffer has two
 *     more bytes, always 0 (so Q past the read is ~0).
 *   - This library's operator new returns zeroed storage. Viterbi1_2's shift-1 decode reads soft_buffer[8192], which work() never
 *     writes: it keeps the 128 of the lock's memset.
 *   - The module's shift test reads viterbi1.getState() twice (module :81); it is kept as written.
 *
 * No reference source is copied here: this file only *calls* the reference code.
 */
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>
#include "common/codings/viterbi/viterbi_1_2.h"
#include "common/codings/rotation.h"
#include "common/codings/deframing/bpsk_ccsds_deframer.h"
#include "common/codings/randomization.h"
#include "common/codings/reedsolomon/reedsolomon.h"
#include "fengyun3/diff.h"

void *operator new(size_t n)
{
    void *p = calloc(n ? n : 1, 1);
    if (!p)
        throw std::bad_alloc();
    return p;
}
void *operator new[](size_t n) { return operator new(n); }
void operator delete(void *p) noexcept { free(p); }
void operator delete(void *p, size_t) noexcept { free(p); }
void operator delete[](void *p) noexcept { free(p); }
void operator delete[](void *p, size_t) noexcept { free(p); }

namespace
{
    constexpr int BUFFER_SIZE = 8192;

    struct RefMpt
    {
        viterbi::Viterbi1_2 viterbi1, viterbi2;
        deframing::BPSK_CCSDS_Deframer deframer;
        fengyun3::FengyunDiff diff;
        reedsolomon::ReedSolomon rs{reedsolomon::RS223};
        std::vector<int8_t> soft_buffer = std::vector<int8_t>(BUFFER_SIZE * 2 + 2), i_soft = std::vector<int8_t>(BUFFER_SIZE),
                            q_soft = std::vector<int8_t>(BUFFER_SIZE);
        std::vector<uint8_t> v1_out = std::vector<uint8_t>(BUFFER_SIZE), v2_out = std::vector<uint8_t>(BUFFER_SIZE),
                             diff_out = std::vector<uint8_t>(BUFFER_SIZE * 20), frame_buffer = std::vector<uint8_t>(1024 * 10);
        int shift = 0, noSyncRuns = 0, viterbiNoSyncRun = 0;
        bool invert_branches = false;
        int errors[4] = {0, 0, 0, 0};
        long reads = 0;
        std::vector<uint8_t> pending;
        RefMpt(float ber, int outsync)
            : viterbi1(ber, outsync, BUFFER_SIZE, {PHASE_0, PHASE_90}), viterbi2(ber, outsync, BUFFER_SIZE, {PHASE_0, PHASE_90})
        {
        }
    };
}

extern "C"
{
    void *ref_mpt_create(float ber, int outsync) { return new RefMpt(ber, outsync); }
    void ref_mpt_destroy(void *h) { delete (RefMpt *)h; }

    /* Appends n soft bytes and runs the module loop over every whole read. Frames (1024 bytes) go to out (cap bytes, *nbytes written);
       one record of 10 floats per read to recs (cap_recs records, *nrecs written): shift, invert_branches, v1, v2, viterbi1 state,
       viterbi2 state, viterbi1 ber, viterbi2 ber, deframer state, RS errors[0] of the read's last frame (-2: none). stats: [0] rs_avg,
       [1] deframer lock, [2] reads so far. Returns 0, or -1 when a buffer is too small. */
    int ref_mpt_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap, long *nbytes, float *recs, long cap_recs, long *nrecs, long *stats)
    {
        RefMpt *r = (RefMpt *)h;
        r->pending.insert(r->pending.end(), (const uint8_t *)soft, (const uint8_t *)soft + n);
        long nb = 0, nr = 0, used = 0;
        int ok = 0;
        while ((long)r->pending.size() - used >= BUFFER_SIZE * 2) {
            int8_t *buf = r->soft_buffer.data();
            memcpy(buf, r->pending.data() + used, BUFFER_SIZE * 2);
            used += BUFFER_SIZE * 2;
            rotate_soft(buf, BUFFER_SIZE * 2, PHASE_0, true);
            for (int i = 0; i < BUFFER_SIZE; i++) {
                r->i_soft[i] = buf[(i + r->shift) * 2 + 0];
                r->q_soft[i] = ~buf[(i + r->shift) * 2 + 1];
            }
            rotate_soft(r->i_soft.data(), BUFFER_SIZE, PHASE_0, true);
            rotate_soft(r->q_soft.data(), BUFFER_SIZE, PHASE_0, true);
            const int v1 = r->viterbi1.work(r->i_soft.data(), BUFFER_SIZE, r->v1_out.data());
            const int v2 = r->viterbi2.work(r->q_soft.data(), BUFFER_SIZE, r->v2_out.data());
            const int vout = std::min(v1, v2);
            if (r->viterbi1.getState() == 0 || r->viterbi1.getState() == 0) { // (sic, module :81)
                r->viterbiNoSyncRun++;
                if (r->viterbiNoSyncRun >= 10)
                    r->shift = r->shift == 0 ? 1 : 0;
            }
            r->diff.work2(r->invert_branches ? r->v1_out.data() : r->v2_out.data(), r->invert_branches ? r->v2_out.data() : r->v1_out.data(), vout,
                          r->diff_out.data());
            float last_rs = -2;
            if (v1 > 0 && v2 > 0) {
                const int frames = r->deframer.work(r->diff_out.data(), vout * 2, r->frame_buffer.data());
                if (r->deframer.getState() == r->deframer.STATE_NOSYNC) {
                    if (++r->noSyncRuns >= 10) {
                        r->invert_branches = !r->invert_branches;
                        r->noSyncRuns = 0;
                    }
                } else
                    r->noSyncRuns = 0;
                for (int i = 0; i < frames; i++) {
                    uint8_t *cadu = &r->frame_buffer[i * 1024];
                    derand_ccsds(&cadu[4], 1024 - 4);
                    r->rs.decode_interlaved(&cadu[4], true, 4, r->errors);
                    if (nb + 1024 > cap)
                        ok = -1;
                    else {
                        memcpy(out + nb, cadu, 1024);
                        nb += 1024;
                    }
                    last_rs = r->errors[0];
                }
            }
            if (nr >= cap_recs)
                ok = -1;
            else {
                float *q = recs + nr * 10;
                q[0] = r->shift;
                q[1] = r->invert_branches;
                q[2] = v1;
                q[3] = v2;
                q[4] = r->viterbi1.getState();
                q[5] = r->viterbi2.getState();
                q[6] = r->viterbi1.ber();
                q[7] = r->viterbi2.ber();
                q[8] = r->deframer.getState();
                q[9] = last_rs;
                nr++;
            }
            r->reads++;
        }
        r->pending.erase(r->pending.begin(), r->pending.begin() + used);
        *nbytes = nb;
        *nrecs = nr;
        stats[0] = (r->errors[0] + r->errors[1] + r->errors[2] + r->errors[3]) / 4;
        stats[1] = r->deframer.getState() == r->deframer.STATE_SYNCED;
        stats[2] = r->reads;
        return ok;
    }
}
