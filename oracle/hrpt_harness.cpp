/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * oracle/_ref HRPT harness: wires the UNMODIFIED reference deframers noaa::NOAADeframer (noaa_metop_support/noaa/noaa_deframer.cpp) and
 * meteor::CADUDeframer (meteor_support/meteor/deframer.cpp), compiled from the reference tree by oracle/Makefile, the way
 *   noaa::NOAAHRPTDecoderModule::process      plugins/noaa_metop_support/noaa/module_noaa_hrpt_decoder.cpp:26-45
 *   meteor::METEORHRPTDecoderModule::process  plugins/meteor_support/meteor/module_meteor_hrpt_decoder.cpp:24-50
 * run them (8192-byte reads, the last read of a piece shorter), and exposes them through a small C ABI for the Python tests
 * (oracle/hrpt.py). The module files pull in ImGui and the pipeline base, so their loops are restated here as wiring.
 *
 * Definitions made here:
 *   - Both deframers leave their shifter uninitialised (a user-provided constructor that does not set it). Each is constructed over
 *     zeroed storage, so the shifter starts at 0; the GPU decoder defines it the same way.
 *   - Records: with `records` set, work() is called once per soft byte, which leaves the machines' behaviour unchanged. An accepted
 *     sync is seen as NOAA's six fixed words or a step of METEOR's getFrameCount(); the state that accepted it is getState() before
 *     that bit. Its inversion is read from a copy of the deframer fed with zero soft bytes (bit 0): the copy's first NOAA word is
 *     0x3FF, or its METEOR frame's byte 4 is 0xFF, exactly when the frame is inverted. Without `records` each read is one work() call,
 *     as in the module.
 *
 * No reference source is copied here: this file only *calls* the reference code.
 */
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>
#include "noaa/noaa_deframer.h"
#include "meteor/deframer.h"

namespace
{
    constexpr int BUFSIZE = 8192, NOAA_WORDS = 11090;

    template <class T, class... A> T *make_zeroed(A... a)
    {
        void *m = std::calloc(1, sizeof(T));
        return new (m) T(a...);
    }
    template <class T> void free_zeroed(T *p)
    {
        if (p) {
            p->~T();
            std::free(p);
        }
    }

    struct RefHrpt
    {
        int meteor = 0;
        noaa::NOAADeframer *noaa = nullptr;
        meteor::CADUDeframer *def = nullptr;
        long stream_bits = 0; // soft bytes consumed so far
        long units = 0;       // NOAA words / METEOR frames written so far
    };
}

extern "C"
{
    /* meteor 0: noaa_hrpt_decoder with deframer_thresold thr; meteor 1: meteor_hrpt_decoder */
    void *ref_hrpt_create(int meteor, int thr)
    {
        RefHrpt *r = new RefHrpt();
        r->meteor = meteor;
        if (meteor)
            r->def = make_zeroed<meteor::CADUDeframer>();
        else
            r->noaa = make_zeroed<noaa::NOAADeframer>(thr);
        return r;
    }
    void ref_hrpt_destroy(void *h)
    {
        RefHrpt *r = (RefHrpt *)h;
        free_zeroed(r->noaa);
        free_zeroed(r->def);
        delete r;
    }

    /* Appends n soft bytes to the stream and runs the module loop over them. Writes what the module writes (NOAA: little-endian uint16
       words; METEOR: 1024-byte CADUs) to out (cap bytes, *nbytes written); with `records`, one record per accepted sync to recs (3 int64:
       stream bit index of the sync's last bit, inverted, the state that accepted it; at most rcap). stats[0] = words / frames written so
       far, stats[1] = getState() (METEOR; NOAA 0). Returns the number of records, or -1 when a buffer is too small. */
    long ref_hrpt_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap, long *nbytes, int records, long long *recs, long rcap,
                      long long *stats)
    {
        RefHrpt *r = (RefHrpt *)h;
        long nb = 0, nrec = 0;
        bool ok = true;
        auto put = [&](const void *src, long len) {
            if (nb + len > cap) {
                ok = false;
                return;
            }
            std::memcpy(out + nb, src, len);
            nb += len;
        };
        auto record = [&](long bit, int inv, int state) {
            if (nrec >= rcap) {
                ok = false;
                return;
            }
            recs[3 * nrec] = bit;
            recs[3 * nrec + 1] = inv;
            recs[3 * nrec + 2] = state;
            nrec++;
        };
        std::vector<int8_t> zeros(8160, 0);
        for (long a = 0; a < n && ok; a += BUFSIZE) {
            const int len = (int)std::min<long>(BUFSIZE, n - a);
            int8_t *buf = const_cast<int8_t *>(soft + a);
            if (!r->meteor) {
                if (!records) {
                    std::vector<uint16_t> w = r->noaa->work(buf, len);
                    put(w.data(), (long)w.size() * 2);
                    r->units += (long)w.size();
                    continue;
                }
                for (int i = 0; i < len && ok; i++) {
                    std::vector<uint16_t> w = r->noaa->work(buf + i, 1);
                    if (w.size() == 6) {
                        noaa::NOAADeframer probe = *r->noaa;
                        record(r->stream_bits + i, probe.work(zeros.data(), 10)[0] == 0x3FF, 0);
                    }
                    put(w.data(), (long)w.size() * 2);
                    r->units += (long)w.size();
                }
            } else {
                auto emit = [&](const std::vector<std::array<uint8_t, meteor::CADU_SIZE>> &fr) {
                    for (const auto &f : fr)
                        put(f.data(), meteor::CADU_SIZE);
                    r->units += (long)fr.size();
                };
                if (!records) {
                    emit(r->def->work(buf, len));
                    continue;
                }
                for (int i = 0; i < len && ok; i++) {
                    const int state = r->def->getState(), count = r->def->getFrameCount();
                    emit(r->def->work(buf + i, 1));
                    if (r->def->getFrameCount() != count) {
                        meteor::CADUDeframer probe = *r->def;
                        record(r->stream_bits + i, probe.work(zeros.data(), 8160).at(0)[4] == 0xFF, state);
                    }
                }
            }
            r->stream_bits += len;
        }
        *nbytes = nb;
        stats[0] = r->units;
        stats[1] = r->meteor ? r->def->getState() : 0;
        return ok ? nrec : -1;
    }
}
