// Host drivers of the bit-serial decoders without FEC inside the decoder object. noaa_hrpt_decoder (B200_FEC_NOAA_HRPT) and
// meteor_hrpt_decoder (B200_FEC_METEOR_HRPT):
// NOAAHRPTDecoderModule::process (plugins/noaa_metop_support/noaa/module_noaa_hrpt_decoder.cpp:26-45) and METEORHRPTDecoderModule::process
// (plugins/meteor_support/meteor/module_meteor_hrpt_decoder.cpp:24-50) over the soft FIFO of Fec. Every push: hard bits, the sync
// candidates of every bit position, the machine's walk, then the gather of what it wrote. noaa_gac_decoder (B200_FEC_NOAA_GAC) and
// dmsp_rtd_decoder (B200_FEC_DMSP_RTD) follow at the end (gac.cuh).
#include "hrpt.cuh"
#include "gac.cuh"
#include "fec_host.h"
#include <algorithm>

namespace b200
{

struct Hrpt : Framed
{
    bool noaa = false;
    int thr = 0;
    long max_seg = 0;
    DevBuf<uint32_t> hw, cand;
    DevBuf<HrptState> st;
    DevBuf<HrptRec> recs;
    DevBuf<HrptSeg> segs;
    DevBuf<HrptOut> out;
    PinnedBuf<HrptState> h_st;
    PinnedBuf<HrptRec> h_recs;
    PinnedBuf<HrptOut> h_out;

    explicit Hrpt(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
};

Hrpt::Hrpt(Fec &f)
{
    noaa = f.cfg.kind == B200_FEC_NOAA_HRPT;
    thr = f.cfg.deframer_thresold;
    if (noaa)
        B200_REQUIRE(thr >= 0 && thr <= 60, B200_EINVAL, "noaa_hrpt_decoder: deframer_thresold must be 0..60 (got %d)", thr);
    B200_REQUIRE(f.cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for the HRPT decoders");
    // one output unit per NOAA word / METEOR CADU, so that frames_out and b200_chain work unchanged
    f.cadu_bytes = noaa ? 2 : MH_CADU;
    f.geom.chunk = 8192; // the modules' read size: what a stream reader of the decoder hands over at a time (b200_fec_chunk_size)
    const int frame_bits = noaa ? NOAA_WORDS * 10 : MH_PERIOD;
    const long fifo = f.cfg.max_soft + 2L * frame_bits;
    // a push accepts at most one sync per frame length, plus the frame left open by the push before
    max_seg = fifo / (noaa ? NOAA_DATA_BITS : MH_PERIOD) + 4;
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    f.framed_storage(frame_bits, noaa ? fifo / 10 + NOAA_WORDS * 2 : max_seg);
    hw.alloc((size_t)fifo / 32 + 8);
    cand.alloc((size_t)fifo / 32 + 8);
    st.alloc(1);
    recs.alloc((size_t)max_seg);
    segs.alloc((size_t)max_seg);
    out.alloc(1);
    h_st.alloc(1);
    h_recs.alloc((size_t)max_seg);
    h_out.alloc(1);
    reset(f);
}

std::unique_ptr<Framed> hrpt_decoder(Fec &f) { return std::make_unique<Hrpt>(f); }

// a fresh deframer: IDLE / state 0, no inversion, the shifter 0 (the reference leaves it uninitialised: DESIGN §9)
void Hrpt::reset(Fec &f)
{
    Framed::reset(f);
    HrptState &S = *h_st.p;
    memset(&S, 0, sizeof(S));
    S.open = HRPT_NONE;
    S.stale_end = HRPT_NONE;
    S.inv_at = HRPT_NONE;
    f.defr_state_now = 0;
    B200_CUDA(cudaMemcpyAsync(st.p, h_st.p, sizeof(HrptState), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void Hrpt::stats(b200_fec_stats *o) { o->deframer_state = h_st.p->state; }

void Hrpt::process(Fec &f)
{
    if (!begin(f, 1))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, nwords = (have + 31) / 32 + 2;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<1><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    if (noaa) {
        k_sync_cand<<<(unsigned)((have + 255) / 256), 256, 0, stream>>>(hw.p, have, NOAA_SYNC, NOAA_MASK, thr, cand.p);
        k_noaa_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, thr, st.p, recs.p, segs.p, out.p);
    } else {
        k_sync_cand<<<(unsigned)((have + 255) / 256), 256, 0, stream>>>(hw.p, have, MH_ASM, 0xffffffffull, 2, cand.p);
        k_meteor_hrpt_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, st.p, recs.p, segs.p, out.p);
    }
    f.launches += 3;
    B200_CUDA(cudaMemcpyAsync(h_out.p, out.p, sizeof(HrptOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_st.p, st.p, sizeof(HrptState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const HrptOut o = *h_out.p;
    B200_REQUIRE(o.nseg <= max_seg && o.nrec <= max_seg, B200_ESTATE, "internal: %d HRPT frames in one push", std::max(o.nseg, o.nrec));
    if (o.nseg > 0) {
        B200_REQUIRE((size_t)(f.out_frames + o.units) * f.cadu_bytes <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        uint8_t *dst = f.frames_out.p + f.out_frames * f.cadu_bytes;
        for (int y0 = 0; y0 < o.nseg; y0 += 65535) { // (gridDim.y <= 65535; a locked METEOR push of 2^30 bytes has 131 000 frames)
            const unsigned ny = (unsigned)std::min(o.nseg - y0, 65535);
            if (noaa)
                k_noaa_gather<<<dim3((NOAA_WORDS + 255) / 256, ny), 256, 0, stream>>>(hw.p, segs.p + y0, (uint16_t *)dst);
            else
                k_meteor_hrpt_gather<<<dim3(MH_CADU / 256, ny), 256, 0, stream>>>(hw.p, segs.p + y0, dst);
            f.launches++;
        }
    }
    if (o.nrec > 0)
        B200_CUDA(cudaMemcpyAsync(h_recs.p, recs.p, sizeof(HrptRec) * o.nrec, cudaMemcpyDeviceToHost, stream));
    // the FIFO keeps the open frame's bits, else the last 63 bits (the windows of the next tests reach back that far)
    const HrptState &S = *h_st.p;
    long keep_from = have - 63;
    if (S.open != HRPT_NONE)
        keep_from = std::min<long>(keep_from, (long)(S.open + 1 - base_off));
    const long used = std::max<long>(0, keep_from);
    f.keep_soft_tail(used);
    B200_CUDA(cudaEventRecord(f.ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
    base_off += used;
    tail_seen = f.soft_have;
    last_nf = o.nrec;
    f.out_frames += o.units;
    f.total_frames += o.units;
    f.total_bits += have - f.soft_have;
    f.defr_state_now = S.state;
}

long Fec::hrpt_frames(b200_hrpt_frame *out, long cap)
{
    const Hrpt &D = framed_as<Hrpt>("not an HRPT decoder");
    B200_REQUIRE(D.last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", D.last_nf);
    for (long k = 0; k < D.last_nf; k++) {
        out[k].bit = D.h_recs.p[k].bit;
        out[k].inverted = D.h_recs.p[k].inverted;
        out[k].state = D.h_recs.p[k].state;
    }
    return D.last_nf;
}

} // namespace b200

// ---------------------------------------------------------------- noaa_gac_decoder, dmsp_rtd_decoder (gac.cuh)
namespace b200
{

// The bytes module_noaa_gac_decoder.cpp:55-63 XORs onto every frame: bits 0 .. 59 zero, bit 60 + i the PN bit i % 1023, MSB first.
// The PN bits are the recurrence b[i] = b[i-1] ^ b[i-5] ^ b[i-6] ^ b[i-8] ^ b[i-11] from 0 0 0 0 0 1 1 1 0 1 0; its entry 1022 is 0, as
// in the module's table (1023 entries, 1022 initialised).
void gac_pn_bytes(uint8_t *pn)
{
    uint8_t b[GAC_PN_LEN] = {0, 0, 0, 0, 0, 1, 1, 1, 0, 1, 0};
    for (int i = 11; i < GAC_PN_LEN; i++)
        b[i] = b[i - 1] ^ b[i - 5] ^ b[i - 6] ^ b[i - 8] ^ b[i - 11];
    memset(pn, 0, GAC_BYTES);
    for (int i = 0; i < GAC_BYTES * 8 - GAC_PN_ZERO; i++) {
        const int bit = i + GAC_PN_ZERO;
        pn[bit / 8] = (uint8_t)(pn[bit / 8] << 1 | b[i % GAC_PN_LEN]);
    }
}

// NOAAGACDecoderModule::process (module_noaa_gac_decoder.cpp:65-102) over the soft FIFO of Fec: every push's hard bits enter the bit FIFO
// (k_gac_bits), the deframer and frame stage of the convolutional decoders run with cadu_size 33270 and the GAC sync word (no
// derandomiser, no RS), and k_gac_post reverses (backward) and descrambles the frames in the output.
struct Gac : Framed
{
    long dropped = 0; // bit FIFO bits dropped by compaction: FIFO bit q is stream bit q - 32 + dropped
    DevBuf<uint8_t> pn;
    PinnedBuf<FrameRec> h_fr;

    explicit Gac(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
};

Gac::Gac(Fec &f)
{
    b200_fec_cfg &c = f.cfg;
    B200_REQUIRE(c.backward == 0 || c.backward == 1, B200_EINVAL, "noaa_gac_decoder: backward must be 0 or 1 (got %d)", c.backward);
    B200_REQUIRE(c.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for noaa_gac_decoder");
    // BPSK_CCSDS_Deframer(33270, backward ? 0x33c3e4a6 : 0xA116FD71), CADU_PADDING = 33270 % 8 (:20-22): (33270 + 6) / 8 = 4159 bytes
    c.cadu_size = GAC_BITS;
    c.asm_sync = c.backward ? GAC_SYNC_BACKWARD : GAC_SYNC;
    c.nrzm = 0;
    c.derandomize = 0;
    c.derand_after_rs = 0;
    c.derand_start = 0;
    c.rs_i = 0;
    c.rs_dualbasis = 0;
    c.rs_type = 0;
    c.rs_fill_bytes = -1;
    c.rs_usecheck = 0;
    f.st_synced = 12;
    f.cadu_bytes = GAC_BYTES;
    f.geom.chunk = 8192; // the module's read size (BUFSIZE)
    check_device(c.device);
    DeviceGuard g(c.device);
    f.framed_storage(1, 0);
    f.deframer_storage(c.max_soft); // one bit per soft byte
    pn.alloc(GAC_BYTES);
    h_fr.alloc((size_t)f.max_frames_push);
    std::vector<uint8_t> h_pn(GAC_BYTES);
    gac_pn_bytes(h_pn.data());
    B200_CUDA(cudaMemcpy(pn.p, h_pn.data(), GAC_BYTES, cudaMemcpyHostToDevice));
    reset(f);
}

std::unique_ptr<Framed> gac_decoder(Fec &f) { return std::make_unique<Gac>(f); }

void Gac::reset(Fec &f)
{
    f.start_stream(64); // the bit FIFO and the deframer
    Framed::reset(f);
    dropped = 0;
    f.done_bits.clear();
    f.pulled_bits.clear();
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void Gac::process(Fec &f)
{
    if (!begin(f, 1))
        return;
    cudaStream_t stream = f.stream;
    const long fb0 = f.fifo_bits;
    f.compact_fifo(false);
    dropped += fb0 - f.fifo_bits;
    const long nbits = f.soft_have;
    B200_REQUIRE(((f.fifo_bits + nbits + 64) >> 5) + 2 < (long)f.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    const long words = (f.fifo_bits + nbits + 31) / 32 - f.fifo_bits / 32;
    k_gac_bits<<<(unsigned)std::min<long>((words + 7) / 8, 132 * 32), 256, 0, stream>>>(f.softbuf.p, nbits, f.fifo.p, f.fifo_bits);
    f.launches++;
    f.last_bits0 = f.fifo_bits;
    f.last_nbits = nbits;
    const long out0 = f.out_frames;
    f.deframe_and_rs(nbits); // (synchronises the stream)
    const int nf = f.last_nf;
    if (nf > 0) {
        k_gac_post<<<nf, 256, 0, stream>>>(f.frames_out.p + out0 * GAC_BYTES, f.cfg.backward, pn.p);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_fr.p, f.frames.p, sizeof(FrameRec) * nf, cudaMemcpyDeviceToHost, stream));
    }
    f.keep_soft_tail(nbits);
    B200_CUDA(cudaEventRecord(f.ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
    f.t_vit -= f.t_frames;
    std::vector<long> bits(nf);
    for (int k = 0; k < nf; k++) // the frame's last bit: its payload's (33270 - 32)th
        bits[k] = h_fr.p[k].pay_bit + (GAC_BITS - 32) - 1 - 32 + dropped;
    f.note_frame_bits(out0, bits);
    tail_seen = f.soft_have;
    f.total_bits += nbits;
}

// DMSPRTDDecoderModule::process (module_dmsp_rtd_decoder.cpp:34-70) with DMSP_Deframer(150, 2) over the soft FIFO of Fec: hard bits, the
// bitmap of exact sync words, the machine's walk, then the gather of its frames.
struct Dmsp : Framed
{
    long max_seg = 0;
    DevBuf<uint32_t> hw, cand;
    DevBuf<DmspState> st;
    DevBuf<DmspRec> recs, segs;
    DevBuf<DmspOut> out;
    PinnedBuf<DmspState> h_st;
    PinnedBuf<DmspRec> h_segs;
    PinnedBuf<DmspOut> h_out;

    explicit Dmsp(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
};

Dmsp::Dmsp(Fec &f)
{
    B200_REQUIRE(f.cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for dmsp_rtd_decoder");
    f.cadu_bytes = DMSP_BYTES;
    f.geom.chunk = 8192; // the module's read size (BUFFER_SIZE)
    const long fifo = f.cfg.max_soft + 2L * DMSP_BITS;
    max_seg = fifo / DMSP_BITS + 4; // accepted syncs are at least a frame apart
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    f.framed_storage(DMSP_BITS, max_seg);
    hw.alloc((size_t)fifo / 32 + 8);
    cand.alloc((size_t)fifo / 32 + 8);
    st.alloc(1);
    recs.alloc((size_t)max_seg);
    segs.alloc((size_t)max_seg);
    out.alloc(1);
    h_st.alloc(1);
    h_segs.alloc((size_t)max_seg);
    h_out.alloc(1);
    reset(f);
}

std::unique_ptr<Framed> dmsp_decoder(Fec &f) { return std::make_unique<Dmsp>(f); }

// a fresh deframer: NOSYNC, no inversion, the shifter 0
void Dmsp::reset(Fec &f)
{
    Framed::reset(f);
    DmspState &S = *h_st.p;
    memset(&S, 0, sizeof(S));
    S.open = HRPT_NONE;
    f.defr_state_now = 0;
    f.done_bits.clear();
    f.pulled_bits.clear();
    B200_CUDA(cudaMemcpyAsync(st.p, h_st.p, sizeof(DmspState), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void Dmsp::process(Fec &f)
{
    if (!begin(f, 1))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, nwords = (have + 31) / 32 + 2;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<1><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    k_sync_cand<<<(unsigned)((have + 255) / 256), 256, 0, stream>>>(hw.p, have, DMSP_ASM, DMSP_MASK, 0, cand.p);
    k_dmsp_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, st.p, recs.p, segs.p, out.p);
    f.launches += 3;
    B200_CUDA(cudaMemcpyAsync(h_out.p, out.p, sizeof(DmspOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_st.p, st.p, sizeof(DmspState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const DmspOut o = *h_out.p;
    B200_REQUIRE(o.nseg <= max_seg && o.nrec <= max_seg, B200_ESTATE, "internal: %d DMSP frames in one push", std::max(o.nseg, o.nrec));
    const long out0 = f.out_frames;
    if (o.nseg > 0) {
        B200_REQUIRE((size_t)(f.out_frames + o.nseg) * f.cadu_bytes <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        k_dmsp_gather<<<(unsigned)(((long)o.nseg * DMSP_BYTES + 255) / 256), 256, 0, stream>>>(hw.p, segs.p, o.nseg,
                                                                                              f.frames_out.p + f.out_frames * f.cadu_bytes);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_segs.p, segs.p, sizeof(DmspRec) * o.nseg, cudaMemcpyDeviceToHost, stream));
    }
    // the FIFO keeps the open frame's bits, else the last 63 bits (the windows of the next tests reach back 12)
    const DmspState &S = *h_st.p;
    long keep_from = have - 63;
    if (S.open != HRPT_NONE)
        keep_from = std::min<long>(keep_from, (long)(S.open + 1 - base_off));
    const long used = std::max<long>(0, keep_from);
    f.keep_soft_tail(used);
    B200_CUDA(cudaEventRecord(f.ev[1], stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    B200_CUDA(cudaGetLastError());
    cudaEventElapsedTime(&f.t_vit, f.ev[0], f.ev[1]);
    std::vector<long> bits(o.nseg);
    for (int k = 0; k < o.nseg; k++)
        bits[k] = (long)h_segs.p[k].bit + DMSP_PAY + base_off;
    f.note_frame_bits(out0, bits);
    base_off += used;
    tail_seen = f.soft_have;
    last_nf = o.nrec;
    f.out_frames += o.nseg;
    f.total_frames += o.nseg;
    f.total_bits += have - f.soft_have;
    f.defr_state_now = S.state;
}

// frames in frames_out [0, out0) keep their bits; what left frames_out without a pull (b200_chain) is forgotten
void Fec::note_frame_bits(long out0, const std::vector<long> &bits)
{
    if ((long)done_bits.size() > out0)
        done_bits.erase(done_bits.begin(), done_bits.end() - out0);
    done_bits.insert(done_bits.end(), bits.begin(), bits.end());
}

long Fec::frame_bits(long *out, long cap)
{
    B200_REQUIRE(cfg.kind == B200_FEC_NOAA_GAC || cfg.kind == B200_FEC_DMSP_RTD, B200_EINVAL,
                 "frame completion bits are kept by noaa_gac_decoder and dmsp_rtd_decoder only");
    const long n = (long)pulled_bits.size();
    B200_REQUIRE(n <= cap, B200_ESTATE, "output buffer too small: need %ld", n);
    std::copy(pulled_bits.begin(), pulled_bits.end(), out);
    return n;
}

} // namespace b200
