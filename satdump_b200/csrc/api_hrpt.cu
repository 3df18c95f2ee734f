// Host driver of noaa_hrpt_decoder (B200_FEC_NOAA_HRPT) and meteor_hrpt_decoder (B200_FEC_METEOR_HRPT) inside the decoder object:
// NOAAHRPTDecoderModule::process (plugins/noaa_metop_support/noaa/module_noaa_hrpt_decoder.cpp:26-45) and METEORHRPTDecoderModule::process
// (plugins/meteor_support/meteor/module_meteor_hrpt_decoder.cpp:24-50) over the soft FIFO of Fec. Every push: hard bits, the sync
// candidates of every bit position, the machine's walk, then the gather of what it wrote.
#include "hrpt.cuh"
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
