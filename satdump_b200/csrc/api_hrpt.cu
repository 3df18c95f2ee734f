// Host drivers of the decoders without a correlator, inside the decoder object.
//   The sync walks: noaa_hrpt_decoder (B200_FEC_NOAA_HRPT), meteor_hrpt_decoder (B200_FEC_METEOR_HRPT) and dmsp_rtd_decoder
//   (B200_FEC_DMSP_RTD), that is NOAAHRPTDecoderModule::process (plugins/noaa_metop_support/noaa/module_noaa_hrpt_decoder.cpp:26-45),
//   METEORHRPTDecoderModule::process (plugins/meteor_support/meteor/module_meteor_hrpt_decoder.cpp:24-50) and DMSPRTDDecoderModule::process
//   (module_dmsp_rtd_decoder.cpp:34-70) with DMSP_Deframer(150, 2), over the soft FIFO of Fec. Every push: hard bits, the sync candidates
//   of every bit position, the machine's walk (hrpt.cuh, gac.cuh), then the gather of the frames it accepted.
//   The bit stages: aqua_db_decoder (B200_FEC_AQUA_DB) and noaa_gac_decoder (B200_FEC_NOAA_GAC), that is AquaDBDecoderModule::process
//   (plugins/eos_support/aqua/module_aqua_db_decoder.cpp:27-83) and NOAAGACDecoderModule::process (module_noaa_gac_decoder.cpp:65-102).
//   Every push: its bits into the bit FIFO, then the deframer and frame stage of the convolutional decoders.
//   The METEOR-M X-band dump decoder: meteor_xband_decoder (B200_FEC_METEOR_XBAND), that is MeteorXBandDecoderModule::process
//   (plugins/meteor_support/meteor/module_meteor_xband_decoder.cpp:62-212), two-level: a record walk and packet gather, then the inner
//   deframers' walk over the packet FIFO and the frame gather (xband.cuh).
#include "hrpt.cuh"
#include "gac.cuh"
#include "xband.cuh"
#include "fec_host.h"
#include <algorithm>

namespace b200
{

struct SyncWalk : Framed
{
    enum Machine { NOAA, METEOR, DMSP } m;
    int thr = 0; // NOAA: deframer_thresold
    long max_seg = 0;
    DevBuf<uint32_t> hw, cand;
    DevBuf<HrptRec> recs;             // every accepted sync
    DevBuf<HrptSeg> segs;             // NOAA / METEOR: what the gathers write
    DevBuf<HrptRec> dmsp_segs;        // DMSP: the syncs of the frames its gather writes
    DevBuf<HrptOut> out;
    DevBuf<HrptState> st;             // the machine between pushes: NOAA / METEOR ...
    DevBuf<DmspState> dmsp_st;        // ... DMSP
    PinnedBuf<HrptState> h_st;
    PinnedBuf<DmspState> h_dmsp_st;
    PinnedBuf<HrptRec> h_recs;        // NOAA / METEOR: the records of the last push; DMSP: the syncs of its frames
    PinnedBuf<HrptOut> h_out;

    explicit SyncWalk(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
    void stats(b200_fec_stats *o) override;
    long records(b200_hrpt_frame *out, long cap) const; // of the last push
};

SyncWalk::SyncWalk(Fec &f)
    : m(f.cfg.kind == B200_FEC_NOAA_HRPT ? NOAA : (f.cfg.kind == B200_FEC_METEOR_HRPT ? METEOR : DMSP))
{
    if (m == NOAA) {
        thr = f.cfg.deframer_thresold;
        B200_REQUIRE(thr >= 0 && thr <= 60, B200_EINVAL, "noaa_hrpt_decoder: deframer_thresold must be 0..60 (got %d)", thr);
    }
    B200_REQUIRE(f.cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for %s", m == DMSP ? "dmsp_rtd_decoder" : "the HRPT decoders");
    // one output unit per NOAA word / METEOR CADU / DMSP frame, so that frames_out and b200_chain work unchanged
    f.cadu_bytes = m == NOAA ? 2 : (m == METEOR ? MH_CADU : DMSP_BYTES);
    f.geom.chunk = 8192; // the modules' read size: what a stream reader of the decoder hands over at a time (b200_fec_chunk_size)
    const int frame_bits = m == NOAA ? NOAA_WORDS * 10 : (m == METEOR ? MH_PERIOD : DMSP_BITS);
    const long fifo = f.cfg.max_soft + 2L * frame_bits;
    // a push accepts at most one sync per frame length (NOAA: per frame's data bits), plus the frame left open by the push before
    max_seg = fifo / (m == NOAA ? NOAA_DATA_BITS : frame_bits) + 4;
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    f.framed_storage(frame_bits, m == NOAA ? fifo / 10 + NOAA_WORDS * 2 : max_seg);
    hw.alloc((size_t)fifo / 32 + 8);
    cand.alloc((size_t)fifo / 32 + 8);
    recs.alloc((size_t)max_seg);
    out.alloc(1);
    h_recs.alloc((size_t)max_seg);
    h_out.alloc(1);
    if (m == DMSP) {
        dmsp_segs.alloc((size_t)max_seg);
        dmsp_st.alloc(1);
        h_dmsp_st.alloc(1);
    } else {
        segs.alloc((size_t)max_seg);
        st.alloc(1);
        h_st.alloc(1);
    }
    reset(f);
}

std::unique_ptr<Framed> sync_walk_decoder(Fec &f) { return std::make_unique<SyncWalk>(f); }

// a fresh deframer: NOSYNC / IDLE / state 0, no inversion, the shifter 0 (the NOAA reference leaves it uninitialised: DESIGN §9)
void SyncWalk::reset(Fec &f)
{
    Framed::reset(f);
    f.defr_state_now = 0;
    if (m == DMSP) {
        memset(h_dmsp_st.p, 0, sizeof(DmspState));
        h_dmsp_st.p->open = HRPT_NONE;
        B200_CUDA(cudaMemcpyAsync(dmsp_st.p, h_dmsp_st.p, sizeof(DmspState), cudaMemcpyHostToDevice, f.stream));
    } else {
        HrptState &S = *h_st.p;
        memset(&S, 0, sizeof(S));
        S.open = S.stale_end = S.inv_at = HRPT_NONE;
        B200_CUDA(cudaMemcpyAsync(st.p, h_st.p, sizeof(HrptState), cudaMemcpyHostToDevice, f.stream));
    }
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

// NOAA / METEOR report the state the last walk left, also when its push failed after the walk; DMSP reports defr_state_now, the state
// after its last complete push
void SyncWalk::stats(b200_fec_stats *o)
{
    if (m != DMSP)
        o->deframer_state = h_st.p->state;
}

void SyncWalk::process(Fec &f)
{
    if (!begin(f, 1))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have, nwords = (have + 31) / 32 + 2;
    const unsigned cand_blocks = (unsigned)((have + 255) / 256);
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<1><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    switch (m) {
    case NOAA:
        k_sync_cand<<<cand_blocks, 256, 0, stream>>>(hw.p, have, NOAA_SYNC, NOAA_MASK, thr, cand.p);
        k_noaa_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, thr, st.p, recs.p, segs.p, out.p);
        break;
    case METEOR:
        k_sync_cand<<<cand_blocks, 256, 0, stream>>>(hw.p, have, MH_ASM, 0xffffffffull, 2, cand.p);
        k_meteor_hrpt_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, st.p, recs.p, segs.p, out.p);
        break;
    case DMSP:
        k_sync_cand<<<cand_blocks, 256, 0, stream>>>(hw.p, have, DMSP_ASM, DMSP_MASK, 0, cand.p);
        k_dmsp_walk<<<1, 32, 0, stream>>>(hw.p, cand.p, have, base_off, dmsp_st.p, recs.p, dmsp_segs.p, out.p);
        break;
    }
    f.launches += 3;
    B200_CUDA(cudaMemcpyAsync(h_out.p, out.p, sizeof(HrptOut), cudaMemcpyDeviceToHost, stream));
    if (m == DMSP)
        B200_CUDA(cudaMemcpyAsync(h_dmsp_st.p, dmsp_st.p, sizeof(DmspState), cudaMemcpyDeviceToHost, stream));
    else
        B200_CUDA(cudaMemcpyAsync(h_st.p, st.p, sizeof(HrptState), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const HrptOut o = *h_out.p;
    B200_REQUIRE(o.nseg <= max_seg && o.nrec <= max_seg, B200_ESTATE, "internal: %d %s frames in one push", std::max(o.nseg, o.nrec),
                 m == DMSP ? "DMSP" : "HRPT");
    if (o.nseg > 0) {
        B200_REQUIRE((size_t)(f.out_frames + o.units) * f.cadu_bytes <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        uint8_t *dst = f.frames_out.p + f.out_frames * f.cadu_bytes;
        if (m == DMSP) {
            k_dmsp_gather<<<(unsigned)(((long)o.nseg * DMSP_BYTES + 255) / 256), 256, 0, stream>>>(hw.p, dmsp_segs.p, o.nseg, dst);
            f.launches++;
        } else
            for (int y0 = 0; y0 < o.nseg; y0 += 65535) { // (gridDim.y <= 65535; a locked METEOR push of 2^30 bytes has 131 000 frames)
                const unsigned ny = (unsigned)std::min(o.nseg - y0, 65535);
                if (m == NOAA)
                    k_noaa_gather<<<dim3((NOAA_WORDS + 255) / 256, ny), 256, 0, stream>>>(hw.p, segs.p + y0, (uint16_t *)dst);
                else
                    k_meteor_hrpt_gather<<<dim3(MH_CADU / 256, ny), 256, 0, stream>>>(hw.p, segs.p + y0, dst);
                f.launches++;
            }
    }
    const int nkeep = m == DMSP ? o.nseg : o.nrec;
    if (nkeep > 0)
        B200_CUDA(cudaMemcpyAsync(h_recs.p, m == DMSP ? dmsp_segs.p : recs.p, sizeof(HrptRec) * nkeep, cudaMemcpyDeviceToHost, stream));
    // the FIFO keeps the open frame's bits, else the last 63 bits (the windows of the next tests reach back that far)
    const long long open = m == DMSP ? h_dmsp_st.p->open : h_st.p->open;
    long keep_from = have - 63;
    if (open != HRPT_NONE)
        keep_from = std::min<long>(keep_from, (long)(open + 1 - base_off));
    const long used = std::max<long>(0, keep_from);
    f.keep_soft_tail(used);
    end(f);
    if (m == DMSP) {
        std::vector<long> bits(o.nseg);
        for (int k = 0; k < o.nseg; k++) // the frame's last bit
            bits[k] = (long)h_recs.p[k].bit + DMSP_PAY + base_off;
        f.note_frame_bits(f.out_frames, bits);
    }
    base_off += used;
    tail_seen = f.soft_have;
    last_nf = o.nrec;
    f.out_frames += o.units;
    f.total_frames += o.units;
    f.total_bits += have - f.soft_have;
    f.defr_state_now = m == DMSP ? h_dmsp_st.p->state : h_st.p->state;
}

long SyncWalk::records(b200_hrpt_frame *out, long cap) const
{
    B200_REQUIRE(m != DMSP, B200_EINVAL, "not an HRPT decoder");
    B200_REQUIRE(last_nf <= cap, B200_ESTATE, "output buffer too small: need %ld records", last_nf);
    for (long k = 0; k < last_nf; k++) {
        out[k].bit = h_recs.p[k].bit;
        out[k].inverted = h_recs.p[k].inverted;
        out[k].state = h_recs.p[k].state;
    }
    return last_nf;
}

// ---------------------------------------------------------------- aqua_db_decoder, noaa_gac_decoder

// The soft FIFO of aqua_db_decoder starts with the previous push's last symbol (at a stream's start, the symbol (0, 0): both rails'
// NRZMDiff::lastBit = 0).
constexpr int AQUA_LEAD = 2;

// Soft pairs (I, Q) -> decoded bits. The module's interleaved hard bits are h(2s) = Q_s > 0 (rail A, demod >> 1) and h(2s + 1) = I_s > 0
// (rail B, demod & 1), that is h(k) = soft[k ^ 1] > 0; each rail's NRZMDiff::decode_bits XORs a bit with the same rail's bit one symbol
// earlier, so decoded bit j = h(j + 2) ^ h(j), with symbol 0 of `soft` the carried one. One warp writes one word of the MSB-first bit
// FIFO, which the stream enters at bit fifo_bits0 (the bits in front of it in the first word are kept).
__global__ void __launch_bounds__(256) k_aqua_bits(const int8_t *__restrict__ soft, long nbits, uint32_t *__restrict__ fifo, long fifo_bits0)
{
    const int lane = threadIdx.x & 31;
    const long w0 = fifo_bits0 >> 5, w1 = (fifo_bits0 + nbits + 31) >> 5;
    const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
    for (long w = w0 + ((long)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < w1; w += nwarps) {
        const long j = (w << 5) - fifo_bits0 + lane;
        const bool in = j >= 0 && j < nbits;
        const bool bit = in && ((soft[(j + 2) ^ 1] > 0) != (soft[j ^ 1] > 0));
        const uint32_t v = __brev(__ballot_sync(0xffffffffu, bit)), mask = __brev(__ballot_sync(0xffffffffu, in));
        if (lane == 0)
            fifo[w] = mask == 0xffffffffu ? v : ((fifo[w] & ~mask) | v);
    }
}

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

// Every push's bits enter the bit FIFO (aqua_db_decoder: k_aqua_bits, noaa_gac_decoder: k_gac_bits), the deframer and frame stage of the
// convolutional decoders run with the decoder's settings, and noaa_gac_decoder's k_gac_post reverses (backward) and descrambles the frames
// in the output.
struct BitStage : Framed
{
    bool gac;
    int F;                            // the soft bytes a push needs (aqua_db_decoder: a complete symbol behind the carried one)
    long dropped = 0;                 // bit FIFO bits dropped by compaction: FIFO bit q is stream bit q - 32 + dropped
    DevBuf<uint8_t> pn;               // noaa_gac_decoder: the bytes XORed onto every frame ...
    PinnedBuf<FrameRec> h_fr;         // ... and the deframer's records of the last push

    explicit BitStage(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
};

BitStage::BitStage(Fec &f) : gac(f.cfg.kind == B200_FEC_NOAA_GAC), F(gac ? 1 : 2 * AQUA_LEAD)
{
    b200_fec_cfg &c = f.cfg;
    if (gac)
        B200_REQUIRE(c.backward == 0 || c.backward == 1, B200_EINVAL, "noaa_gac_decoder: backward must be 0 or 1 (got %d)", c.backward);
    B200_REQUIRE(c.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for %s", gac ? "noaa_gac_decoder" : "aqua_db_decoder");
    // The deframer and frame stage. aqua_db_decoder: BPSK_CCSDS_Deframer(8192, 0x1ACFFC1D) with STATE_SYNCED = 10 (:20-21),
    // derand_ccsds(&cadu[4], 1020), decode_interlaved(&cadu[4], true, 4). noaa_gac_decoder: BPSK_CCSDS_Deframer(33270, backward ?
    // 0x33c3e4a6 : 0xA116FD71), CADU_PADDING = 33270 % 8 (:20-22): (33270 + 6) / 8 = 4159 bytes, no derandomiser, no RS. chunk: the
    // module's read size (BUFFER_SIZE, BUFSIZE), what a stream reader of the decoder hands over at a time.
    struct Stage { int cadu_size; unsigned asm_sync; int derandomize, derand_start, rs_i, rs_dualbasis, st_synced, cadu_bytes, chunk; };
    //                          cadu_size asm_sync                                   derandomize derand_start rs_i rs_dualbasis st_synced cadu_bytes chunk
    const Stage s = gac ? Stage{GAC_BITS, c.backward ? GAC_SYNC_BACKWARD : GAC_SYNC, 0,          0,           0,   0,           12,       GAC_BYTES, 8192}
                        : Stage{8192,     0x1ACFFC1Du,                               1,          4,           4,   1,           10,       1024,      65536};
    c.cadu_size = s.cadu_size;
    c.asm_sync = s.asm_sync;
    c.derandomize = s.derandomize;
    c.derand_start = s.derand_start;
    c.rs_i = s.rs_i;
    c.rs_dualbasis = s.rs_dualbasis;
    c.nrzm = c.derand_after_rs = c.rs_type = c.rs_usecheck = 0;
    c.rs_fill_bytes = -1;
    f.st_synced = s.st_synced;
    f.cadu_bytes = s.cadu_bytes;
    f.geom.chunk = s.chunk;
    check_device(c.device);
    DeviceGuard g(c.device);
    f.framed_storage(F, 0);
    f.deframer_storage(c.max_soft + (gac ? 0 : 2 * AQUA_LEAD)); // one bit per soft byte
    if (gac) {
        pn.alloc(GAC_BYTES);
        h_fr.alloc((size_t)f.max_frames_push);
        std::vector<uint8_t> h_pn(GAC_BYTES);
        gac_pn_bytes(h_pn.data());
        B200_CUDA(cudaMemcpy(pn.p, h_pn.data(), GAC_BYTES, cudaMemcpyHostToDevice));
    }
    reset(f);
}

std::unique_ptr<Framed> bit_stage_decoder(Fec &f) { return std::make_unique<BitStage>(f); }

void BitStage::reset(Fec &f)
{
    f.start_stream(64); // the bit FIFO and the deframer
    Framed::reset(f);
    dropped = 0;
    if (!gac) {
        B200_CUDA(cudaMemsetAsync(f.softbuf.p, 0, AQUA_LEAD, f.stream));
        f.soft_have = AQUA_LEAD;
    }
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void BitStage::process(Fec &f)
{
    if (!begin(f, F))
        return;
    cudaStream_t stream = f.stream;
    const long fb0 = f.fifo_bits;
    f.compact_fifo(false);
    dropped += fb0 - f.fifo_bits;
    const long nbits = gac ? f.soft_have : (f.soft_have / 2 - 1) * 2;
    B200_REQUIRE(((f.fifo_bits + nbits + 64) >> 5) + 2 < (long)f.fifo.n, B200_ESTATE, "internal: bit FIFO too small");
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    const long words = (f.fifo_bits + nbits + 31) / 32 - f.fifo_bits / 32;
    const auto bits_kernel = gac ? k_gac_bits : k_aqua_bits;
    bits_kernel<<<(unsigned)std::min<long>((words + 7) / 8, 132 * 32), 256, 0, stream>>>(f.softbuf.p, nbits, f.fifo.p, f.fifo_bits);
    f.launches++;
    f.last_bits0 = f.fifo_bits;
    f.last_nbits = nbits;
    const long out0 = f.out_frames;
    f.deframe_and_rs(nbits); // (synchronises the stream)
    const int nf = f.last_nf;
    if (gac && nf > 0) {
        k_gac_post<<<nf, 256, 0, stream>>>(f.frames_out.p + out0 * GAC_BYTES, f.cfg.backward, pn.p);
        f.launches++;
        B200_CUDA(cudaMemcpyAsync(h_fr.p, f.frames.p, sizeof(FrameRec) * nf, cudaMemcpyDeviceToHost, stream));
    }
    f.keep_soft_tail(nbits); // (aqua_db_decoder: the last symbol, the next push's predecessor, and an odd byte stay)
    end(f);
    f.t_vit -= f.t_frames;
    if (gac) {
        std::vector<long> bits(nf);
        for (int k = 0; k < nf; k++) // the frame's last bit: its payload's (33270 - 32)th
            bits[k] = h_fr.p[k].pay_bit + (GAC_BITS - 32) - 1 - 32 + dropped;
        f.note_frame_bits(out0, bits);
    }
    tail_seen = f.soft_have;
    f.total_bits += nbits;
}

// ---------------------------------------------------------------- meteor_xband_decoder

// The soft FIFO starts with the byte before the first bit not decoded yet (its hard bit is NRZMDiff::lastBit); FIFO bit q >= 1 is padded
// stream bit q + pos0 - 1 (xband.cuh). At a stream's start the FIFO holds that byte and PAD zero bytes: the zeroed shift buffers, lastBit 0.
// A push decodes the module's whole 8192-byte reads: the record walk tests the window starts [next, R) with R the soft bytes of those
// reads, its records' packets enter the packet FIFO (32-bit words MSB first, whole records, each with its read), and the inner deframers
// walk the new packet bits. The inner frames come out ordered by (read, deframer, position), as the module writes them.
struct XBand : Framed
{
    bool kmss;
    int pad, npb, ndef, frm_bytes;
    long rec_cap = 0, frm_cap = 0, pk_cap = 0;
    long long pos0 = 0, pbase = 0;    // padded bit of FIFO bit 1; packet-stream bit of packet FIFO bit 0
    long pk_bytes = 0;                // bytes in the packet FIFO
    DevBuf<uint32_t> hw, db, cand, pk, pcand, pk_read, pk_tmp;
    DevBuf<XbRec> recs;
    DevBuf<XbFrame> frm;
    DevBuf<int> order;
    DevBuf<XbState> st;
    DevBuf<XbInner> inner;
    DevBuf<XbOut> out;
    PinnedBuf<XbOut> h_out;
    PinnedBuf<XbState> h_st;
    PinnedBuf<XbInner> h_inner;
    PinnedBuf<XbFrame> h_frm;
    PinnedBuf<int> h_order;

    explicit XBand(Fec &f);
    void process(Fec &f) override;
    void reset(Fec &f) override;
};

XBand::XBand(Fec &f)
    : kmss(f.cfg.instrument_type == 1), pad(kmss ? KMSS_PAD : MTVZA_PAD), npb(8 * (kmss ? KMSS_PKT : MTVZA_PKT)), ndef(kmss ? 3 : 1),
      frm_bytes(kmss ? KMSS_FRM : MTVZA_FRM)
{
    B200_REQUIRE(f.cfg.instrument_type == 0 || f.cfg.instrument_type == 1, B200_EINVAL, "Invalid METEOR instrument type!");
    B200_REQUIRE(f.cfg.max_soft <= (1L << 30), B200_EINVAL, "max_soft must be <= 2^30 for meteor_xband_decoder");
    f.cadu_bytes = frm_bytes;
    f.geom.chunk = XB_READ;
    const int F = pad + XB_READ + 64;    // what the FIFO keeps: the carried byte, the windows' reach and a partial read
    const long fifo = f.cfg.max_soft + 2L * F;
    // records a push can accept: kmss_bpsk one per 12288 tests; mtvza one per 3072 tests when locked (the cap allows 8 times that)
    rec_cap = kmss ? fifo / KMSS_REC + 4 : fifo / 384 + 8;
    // inner frames: one per 481280 / 3040 packet bits when locked, plus the open ones (the cap allows about 7 times that)
    const long pk_new = rec_cap * npb;
    frm_cap = kmss ? pk_new / 8192 + 8 : pk_new / 64 + 8;
    pk_cap = pk_new + (kmss ? KMSS_FRM : MTVZA_FRM) + 2L * npb + 64;
    check_device(f.cfg.device);
    DeviceGuard g(f.cfg.device);
    f.framed_storage(F, frm_cap * ndef);
    const size_t words = (size_t)fifo / 32 + 8, pwords = (size_t)pk_cap / 4 + 8;
    hw.alloc(words);
    db.alloc(words);
    cand.alloc(words);
    pk.alloc(pwords);
    pk_tmp.alloc(pwords);
    pcand.alloc((pwords + 8) * ndef);
    pk_read.alloc((size_t)pk_cap / npb + 8);
    recs.alloc((size_t)rec_cap);
    frm.alloc((size_t)frm_cap * ndef);
    order.alloc((size_t)frm_cap * ndef);
    st.alloc(1);
    inner.alloc(3);
    out.alloc(1);
    h_out.alloc(1);
    h_st.alloc(1);
    h_inner.alloc(3);
    h_frm.alloc((size_t)frm_cap * ndef);
    h_order.alloc((size_t)frm_cap * ndef);
    reset(f);
}

std::unique_ptr<Framed> xband_decoder(Fec &f) { return std::make_unique<XBand>(f); }

// a fresh module: lastBit 0, zeroed shift buffers, not synced, runs_since_sync and skip_bits 0, no open inner frame
void XBand::reset(Fec &f)
{
    Framed::reset(f);
    B200_CUDA(cudaMemsetAsync(f.softbuf.p, 0, (size_t)pad + 1, f.stream));
    f.soft_have = pad + 1;
    pos0 = pbase = 0;
    pk_bytes = 0;
    *h_st.p = XbState{0, 0, 0};
    for (int d = 0; d < 3; d++)
        h_inner.p[d] = XbInner{0, HRPT_NONE};
    B200_CUDA(cudaMemcpyAsync(st.p, h_st.p, sizeof(XbState), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaMemcpyAsync(inner.p, h_inner.p, 3 * sizeof(XbInner), cudaMemcpyHostToDevice, f.stream));
    B200_CUDA(cudaStreamSynchronize(f.stream));
}

void XBand::process(Fec &f)
{
    if (!begin(f, 1))
        return;
    cudaStream_t stream = f.stream;
    const long have = f.soft_have;
    const long long R = (pos0 + have - 1 - pad) / XB_READ * XB_READ; // (pos0 + have - 1: the padded bits in the FIFO)
    if (R <= pos0) {
        tail_seen = have;
        return;
    }
    const long long base = pos0 - 1, qend = R - base;
    const long nwords = (have + 31) / 32 + 2;
    B200_CUDA(cudaEventRecord(f.ev[0], stream));
    k_hard_pack<1><<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, stream>>>(f.softbuf.p, have, nwords, hw.p);
    k_nrzm_words<<<(unsigned)((nwords + 255) / 256), 256, 0, stream>>>(hw.p, nwords, db.p);
    k_xband_cand<<<(unsigned)((qend + 255) / 256), 256, 0, stream>>>(db.p, qend, kmss, cand.p);
    k_xband_rec_walk<<<1, 32, 0, stream>>>(db.p, cand.p, base, R, kmss, st.p, recs.p, (int)rec_cap, out.p);
    f.launches += 4;
    B200_CUDA(cudaMemcpyAsync(h_out.p, out.p, sizeof(XbOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    const int nrec = h_out.p->nrec;
    B200_REQUIRE(nrec <= rec_cap && pk_bytes + (long)nrec * npb <= pk_cap, B200_ESTATE,
                 "meteor_xband_decoder: %d records in one push (at most %ld): push less at a time", nrec, rec_cap);
    if (nrec > 0) {
        k_xband_packets<<<(unsigned)(((long)nrec * npb + 255) / 256), 256, 0, stream>>>(db.p, base, recs.p, nrec, kmss, (uint8_t *)pk.p,
                                                                                       pk_bytes, pk_read.p, pk_bytes / npb);
        f.launches++;
    }
    pk_bytes += (long)nrec * npb;
    const long long pbits = 8LL * pk_bytes;
    const long cwords = (long)(pbits / 32) + 2;
    for (int d = 0; d < ndef && pbits > 0; d++)
        k_sync_cand<<<(unsigned)((pbits + 255) / 256), 256, 0, stream>>>(pk.p, pbits, kmss ? kmss_sync(d) : MTVZA_SYNC,
                                                                       kmss ? (1ull << 56) - 1 : 0xFFFFFFFFull, 0, pcand.p + d * cwords);
    k_xband_inner_walk<<<ndef, 32, 0, stream>>>(pk.p, pcand.p, cwords, pbits, pbase, kmss, pk_read.p, inner.p, frm.p, (int)frm_cap, out.p);
    f.launches += (pbits > 0 ? ndef : 0) + 1;
    B200_CUDA(cudaMemcpyAsync(h_out.p, out.p, sizeof(XbOut), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaMemcpyAsync(h_inner.p, inner.p, 3 * sizeof(XbInner), cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    long nf = 0;
    for (int d = 0; d < ndef; d++) {
        B200_REQUIRE(h_out.p->nfrm[d] <= frm_cap, B200_ESTATE, "meteor_xband_decoder: %d frames in one push (at most %ld): push less at a time",
                     h_out.p->nfrm[d], frm_cap);
        nf += h_out.p->nfrm[d];
    }
    if (nf > 0) {
        B200_REQUIRE((size_t)(f.out_frames + nf) * f.cadu_bytes <= f.frames_out.n, B200_ESTATE,
                     "%ld frames not pulled yet: pull the frames between pushes", f.out_frames);
        uint8_t *dst = f.frames_out.p + f.out_frames * f.cadu_bytes;
        if (kmss) {
            // the module runs deframer 1, 2, 3 over each read's packets and writes their frames in that order
            for (int d = 0; d < 3; d++)
                if (h_out.p->nfrm[d] > 0)
                    B200_CUDA(cudaMemcpyAsync(h_frm.p + d * frm_cap, frm.p + d * frm_cap, sizeof(XbFrame) * h_out.p->nfrm[d],
                                              cudaMemcpyDeviceToHost, stream));
            B200_CUDA(cudaStreamSynchronize(stream));
            long k = 0, at[3] = {0, 0, 0};
            while (k < nf) {
                int best = -1;
                for (int d = 0; d < 3; d++)
                    if (at[d] < h_out.p->nfrm[d] && (best < 0 || h_frm.p[d * frm_cap + at[d]].read < h_frm.p[best * frm_cap + at[best]].read))
                        best = d;
                h_order.p[k++] = (int)(best * frm_cap + at[best]++);
            }
            B200_CUDA(cudaMemcpyAsync(order.p, h_order.p, sizeof(int) * nf, cudaMemcpyHostToDevice, stream));
            k_kmss_frames<<<(unsigned)((nf * KMSS_FRM + 255) / 256), 256, 0, stream>>>(pk.p, pbase, frm.p, order.p, nf, dst);
        } else {
            k_mtvza_frames<<<(unsigned)((nf * MTVZA_FRM + 255) / 256), 256, 0, stream>>>(pk.p, pbase, frm.p, nf, dst);
        }
        f.launches++;
    }
    // the packet FIFO keeps whole records from the first open frame's sync, else from 64 bits before the next test
    long long keep = pbits;
    for (int d = 0; d < ndef; d++)
        keep = std::min(keep, (h_inner.p[d].open != HRPT_NONE ? h_inner.p[d].open : h_inner.p[d].next) - 64 - pbase);
    const long drop_recs = (long)(std::max(0LL, keep) / 8 / npb);
    if (drop_recs > 0) {
        const long drop = drop_recs * npb, kept = pk_bytes - drop, nrecs = kept / npb;
        if (kept > 0) {
            B200_CUDA(cudaMemcpyAsync(pk_tmp.p, (uint8_t *)pk.p + drop, kept, cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(pk.p, pk_tmp.p, kept, cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(pk_tmp.p, pk_read.p + drop_recs, nrecs * 4, cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemcpyAsync(pk_read.p, pk_tmp.p, nrecs * 4, cudaMemcpyDeviceToDevice, stream));
        }
        pk_bytes = kept;
        pbase += 8LL * drop;
    }
    const long used = (long)(R - pos0);
    f.keep_soft_tail(used);
    end(f);
    pos0 = R;
    tail_seen = f.soft_have;
    last_nf = nrec;
    f.out_frames += nf;
    f.total_frames += nf;
    f.total_bits += used;
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

using namespace b200;

extern "C" int b200_fec_debug_hrpt_frames(b200_fec *h, b200_hrpt_frame *out, long cap, long *n_out)
{
    return guarded([&] {
        B200_REQUIRE(h && out && n_out, B200_EINVAL, "NULL argument");
        *n_out = h->f->framed_as<SyncWalk>("not an HRPT decoder").records(out, cap);
    });
}
